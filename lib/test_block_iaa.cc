// test_block_iaa.cc - exercises set_estimator(4 = IAA) and set_iaa_iterations() on the three gr::sync_block fronts as a
// flowgraph would: factory -> setters -> one work() call with every output connected.  Reads a test vector file written
// by tests/test_gpu_iaa.py and writes the outputs next to it; the Python test compares them with the Python blocks.
//   in file (little endian): u32 kind (0 = baz_music_doa, 1 = baz_music_doa_azel, 2 = baz_music_doa_channels), m, n,
//                            nsamples, nwindows, iterations, peak_mode; f64 loading; then per kind
//     0: u32 resolution; f64 wavelength; positions[m][2] (metres)
//     1: u32 n_az, n_el; f64 el_lo, el_hi, wavelength; positions[m][3] (metres)
//     2: u32 resolution, nfft, chan_first, chan_count, combine; f64 centre_frequency, sample_rate; positions[m][2] (metres)
//   and in[nwindows * nsamples * 2] f32
//   out file: angles (azimuths) [nwindows][rows][n] f32; elevations [nwindows][n] f32 (kind 1 only); levels
//             [nwindows][rows][n] f32; spectrum [nwindows][rows][K] f32; bins [nwindows][rows][n] i32
//             (rows = chan_count for a separate channel block, else 1)
#include <baz_music_doa.h>
#include <baz_music_doa_azel.h>
#include <baz_music_doa_channels.h>

#include <cstdio>
#include <stdexcept>
#include <vector>

namespace {

template <class T>
bool get(FILE *f, T *p, size_t count) { return fread(p, sizeof(T), count, f) == count; }

// the IAA setters' argument checks follow the library convention (std::invalid_argument)
template <class B>
int check_refusals(B &blk)
{
    for (int bad : {0, 65}) {
        bool threw = false;
        try { blk->set_iaa_iterations(bad); } catch (const std::invalid_argument &) { threw = true; }
        if (!threw) { fprintf(stderr, "expected invalid_argument for %d IAA iterations\n", bad); return 3; }
    }
    bool threw = false;
    try { blk->set_estimator(4, -1.0); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for a negative IAA loading\n"); return 3; }
    return 0;
}

template <class B>
int run(B &blk, unsigned W, unsigned iters, int peak, double loading, std::vector<float> &in, std::vector<std::vector<float> > &outs_f)
{
    if (const int rc = check_refusals(blk)) return rc;
    blk->set_estimator(4, loading);
    blk->set_iaa_iterations((int)iters);
    blk->set_peak_mode(peak, 0);
    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    for (auto &o : outs_f) outs.push_back(o.data());
    return blk->work((int)W, ins, outs) == (int)W ? 0 : 5;
}

}  // namespace

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[7];
    double loading;
    if (!get(f, hdr, 7) || !get(f, &loading, 1)) return 2;
    const unsigned kind = hdr[0], m = hdr[1], n = hdr[2], ns = hdr[3], W = hdr[4], iters = hdr[5];
    const int peak = (int)hdr[6];
    std::vector<std::vector<float> > outs;
    std::vector<int> bins;
    std::vector<float> in;
    if (kind == 0) {
        unsigned K;
        double lam;
        std::vector<double> p(2 * (size_t)m);
        if (!get(f, &K, 1) || !get(f, &lam, 1) || !get(f, p.data(), p.size())) return 2;
        in.resize((size_t)W * ns * 2);
        if (!get(f, in.data(), in.size())) return 2;
        std::vector<std::vector<double> > pos(m, std::vector<double>(2));
        for (unsigned i = 0; i < m; ++i) pos[i] = {p[2 * i], p[2 * i + 1]};
        array_response_t table(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)));
        baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, table, K);
        blk->set_array_geometry(pos, lam);
        outs = {std::vector<float>((size_t)W * n), std::vector<float>((size_t)W * n), std::vector<float>((size_t)W * K)};
        if (const int rc = run(blk, W, iters, peak, loading, in, outs)) return rc;
        bins = blk->last_bins();
    } else if (kind == 1) {
        unsigned g[2];
        double dv[3];
        std::vector<double> p(3 * (size_t)m);
        if (!get(f, g, 2) || !get(f, dv, 3) || !get(f, p.data(), p.size())) return 2;
        in.resize((size_t)W * ns * 2);
        if (!get(f, in.data(), in.size())) return 2;
        std::vector<std::vector<double> > pos(m, std::vector<double>(3));
        for (unsigned i = 0; i < m; ++i) pos[i] = {p[3 * i], p[3 * i + 1], p[3 * i + 2]};
        baz_music_doa_azel_sptr blk = baz_make_music_doa_azel(m, n, ns, g[0], g[1], dv[0], dv[1], pos, dv[2]);
        outs = {std::vector<float>((size_t)W * n), std::vector<float>((size_t)W * n), std::vector<float>((size_t)W * n),
                std::vector<float>((size_t)W * g[0] * g[1])};
        if (const int rc = run(blk, W, iters, peak, loading, in, outs)) return rc;
        bins = blk->last_bins();
    } else if (kind == 2) {
        unsigned c[5];
        double dv[2];
        std::vector<double> p(2 * (size_t)m);
        if (!get(f, c, 5) || !get(f, dv, 2) || !get(f, p.data(), p.size())) return 2;
        in.resize((size_t)W * ns * 2);
        if (!get(f, in.data(), in.size())) return 2;
        std::vector<std::vector<double> > pos(m, std::vector<double>(2));
        for (unsigned i = 0; i < m; ++i) pos[i] = {p[2 * i], p[2 * i + 1]};
        const unsigned K = c[0], rows = c[4] == 0 ? c[3] : 1;
        baz_music_doa_channels_sptr blk = baz_make_music_doa_channels(m, n, ns, K, c[1], c[2], c[3], 1, (int)c[4], pos, 1.0, dv[0], dv[1]);
        outs = {std::vector<float>((size_t)W * rows * n), std::vector<float>((size_t)W * rows * n),
                std::vector<float>((size_t)W * rows * K)};
        if (const int rc = run(blk, W, iters, peak, loading, in, outs)) return rc;
        bins = blk->last_bins();
    } else {
        return 2;
    }
    fclose(f);
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    for (const auto &v : outs) fwrite(v.data(), 4, v.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fclose(o);
    return 0;
}
