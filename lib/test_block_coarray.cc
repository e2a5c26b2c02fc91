// test_block_coarray.cc - exercises baz_make_music_doa_coarray() as a flowgraph would: factory -> the refused setters
// (each must throw) -> the retune -> setters -> one work() call with every output connected.  Reads a test vector file
// written by tests/test_gpu_coarray.py and writes the outputs next to it; the Python test compares them with the Python
// block's.
//   in file (little endian): u32 m, n, nsamples, nwindows, resolution, mv, peak_mode, refine_mode, calibrated;
//                            f64 step[2], wavelength; i32 positions[m]; f64 gains[m][2]; in[nwindows * nsamples * 2] f32
//   out file: angles [nwindows][n] f32; levels [nwindows][n] f32; spectrum [nwindows][K] f32; bins [nwindows][n] i32
#include <baz_music_doa.h>

#include <complex>
#include <cstdio>
#include <stdexcept>
#include <vector>

namespace {

template <class T>
bool get(FILE *f, T *p, size_t count) { return fread(p, sizeof(T), count, f) == count; }

// whether f() throws E
template <class E, class F>
bool throws(F f)
{
    try { f(); } catch (const E &) { return true; }
    return false;
}

}  // namespace

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[9];
    double dv[3];
    if (!get(f, hdr, 9) || !get(f, dv, 3)) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], W = hdr[3], K = hdr[4], mv = hdr[5];
    const int peak = (int)hdr[6], refine = (int)hdr[7];
    const bool calibrated = hdr[8] != 0;
    std::vector<int> pos(m);
    std::vector<double> g(2 * (size_t)m);
    std::vector<float> in((size_t)W * ns * 2);
    if (!get(f, pos.data(), m) || !get(f, g.data(), g.size()) || !get(f, in.data(), in.size())) return 2;
    fclose(f);
    const std::vector<double> step = {dv[0], dv[1]};
    baz_music_doa_sptr blk = baz_make_music_doa_coarray(m, n, ns, K, pos, step, dv[2], mv);
    // what a co-array handle does not serve throws, and leaves the block as it was
    if (!throws<std::invalid_argument>([&] { blk->set_estimator(1, 0.1); })) { fprintf(stderr, "MVDR accepted\n"); return 3; }
    if (!throws<std::invalid_argument>([&] { blk->set_source_rule(1); })) { fprintf(stderr, "MDL accepted\n"); return 3; }
    if (!throws<std::invalid_argument>([&] { blk->set_peak_mode(4, 0); })) { fprintf(stderr, "DML accepted\n"); return 3; }
    if (!throws<std::invalid_argument>([&] { blk->set_beamformer(1, 0.0); })) { fprintf(stderr, "beams accepted\n"); return 3; }
    if (!throws<std::runtime_error>([&] { blk->set_array_response(array_response_t(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)))); })) {
        fprintf(stderr, "set_array_response accepted\n");
        return 3;
    }
    if (!throws<std::invalid_argument>([&] { blk->set_coarray_geometry(std::vector<double>{dv[2], 0.0}, dv[2]); })) {
        fprintf(stderr, "a step of one wavelength accepted\n");
        return 3;
    }
    if (!throws<std::runtime_error>([&] { blk->calibrate(0.0, 2, (int)W); }) ||
        !throws<std::runtime_error>([&] { blk->calibrate_blind(1, 2, (int)W, 1); })) {
        fprintf(stderr, "calibration estimation accepted\n");
        return 3;
    }
    blk->set_coarray_geometry(step, dv[2]);
    blk->set_peak_mode(peak, 0);
    blk->set_refine_mode(refine);
    if (calibrated) {
        std::vector<std::complex<double> > gains(m);
        for (unsigned i = 0; i < m; ++i) gains[i] = std::complex<double>(g[2 * i], g[2 * i + 1]);
        blk->set_calibration(gains);
    }
    std::vector<std::vector<float> > outs = {std::vector<float>((size_t)W * n), std::vector<float>((size_t)W * n),
                                             std::vector<float>((size_t)W * K)};
    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star o;
    for (auto &v : outs) o.push_back(v.data());
    if (blk->work((int)W, ins, o) != (int)W) return 5;
    FILE *out = fopen(argv[2], "wb");
    if (!out) return 2;
    for (const auto &v : outs) fwrite(v.data(), 4, v.size(), out);
    fwrite(blk->last_bins().data(), 4, blk->last_bins().size(), out);
    fclose(out);
    return 0;
}
