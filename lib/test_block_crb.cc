// test_block_crb.cc - exercises baz_music_doa::set_crb() as a flowgraph would: factory -> set_array_geometry() ->
// local-maximum peaks with refinement -> (a delay-and-sum beamformer) -> covariance integration -> set_crb(true) ->
// two work() calls, the integrated covariance carried from the first to the second.  Reads a test vector file written by
// tests/test_gpu_crb.py and writes the results next to it; the Python test compares them with the Python block, whose
// work() makes one library call per call (a second call would advance the integration again).
//   in file (little endian): u32 m, n, nsamples, resolution, nwin, beam_rule; f64 alpha, wavelength;
//                            positions[m][2] f64; in[nwin * nsamples * 2] f32
//   out file: angles [nwin][n] f32; crb [nwin][n] f32; beams [nwin][n][nsamples / m] complex64 (beam_rule != 0 only)
#include <baz_music_doa.h>

#include <algorithm>
#include <cstdio>
#include <vector>

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[6];
    double ld[2];
    if (fread(hdr, 4, 6, f) != 6 || fread(ld, 8, 2, f) != 2) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], W = hdr[4], rule = hdr[5];
    std::vector<double> pos((size_t)m * 2);
    std::vector<float> in((size_t)W * ns * 2);
    if (fread(pos.data(), 8, pos.size(), f) != pos.size() || fread(in.data(), 4, in.size(), f) != in.size()) return 2;
    fclose(f);
    array_response_t table(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)));
    baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, table, K);
    std::vector<std::vector<double> > geo(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i) { geo[i][0] = pos[2 * i]; geo[i][1] = pos[2 * i + 1]; }
    blk->set_array_geometry(geo, ld[1]);
    blk->set_peak_mode(1, 0);
    blk->set_refine(true);
    if (rule) blk->set_beamformer((int)rule, 0.0);
    blk->set_integration(ld[0]);
    blk->set_crb(true);

    const size_t N = ns / m;
    std::vector<float> ang((size_t)W * n), lvl((size_t)W * n), crb((size_t)W * n);
    std::vector<gr_complex> beams(rule ? (size_t)W * n * N : 0);
    const unsigned half = W / 2;
    for (unsigned w0 = 0; w0 < W; w0 += half) {
        const unsigned cnt = std::min(half, W - w0);
        gr_vector_const_void_star ins(1, in.data() + (size_t)w0 * ns * 2);
        gr_vector_void_star outs;
        outs.push_back(ang.data() + (size_t)w0 * n);
        outs.push_back(lvl.data() + (size_t)w0 * n);
        if (blk->work((int)cnt, ins, outs) != (int)cnt) return 5;
        const std::vector<float> &c = blk->last_crb();
        if (c.size() != (size_t)cnt * n) return 6;
        std::copy(c.begin(), c.end(), crb.begin() + (size_t)w0 * n);
        if (rule) {
            const std::vector<gr_complex> &b = blk->last_beams();
            if (b.size() != (size_t)cnt * n * N) return 7;
            std::copy(b.begin(), b.end(), beams.begin() + (size_t)w0 * n * N);
        }
    }
    blk->set_crb(false);
    {
        gr_vector_const_void_star ins(1, in.data());
        gr_vector_void_star outs(1, lvl.data());
        if (blk->work(1, ins, outs) != 1 || !blk->last_crb().empty()) return 8;
    }
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(ang.data(), 4, ang.size(), o);
    fwrite(crb.data(), 4, crb.size(), o);
    if (rule) fwrite(beams.data(), 8, beams.size(), o);
    fclose(o);
    return 0;
}
