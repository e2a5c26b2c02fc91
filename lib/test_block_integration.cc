// test_block_integration.cc - exercises baz_music_doa::set_integration() as a flowgraph would: factory ->
// set_array_geometry() -> set_source_rule() -> set_integration() -> work() calls of `chunk` items each, the integrated
// covariance carried from one call to the next -> reset_integration() -> the same items again.  Reads a test vector file
// written by tests/test_gpu_integration.py and writes the results next to it; the Python test compares them with the
// Python block.
//   in file (little endian): u32 m, n, nsamples, resolution, nwin, rule, chunk; f64 alpha, wavelength;
//                            positions[m][2] f64; in[nwin * nsamples * 2] f32
//   out file: angles [2][nwin][n] f32; bins [2][nwin][n] i32; counts [2][nwin] i32 (before and after the reset)
#include <baz_music_doa.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <limits>
#include <stdexcept>
#include <vector>

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[7];
    double ld[2];
    if (fread(hdr, 4, 7, f) != 7 || fread(ld, 8, 2, f) != 2) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], W = hdr[4], chunk = hdr[6];
    std::vector<double> pos((size_t)m * 2);
    std::vector<float> in((size_t)W * ns * 2);
    if (fread(pos.data(), 8, pos.size(), f) != pos.size() || fread(in.data(), 4, in.size(), f) != in.size()) return 2;
    fclose(f);
    array_response_t table(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)));
    baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, table, K);
    std::vector<std::vector<double> > geo(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i) { geo[i][0] = pos[2 * i]; geo[i][1] = pos[2 * i + 1]; }
    blk->set_array_geometry(geo, ld[1]);
    blk->set_source_rule((int)hdr[5]);

    // forgetting factors outside [0, 1) are refused
    const double bad[3] = {-0.25, 1.0, std::numeric_limits<double>::quiet_NaN()};
    for (int b = 0; b < 3; ++b) {
        bool threw = false;
        try { blk->set_integration(bad[b]); } catch (const std::invalid_argument &) { threw = true; }
        if (!threw) { fprintf(stderr, "expected invalid_argument for alpha = %g\n", bad[b]); return 3; }
    }
    blk->set_integration(ld[0]);

    std::vector<float> ang((size_t)2 * W * n), lvl((size_t)W * n);
    std::vector<int> bins((size_t)2 * W * n), counts((size_t)2 * W);
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1) blk->reset_integration();
        for (unsigned w0 = 0; w0 < W; w0 += chunk) {
            const unsigned cnt = std::min(chunk, W - w0);
            gr_vector_const_void_star ins(1, in.data() + (size_t)w0 * ns * 2);
            gr_vector_void_star outs;
            outs.push_back(ang.data() + ((size_t)pass * W + w0) * n);
            outs.push_back(lvl.data() + (size_t)w0 * n);
            if (blk->work((int)cnt, ins, outs) != (int)cnt) return 5;
            const std::vector<int> &b = blk->last_bins();
            const std::vector<int> &c = blk->last_counts();
            std::copy(b.begin(), b.begin() + (size_t)cnt * n, bins.begin() + ((size_t)pass * W + w0) * n);
            std::copy(c.begin(), c.begin() + cnt, counts.begin() + (size_t)pass * W + w0);
        }
    }
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(ang.data(), 4, ang.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fwrite(counts.data(), 4, counts.size(), o);
    fclose(o);
    return 0;
}
