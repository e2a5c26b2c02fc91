// test_block_calib_blind.cc - exercises baz_music_doa::calibrate_blind() as a flowgraph would: factory ->
// set_array_geometry() -> calibrate_blind() -> the calibration items over several work() calls whose sizes need not be
// whole segments -> more work() calls on other items with the gains the block applied.  Reads a test vector file
// written by tests/test_gpu_calib_blind.py and writes the results next to it; the Python test compares them with the
// Python block.
//   in file (little endian): u32 m, n, nsamples, resolution, ncal, nwin, nsources, kind, segment, chunk; f64 wavelength;
//                            positions[m][2] f64; cal[ncal * nsamples * 2] f32; in[nwin * nsamples * 2] f32
//   out file: gains [m] (re, im) f64; misfit f64; angles [nwin][n] f32; bins [nwin][n] i32
#include <baz_music_doa.h>

#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdio>
#include <stdexcept>
#include <vector>

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[10];
    double lam;
    if (fread(hdr, 4, 10, f) != 10 || fread(&lam, 8, 1, f) != 1) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], C = hdr[4], W = hdr[5], seg = hdr[8], chunk = hdr[9];
    std::vector<double> pos((size_t)m * 2);
    std::vector<float> cal((size_t)C * ns * 2), in((size_t)W * ns * 2);
    if (fread(pos.data(), 8, pos.size(), f) != pos.size() || fread(cal.data(), 4, cal.size(), f) != cal.size() ||
        fread(in.data(), 4, in.size(), f) != in.size())
        return 2;
    fclose(f);
    array_response_t table(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)));
    baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, table, K);
    std::vector<std::vector<double> > geo(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i) { geo[i][0] = pos[2 * i]; geo[i][1] = pos[2 * i + 1]; }
    blk->set_array_geometry(geo, lam);

    // an item count that is not a multiple of the segment, and an unknown kind, are refused
    bool threw = false;
    try { blk->calibrate_blind((int)hdr[6], (int)hdr[7], (int)seg + 1, (int)seg); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw || seg < 2) { fprintf(stderr, "expected invalid_argument for a ragged item count\n"); return 3; }
    threw = false;
    try { blk->calibrate_blind((int)hdr[6], 7, (int)C, (int)seg); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for an unknown kind\n"); return 3; }

    blk->calibrate_blind((int)hdr[6], (int)hdr[7], (int)C, (int)seg);
    std::vector<float> ang((size_t)std::max(C, W) * n), lvl(ang.size());
    for (unsigned c0 = 0; c0 < C; c0 += chunk) {
        const unsigned cnt = std::min(chunk, C - c0);
        gr_vector_const_void_star ins(1, cal.data() + (size_t)c0 * ns * 2);
        gr_vector_void_star outs;
        outs.push_back(ang.data()); outs.push_back(lvl.data());
        if (blk->work((int)cnt, ins, outs) != (int)cnt) return 5;
        if (c0 + cnt < C && !std::isnan(blk->last_calibration_residual())) { fprintf(stderr, "solved too early\n"); return 6; }
    }
    const double misfit = blk->last_calibration_residual();
    if (!(misfit >= 0.0)) { fprintf(stderr, "self-calibration failed\n"); return 7; }
    const std::vector<std::complex<double> > g = blk->calibration();

    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    outs.push_back(ang.data()); outs.push_back(lvl.data());
    if (blk->work((int)W, ins, outs) != (int)W) return 5;
    const std::vector<int> bins = blk->last_bins();
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(g.data(), 16, g.size(), o);
    fwrite(&misfit, 8, 1, o);
    fwrite(ang.data(), 4, (size_t)W * n, o);
    fwrite(bins.data(), 4, (size_t)W * n, o);
    fclose(o);
    return 0;
}
