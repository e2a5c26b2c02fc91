// test_block_calibration.cc - exercises baz_music_doa::calibrate() as a flowgraph would: factory -> set_array_geometry()
// -> set_peak_mode() -> calibrate() -> the calibration items over several work() calls -> more work() calls on other
// items with the gains the block applied.  Reads a test vector file written by tests/test_gpu_calibration.py and writes
// the results next to it; the Python test compares them with the Python block.
//   in file (little endian): u32 m, n, nsamples, resolution, ncal, nwin, peak_mode, kind, chunk; f64 angle, wavelength;
//                            positions[m][2] f64; cal[ncal * nsamples * 2] f32; in[nwin * nsamples * 2] f32
//   out file: gains [m] (re, im) f64; residual f64; angles [nwin][n] f32; bins [nwin][n] i32
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
    unsigned hdr[9];
    double ld[2];
    if (fread(hdr, 4, 9, f) != 9 || fread(ld, 8, 2, f) != 2) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], C = hdr[4], W = hdr[5], chunk = hdr[8];
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
    blk->set_array_geometry(geo, ld[1]);
    blk->set_peak_mode((int)hdr[6], 0);

    // a gain vector of the wrong size and an unknown kind are refused; no calibration: all gains 1, residual NaN
    bool threw = false;
    try { blk->set_calibration(std::vector<std::complex<double> >(m + 1, 1.0)); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for a wrong gain count\n"); return 3; }
    threw = false;
    try { blk->calibrate(ld[0], 7, (int)C); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for an unknown kind\n"); return 3; }
    const std::vector<std::complex<double> > g1 = blk->calibration();
    for (unsigned i = 0; i < m; ++i)
        if (g1[i] != std::complex<double>(1.0, 0.0)) { fprintf(stderr, "uncalibrated gains must be 1\n"); return 4; }
    if (!std::isnan(blk->last_calibration_residual())) return 4;

    blk->calibrate(ld[0], (int)hdr[7], (int)C);
    std::vector<float> ang((size_t)std::max(C, W) * n), lvl(ang.size());
    for (unsigned c0 = 0; c0 < C; c0 += chunk) {
        const unsigned cnt = std::min(chunk, C - c0);
        gr_vector_const_void_star ins(1, cal.data() + (size_t)c0 * ns * 2);
        gr_vector_void_star outs;
        outs.push_back(ang.data()); outs.push_back(lvl.data());
        if (blk->work((int)cnt, ins, outs) != (int)cnt) return 5;
        if (c0 + cnt < C && !std::isnan(blk->last_calibration_residual())) { fprintf(stderr, "solved too early\n"); return 6; }
    }
    const double rho = blk->last_calibration_residual();
    if (!(rho >= 0.0)) { fprintf(stderr, "calibration failed\n"); return 7; }
    const std::vector<std::complex<double> > g = blk->calibration();

    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    outs.push_back(ang.data()); outs.push_back(lvl.data());
    if (blk->work((int)W, ins, outs) != (int)W) return 5;
    const std::vector<int> bins = blk->last_bins();
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(g.data(), 16, g.size(), o);
    fwrite(&rho, 8, 1, o);
    fwrite(ang.data(), 4, (size_t)W * n, o);
    fwrite(bins.data(), 4, (size_t)W * n, o);
    fclose(o);
    return 0;
}
