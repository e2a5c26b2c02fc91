// test_block_beams.cc - exercises baz_music_doa::set_beamformer() as a flowgraph would: factory -> set_array_geometry()
// -> set_peak_mode() -> set_beamformer() -> one work() call with all 3 outputs connected.  Reads a test vector file
// written by tests/test_gpu_beams.py and writes the outputs next to it; the Python test compares them with the Python
// block.
//   in file (little endian): u32 m, n, nsamples, resolution, nwindows, peak_mode, rule; f64 loading, wavelength;
//                            positions[m][2] f64; in[nwindows * nsamples * 2] f32
//   out file: angles, levels [nwindows][n] f32; spectrum [nwindows][resolution] f32; bins [nwindows][n] i32;
//             beams [nwindows][n][nsamples / m] c64
#include <baz_music_doa.h>

#include <cstdio>
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
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], W = hdr[4];
    std::vector<double> pos((size_t)m * 2);
    std::vector<float> in((size_t)W * ns * 2);
    if (fread(pos.data(), 8, pos.size(), f) != pos.size() || fread(in.data(), 4, in.size(), f) != in.size()) return 2;
    fclose(f);
    array_response_t table(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)));
    baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, table, K);
    std::vector<std::vector<double> > geo(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i) { geo[i][0] = pos[2 * i]; geo[i][1] = pos[2 * i + 1]; }
    blk->set_array_geometry(geo, ld[1]);
    blk->set_peak_mode((int)hdr[5], 0);

    // loading with delay-and-sum is refused
    bool threw = false;
    try { blk->set_beamformer(1, 0.5); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for DAS with loading\n"); return 3; }
    blk->set_beamformer((int)hdr[6], ld[0]);

    std::vector<float> ang((size_t)W * n), lvl((size_t)W * n), spec((size_t)W * K);
    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    outs.push_back(ang.data()); outs.push_back(lvl.data()); outs.push_back(spec.data());
    if (blk->work((int)W, ins, outs) != (int)W) return 5;
    const std::vector<int> bins = blk->last_bins();
    const std::vector<gr_complex> beams = blk->last_beams();
    if (beams.size() != (size_t)W * n * (ns / m)) return 6;
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(ang.data(), 4, ang.size(), o);
    fwrite(lvl.data(), 4, lvl.size(), o);
    fwrite(spec.data(), 4, spec.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fwrite(beams.data(), 8, beams.size(), o);
    fclose(o);
    return 0;
}
