// test_block_roots.cc - exercises baz_music_doa::set_peak_mode(2, 0) (root-MUSIC) as a flowgraph would: factory ->
// setters -> one work() call with all 3 outputs connected.  Reads a test vector file written by
// tests/test_gpu_root_music.py and writes the outputs next to it; the Python test compares them with the Python block.
//   in file (little endian): u32 m, n, nsamples, resolution, nwindows, source_rule; f64 wavelength, positions[m][2];
//                            in[nwindows * nsamples * 2] f32
//   out file: angles, levels [nwindows][n] f32; spectrum [nwindows][resolution] f32; bins [nwindows][n] i32;
//             counts [nwindows] i32
#include <baz_music_doa.h>

#include <cstdio>
#include <stdexcept>
#include <vector>

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[6];
    double lambda;
    if (fread(hdr, 4, 6, f) != 6 || fread(&lambda, 8, 1, f) != 1) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], W = hdr[4];
    std::vector<double> p(2 * (size_t)m);
    std::vector<float> in((size_t)W * ns * 2);
    if (fread(p.data(), 8, p.size(), f) != p.size() || fread(in.data(), 4, in.size(), f) != in.size()) return 2;
    fclose(f);
    std::vector<std::vector<double> > pos(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i)
        for (int c = 0; c < 2; ++c) pos[i][c] = p[2 * i + c];

    array_response_t table(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)));
    baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, table, K);

    // without a geometry (a set_array_response() table) and with an exclusion the root mode is refused
    bool threw = false;
    try { blk->set_peak_mode(2, 0); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for the root mode without a geometry\n"); return 3; }
    blk->set_array_geometry(pos, lambda);
    threw = false;
    try { blk->set_peak_mode(2, 1); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for the root mode with exclusion_bins\n"); return 3; }

    blk->set_peak_mode(2, 0);
    blk->set_source_rule((int)hdr[5]);

    std::vector<float> ang((size_t)W * n), lvl((size_t)W * n), spec((size_t)W * K);
    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    outs.push_back(ang.data()); outs.push_back(lvl.data()); outs.push_back(spec.data());
    if (blk->work((int)W, ins, outs) != (int)W) return 5;
    const std::vector<int> bins = blk->last_bins(), counts = blk->last_counts();
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(ang.data(), 4, ang.size(), o);
    fwrite(lvl.data(), 4, lvl.size(), o);
    fwrite(spec.data(), 4, spec.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fwrite(counts.data(), 4, counts.size(), o);
    fclose(o);
    return 0;
}
