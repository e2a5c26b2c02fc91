// test_block_azel.cc - exercises the az-el gr::sync_block front (baz_music_doa_azel) as the GNU Radio scheduler would:
// factory -> setters -> one work() call with all 4 outputs connected.  Reads a test vector file written by
// tests/test_gpu_azel.py and writes the outputs next to it; the Python test compares them with the Python block.
//   in file (little endian): u32 m, n, nsamples, n_az, n_el, nwindows, peak_mode, exclusion, source_rule, refine;
//                            f64 el_lo, el_hi, wavelength, positions[m][3]; in[nwindows * nsamples * 2] f32
//   out file: azimuth, elevation, level [nwindows][n] f32; spectrum [nwindows][n_el * n_az] f32; bins [nwindows][n] i32;
//             counts [nwindows] i32
#include <baz_music_doa_azel.h>

#include <cstdio>
#include <stdexcept>
#include <vector>

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[10];
    double dv[3];
    if (fread(hdr, 4, 10, f) != 10 || fread(dv, 8, 3, f) != 3) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], n_az = hdr[3], n_el = hdr[4], W = hdr[5];
    std::vector<double> p(3 * (size_t)m);
    std::vector<float> in((size_t)W * ns * 2);
    if (fread(p.data(), 8, p.size(), f) != p.size() || fread(in.data(), 4, in.size(), f) != in.size()) return 2;
    fclose(f);
    std::vector<std::vector<double> > pos(m, std::vector<double>(3));
    for (unsigned i = 0; i < m; ++i)
        for (int c = 0; c < 3; ++c) pos[i][c] = p[3 * i + c];

    // constructor argument checks follow the library convention (std::invalid_argument)
    bool threw = false;
    try { baz_make_music_doa_azel(m, n, ns, n_az, n_el, dv[1], dv[0], pos, dv[2]); } catch (const std::invalid_argument &) { threw = true; }
    if (n_el >= 2 && !threw) { fprintf(stderr, "expected invalid_argument for el_lo > el_hi\n"); return 3; }

    baz_music_doa_azel_sptr blk = baz_make_music_doa_azel(m, n, ns, n_az, n_el, dv[0], dv[1], pos, dv[2]);
    if (blk->input_signature()->sizeof_stream_item(0) != (int)(ns * 8)) return 4;
    if (blk->output_signature()->min_streams() != 2 || blk->output_signature()->max_streams() != 4 ||
        blk->output_signature()->sizeof_stream_item(2) != (int)(n * 4) || blk->output_signature()->sizeof_stream_item(3) != (int)(n_az * n_el * 4))
        return 4;
    blk->set_array_geometry(pos, dv[2]);
    blk->set_peak_mode((int)hdr[6], hdr[7]);
    blk->set_source_rule((int)hdr[8]);
    blk->set_refine(hdr[9] != 0);

    std::vector<float> az((size_t)W * n), el((size_t)W * n), lvl((size_t)W * n), spec((size_t)W * n_az * n_el);
    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    outs.push_back(az.data()); outs.push_back(el.data()); outs.push_back(lvl.data()); outs.push_back(spec.data());
    if (blk->work((int)W, ins, outs) != (int)W) return 5;
    const std::vector<int> bins = blk->last_bins(), counts = blk->last_counts();
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(az.data(), 4, az.size(), o);
    fwrite(el.data(), 4, el.size(), o);
    fwrite(lvl.data(), 4, lvl.size(), o);
    fwrite(spec.data(), 4, spec.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fwrite(counts.data(), 4, counts.size(), o);
    fclose(o);
    return 0;
}
