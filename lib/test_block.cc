// test_block.cc - exercises the gr::sync_block front exactly as the GNU Radio scheduler would:
// factory -> work(noutput_items, input_items, output_items) with 1, 2 and 3 connected outputs ->
// set_array_response().  Reads a test vector file written by tests/test_cpp_block.py, writes the
// outputs next to it; the Python test compares them with the oracle.
//   file layout (little endian): u32 m, n, nsamples, resolution, nwindows;
//                                table[resolution*m*2] f32; table2[resolution*m*2] f32; in[nwindows*nsamples*2] f32
// With a third argument RULE (1 = MDL, 2 = AIC) it instead runs one work() call with 3 outputs under that source rule
// and writes angles, levels, spectrum, bins and the per-window counts (table2 is not used).  With a fourth argument
// GEOM (a file of m (x, y) f64 positions in metres followed by the f64 wavelength) it also installs that geometry with
// set_array_geometry() and turns the peak refinement on before the work() call (RULE 0 keeps the fixed source count).
#include <baz_music_doa.h>

#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>

static array_response_t to_response(const float *t, unsigned K, unsigned m)
{
    array_response_t r(K, antenna_response_t(m));
    for (unsigned k = 0; k < K; ++k)
        for (unsigned i = 0; i < m; ++i) r[k][i] = gr_complex(t[2 * (k * m + i)], t[2 * (k * m + i) + 1]);
    return r;
}

// geometry file -> set_array_geometry(), then set_refine(true); the table-only block must refuse the refinement first
static int install_geometry_and_refine(baz_music_doa_sptr blk, unsigned m, const char *geom_path)
{
    FILE *g = fopen(geom_path, "rb");
    if (!g) return 2;
    std::vector<double> v(2 * (size_t)m + 1);
    const size_t got = fread(v.data(), 8, v.size(), g);
    fclose(g);
    if (got != v.size()) return 2;
    bool threw = false;
    try { blk->set_refine(true); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for set_refine on a table without geometry\n"); return 3; }
    std::vector<std::vector<double> > pos(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i) { pos[i][0] = v[2 * i]; pos[i][1] = v[2 * i + 1]; }
    blk->set_array_geometry(pos, v[2 * (size_t)m]);
    blk->set_refine(true);
    return 0;
}

static int run_source_rule(baz_music_doa_sptr blk, int rule, unsigned n, unsigned K, unsigned W, const std::vector<float> &in,
                           const char *out_path)
{
    bool threw = false;
    try { blk->set_source_rule(7); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for source rule 7\n"); return 3; }
    blk->set_source_rule(rule);
    std::vector<float> ang((size_t)W * n), lvl((size_t)W * n), spec((size_t)W * K);
    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    outs.push_back(ang.data()); outs.push_back(lvl.data()); outs.push_back(spec.data());
    if (blk->work((int)W, ins, outs) != (int)W) return 5;
    const std::vector<int> bins = blk->last_bins(), counts = blk->last_counts();
    if (counts.size() != W) return 5;
    FILE *o = fopen(out_path, "wb");
    if (!o) return 2;
    fwrite(ang.data(), 4, ang.size(), o);
    fwrite(lvl.data(), 4, lvl.size(), o);
    fwrite(spec.data(), 4, spec.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fwrite(counts.data(), 4, counts.size(), o);
    fclose(o);
    return 0;
}

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[5];
    if (fread(hdr, 4, 5, f) != 5) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], W = hdr[4];
    std::vector<float> t1((size_t)K * m * 2), t2((size_t)K * m * 2), in((size_t)W * ns * 2);
    if (fread(t1.data(), 4, t1.size(), f) != t1.size() || fread(t2.data(), 4, t2.size(), f) != t2.size() ||
        fread(in.data(), 4, in.size(), f) != in.size())
        return 2;
    fclose(f);

    // constructor argument checks follow the library convention (std::invalid_argument)
    bool threw = false;
    try { baz_make_music_doa(m, m, ns, to_response(t1.data(), K, m), K); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for n == m\n"); return 3; }

    baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, to_response(t1.data(), K, m), K);
    if (argc > 4) {
        const int rc = install_geometry_and_refine(blk, m, argv[4]);
        if (rc) return rc;
    }
    if (argc > 3) return run_source_rule(blk, atoi(argv[3]), n, K, W, in, argv[2]);
    if (blk->input_signature()->sizeof_stream_item(0) != (int)(ns * sizeof(gr_complex))) return 4;
    if (blk->output_signature()->max_streams() != 3 || blk->output_signature()->sizeof_stream_item(2) != (int)(K * 4)) return 4;

    std::vector<float> ang3((size_t)W * n), lvl3((size_t)W * n), spec3((size_t)W * K), ang1((size_t)W * n), ang_t2((size_t)W * n), lvl_t2((size_t)W * n);
    gr_vector_const_void_star ins(1, in.data());
    {
        gr_vector_void_star outs;
        outs.push_back(ang3.data()); outs.push_back(lvl3.data()); outs.push_back(spec3.data());
        if (blk->work((int)W, ins, outs) != (int)W) return 5;
    }
    std::vector<int> bins = blk->last_bins();
    {
        gr_vector_void_star outs(1, ang1.data());  // only port 0 connected
        if (blk->work((int)W, ins, outs) != (int)W) return 5;
    }
    blk->set_array_response(to_response(t2.data(), K, m));
    {
        gr_vector_void_star outs;
        outs.push_back(ang_t2.data()); outs.push_back(lvl_t2.data());
        if (blk->work((int)W, ins, outs) != (int)W) return 5;
    }
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(ang3.data(), 4, ang3.size(), o);
    fwrite(lvl3.data(), 4, lvl3.size(), o);
    fwrite(spec3.data(), 4, spec3.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fwrite(ang1.data(), 4, ang1.size(), o);
    fwrite(ang_t2.data(), 4, ang_t2.size(), o);
    fwrite(lvl_t2.data(), 4, lvl_t2.size(), o);
    fclose(o);
    return 0;
}
