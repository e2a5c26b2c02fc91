// test_block_focus.cc - exercises the channel gr::sync_block front (baz_music_doa_channels) with the coherent combine as
// the GNU Radio scheduler would: factory -> setters -> one work() call with all 3 outputs connected.  Reads a test vector
// file written by tests/test_gpu_focus.py and writes the outputs next to it; the Python test compares them with the
// Python block's.
//   in file (little endian): u32 m, n, nsamples, resolution, nfft, chan_first, chan_count, taper, nwindows, peak_mode,
//                            exclusion, source_rule, estimator, focus_first, focus_count (0: the whole grid);
//                            f64 loading, centre_frequency, sample_rate, positions[m][2] (metres); in[nwindows * nsamples * 2] f32
//   out file: angle, level [nwindows][n] f32; spectrum [nwindows][resolution] f32; bins [nwindows][n] i32;
//             counts [nwindows] i32; focusing errors [chan_count] f64
#include <baz_music_doa_channels.h>

#include <cstdio>
#include <stdexcept>
#include <vector>

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[15];
    double dv[3];
    if (fread(hdr, 4, 15, f) != 15 || fread(dv, 8, 3, f) != 3) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], F = hdr[4], first = hdr[5], C = hdr[6], W = hdr[8];
    const int taper = (int)hdr[7];
    std::vector<double> p(2 * (size_t)m);
    std::vector<float> in((size_t)W * ns * 2);
    if (fread(p.data(), 8, p.size(), f) != p.size() || fread(in.data(), 4, in.size(), f) != in.size()) return 2;
    fclose(f);
    std::vector<std::vector<double> > pos(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i)
        for (int c = 0; c < 2; ++c) pos[i][c] = p[2 * i + c];

    baz_music_doa_channels_sptr blk = baz_make_music_doa_channels(m, n, ns, K, F, first, C, taper, 2, pos, 1.0, dv[1], dv[2]);
    if (blk->output_signature()->sizeof_stream_item(1) != (int)(n * 4) || blk->output_signature()->sizeof_stream_item(2) != (int)(K * 4))
        return 4;
    // an empty sector is refused with the library convention (std::invalid_argument)
    bool threw = false;
    try { blk->set_focusing(0, 0); } catch (const std::invalid_argument &) { threw = true; }
    if (!threw) { fprintf(stderr, "expected invalid_argument for an empty focusing sector\n"); return 3; }
    if (hdr[14]) blk->set_focusing(hdr[13], hdr[14]);
    blk->set_estimator((int)hdr[12], dv[0]);
    blk->set_source_rule((int)hdr[11]);
    blk->set_peak_mode((int)hdr[9], hdr[10]);

    std::vector<float> ang((size_t)W * n), lvl((size_t)W * n), spec((size_t)W * K);
    gr_vector_const_void_star ins(1, in.data());
    gr_vector_void_star outs;
    outs.push_back(ang.data()); outs.push_back(lvl.data()); outs.push_back(spec.data());
    if (blk->work((int)W, ins, outs) != (int)W) return 5;
    const std::vector<int> bins = blk->last_bins(), counts = blk->last_counts();
    const std::vector<double> err = blk->focusing_error();
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 2;
    fwrite(ang.data(), 4, ang.size(), o);
    fwrite(lvl.data(), 4, lvl.size(), o);
    fwrite(spec.data(), 4, spec.size(), o);
    fwrite(bins.data(), 4, bins.size(), o);
    fwrite(counts.data(), 4, counts.size(), o);
    fwrite(err.data(), 8, err.size(), o);
    fclose(o);
    return 0;
}
