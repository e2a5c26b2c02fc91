// test_block_tracks.cc - exercises baz_music_doa::set_tracking() as a flowgraph would: factory -> set_array_geometry() ->
// local-maximum peaks with refinement -> tracking under CRB variance -> two work() calls, the tracks carried from the
// first to the second.  Reads a test vector file written by tests/test_gpu_tracks.py and writes the results next to it;
// the Python test compares them with one device call over all windows.
//   in file (little endian): u32 m, n, nsamples, resolution, nwin, max_tracks; f64 wavelength, q, rate_std0, floor_deg,
//                            crb_scale, gate; u32 confirm_hits, confirm_window, max_misses; positions[m][2] f64;
//                            in[nwin * nsamples * 2] f32
//   out file: slot_track [nwin][n] i32; track_ids [nwin][max_tracks] i32; track_state [nwin][max_tracks][3] f32
#include <baz_music_doa.h>

#include <algorithm>
#include <cstdio>
#include <vector>

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s in.bin out.bin\n", argv[0]); return 2; }
    FILE *f = fopen(argv[1], "rb");
    if (!f) return 2;
    unsigned hdr[6], cfg[3];
    double d[6];
    if (fread(hdr, 4, 6, f) != 6 || fread(d, 8, 6, f) != 6 || fread(cfg, 4, 3, f) != 3) return 2;
    const unsigned m = hdr[0], n = hdr[1], ns = hdr[2], K = hdr[3], W = hdr[4], T = hdr[5];
    std::vector<double> pos((size_t)m * 2);
    std::vector<float> in((size_t)W * ns * 2);
    if (fread(pos.data(), 8, pos.size(), f) != pos.size() || fread(in.data(), 4, in.size(), f) != in.size()) return 2;
    fclose(f);
    array_response_t table(K, antenna_response_t(m, gr_complex(1.0f, 0.0f)));
    baz_music_doa_sptr blk = baz_make_music_doa(m, n, ns, table, K);
    std::vector<std::vector<double> > geo(m, std::vector<double>(2));
    for (unsigned i = 0; i < m; ++i) { geo[i][0] = pos[2 * i]; geo[i][1] = pos[2 * i + 1]; }
    blk->set_array_geometry(geo, d[0]);
    blk->set_peak_mode(1, 0);
    blk->set_refine(true);
    blk->set_tracking(2 /* MUSIC_B200_TRACK_CRB */, d[1], d[2], d[3], d[4], d[5], cfg[0], cfg[1], cfg[2], T);

    std::vector<float> ang((size_t)W * n), lvl((size_t)W * n), state((size_t)W * T * 3);
    std::vector<int> slot((size_t)W * n), ids((size_t)W * T);
    const unsigned half = W / 2;
    for (unsigned w0 = 0; w0 < W; w0 += half) {
        const unsigned cnt = std::min(half, W - w0);
        gr_vector_const_void_star ins(1, in.data() + (size_t)w0 * ns * 2);
        gr_vector_void_star outs;
        outs.push_back(ang.data() + (size_t)w0 * n);
        outs.push_back(lvl.data() + (size_t)w0 * n);
        if (blk->work((int)cnt, ins, outs) != (int)cnt) return 5;
        if (blk->last_slot_track().size() != (size_t)cnt * n || blk->last_track_ids().size() != (size_t)cnt * T ||
            blk->last_track_state().size() != (size_t)cnt * T * 3)
            return 6;
        std::copy(blk->last_slot_track().begin(), blk->last_slot_track().end(), slot.begin() + (size_t)w0 * n);
        std::copy(blk->last_track_ids().begin(), blk->last_track_ids().end(), ids.begin() + (size_t)w0 * T);
        std::copy(blk->last_track_state().begin(), blk->last_track_state().end(), state.begin() + (size_t)w0 * T * 3);
    }
    FILE *o = fopen(argv[2], "wb");
    if (!o) return 3;
    fwrite(slot.data(), 4, slot.size(), o);
    fwrite(ids.data(), 4, ids.size(), o);
    fwrite(state.data(), 4, state.size(), o);
    fclose(o);
    return 0;
}
