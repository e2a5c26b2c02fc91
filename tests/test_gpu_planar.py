"""GPU: planar antenna streams with windows formed by pointer arithmetic (music_b200_process_planar_*,
SURVEY.md section 8(f) rank 2) against the oracle run on the windows the reference flowgraph would build on
the CPU: x_w(r, c) = stream_r[w * hop + c] (interleave /root/reference/lib/baz_interleaver.cc:152-229,
overlap /root/reference/lib/baz_overlap.cc:107-129, reshape /root/reference/lib/baz_music_doa.cc:82-84)."""
import numpy as np
import pytest
import torch

from gr_baz_b200 import synth
from gr_baz_b200._capi import MusicB200Error
from gr_baz_b200.music_doa import music_doa
from oracle import c_oracle as co

import helpers
from helpers import form_windows, streams_for

pytestmark = pytest.mark.gpu

P_RTOL = 1e-5


CASES = [  # base config, overrides, hop (None = N), windows
    (1, {}, None, 9), (1, {}, 256, 21), (1, {}, 1, 40), (1, {}, 1500, 5),
    (2, {"snapshots": 1024, "resolution": 720}, 512, 33),
    (4, {"snapshots": 512}, 128, 17), (4, {"snapshots": 512, "n": 3}, None, 8),
    (5, {"snapshots": 512, "resolution": 720}, 384, 9),
    (1, {"m": 6, "geometry": "uca", "n": 2}, 100, 12), (1, {"m": 5, "geometry": "ula_y"}, None, 7),
]


@pytest.mark.parametrize("base,over,hop,W", CASES)
def test_planar_host_matches_oracle_on_formed_windows(base, over, hop, W):
    cfg = synth.config(base, **over)
    N = cfg["snapshots"]
    hop_ = N if hop is None else hop
    table = helpers.table_for(cfg)
    streams = streams_for(cfg, 1234 + base, (W - 1) * hop_ + N)
    x = form_windows(streams, hop_, W, N)
    ref = co.work_batch(x, cfg["m"], cfg["n"], table, want_spectrum=True)
    blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], table.tolist(), cfg["resolution"])
    ang = np.full((W, cfg["n"]), -7, np.float32)
    lvl = np.full((W, cfg["n"]), -7, np.float32)
    spec = np.zeros((W, cfg["resolution"]), np.float32)
    assert blk.work_planar(W, streams, [ang, lvl, spec], hop=hop) == W
    assert np.array_equal(blk.last_bins(), ref["bins"])
    assert np.array_equal(ang, ref["angles"])
    assert helpers.rel_err(lvl, ref["levels"]) <= P_RTOL
    assert helpers.rel_err(spec, ref["spectrum"]) <= P_RTOL
    # and the same bins as the interleaved entry on the copied windows
    ang2 = np.zeros_like(ang)
    assert blk.work(W, [x], [ang2]) == W and np.array_equal(ang2, ang)


def test_planar_device_entry_many_windows_with_overlap():
    """device-resident streams, 50 % overlap, enough windows to take several chunks of the scan"""
    cfg = synth.config(2, snapshots=1024)
    N, hop, W = 1024, 512, 1500
    table = helpers.table_for(cfg)
    streams = streams_for(cfg, 77, (W - 1) * hop + N)
    x = form_windows(streams, hop, W, N)
    ref = co.work_batch(x, cfg["m"], cfg["n"], table)
    blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], table.tolist(), cfg["resolution"])
    dev = torch.device("cuda:0")
    d_streams = [torch.from_numpy(s.view(np.float32)).to(dev) for s in streams]
    d_ang = torch.zeros(W, 1, dtype=torch.float32, device=dev)
    d_lvl = torch.zeros(W, 1, dtype=torch.float32, device=dev)
    d_bins = torch.zeros(W, 1, dtype=torch.int32, device=dev)
    blk.process_planar_device([t.data_ptr() for t in d_streams], hop, W, d_ang.data_ptr(), d_lvl.data_ptr(), None,
                              d_bins.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ties = helpers.assert_bins_equal_up_to_exact_ties(d_bins.cpu().numpy(), ref)
    if ties == 0:
        assert np.array_equal(d_ang.cpu().numpy(), ref["angles"])
    assert helpers.rel_err(d_lvl.cpu().numpy(), ref["levels"]) <= P_RTOL
    # unaligned stream start (odd snapshot offset: 8-byte but not 16-byte aligned) gives the shifted windows
    blk.process_planar_device([t.data_ptr() + 8 for t in d_streams], hop, W - 1, d_ang.data_ptr(), d_lvl.data_ptr(), None,
                              d_bins.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    x1 = form_windows([s[1:] for s in streams], hop, W - 1, N)
    ref1 = co.work_batch(x1, cfg["m"], cfg["n"], table)
    helpers.assert_bins_equal_up_to_exact_ties(d_bins.cpu().numpy()[:W - 1], ref1)


@pytest.mark.parametrize("N,hop,W", [(1000, 1000, 300), (1000, 500, 300), (1024, 2, 260), (1000, 334, 120), (1000, 333, 120), (130, 64, 1100)])
def test_planar_fused_path_m4(N, hop, W):
    """M = 4, n = 1, peak outputs only: planar streams go through the fused persistent kernel (four 1 KiB bulk copies
    per stage) when hop and N are even, else through cov_planar_kernel; both must match the oracle.  N = 1000 / 130
    leave a partial last stage; W > 8 * 132 (eight covariance warps per H100 SM) exercises the dynamic tickets."""
    cfg = synth.config(2, snapshots=N, resolution=720)
    table = helpers.table_for(cfg)
    streams = streams_for(cfg, 4321 + hop, (W - 1) * hop + N)
    x = form_windows(streams, hop, W, N)
    ref = co.work_batch(x, cfg["m"], cfg["n"], table)
    blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], table.tolist(), cfg["resolution"])
    ang = np.full((W, 1), -7, np.float32)
    lvl = np.full((W, 1), -7, np.float32)
    l0 = blk.launch_count()
    assert blk.work_planar(W, streams, [ang, lvl], hop=hop) == W
    launches = blk.launch_count() - l0
    fusable = hop % 2 == 0 and N % 2 == 0
    assert (launches <= 2) if fusable else (launches >= 3)  # one fused launch per host chunk vs cov + eig + scan
    helpers.assert_bins_equal_up_to_exact_ties(blk.last_bins(), ref)
    ok = np.all(blk.last_bins() == ref["bins"], axis=1)
    assert np.array_equal(ang[ok], ref["angles"][ok])
    assert helpers.rel_err(lvl[ok], ref["levels"][ok]) <= P_RTOL


def test_planar_device_entry_uca_overlap_is_bit_exact():
    """same as above on a circular array (no mirror symmetry, hence no exact ties): bins bit-exact"""
    cfg = synth.config(4, snapshots=512, resolution=1800)
    N, hop, W = 512, 128, 900
    table = helpers.table_for(cfg)
    streams = streams_for(cfg, 78, (W - 1) * hop + N)
    x = form_windows(streams, hop, W, N)
    ref = co.work_batch(x, cfg["m"], cfg["n"], table)
    blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], table.tolist(), cfg["resolution"])
    dev = torch.device("cuda:0")
    d_streams = [torch.from_numpy(s.view(np.float32)).to(dev) for s in streams]
    d_ang = torch.zeros(W, 1, dtype=torch.float32, device=dev)
    d_bins = torch.zeros(W, 1, dtype=torch.int32, device=dev)
    blk.process_planar_device([t.data_ptr() for t in d_streams], hop, W, d_ang.data_ptr(), None, None,
                              d_bins.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_bins.cpu().numpy(), ref["bins"])
    assert np.array_equal(d_ang.cpu().numpy(), ref["angles"])


def test_planar_argument_errors():
    cfg = synth.config(1)
    table = helpers.table_for(cfg)
    blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], table.tolist(), cfg["resolution"])
    streams = streams_for(cfg, 5, 2 * cfg["snapshots"])
    ang = np.zeros((2, 1), np.float32)
    with pytest.raises(ValueError):
        blk.work_planar(2, streams[:-1], [ang])
    with pytest.raises(ValueError):
        blk.work_planar(3, streams, [np.zeros((3, 1), np.float32)])  # streams too short for 3 windows
    with pytest.raises(ValueError):
        blk.work_planar(2, streams, [ang], hop=0)
    with pytest.raises(MusicB200Error):
        blk.process_planar_device([0] * cfg["m"], 16, 1, ang.ctypes.data)
    with pytest.raises(MusicB200Error):
        blk.process_planar_device([4] * cfg["m"], 16, 1, ang.ctypes.data)  # misaligned
    assert blk.work_planar(0, streams, [ang]) == 0
