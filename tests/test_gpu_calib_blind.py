"""GPU: receiver self-calibration without a known source (music_b200_calib_blind_*) against its fp64 definition
(tests/calib_blind_oracle.py), end to end against the truth, its refusals and the multi-device handle."""
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200.music_doa_azel import music_doa_azel

import calib_blind_oracle as cb
import gpu_harness as gh
from helpers import LAM, array_wl, circ, corrupt, random_gains, ula
from test_gpu_calibration import windows

pytestmark = pytest.mark.gpu


def moving_windows(pos, S, seg, d, seed, snaps, snr_db=20.0):
    """S segments of `seg` windows each, d sources per segment at directions spread over the circle (segment s near
    360 s / S), unit noise"""
    rng = np.random.default_rng(seed)
    degs = []
    for s in range(S):
        t0 = 360.0 * s / S + rng.uniform(0.0, 360.0 / S)
        degs += [[(t0 + 360.0 * j / (d + 1) + rng.uniform(0.0, 20.0)) % 360.0 for j in range(d)]] * seg
    return windows(pos, degs, seed + 1, snaps, snr_db)


def segment_covariances(blk, x, seg):
    """the device's raw per-window R (process_device_ex d_R, the same covariance kernels), averaged per segment in fp64"""
    R = gh.device_call(blk, x, ("R",))[0]["R"]
    return cb.segments(R, seg)


# ---- 1. the solve against the oracle on the device's own R ------------------------------------------------------------
CASES = [(4, 1, 16, 2), (8, 1, 16, 2), (8, 2, 16, 1), (5, 2, 12, 2)]  # (m, d, S, windows per segment)


@pytest.mark.parametrize("m,d,S,seg", CASES)
def test_solve_matches_oracle(m, d, S, seg):
    """the same winning start (up to starts tied in J to 1e-9), the same final bins (except where the oracle's P is tied to 1e-9 between the two),
    gains within 1e-8, the misfit to 1e-6 relative, polish iterations within one; PHASE gives the unit-modulus phases"""
    K, snaps = 720, 256
    pos = array_wl("uca", m)
    rng = np.random.default_rng(300 + 10 * m + d)
    g = random_gains(rng, m)
    x = corrupt(moving_windows(pos, S, seg, d, 310 + m + d, snaps), g)
    blk = gh.make_block(m, 1, snaps, K, pos=pos)
    got, ang, st = blk.calibrate_blind(x, d, seg, starts=32, seed=7)
    table = blk.array_response_c64().astype(np.complex128)
    Rs = segment_covariances(blk, x, seg)
    ref, ang_ref, mis_ref, used_ref, win_ref, Js, bins_ref = cb.solve(Rs, table, d, cb.GAIN_PHASE, 32, 7, pos, trace=True)
    # the same winner, unless the two starts reached the same point and their J differ by rounding alone
    assert st["start"] == win_ref or abs(Js[st["start"]] - Js[win_ref]) <= 1e-9 * Js[win_ref] + 1e-15, (st, win_ref)
    assert abs(st["polish"] - used_ref) <= 1
    assert np.max(np.abs(got - ref)) <= 1e-8, (got, ref)
    assert abs(st["misfit"] - mis_ref) <= 1e-6 * mis_ref + 1e-15
    bins = np.where(np.isnan(ang), -1, np.rint(np.nan_to_num(ang) * K / 360.0)).astype(np.int64)
    if not np.array_equal(bins, bins_ref):
        P = cb.spectra(cb.noise_bases(Rs, cb.magnitudes(Rs), d), got / np.abs(got), table)
        for s, i in zip(*np.nonzero(bins != bins_ref)):
            a, b = P[s, bins[s, i]], P[s, bins_ref[s, i]]
            assert abs(a - b) <= 1e-9 * max(a, b), (s, i, bins[s, i], bins_ref[s, i], a, b)
    # the segments are kept; PHASE reports phi alone
    ph, _, _ = blk.calib_blind_solve(d, "phase", 32, 7)
    assert np.max(np.abs(ph - ref / np.abs(ref))) <= 1e-8 and np.allclose(np.abs(ph), 1.0, atol=1e-15)
    blk.close()


def test_split_invariance_and_device_entry():
    """segments accumulated through the device entry in uneven calls (whole segments each) solve to the same bits as
    one host call"""
    m, d, S, seg, K, snaps = 8, 1, 12, 3, 720, 256
    pos = array_wl("uca", m)
    g = random_gains(np.random.default_rng(41), m)
    x = corrupt(moving_windows(pos, S, seg, d, 42, snaps), g)
    blk = gh.make_block(m, 1, snaps, K, pos=pos)
    ga, aa, sa = blk.calibrate_blind(x, d, seg)
    blk.calib_blind_reset()
    d_in = torch.from_numpy(x.view(np.float32).reshape(-1)).to(gh.DEV)
    step = m * snaps * 2
    for lo, hi in ((0, 3), (3, 15), (15, 36)):
        blk.calib_blind_accumulate_device(d_in[lo * step:].data_ptr(), hi - lo, seg, stream=gh.stream())
    gb, ab, sb = blk.calib_blind_solve(d)
    assert np.array_equal(ga, gb) and np.array_equal(aa, ab, equal_nan=True) and sa == sb
    blk.close()


# ---- 2. end to end: calibrate on unknown emitters, then MUSIC on fresh windows ----------------------------------------
def test_doa_restored():
    """gains from windows of an emitter moving around the array (its directions unknown to the solve) correct the DOA:
    fresh windows of a source on a grid bin come back within one grid step, while the uncorrected handle misses"""
    m, K, snaps, S, seg = 8, 360, 256, 16, 2
    pos = array_wl("uca", m)
    rng = np.random.default_rng(501)
    g = random_gains(rng, m)
    blk = gh.make_block(m, 1, snaps, K, pos=pos)
    gains, _, st = blk.calibrate_blind(corrupt(moving_windows(pos, S, seg, 1, 502, snaps), g), 1, seg)
    assert st["misfit"] < 0.05, st
    truth = rng.integers(0, K, 24) * (360.0 / K)
    xr = corrupt(windows(pos, [[t] for t in truth], 503, snaps), g)

    def errors():
        ang = np.zeros((len(truth), 1), np.float32)
        blk.work(len(truth), [xr], [ang])
        return circ(ang[:, 0], truth)

    raw = errors()
    blk.set_calibration(gains)
    fixed = errors()
    assert np.max(fixed) <= 360.0 / K + 1e-4, fixed
    assert np.max(raw) > 360.0 / K, raw
    blk.close()


# ---- 3. refusals ---------------------------------------------------------------------------------------------------------
def test_refusals():
    L = _capi.load()
    EINVAL = _capi.EINVAL
    m, K, snaps = 4, 360, 64
    pos = array_wl("uca", m)
    blk = gh.make_block(m, 1, snaps, K, pos=pos)
    x = windows(pos, [[10.0 * w] for w in range(8)], 5, snaps)
    out, ang, st = np.full(2 * m, -3.0), np.full(8, -3.0), np.full(4, -3.0)

    def solve(h, d=1, kind=2, starts=32):
        return L.music_b200_calib_blind_solve(h._h, d, kind, starts, 0, out.ctypes.data, ang.ctypes.data, st.ctypes.data)

    blk.calib_blind_reset()
    assert solve(blk) == EINVAL  # no segments
    # accumulate: segment 0, a window count that is not a multiple of the segment
    assert L.music_b200_calib_blind_accumulate_host(blk._h, x.ctypes.data, 8, 0) == EINVAL
    assert L.music_b200_calib_blind_accumulate_host(blk._h, x.ctypes.data, 7, 2) == EINVAL
    blk.calib_blind_accumulate(x, 1)
    for d in (0, m - 1):
        assert solve(blk, d=d) == EINVAL
    for starts in (0, 257):
        assert solve(blk, starts=starts) == EINVAL
    assert solve(blk, kind=3) == EINVAL
    assert np.all(out == -3.0) and np.all(ang == -3.0) and np.all(st == -3.0)  # nothing written
    assert solve(blk, starts=1) == _capi.OK
    # more than MUSIC_B200_CALIB_MAX_SEGMENTS segments
    big = np.repeat(x[:1], 1024 - 7, axis=0)
    assert L.music_b200_calib_blind_accumulate_host(blk._h, big.ctypes.data, len(big), 1) == EINVAL
    blk.calib_blind_accumulate(big[:-1], 1)
    assert L.music_b200_calib_blind_accumulate_host(blk._h, x.ctypes.data, 1, 1) == EINVAL
    # non-finite data, a dead element
    blk.calib_blind_reset()
    bad = x.copy()
    bad[3, 5] = np.nan
    blk.calib_blind_accumulate(bad, 2)
    out[:] = -3.0
    assert solve(blk) == EINVAL and np.all(out == -3.0)
    blk.calib_blind_reset()
    blk.calib_blind_accumulate(corrupt(x, np.r_[1.0, 0.0, 1.0, 1.0]), 2)
    assert solve(blk) == EINVAL
    # a set_table() table
    blk.calib_blind_reset()
    blk.calib_blind_accumulate(x, 2)
    blk.set_array_response(np.ones((K, m), np.complex64))
    assert solve(blk) == EINVAL
    blk.close()
    # collinear elements, m < 3
    for p in (ula(4, "oblique"), ula(2, "x")):
        h = gh.make_block(len(p), 1, snaps, K, pos=p)
        h.calib_blind_accumulate(windows(p, [[20.0]] * 2, 6, snaps), 1)
        assert solve(h) == EINVAL
        h.close()
    # an az-el handle
    p3 = np.c_[pos, np.zeros(m)]
    az = music_doa_azel(m, 1, m * snaps, 36, 3, (0.0, 40.0), p3, LAM)
    assert L.music_b200_calib_blind_reset(az._h) == EINVAL
    assert L.music_b200_calib_blind_accumulate_host(az._h, x.ctypes.data, 8, 1) == EINVAL
    assert solve(az) == EINVAL
    az.close()


# ---- 4. multi-device handle -----------------------------------------------------------------------------------------------
def test_multi_device():
    """devices[0] serves the segments and the solve: the same bits as a single-device handle"""
    m, d, S, seg, K, snaps = 8, 1, 8, 2, 360, 256
    pos = array_wl("uca", m)
    x = corrupt(moving_windows(pos, S, seg, d, 61, snaps), random_gains(np.random.default_rng(60), m))
    one = gh.make_block(m, 1, snaps, K, pos=pos)
    multi = gh.make_block(m, 1, snaps, K, pos=pos, devices=list(range(torch.cuda.device_count())))
    ra, rb = one.calibrate_blind(x, d, seg), multi.calibrate_blind(x, d, seg)
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1], equal_nan=True) and ra[2] == rb[2]
    one.close()
    multi.close()


def test_default_path_unchanged():
    """a handle that has run a self-calibration (and holds its segments) processes windows with the same launches and
    the same bytes as one that never did"""
    m, K, snaps = 8, 360, 256
    pos = array_wl("uca", m)
    x = windows(pos, [[30.0 * w] for w in range(8)], 71, snaps)
    a, b = gh.make_block(m, 1, snaps, K, pos=pos), gh.make_block(m, 1, snaps, K, pos=pos)
    b.calibrate_blind(moving_windows(pos, 8, 1, 1, 72, snaps), 1, 1)
    ra, la = gh.device_call(a, x, ("levels", "bins"))
    rb, lb = gh.device_call(b, x, ("levels", "bins"))
    assert la == lb and all(ra[k].tobytes() == rb[k].tobytes() for k in ra)
    a.close()
    b.close()


# ---- 5. C++ block ----------------------------------------------------------------------------------------------------------
def test_cpp_block():
    """calibrate_blind() armed on the C++ block, the calibration items over work() calls that split segments: the gains it
    applies and its misfit equal the Python block's calibrate_blind on the same items, and its later DOA outputs equal
    the Python block's with those gains"""
    m, n, K, snaps, S, seg, chunk, W = 8, 1, 360, 256, 12, 2, 5, 10
    pos = array_wl("uca", m)
    rng = np.random.default_rng(811)
    g = random_gains(rng, m)
    cal = corrupt(moving_windows(pos, S, seg, 1, 812, snaps), g)
    x = corrupt(windows(pos, [[t] for t in rng.uniform(0, 360, W)], 813, snaps), g)
    c = gh.run_cpp_block("test_block_calib_blind", struct.pack("<10I", m, n, m * snaps, K, S * seg, W, 1, 2, seg, chunk) +
                         struct.pack("<d", LAM), [np.ascontiguousarray(pos, np.float64), cal, x],
                         [("g", np.complex128, m), ("misfit", np.float64, 1), ("a", np.float32, W * n), ("b", np.int32, W * n)])
    blk = gh.make_block(m, n, snaps, K, pos=pos)
    pg, _, st = blk.calibrate_blind(cal, 1, seg)
    assert np.array_equal(c["g"], pg) and c["misfit"][0] == st["misfit"]
    blk.set_calibration(pg)
    ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    blk.work(W, [x], [ang, lvl])
    assert np.array_equal(c["a"], ang.ravel()) and np.array_equal(c["b"], blk.last_bins().ravel())
    blk.close()
