"""Angle tracking on the device (music_b200_set_tracking, the *_tracks entries, music_track.cuh): off is off; against the
literal restatement (tests/track_oracle.py) fed the device's own angles, bins and CRB under every kind of peak mode;
the assignment under stress; split invariance; the reset rules and refusals; sources crossing against the truth; the
blocks."""
import ctypes
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200._capi import MusicB200Error
from gr_baz_b200.music_doa_azel import music_doa_azel
from gr_baz_b200.music_doa_channels import music_doa_channels

import crb_oracle as co
import gpu_harness as gh
import helpers
import track_oracle as to
from helpers import LAM

pytestmark = pytest.mark.gpu

SNAPS = 64


def tracks_device(blk, x, stream=None, std=True, fill=gh.SENTINEL):
    """one process_device_tracks (az-el: process_azel_device_tracks) call on the windows x asking for every output (the
    CRB too when `std`): numpy outputs, launches"""
    W, n = x.shape[0], blk.n
    T = blk._tracking[1]
    azel = isinstance(blk, music_doa_azel)
    t = lambda shape, dt: torch.full(shape, fill, dtype=dt, device=gh.DEV)
    o = {"levels": t((W, n), torch.float32), "bins": t((W, n), torch.int32), "counts": t((W,), torch.int32),
         "slot_track": t((W, n), torch.int32), "track_ids": t((W, T), torch.int32),
         "track_state": t((W, T, 6 if azel else 3), torch.float32)}
    if std:
        o["std"] = t((W, n, 3) if azel else (W, n), torch.float32)
    p = lambda k: o[k].data_ptr() if k in o else None
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    st = gh.stream() if stream is None else stream.cuda_stream
    l0 = blk.launch_count()
    if azel:
        o.update(azimuth=t((W, n), torch.float32), elevation=t((W, n), torch.float32))
        blk.process_device_tracks(d_in.data_ptr(), W, p("azimuth"), p("elevation"), p("slot_track"), p("levels"), None, p("bins"),
                                  p("counts"), p("std"), p("track_ids"), p("track_state"), stream=st)
    else:
        o.update(angles=t((W, n), torch.float32))
        blk.process_device_tracks(d_in.data_ptr(), W, p("angles"), p("slot_track"), p("levels"), None, p("bins"), p("counts"),
                                  None, None, p("std"), p("track_ids"), p("track_state"), stream=st)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}, blk.launch_count() - l0


def oracle_run(params, got, azel=False, tr=None):
    tr = tr or to.Tracker(params, azel=azel)
    ang = got["azimuth"] if azel else got["angles"]
    crb = got.get("std") if params.variance == to.CRB else None
    out = tr.run(ang, got["bins"], got.get("elevation"), crb)
    return tr, out


def assert_matches(blk, got, tr, out, ctx):
    st, ids, state = out
    assert np.array_equal(got["slot_track"], st), ctx
    assert np.array_equal(got["track_ids"], ids), ctx
    g, r = got["track_state"].astype(np.float64), state.astype(np.float64)
    ulp = np.spacing(np.abs(state)).astype(np.float64)
    bad = np.abs(g - r) > ulp
    assert not bad.any(), (ctx, np.argwhere(bad)[:5], g[bad][:5], r[bad][:5])
    rows, sstate, nxt = blk.tracks()
    orows, ostate, onxt = tr.snapshot()
    assert np.array_equal(rows, orows) and nxt == onxt, ctx
    scale = np.maximum(np.abs(ostate).max(1, keepdims=True), 1e-300)
    err = np.abs(sstate - ostate) / scale
    assert err.max() <= 1e-12, (ctx, err.max())


def moving_windows(pos_wl, W, seed, tracks, snr_db=20.0):
    th = [[(a + r * w) % 360.0 for a, r in tracks] for w in range(W)]
    return helpers.angle_windows(pos_wl, th, False, W, seed, snr_db=snr_db, snaps=SNAPS)


def _ura(rows, cols, step=0.5):
    return np.array([[c * step, r * step, 0.0] for r in range(rows) for c in range(cols)])


def azel_windows(pos_wl, paths, W, seed, snr_db=20.0):
    """sources on straight (az, el) paths: paths = [((az0, el0), (daz, del)), ...] per window"""
    rng = np.random.default_rng(seed)
    m = pos_wl.shape[0]
    X = (rng.standard_normal((W, SNAPS, m)) + 1j * rng.standard_normal((W, SNAPS, m))) / math.sqrt(2.0)
    w = np.arange(W)
    for (az0, el0), (daz, dele) in paths:
        A = np.stack([co.steer_azel(pos_wl, 1.0, math.radians(az0 + daz * k), math.radians(el0 + dele * k))[0] for k in w])
        s = 10 ** (snr_db / 20) * (rng.standard_normal((W, SNAPS)) + 1j * rng.standard_normal((W, SNAPS))) / math.sqrt(2.0)
        X = X + s[..., None] * A[:, None, :]
    return X.reshape(W, SNAPS * m).astype(np.complex64)


def set_tracking(blk, params):
    blk.set_tracking(["off", "fixed", "crb"][params.variance], params.q, params.rate_std0, params.floor_deg, params.crb_scale,
                     params.gate, params.confirm_hits, params.confirm_window, params.max_misses, params.max_tracks)


CRB_P = to.Params(variance=to.CRB, q=1e-3, rate_std0=1.0, floor_deg=0.05, crb_scale=2.0, gate=16.0, confirm_hits=3,
                  confirm_window=4, max_misses=4, max_tracks=6)
FIXED_P = to.Params(variance=to.FIXED, q=1e-3, rate_std0=1.0, floor_deg=0.7, gate=16.0, confirm_hits=2, confirm_window=3,
                    max_misses=3, max_tracks=6)

ONE_D = [  # (name, geometry, n, block settings, params)
    ("uca_local_newton", "uca", 2, dict(mode="local_maxima", refine=True), CRB_P),
    ("ula_roots", "x", 2, dict(mode="roots"), CRB_P),
    ("ula_esprit", "x", 2, dict(mode="esprit"), CRB_P),
    ("uca_dml", "uca", 2, dict(mode="dml"), CRB_P),
    ("uca_mvdr", "uca", 2, dict(mode="local_maxima", est=("mvdr", 0.01)), FIXED_P),
    ("set_table_fixed", "uca", 2, dict(mode="local_maxima"), FIXED_P),
]


@pytest.mark.parametrize("name,geom,n,settings,params", ONE_D, ids=[c[0] for c in ONE_D])
def test_against_oracle_1d(name, geom, n, settings, params):
    m, W = 8, 300
    pos_wl = helpers.array_wl(geom, m)
    paths = [(40.0, 0.2), (140.0, -0.15)] if geom == "x" else [(60.0, 0.3), (200.0, -0.2)]
    x = moving_windows(pos_wl, W, 11, paths)
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos_wl * LAM, **settings)
    if name == "set_table_fixed":
        blk.set_array_response(helpers.table_wl(pos_wl))
    set_tracking(blk, params)
    tr = None
    for w0, w1 in ((0, 120), (120, W)):  # the carry across two calls
        got, _ = tracks_device(blk, x[w0:w1], std=params.variance == to.CRB)
        tr, out = oracle_run(params, got, tr=tr)
        assert_matches(blk, got, tr, out, (name, w0))
    assert (got["track_ids"] >= 0).sum(1).max() >= 2, name


@pytest.mark.parametrize("kind", ["esprit2d", "grid_local"])
def test_against_oracle_azel(kind):
    pos_wl = _ura(4, 4)
    m, n, W = 16, 2, 240
    x = azel_windows(pos_wl, [((40.0, 30.0), (0.3, 0.05)), ((200.0, 55.0), (-0.2, -0.05))], W, 13)
    blk = music_doa_azel(m, n, m * SNAPS, 72, 19, (0.0, 90.0), pos_wl * LAM, LAM)
    if kind == "esprit2d":
        blk.set_peak_mode("esprit", 0)
    else:
        blk.set_peak_mode("local_maxima", 2)
        blk.set_refine(True)
    set_tracking(blk, CRB_P)
    got, _ = tracks_device(blk, x)
    tr, out = oracle_run(CRB_P, got, azel=True)
    assert_matches(blk, got, tr, out, kind)
    assert (got["track_ids"] >= 0).sum(1).max() >= 2


def test_assignment_stress():
    # noise only, 15 slots, 32 rows, a wide gate: ambiguous clusters in every window
    m, n, W = 16, 15, 200
    rng = np.random.default_rng(17)
    x = ((rng.standard_normal((W, SNAPS * m)) + 1j * rng.standard_normal((W, SNAPS * m))) / math.sqrt(2)).astype(np.complex64)
    blk = gh.make_block(m, n, SNAPS, K=720, pos=helpers.array_wl("uca", m) * LAM, mode="local_maxima")
    p = to.Params(variance=to.FIXED, q=1.0, rate_std0=3.0, floor_deg=5.0, gate=30.0, confirm_hits=2, confirm_window=4,
                  max_misses=2, max_tracks=32)
    set_tracking(blk, p)
    got, _ = tracks_device(blk, x, std=False)
    tr, out = oracle_run(p, got)
    assert_matches(blk, got, tr, out, "stress")
    assert (got["slot_track"] >= 0).mean() > 0.5


def _split_block(K=3600):
    pos = helpers.array_wl("uca", 4) * LAM
    blk = gh.make_block(4, 2, 16, K=K, pos=pos, mode="local_maxima", refine=True)
    set_tracking(blk, FIXED_P)
    return blk


def test_split_invariance():
    W = 30000
    pos_wl = helpers.array_wl("uca", 4)
    rng = np.random.default_rng(3)
    th = [[(50 + 0.01 * w) % 360, (250 - 0.02 * w) % 360] for w in range(W)]
    x = helpers.angle_windows(pos_wl, th, False, W, 19, snr_db=15.0, snaps=16)
    keys = ("angles", "bins", "slot_track", "track_ids", "track_state")
    blk = _split_block()
    one, launches = tracks_device(blk, x, std=False)
    ref = {k: one[k].tobytes() for k in keys}
    ref_tracks = blk.tracks()
    assert launches > 8  # several sub-batches
    # many device calls of random sizes
    blk = _split_block()
    parts, w0 = [], 0
    while w0 < W:
        k = int(min(W - w0, rng.integers(1, 4000)))
        parts.append(tracks_device(blk, x[w0:w0 + k], std=False)[0])
        w0 += k
    for k in keys:
        assert np.concatenate([p[k] for p in parts]).tobytes() == ref[k], k
    # two caller streams alternating
    blk = _split_block()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    parts = [tracks_device(blk, x[w0:w0 + 5000], stream=streams[i % 2], std=False)[0] for i, w0 in enumerate(range(0, W, 5000))]
    for k in keys:
        assert np.concatenate([p[k] for p in parts]).tobytes() == ref[k], k
    assert [np.array_equal(a, b) for a, b in zip(blk.tracks(), ref_tracks)] == [True] * 3
    # the host entry (each call's chunks on the two staging streams), through work() in three calls of 2000 windows
    blk = _split_block()
    got = {k: [] for k in ("angles", "slot_track", "track_ids", "track_state")}
    for w0 in range(0, 6000, 2000):
        a = np.zeros((2000, 2), np.float32)
        blk.work(2000, [np.ascontiguousarray(x[w0:w0 + 2000])], [a])
        got["angles"].append(a)
        for k, v in zip(("slot_track", "track_ids", "track_state"), blk.last_tracks()):
            got[k].append(v)
    for k, v in got.items():
        assert np.concatenate(v).tobytes() == one[k][:6000].tobytes(), k


def test_off_is_off():
    m, n, W = 8, 2, 64
    pos_wl = helpers.array_wl("uca", m)
    x = moving_windows(pos_wl, W, 5, [(60.0, 0.3), (200.0, -0.2)])
    outs = ("levels", "bins", "counts")
    plain = gh.make_block(m, n, SNAPS, K=360, pos=pos_wl * LAM, mode="local_maxima", refine=True)
    ref, ref_l = gh.device_call(plain, x, outs)
    ref_host = gh.host_call(plain, x)
    ref_ex, ref_exl = gh.device_call(plain, x, ("levels", "bins", "R"))
    for variance in ("off", "fixed", "crb"):
        blk = gh.make_block(m, n, SNAPS, K=360, pos=pos_wl * LAM, mode="local_maxima", refine=True)
        blk.set_tracking(variance)
        got, l = gh.device_call(blk, x, outs)
        assert l == ref_l and all(got[k].tobytes() == ref[k].tobytes() for k in ("angles",) + outs), variance
        if variance == "off":
            h = gh.host_call(blk, x)
            assert blk.last_tracks() is None
            assert all(h[k].tobytes() == ref_host[k].tobytes() for k in ("angles", "levels", "bins", "counts"))
        else:
            # the carry is untouched by the other entries
            assert blk.tracks()[2] == 0
            # the tracks call's other outputs equal the unfused call's
            tr, _ = tracks_device(blk, x)
            for k in ("angles", "levels", "bins"):
                assert tr[k].tobytes() == ref_ex[k].tobytes(), (variance, k)
        blk.close()


def _reset_pair(setter, resets):
    """call A, `setter`, call B on one block; B against a block that ran A and B without the setter (kept carry) or
    B alone (reset carry)"""
    m, n = 8, 2
    pos_wl = helpers.array_wl("uca", m)
    x = moving_windows(pos_wl, 80, 23, [(60.0, 0.3), (200.0, -0.2)])
    mk = lambda: gh.make_block(m, n, SNAPS, K=360, pos=pos_wl * LAM, mode="local_maxima", refine=True)
    blk = mk()
    set_tracking(blk, FIXED_P)
    tracks_device(blk, x[:40], std=False)
    nxt = blk.tracks()[2]
    assert nxt >= 2
    setter(blk, pos_wl)
    got, _ = tracks_device(blk, x[40:], std=False)
    ref = mk()
    set_tracking(ref, FIXED_P)
    if not resets:
        tracks_device(ref, x[:40], std=False)
    want, _ = tracks_device(ref, x[40:], std=False)
    for k in ("slot_track", "track_ids", "track_state"):
        assert got[k].tobytes() == want[k].tobytes(), k
    if resets:
        assert got["slot_track"][got["slot_track"] >= 0].min() == 0


def _no_windows(blk):
    """a tracks call with nwindows = 0 (its outputs are never written)"""
    out = torch.zeros(16, dtype=torch.int32, device=gh.DEV)
    blk.process_device_tracks(0, 0, out.data_ptr(), out.data_ptr())


RESETS = {
    "reset_tracks": (lambda b, p: b.reset_tracks(), True),
    "set_tracking_same": (lambda b, p: set_tracking(b, FIXED_P), True),
    "set_array_geometry": (lambda b, p: b.set_array_geometry(p * LAM, LAM), True),
    "set_peak_mode": (lambda b, p: b.set_peak_mode("local_maxima", 0), False),
    "set_estimator": (lambda b, p: b.set_estimator("music"), False),
    "set_source_rule": (lambda b, p: b.set_source_rule("fixed"), False),
    "set_refine": (lambda b, p: b.set_refine(True), False),
    "set_beamformer": (lambda b, p: b.set_beamformer("off"), False),
    "set_integration": (lambda b, p: b.set_integration(0.0), False),
    "set_calibration": (lambda b, p: b.set_calibration(None), False),
    "zero_windows": (lambda b, p: _no_windows(b), False),
}


@pytest.mark.parametrize("name", sorted(RESETS))
def test_reset_rules(name):
    setter, resets = RESETS[name]
    _reset_pair(setter, resets)


def test_set_table_resets():
    m, n = 8, 2
    pos_wl = helpers.array_wl("uca", m)
    x = moving_windows(pos_wl, 60, 29, [(60.0, 0.3), (200.0, -0.2)])
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos_wl * LAM, mode="local_maxima")
    set_tracking(blk, FIXED_P)
    tracks_device(blk, x[:30], std=False)
    assert blk.tracks()[2] >= 2
    blk.set_array_response(helpers.table_wl(pos_wl))
    assert blk.tracks()[2] == 0 and np.all(blk.tracks()[0][:, 0] == -1)
    got, _ = tracks_device(blk, x[30:], std=False)
    assert got["slot_track"][got["slot_track"] >= 0].min() == 0


def _next_id(L, h):
    """the handle's next track id, read without the rows (this test sets the tracker through the C ABI, so the block's own
    record of the row count is not current)"""
    nxt = ctypes.c_uint32(0)
    assert L.music_b200_get_tracks(h, None, None, ctypes.byref(nxt)) == _capi.OK
    return nxt.value


def test_refusals_and_untouched_carry():
    m, n, W = 8, 2, 8
    pos = helpers.array_wl("uca", m) * LAM
    x = moving_windows(pos / LAM, W, 3, [(60.0, 0.3), (200.0, -0.2)])
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima")
    L, h = blk._lib, blk._h
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    ang = torch.zeros((W, n), dtype=torch.float32, device=gh.DEV)
    buf = torch.zeros((W * 32 * 6 + 8,), dtype=torch.int32, device=gh.DEV)
    b = buf.data_ptr()
    call = lambda hh, st, ids=None, state=None, std=None: L.music_b200_process_device_tracks(
        hh, d_in.data_ptr(), W, ang.data_ptr(), None, None, None, None, None, None, std, st, ids, state, None)
    assert call(h, b) == _capi.EINVAL  # tracking off
    good = FIXED_P.args()
    bad = [dict(variance=3), dict(q=-1.0), dict(q=float("nan")), dict(rate_std0=-1.0), dict(floor_deg=float("inf")),
           dict(gate=0.0), dict(gate=float("inf")), dict(floor_deg=0.0), dict(variance=to.CRB, crb_scale=0.0),
           dict(confirm_hits=0), dict(confirm_hits=4, confirm_window=3), dict(confirm_window=65), dict(max_misses=0),
           dict(max_tracks=0), dict(max_tracks=33)]
    for kw in bad:
        p = to.Params(**{**FIXED_P.__dict__, **kw})
        assert L.music_b200_set_tracking(h, *p.args()) == _capi.EINVAL, kw
    assert call(h, b) == _capi.EINVAL  # the old setting (off) is kept
    assert L.music_b200_set_tracking(h, *good) == _capi.OK
    assert call(h, None) == _capi.EINVAL
    assert call(h, b, ids=b) == _capi.EINVAL
    assert call(h, b + 2) == _capi.EINVAL
    assert call(h, b, ids=b, state=b + 2) == _capi.EINVAL
    assert _next_id(L, h) == 0  # refused calls left the carry untouched
    assert call(h, b) == _capi.OK
    torch.cuda.synchronize()
    nxt = _next_id(L, h)
    assert nxt >= 1
    assert L.music_b200_process_azel_device_tracks(h, d_in.data_ptr(), W, ang.data_ptr(), ang.data_ptr(), None, None, None, None,
                                                   None, b, None, None, None) == _capi.EINVAL
    assert _next_id(L, h) == nxt
    # CRB variance needs a geometric table: at the setter and at the call
    blk.set_array_response(helpers.table_wl(pos / LAM))
    crb = to.Params(**{**FIXED_P.__dict__, "variance": to.CRB})
    assert L.music_b200_set_tracking(h, *crb.args()) == _capi.EINVAL
    blk.set_array_geometry(pos, LAM)
    assert L.music_b200_set_tracking(h, *crb.args()) == _capi.OK
    blk.set_array_response(helpers.table_wl(pos / LAM))
    assert call(h, b) == _capi.EINVAL
    assert "geometry" in L.music_b200_last_error(h).decode()
    # the reverse: a 1-D entry on an az-el handle
    az = music_doa_azel(m, n, m * SNAPS, 36, 4, (0.0, 45.0), np.c_[pos, np.zeros(m)], LAM)
    assert L.music_b200_set_tracking(az._h, *good) == _capi.OK
    assert call(az._h, b) == _capi.EINVAL
    # multi-device and channel handles refuse the setting
    mb = gh.make_block(m, n, SNAPS, K=360, pos=pos, devices=[0])
    assert L.music_b200_set_tracking(mb._h, *good) == _capi.EINVAL
    assert L.music_b200_reset_tracks(mb._h) == _capi.EINVAL
    ch = music_doa_channels(m, n, m * SNAPS, 90, 16, (14, 5), "hann", "separate", np.asarray(pos / LAM), 0.3, 400e6, 56e6)
    with pytest.raises(MusicB200Error):
        ch.set_tracking("fixed")
    assert L.music_b200_set_tracking(ch._h, *good) == _capi.EINVAL


def _follow(truth, state, ids, wins):
    """per truth column k and window in wins: the id of the confirmed track nearest in angle"""
    out = np.full((len(wins), truth.shape[1]), -1)
    for a, w in enumerate(wins):
        live = ids[w] >= 0
        if not live.any():
            continue
        for k in range(truth.shape[1]):
            d = np.abs(to.wrap180(state[w, live, 0].astype(np.float64) - truth[w, k]))
            out[a, k] = ids[w, live][np.argmin(d)]
    return out


@pytest.mark.parametrize("azel", [False, True])
def test_crossing_against_truth(azel):
    W = 400 if azel else 280  # the line array's sources stay inside (20, 160) degrees, away from end-fire
    w = np.arange(W)
    p = to.Params(variance=to.CRB, q=1e-5, rate_std0=1.0, floor_deg=0.02, crb_scale=1.5, gate=16.0, confirm_hits=3,
                  confirm_window=5, max_misses=12, max_tracks=8)
    # gridless modes: two measurements near the crossing rather than one merged grid peak and a noise peak elsewhere
    if azel:
        pos_wl = _ura(4, 4)
        paths = [((40.0, 30.0), (0.25, 0.05)), ((140.0, 50.0), (-0.25, -0.05))]  # meet at (90, 40) at window 200
        x = azel_windows(pos_wl, paths, W, 41)
        blk = music_doa_azel(16, 2, 16 * SNAPS, 72, 19, (0.0, 90.0), pos_wl * LAM, LAM)
        blk.set_peak_mode("esprit", 0)
        truth = np.stack([p0[0] + d[0] * w for p0, d in paths], 1)
    else:
        pos_wl = helpers.array_wl("x", 8)
        tracks = [(50.0, 0.35), (130.0, -0.25)]  # cross at window 133
        x = moving_windows(pos_wl, W, 41, tracks)
        blk = gh.make_block(8, 2, SNAPS, K=360, pos=pos_wl * LAM, mode="esprit")
        truth = np.stack([a + r * w for a, r in tracks], 1)
    set_tracking(blk, p)
    got, _ = tracks_device(blk, x)
    ids, state = got["track_ids"], got["track_state"]
    sep = np.abs(to.wrap180(truth[:, 0] - truth[:, 1]))
    wc = int(np.argmin(sep))
    clear = (sep > 15.0) & (w >= 10)
    before, after = w[clear & (w < wc)], w[clear & (w > wc)]
    assert np.all((ids[before] >= 0).sum(1) == 2) and np.all((ids[after] >= 0).sum(1) == 2)
    fb, fa = _follow(truth, state, ids, before), _follow(truth, state, ids, after)
    for k in range(2):
        assert len(set(fb[:, k])) == 1 and len(set(fa[:, k])) == 1, (k, set(fb[:, k]), set(fa[:, k]))
        assert fb[0, k] == fa[0, k]
    assert fb[0, 0] != fb[0, 1]
    # track error against raw measurement error outside the crossing
    outside = np.concatenate([before, after])
    trk_err, raw_err, nees = [], [], []  # nees: the angle's squared error over its reported variance
    ang = got["azimuth"] if azel else got["angles"]
    for wi in outside:
        for k in range(2):
            r = np.flatnonzero(ids[wi] == fb[0, k])[0]
            e = to.wrap180(float(state[wi, r, 0]) - truth[wi, k])
            trk_err.append(e)
            raw_err.append(np.min(np.abs(to.wrap180(ang[wi].astype(np.float64) - truth[wi, k]))))
            nees.append(e * e / float(state[wi, r, 2 if not azel else 4]) ** 2)
    rms_trk, rms_raw = np.sqrt(np.mean(np.square(trk_err))), np.sqrt(np.mean(np.square(raw_err)))
    print("crossing azel=%s: rms track %.4f deg, rms raw %.4f deg, mean normalised angle error^2 %.3f"
          % (azel, rms_trk, rms_raw, float(np.mean(nees))))
    assert rms_trk < rms_raw


def test_python_work_equals_device_call():
    m, n, W = 8, 2, 90
    pos_wl = helpers.array_wl("uca", m)
    x = moving_windows(pos_wl, W, 7, [(60.0, 0.3), (200.0, -0.2)])
    mk = lambda: gh.make_block(m, n, SNAPS, K=360, pos=pos_wl * LAM, mode="local_maxima", refine=True, beamformer=("das", 0.0))
    ref_blk = mk()
    set_tracking(ref_blk, CRB_P)
    ref, _ = tracks_device(ref_blk, x)
    blk = mk()
    set_tracking(blk, CRB_P)
    blk.set_crb(True)
    parts = []
    for w0 in range(0, W, 30):
        blk.work(30, [x[w0:w0 + 30]], [np.zeros((30, n), np.float32)])
        parts.append(tuple(a.copy() for a in blk.last_tracks()) + (blk.last_crb().copy(),))
    for i, k in enumerate(("slot_track", "track_ids", "track_state", "std")):
        assert np.concatenate([p[i] for p in parts]).tobytes() == ref[k].tobytes(), k


def test_cpp_block():
    m, n, W = 8, 2, 60
    pos = helpers.array_wl("uca", m) * LAM
    x = moving_windows(pos / LAM, W, 8, [(60.0, 0.3), (200.0, -0.2)])
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima", refine=True)
    set_tracking(blk, CRB_P)
    ref, _ = tracks_device(blk, x)
    T = CRB_P.max_tracks
    header = struct.pack("<6I", m, n, m * SNAPS, 360, W, T) + struct.pack("<6d", LAM, CRB_P.q, CRB_P.rate_std0, CRB_P.floor_deg,
                                                                        CRB_P.crb_scale, CRB_P.gate)
    header += struct.pack("<3I", CRB_P.confirm_hits, CRB_P.confirm_window, CRB_P.max_misses)
    layout = [("slot_track", np.int32, W * n), ("track_ids", np.int32, W * T), ("track_state", np.float32, W * T * 3)]
    out = gh.run_cpp_block("test_block_tracks", header, [pos.astype(np.float64), x], layout)
    for k, _, _ in layout:
        assert out[k].tobytes() == ref[k].tobytes(), k
