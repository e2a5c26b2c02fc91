"""The stochastic CRB of every filled slot on the device (music_b200_process_*_crb, music_crb.cuh): against the literal
fp64 restatement (tests/crb_oracle.py) on the device's own covariance, angles and bins under every peak mode that takes a
geometric table; the other outputs unchanged; integration and calibration; the entries and splits; az-el; the spread of
the GPU's own estimates against the reported bound; the refusals and the blocks."""
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
import test_crb_oracle as tco
from helpers import LAM

pytestmark = pytest.mark.gpu

SNAPS = 256
RTOL = 1e-6
COND_MAX = 1e8  # rtol holds where the oracle's Fisher matrix has cond(F) <= COND_MAX
CLEAR = 4.0  # NaN / finite must agree where the oracle's deciding check is this far from its threshold


def crb_device(blk, x, beams=False, fill=gh.SENTINEL):
    """one process_device_crb (az-el: process_azel_device_crb) call on the windows x: every output plus the bound,
    (numpy outputs, launches)"""
    W, n = x.shape[0], blk.n
    azel = isinstance(blk, music_doa_azel)
    t = lambda shape, dt: torch.full(shape, fill, dtype=dt, device=gh.DEV)
    o = {"levels": t((W, n), torch.float32), "bins": t((W, n), torch.int32), "counts": t((W,), torch.int32)}
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    l0 = blk.launch_count()
    if azel:
        o.update(azimuth=t((W, n), torch.float32), elevation=t((W, n), torch.float32), crb=t((W, n, 3), torch.float32))
        blk.process_device_crb(d_in.data_ptr(), W, o["azimuth"].data_ptr(), o["elevation"].data_ptr(), o["crb"].data_ptr(),
                               o["levels"].data_ptr(), None, o["bins"].data_ptr(), o["counts"].data_ptr(), stream=gh.stream())
    else:
        o.update(angles=t((W, n), torch.float32), std=t((W, n), torch.float32))
        if beams:
            o.update(weights=t((W, n, blk.m, 2), torch.float64), beams=t((W, n, blk.nsamples // blk.m, 2), torch.float32))
        p = lambda k: o[k].data_ptr() if k in o else None
        blk.process_device_crb(d_in.data_ptr(), W, p("angles"), p("std"), p("levels"), None, p("bins"), p("counts"),
                               p("weights"), p("beams"), stream=gh.stream())
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    for k in ("weights", "beams"):
        if k in out:
            out[k] = out[k][..., 0] + 1j * out[k][..., 1]
    if "beams" in out:
        out["beams"] = out["beams"].astype(np.complex64)
    return out, blk.launch_count() - l0


def assert_matches_oracle(got, ref, info, ctx):
    """got / ref (W, n) or (W, n, 3): rtol where the oracle's F is well conditioned, NaN-ness where its deciding check is
    clear of the threshold"""
    checked = 0
    for w, r in enumerate(info):
        if r is None:
            assert np.all(got[w] == 0), (ctx, w, got[w])
            continue
        clear = r["margin"] >= CLEAR or r["margin"] <= 1.0 / CLEAR
        if clear:
            assert np.array_equal(np.isnan(got[w]), np.isnan(ref[w])), (ctx, w, got[w], ref[w], r["margin"])
        if r["ok"] and r["cond_F"] <= COND_MAX and not np.any(np.isnan(got[w])):
            np.testing.assert_allclose(got[w], ref[w], rtol=RTOL, atol=0, err_msg="%s window %d" % (ctx, w))
            checked += 1
    return checked


def two_source_windows(pos_wl, W, seed, lo=20.0, hi=160.0, snr_db=20.0, snaps=SNAPS):
    rng = np.random.default_rng(seed)
    th = [sorted(rng.uniform(lo, hi, 2)) for _ in range(W)]
    for t in th:
        if t[1] - t[0] < 25.0:
            t[1] = t[0] + 25.0
    return helpers.angle_windows(pos_wl, th, False, W, seed, snr_db=snr_db, snaps=snaps)


def oracle_for(blk, x, pos, N=SNAPS, R=None):
    """the oracle's bound on the device's own R (process_device_ex), angles and bins of the same windows"""
    ex, _ = gh.device_call(blk, x, ("levels", "bins", "R"))
    R = ex["R"] if R is None else R
    return co.crb_outputs(R, ex["angles"], ex["bins"], N, pos, LAM)


MODES = [("local_maxima", "uca", 2), ("top_bins", "uca", 1), ("roots", "x", 2), ("esprit", "x", 2), ("dml", "uca", 2),
         ("manifold", "uca", 2)]


@pytest.mark.parametrize("m", [3, 4, 5, 8, 12, 16])
@pytest.mark.parametrize("mode,geom,n", MODES)
def test_against_oracle_every_peak_mode(m, mode, geom, n):
    grid = mode in ("local_maxima", "top_bins")
    pos_wl = helpers.array_wl(geom, m)
    pos = pos_wl * LAM
    x = two_source_windows(pos_wl, 24, 100 + m)
    checked = 0
    for est in (("music", 0.0), ("mvdr", 0.01), ("bartlett", 0.0)) if grid else (None,):
        for refine in (False, True) if grid else (False,):
            blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, est=est, mode=mode, refine=refine)
            ref, info = oracle_for(blk, x, pos)
            got, _ = crb_device(blk, x)
            checked += assert_matches_oracle(got["std"], ref, info, (m, mode, est, refine))
            blk.close()
    assert checked > 0


@pytest.mark.parametrize("beams", [False, True])
def test_other_outputs_unchanged(beams):
    m, n = 8, 2
    pos_wl = helpers.array_wl("uca", m)
    x = two_source_windows(pos_wl, 40, 7)
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos_wl * LAM, mode="local_maxima", refine=True,
                        beamformer=("lcmv", 0.01) if beams else None)
    if beams:
        ref, _ = gh.device_call(blk, x, ("levels", "bins", "counts", "weights", "beams"))
    else:
        ref, _ = gh.device_call(blk, x, ("levels", "bins", "R"))
    got, launches = crb_device(blk, x, beams=beams)
    for k in ("angles", "levels", "bins") + (("counts", "weights", "beams") if beams else ()):
        assert got[k].tobytes() == ref[k].tobytes(), k
    assert launches >= 1


def test_integration_uses_neff_per_window():
    m, n, alpha = 8, 2, 0.9
    pos_wl = helpers.array_wl("uca", m)
    pos = pos_wl * LAM
    x = helpers.angle_windows(pos_wl, [[50.0, 130.0]] * 48, False, 48, 21, snr_db=0.0, snaps=SNAPS)
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima", refine=True)
    blk.set_integration(alpha)
    ex, _ = gh.device_call(blk, x, ("levels", "bins", "R"))  # Rbar from a fresh carry
    blk.reset_integration()
    got, _ = crb_device(blk, x)
    j = np.arange(x.shape[0], dtype=np.float64)
    c = (1.0 - alpha ** (j + 1)) / (1.0 - alpha)
    q = (1.0 - alpha ** (2 * (j + 1))) / (1.0 - alpha ** 2)
    ref, info = co.crb_outputs(ex["R"], ex["angles"], ex["bins"], SNAPS * c * c / q, pos, LAM)
    assert assert_matches_oracle(got["std"], ref, info, "integration") > 0
    # the bound shrinks as N_eff grows
    assert np.nanmedian(got["std"][-8:]) < 0.5 * np.nanmedian(got["std"][:1])


def test_calibration_uses_corrected_R():
    m, n = 8, 2
    pos_wl = helpers.array_wl("uca", m)
    pos = pos_wl * LAM
    rng = np.random.default_rng(4)
    g = helpers.random_gains(rng, m)
    x = helpers.corrupt(two_source_windows(pos_wl, 32, 22), g)
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima", refine=True, calibration=g)
    ref, info = oracle_for(blk, x, pos)
    got, _ = crb_device(blk, x)
    assert assert_matches_oracle(got["std"], ref, info, "calibration") > 0


def test_entries_and_splits_agree():
    m, n = 8, 2
    pos_wl = helpers.array_wl("uca", m)
    pos = pos_wl * LAM
    x = two_source_windows(pos_wl, 60, 23)
    make = lambda devices=None: gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima", refine=True, devices=devices)
    blk = make()
    dev, _ = crb_device(blk, x)
    a, b = crb_device(blk, x[:25])[0], crb_device(blk, x[25:])[0]
    assert np.concatenate([a["std"], b["std"]]).tobytes() == dev["std"].tobytes()
    blk.set_crb(True)
    ang = np.zeros((60, n), np.float32)
    blk.work(60, [x], [ang])
    assert blk.last_crb().tobytes() == dev["std"].tobytes()
    assert ang.tobytes() == dev["angles"].tobytes()
    for devices in ([0], list(range(torch.cuda.device_count()))):
        mb = make(devices=devices)
        mb.set_crb(True)
        mb.work(60, [x], [np.zeros((60, n), np.float32)])
        assert mb.last_crb().tobytes() == dev["std"].tobytes(), devices
        assert crb_device(mb, x)[0]["std"].tobytes() == dev["std"].tobytes()
        mb.close()


def _ura(rows, cols, step=0.5):
    return np.array([[c * step, r * step, 0.0] for r in range(rows) for c in range(cols)])


def azel_windows(pos_wl, pairs, W, seed, snr_db=20.0, snaps=SNAPS):
    rng = np.random.default_rng(seed)
    m = pos_wl.shape[0]
    X = (rng.standard_normal((W, snaps, m)) + 1j * rng.standard_normal((W, snaps, m))) / math.sqrt(2.0)
    for az, el in pairs:
        a = co.steer_azel(pos_wl, 1.0, math.radians(az), math.radians(el))[0]
        s = 10 ** (snr_db / 20) * (rng.standard_normal((W, snaps)) + 1j * rng.standard_normal((W, snaps))) / math.sqrt(2.0)
        X = X + s[..., None] * a
    return X.reshape(W, snaps * m).astype(np.complex64)


@pytest.mark.parametrize("kind", ["grid_newton", "esprit2d", "random3d"])
def test_azel_against_oracle(kind):
    if kind == "random3d":
        pos_wl = np.random.default_rng(9).uniform(-0.6, 0.6, (8, 3))
    else:
        pos_wl = _ura(4, 4)
    m, n = pos_wl.shape[0], 2
    pos = pos_wl * LAM
    x = azel_windows(pos_wl, [(40.0, 30.0), (150.0, 50.0)], 24, 31)
    blk = music_doa_azel(m, n, m * SNAPS, 72, 19, (0.0, 90.0), pos, LAM)
    if kind == "esprit2d":
        blk.set_peak_mode("esprit", 0)
    else:
        blk.set_peak_mode("local_maxima", 2)
        blk.set_refine(True)
    got, _ = crb_device(blk, x)
    # the covariance of a 1-D handle of the same shape is the same kernel on the same windows
    R = gh.device_call(gh.make_block(m, 1, SNAPS, K=360), x, ("R",))[0]["R"]
    ref, info = co.crb_outputs(R, got["azimuth"], got["bins"], SNAPS, pos, LAM, elev=got["elevation"])
    assert assert_matches_oracle(got["crb"], ref, info, kind) > 0
    blk.set_crb(True)
    outs = [np.zeros((24, n), np.float32) for _ in range(3)]
    blk.work(24, [x], outs)
    assert blk.last_crb().tobytes() == got["crb"].tobytes()


@pytest.mark.parametrize("theta", [0.0, 180.0])
def test_ula_end_fire_is_nan(theta):
    # sin(pi) is 1.2e-16 in fp64, not 0: both end-fire directions must fail by the derivative-scale test, not only 0
    m = 8
    pos_wl = helpers.array_wl("x", m)
    pos = pos_wl * LAM
    x = helpers.angle_windows(pos_wl, [[theta]] * 16, False, 16, 41, snr_db=30.0, snaps=SNAPS)
    blk = gh.make_block(m, 1, SNAPS, K=360, pos=pos)
    got, _ = crb_device(blk, x)
    at = got["angles"][:, 0] == theta
    assert at.sum() > 0
    assert np.all(np.isnan(got["std"][at, 0]))
    ref, info = oracle_for(blk, x, pos)
    assert_matches_oracle(got["std"], ref, info, ("end-fire", theta))


def test_azel_planar_at_zero_elevation_is_nan():
    pos_wl = _ura(3, 3)
    pos = pos_wl * LAM
    x = azel_windows(pos_wl, [(70.0, 0.0)], 16, 32, snr_db=30.0)
    blk = music_doa_azel(9, 1, 9 * SNAPS, 72, 13, (0.0, 60.0), pos, LAM)
    got, _ = crb_device(blk, x)
    at0 = got["elevation"][:, 0] == 0.0
    assert at0.sum() > 0
    assert np.all(np.isnan(got["crb"][at0, 0]))
    assert np.all(np.isfinite(got["crb"][~at0, 0]))


def _stat_windows(pos_wl, truth, W, seed, snr_db=20.0):
    rng = np.random.default_rng(seed)
    A = np.stack([co.steer_1d(pos_wl, 1.0, math.radians(t))[0] for t in truth], 1)
    X = co.sample_windows(rng, A, 10 ** (snr_db / 10) * np.eye(len(truth)), 1.0, SNAPS, W)
    return np.ascontiguousarray(np.swapaxes(X, 1, 2).reshape(W, -1))


@pytest.mark.parametrize("mode,geom,refine,alpha", [("esprit", "x", False, 0.0), ("roots", "x", False, 0.0),
                                                    ("manifold", "uca", False, 0.0), ("local_maxima", "uca", True, 0.0),
                                                    ("esprit", "x", False, 0.9)])
def test_gpu_estimates_spread_at_the_bound(mode, geom, refine, alpha):
    m, W = 8, 300
    truth = np.array([60.0, 80.0]) if geom == "x" else np.array([60.0, 100.0])
    pos_wl = helpers.array_wl(geom, m)
    x = _stat_windows(pos_wl, truth, W, 77)
    blk = gh.make_block(m, 2, SNAPS, K=360, pos=pos_wl * LAM, mode=mode, refine=refine)
    if alpha:
        blk.set_integration(alpha)
    got, _ = crb_device(blk, x)
    skip = 40 if alpha else 0  # the first windows of an integration have not reached N_eff's limit
    ang, std = got["angles"][skip:], got["std"][skip:]
    order = np.argsort(ang, axis=1)
    ang, std = np.take_along_axis(ang, order, 1), np.take_along_axis(std, order, 1)
    assert np.all(np.abs(ang - truth) < 5.0)
    ratio = np.std(ang.astype(np.float64) - truth, axis=0) / np.median(std, axis=0)
    lo, hi = (tco.RATIO_LO_INTEG, tco.RATIO_HI_INTEG) if alpha else (tco.RATIO_LO, tco.RATIO_HI)
    print("crb ratio", mode, refine, alpha, ratio)
    assert np.all(ratio >= lo) and np.all(ratio <= hi), ratio


def test_refusals():
    m, n, W = 8, 2, 4
    pos = helpers.array_wl("uca", m) * LAM
    x = two_source_windows(pos / LAM, W, 3)
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima")
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    buf = torch.zeros((W * n * 3 + 4,), dtype=torch.float32, device=gh.DEV)
    ang = torch.zeros((W, n), dtype=torch.float32, device=gh.DEV)
    L = blk._lib
    call = lambda h, std, wts=None: L.music_b200_process_device_crb(h, d_in.data_ptr(), W, ang.data_ptr(), None, None, None, None,
                                                                     wts, None, std, None)
    assert call(blk._h, None) == _capi.EINVAL
    assert call(blk._h, buf.data_ptr() + 2) == _capi.EINVAL  # misaligned
    wts = torch.zeros((W, n, m, 2), dtype=torch.float64, device=gh.DEV)
    assert call(blk._h, buf.data_ptr(), wts.data_ptr()) == _capi.EINVAL  # no beamformer
    assert L.music_b200_process_host_crb(blk._h, x.ctypes.data, W, np.zeros((W, n), np.float32).ctypes.data, None, None, None,
                                         None, None, None, None) == _capi.EINVAL
    assert L.music_b200_process_azel_device_crb(blk._h, d_in.data_ptr(), W, ang.data_ptr(), ang.data_ptr(), None, None, None, None,
                                                buf.data_ptr(), None) == _capi.EINVAL
    assert call(blk._h, buf.data_ptr()) == _capi.OK
    # a table from set_table(): no geometry
    blk.set_array_response(helpers.table_wl(pos / LAM))
    assert call(blk._h, buf.data_ptr()) == _capi.EINVAL
    assert "geometry" in L.music_b200_last_error(blk._h).decode()
    blk.set_crb(True)
    with pytest.raises(MusicB200Error):
        blk.work(W, [x], [np.zeros((W, n), np.float32)])
    # the reverse: a 1-D entry on an az-el handle
    az = music_doa_azel(m, n, m * SNAPS, 36, 4, (0.0, 45.0), np.c_[pos, np.zeros(m)], LAM)
    assert call(az._h, buf.data_ptr()) == _capi.EINVAL
    assert L.music_b200_process_host_crb(az._h, x.ctypes.data, W, np.zeros((W, n), np.float32).ctypes.data, None, None, None, None,
                                         None, None, np.zeros((W, n), np.float32).ctypes.data) == _capi.EINVAL
    # channel handles, COHERENT included
    for combine in ("separate", "coherent"):
        ch = music_doa_channels(m, n, m * SNAPS, 90, 16, (14, 5), "hann", combine, np.asarray(pos / LAM), 0.3, 400e6, 56e6)
        with pytest.raises(ValueError):
            ch.set_crb(True)
        assert not ch.crb() and ch.last_crb() is None
        assert call(ch._h, buf.data_ptr()) == _capi.EINVAL
        assert L.music_b200_process_azel_device_crb(ch._h, d_in.data_ptr(), W, ang.data_ptr(), ang.data_ptr(), None, None, None,
                                                    None, buf.data_ptr(), None) == _capi.EINVAL
        ch.close()


class _CountingLib:
    """the block's ctypes library, counting the process_* calls made through it"""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if not name.startswith("music_b200_process"):
            return f

        def wrapped(*a):
            self.calls.append(name)
            return f(*a)
        return wrapped


@pytest.mark.parametrize("beamformer", [None, ("das", 0.0)])
def test_python_block_one_call_per_work(beamformer):
    m, n, W = 8, 2, 30
    pos = helpers.array_wl("uca", m) * LAM
    x = two_source_windows(pos / LAM, W, 5)
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima", refine=True, beamformer=beamformer)
    ref, _ = crb_device(blk, x, beams=beamformer is not None)
    blk.set_crb(True)
    blk._lib = _CountingLib(blk._lib)
    ang = np.zeros((W, n), np.float32)
    blk.work(W, [x], [ang])
    assert blk._lib.calls == ["music_b200_process_host_crb"]
    assert blk.last_crb().tobytes() == ref["std"].tobytes()
    if beamformer:
        assert blk.last_beams().tobytes() == ref["beams"].tobytes()
    blk.set_crb(False)
    blk.work(W, [x], [ang])
    assert blk.last_crb() is None


@pytest.mark.parametrize("rule", [0, 1])
def test_cpp_block(rule):
    # two work() calls under integration: a block that made two library calls per work() would advance the carry twice
    m, n, W, alpha = 8, 2, 30, 0.8
    pos = helpers.array_wl("uca", m) * LAM
    x = two_source_windows(pos / LAM, W, 6)
    blk = gh.make_block(m, n, SNAPS, K=360, pos=pos, mode="local_maxima", refine=True, beamformer=("das", 0.0) if rule else None)
    blk.set_integration(alpha)
    blk.set_crb(True)
    ang, crb, beams = np.zeros((W, n), np.float32), [], []
    for w0 in (0, W // 2):
        blk.work(W // 2, [x[w0:w0 + W // 2]], [ang[w0:w0 + W // 2], np.zeros((W // 2, n), np.float32)])
        crb.append(blk.last_crb().copy())
        if rule:
            beams.append(blk.last_beams().copy())
    header = struct.pack("<6I", m, n, m * SNAPS, 360, W, rule) + struct.pack("<2d", alpha, LAM)
    layout = [("angles", np.float32, W * n), ("crb", np.float32, W * n)]
    if rule:
        layout.append(("beams", np.complex64, W * n * SNAPS))
    out = gh.run_cpp_block("test_block_crb", header, [pos.astype(np.float64), x], layout)
    assert out["angles"].tobytes() == ang.tobytes()
    assert out["crb"].tobytes() == np.concatenate(crb).tobytes()
    if rule:
        assert out["beams"].tobytes() == np.concatenate(beams).tobytes()
