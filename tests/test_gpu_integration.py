"""Covariance integration across windows on the device (music_b200_set_integration): off is off, the integrated
covariance against the sequential fp64 recurrence (tests/integration_oracle.py) on the raw covariances of an alpha = 0
handle, split and stream invariance, the reset rules, every stage downstream reading Rbar, the refusals, the weak-source
benefit and the C++ block."""
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200._capi import MusicB200Error
from gr_baz_b200.music_doa_azel import music_doa_azel
from gr_baz_b200.music_doa_channels import music_doa_channels

import azel_oracle as ao
import beams_oracle as bo
import estimator_oracle as eo
import gpu_harness as gh
import helpers
import integration_oracle as io
import source_count_oracle as sco
from helpers import LAM

pytestmark = pytest.mark.gpu

WORST = {}  # worst observed max |Rbar_gpu - Rbar_ref| / max |Rbar_ref| per case (printed with -s)


def noise_windows(m, snaps, W, seed, theta=None, pos=None, snr_db=0.0):
    """complex64 [W][m * snaps]: unit white noise, plus one source at theta (degrees) of a geometry in metres"""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((W, snaps, m)) + 1j * rng.standard_normal((W, snaps, m))) / math.sqrt(2.0)
    if theta is not None:
        a = helpers.steering_wl(pos / LAM, theta)
        s = 10.0 ** (snr_db / 20.0) * (rng.standard_normal((W, snaps)) + 1j * rng.standard_normal((W, snaps))) / math.sqrt(2.0)
        x = x + s[..., None] * a
    return x.reshape(W, snaps * m).astype(np.complex64)


def raw_R(make, x):
    blk = make()
    out, _ = gh.device_call(blk, x, ("R",))
    blk.close()
    return out["R"]


def check_R(got, ref, case):
    err = io.rel_err(got, ref)
    WORST[case] = float(np.max(err))
    print("integration %s: worst relative error %.3g" % (case, WORST[case]))
    assert np.all(err <= io.REL_BOUND), (case, float(np.max(err)))


def music_P(R, table, n):
    a = np.asarray(table, np.complex128)
    _, V = np.linalg.eigh(R)
    G = V[:, : R.shape[0] - n]
    return 1.0 / np.sum(np.abs(a.conj() @ G) ** 2, axis=1)


def assert_bins_close(got, P_rows, n, rel=1e-9):
    """the device's bins against the oracle's top-n picks on the same fp64 P, up to ties within `rel`"""
    for w, P in enumerate(P_rows):
        ref = eo.picks(P, n, len(P))[2]
        for g, r in zip(got[w], ref):
            assert g == r or abs(P[g] - P[r]) <= rel * P[r], (w, g, r)


# ---- off is off ----
@pytest.mark.parametrize("m,snaps", [(4, 256), (8, 256)])
def test_off_is_off_on_the_fused_paths(m, snaps):
    pos = helpers.positions("uca", m)
    x = noise_windows(m, snaps, 64, 11, theta=40.0, pos=pos, snr_db=10.0)
    table = helpers.table_wl(pos / LAM)
    fresh = gh.make_block(m, 1, snaps, table=table)
    ref, l_ref = gh.device_call(fresh, x, ("levels", "bins"))
    ref_host = gh.host_call(fresh, x)
    rt = gh.make_block(m, 1, snaps, table=table)
    rt.set_integration(0.0)
    a, l_a = gh.device_call(rt, x, ("levels", "bins"))
    rt.set_integration(0.9)
    rt.set_integration(0.0)
    b, l_b = gh.device_call(rt, x, ("levels", "bins"))
    h = gh.host_call(rt, x)
    assert l_ref == 1 and l_a == l_ref and l_b == l_ref  # one fused launch each
    for k in ref:
        assert np.array_equal(a[k], ref[k]) and np.array_equal(b[k], ref[k]), k
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(h[k], ref_host[k]), k
    on = gh.make_block(m, 1, snaps, table=table)
    on.set_integration(0.5)
    _, l_on = gh.device_call(on, x, ("levels", "bins"))
    assert l_on > 1  # integration runs the unfused kernels
    for blk in (fresh, rt, on):
        blk.close()


# ---- against the oracle ----
@pytest.mark.parametrize("m", [2, 3, 4, 5, 8, 12, 16])
@pytest.mark.parametrize("alpha", [0.5, 0.9, 0.99])
def test_against_the_oracle(m, alpha):
    W, snaps = 300, 32
    x = noise_windows(m, snaps, W, 100 + m)
    make = lambda: gh.make_block(m, 1, snaps, K=90)
    R = raw_R(make, x)
    blk = make()
    blk.set_integration(alpha)
    first, _ = gh.device_call(blk, x[:170], ("R",))  # the carry crosses a call inside a tile
    second, _ = gh.device_call(blk, x[170:], ("R",))
    got = np.concatenate([first["R"], second["R"]])
    ref, _ = io.integrate(R, alpha)
    assert np.array_equal(got[0], R[0])
    assert np.array_equal(got, np.conj(np.swapaxes(got, 1, 2)))  # exactly Hermitian, as R is
    assert np.all(got[:, np.arange(m), np.arange(m)].imag == 0.0)
    check_R(got, ref, "m=%d alpha=%g" % (m, alpha))
    blk.close()


def test_across_sub_batches():
    # m = 16, n = 2 under TOP_BINS keeps the fp64 spectrum of K = 65536 bins: about 750 windows per sub-batch
    m, n, snaps, K, W = 16, 2, 32, 65536, 2000
    x = noise_windows(m, snaps, W, 5)
    make = lambda: gh.make_block(m, n, snaps, K=K)
    R = raw_R(make, x)
    blk = make()
    blk.set_integration(0.99)
    got, _ = gh.device_call(blk, x, ("R",))
    check_R(got["R"], io.integrate(R, 0.99)[0], "m=16 K=65536 W=2000")
    blk.close()


# ---- split and stream invariance ----
def test_split_invariance_across_entries():
    # every input below 1 MiB: the host entries register larger caller buffers with the driver for as long as the
    # handle lives, and a freed slice's pages could come back as the next slice
    m, snaps, W = 4, 64, 700
    pos = helpers.positions("uca", m)
    table = helpers.table_wl(pos / LAM)
    x = noise_windows(m, snaps, W, 21, theta=123.0, pos=pos, snr_db=-5.0)
    make = lambda: gh.make_block(m, 1, snaps, table=table, pos=pos)
    whole_blk = make()
    whole_blk.set_integration(0.9)
    whole, _ = gh.device_call(whole_blk, x, ("R", "bins"))
    R_raw = raw_R(make, x)
    check_R(whole["R"], io.integrate(R_raw, 0.9)[0], "split: one call")
    blk = make()
    blk.set_integration(0.9)
    a, _ = gh.device_call(blk, x[:1], ("R", "bins"))                                   # device, 1 window
    s = helpers.antenna_streams(x[1:8], m)
    pa, pl = np.zeros((7, 1), np.float32), np.zeros((7, 1), np.float32)
    blk.work_planar(7, s, [pa, pl])                                                    # planar host, 7 windows
    b_bins = blk.last_bins().copy()
    h = gh.host_call(blk, x[8:264])                                                    # host, 256 (two staging streams)
    c, _ = gh.device_call(blk, x[264:], ("R", "bins"))                                 # device, the rest
    ref = whole["R"]
    check_R(np.concatenate([a["R"], c["R"]]), np.concatenate([ref[:1], ref[264:]]), "split: 1 / 7 / 256 / rest")
    bins = np.concatenate([a["bins"], b_bins, h["bins"], c["bins"]])
    assert_bins_close(bins, [music_P(R, table, 1) for R in ref], 1)
    for blk_ in (whole_blk, blk):
        blk_.close()


def test_two_streams_integrate_in_call_order():
    m, snaps, W = 8, 64, 512
    x = noise_windows(m, snaps, W, 31)
    make = lambda: gh.make_block(m, 1, snaps, K=90)
    ref = io.integrate(raw_R(make, x), 0.95)[0]
    blk = make()
    blk.set_integration(0.95)
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    R = torch.zeros((W, m, m, 2), dtype=torch.float64, device=gh.DEV)
    ang = torch.zeros((W, 1), dtype=torch.float32, device=gh.DEV)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    half = W // 2
    per = m * snaps * 2
    torch.cuda.synchronize()  # the inputs and zeroed outputs are in place before the two streams start
    blk.process_device(d_in.data_ptr(), half, ang.data_ptr(), stream=s1.cuda_stream, d_R=R.data_ptr())
    blk.process_device(d_in.data_ptr() + half * per * 4, W - half, ang[half:].data_ptr(), stream=s2.cuda_stream,
                       d_R=R[half:].data_ptr())
    torch.cuda.synchronize()
    got = R.cpu().numpy()
    check_R(got[..., 0] + 1j * got[..., 1], ref, "two streams")
    blk.close()


# ---- resets ----
def test_resets():
    m, snaps = 4, 64
    pos = helpers.ula(m, "x") * LAM
    table = helpers.table_wl(pos / LAM)
    x = noise_windows(m, snaps, 40, 41)
    R = raw_R(lambda: gh.make_block(m, 1, snaps, table=table, pos=pos), x)
    blk = gh.make_block(m, 1, snaps, table=table, pos=pos)
    blk.set_integration(0.8)
    step = lambda: gh.device_call(blk, x[10:11], ("R",))[0]["R"][0]
    gh.device_call(blk, x[:10], ("R",))
    resets = {"reset_integration": lambda: blk.reset_integration(),
              "set_integration": lambda: blk.set_integration(0.8),
              "set_array_response": lambda: blk.set_array_response(table),
              "set_array_geometry": lambda: blk.set_array_geometry(pos, LAM),
              "set_calibration": lambda: blk.set_calibration(np.ones(m))}
    for name, fn in resets.items():
        gh.device_call(blk, x[:10], ("R",))
        fn()
        assert np.array_equal(step(), R[10]), name
    blk.set_calibration(None)
    blk.set_array_geometry(pos, LAM)
    keeps = {"set_peak_mode": lambda: blk.set_peak_mode("local_maxima"),
             "set_estimator": lambda: blk.set_estimator("mvdr", 0.01),
             "set_source_rule": lambda: blk.set_source_rule("mdl"),
             "set_refine": lambda: blk.set_refine(True),
             "set_beamformer": lambda: blk.set_beamformer("das")}
    for name, fn in keeps.items():
        blk.reset_integration()
        gh.device_call(blk, x[:10], ("R",))
        fn()
        assert not np.array_equal(step(), R[10]), name
    blk.close()


def test_empty_and_refused_calls_leave_the_carry():
    m, snaps = 4, 64
    x = noise_windows(m, snaps, 20, 43)
    make = lambda: gh.make_block(m, 1, snaps, K=90)
    ref = io.integrate(raw_R(make, x), 0.7)[0]
    blk = make()
    blk.set_integration(0.7)
    gh.device_call(blk, x[:10], ("R",))
    blk.process_device(0, 0, 0)  # nwindows = 0
    with pytest.raises(MusicB200Error):
        blk.process_device(1, 4, 0)  # refused before anything is enqueued (NULL angles)
    got, _ = gh.device_call(blk, x[10:], ("R",))
    check_R(got["R"], ref[10:], "empty and refused calls")
    blk.close()


# ---- downstream stages read Rbar ----
def test_downstream_grid_estimators_counts_and_calibration():
    m, snaps, W, alpha = 8, 32, 200, 0.9
    pos = helpers.positions("uca", m)
    table = helpers.table_wl(pos / LAM)
    x = noise_windows(m, snaps, W, 51, theta=73.0, pos=pos, snr_db=-6.0)
    rng = np.random.default_rng(3)
    gains = np.exp(1j * rng.uniform(-1, 1, m)) * rng.uniform(0.8, 1.2, m)
    for kind, loading, peak in (("music", 0.0, "top_bins"), ("music", 0.0, "local_maxima"), ("mvdr", 0.01, "top_bins"),
                                ("bartlett", 0.0, "top_bins")):
        for cal in (None, gains):
            blk = gh.make_block(m, 2, snaps, table=table, pos=pos, est=(kind, loading), mode=peak, calibration=cal)
            blk.set_integration(alpha)
            out, _ = gh.device_call(blk, x, ("R", "P64", "bins"))
            for w in range(0, W, 7):
                R = out["R"][w]
                P = music_P(R, table, 2) if kind == "music" else eo.spectrum(R, table, kind, loading)
                assert np.allclose(out["P64"][w], P, rtol=1e-8, atol=0), (kind, peak, w)
                ref = eo.picks(P, 2, len(P), "local" if peak == "local_maxima" else "top")[2]
                for g, r in zip(out["bins"][w], ref):
                    assert g == r or abs(P[g] - P[r]) <= 1e-9 * abs(P[r]), (kind, peak, w)
            blk.close()
    # MDL with N_eff: the device's own eigenvalues, the counts of an identical handle on the same windows
    ev_blk = gh.make_block(m, m - 1, snaps, table=table, rule="mdl")
    cnt_blk = gh.make_block(m, m - 1, snaps, table=table, rule="mdl")
    for b in (ev_blk, cnt_blk):
        b.set_integration(alpha)
    ev = gh.device_call(ev_blk, x, ("eigvals",))[0]["eigvals"]
    counts = gh.device_call(cnt_blk, x, ("counts",))[0]["counts"]
    ref = [sco.estimate_source_count(ev[w], io.n_eff(snaps, alpha, w), m - 1, "mdl")[0] for w in range(W)]
    assert np.array_equal(counts, ref)
    assert np.mean(counts[50:] == 1) >= 0.9  # what N_eff buys on a -6 dB source
    ev_blk.close()
    cnt_blk.close()


def test_downstream_beams():
    m, snaps, W = 4, 64, 64
    pos = helpers.positions("uca", m)
    table = helpers.table_wl(pos / LAM)
    x = noise_windows(m, snaps, W, 61, theta=200.0, pos=pos, snr_db=0.0)
    for rule, loading in (("das", 0.0), ("mvdr", 0.01)):
        blk = gh.make_block(m, 1, snaps, table=table, pos=pos, beamformer=(rule, loading))
        code = {"das": bo.DAS, "mvdr": bo.MVDR}[rule]
        blk.set_integration(0.9)
        out, _ = gh.device_call(blk, x, ("bins", "weights", "beams"))
        ref_blk = gh.make_block(m, 1, snaps, table=table, pos=pos)
        ref_blk.set_integration(0.9)
        R = gh.device_call(ref_blk, x, ("R",))[0]["R"]
        for w in range(W):
            wt = bo.weights(R[w], out["angles"][w], out["bins"][w], code, loading, pos=pos, lam=LAM)
            assert np.allclose(out["weights"][w], wt, rtol=1e-9, atol=1e-12), (rule, w)
        helpers.check_beams(x, out["weights"], out["beams"])  # formed from each window's own samples
        blk.close()
        ref_blk.close()


def _angle_err(a, t):
    return np.abs((np.asarray(a, np.float64) - t + 180.0) % 360.0 - 180.0)


@pytest.mark.parametrize("mode,refine", [("roots", False), ("esprit", False), ("dml", False), ("top_bins", True)])
def test_downstream_gridless_dml_and_refinement_find_a_weak_source(mode, refine):
    # one -10 dB source at 63.3 degrees on an x-axis ULA: integrated windows place it, single windows often do not
    m, snaps, W = 8, 32, 300
    pos = helpers.ula(m, "x") * LAM
    table = helpers.table_wl(pos / LAM)
    x = noise_windows(m, snaps, W, 71, theta=63.3, pos=pos, snr_db=-10.0)
    errs = {}
    for alpha in (0.0, 0.95):
        blk = gh.make_block(m, 1, snaps, table=table, pos=pos, mode=mode, refine=refine)
        blk.set_integration(alpha)
        out, _ = gh.device_call(blk, x, ("bins",))
        e = _angle_err(out["angles"][100:, 0], 63.3)
        e = np.minimum(e, _angle_err(out["angles"][100:, 0], -63.3))  # the x-axis ULA's mirror
        errs[alpha] = float(np.mean(e <= 1.0))
        blk.close()
    print("integration %s%s: share within 1 degree, alpha 0 %.2f, alpha 0.95 %.2f" % (mode, "+newton" if refine else "",
                                                                                   errs[0.0], errs[0.95]))
    assert errs[0.95] >= 0.9 and errs[0.95] >= errs[0.0]


def test_downstream_azel_esprit2d():
    pos = ao.ura_xyz(4, 4, LAM)
    m, snaps, W = 16, 32, 200
    az, el = 140.0, 35.0
    ca, sa, ce, se = (math.cos(math.radians(az)), math.sin(math.radians(az)), math.cos(math.radians(el)),
                      math.sin(math.radians(el)))
    a = np.exp(-2j * math.pi / LAM * (pos[:, 0] * ce * ca + pos[:, 1] * ce * sa + pos[:, 2] * se))
    rng = np.random.default_rng(81)
    s = 10 ** (-12 / 20) * (rng.standard_normal((W, snaps)) + 1j * rng.standard_normal((W, snaps))) / math.sqrt(2)
    nz = (rng.standard_normal((W, snaps, m)) + 1j * rng.standard_normal((W, snaps, m))) / math.sqrt(2)
    x = (s[..., None] * a + nz).reshape(W, snaps * m).astype(np.complex64)
    share = {}
    for alpha in (0.0, 0.95):
        blk = music_doa_azel(m, 1, m * snaps, 360, 91, (0.0, 90.0), pos, LAM)
        blk.set_peak_mode("esprit", 0)
        blk.set_integration(alpha)
        out, _ = gh.device_call(blk, x)
        ok = (_angle_err(out["azimuth"][100:, 0], az) <= 2.0) & (np.abs(out["elevation"][100:, 0] - el) <= 2.0)
        share[alpha] = float(np.mean(ok))
        blk.close()
    print("integration 2-D ESPRIT: share within 2 degrees, alpha 0 %.2f, alpha 0.95 %.2f" % (share[0.0], share[0.95]))
    assert share[0.95] >= 0.9 and share[0.95] >= share[0.0]


# ---- refusals ----
def test_refusals():
    blk = gh.make_block(4, 1, 64, K=90)
    blk.set_integration(0.5)
    for bad in (-0.1, 1.0, 1.5, float("nan"), float("inf")):
        with pytest.raises(MusicB200Error):
            blk.set_integration(bad)
    blk.close()
    multi = gh.make_block(4, 1, 64, K=90, devices=[0])
    with pytest.raises(MusicB200Error):
        multi.set_integration(0.5)
    with pytest.raises(MusicB200Error):
        multi.reset_integration()
    multi.close()
    pos = np.random.default_rng(1).uniform(-0.3, 0.3, (4, 2))
    chan = music_doa_channels(4, 1, 4 * 64, 90, 16, (0, 4), "hann", "separate", pos, 1.0, 400e6, 56e6)
    with pytest.raises(MusicB200Error):
        chan.set_integration(0.5)
    chan.close()


# ---- the benefit ----
def test_weak_source_benefit_through_the_block():
    m, N, W = 8, 32, 400
    pos = io.uca_wl(m) * LAM
    x = io.weak_source_windows(W, 2026, m, N)
    res = {}
    for alpha in (0.0, 0.9, 0.95):
        blk = gh.make_block(m, 1, N, K=360, pos=pos, rule="mdl")
        blk.set_integration(alpha)
        h = gh.host_call(blk, x)
        err = _angle_err(h["angles"][200:, 0], 73.0)
        res[alpha] = (float(np.mean((err <= 2.0) & (h["bins"][200:, 0] >= 0))), float(np.mean(h["counts"][200:] == 1)))
        blk.close()
    # the count-aware peak: under MDL a window counted 0 reports no peak (bin -1)
    print("integration weak source (UCA-8, -12 dB, N = 32, windows 200-399): peak within 2 deg / MDL = 1: %s" % res)
    assert res[0.0][0] <= 0.5 and res[0.0][1] <= 0.1
    assert res[0.95][0] >= 0.9 and res[0.95][1] >= 0.9


# ---- the C++ block ----
def test_cpp_block():
    m, n, N, W, K, chunk, alpha = 8, 1, 32, 300, 360, 64, 0.95
    pos = io.uca_wl(m) * LAM
    x = io.weak_source_windows(W, 7, m, N)
    hdr = struct.pack("<7I2d", m, n, m * N, K, W, 1, chunk, alpha, LAM)
    out = gh.run_cpp_block("test_block_integration", hdr, [pos.astype(np.float64), x],
                           [("angles", np.float32, 2 * W * n), ("bins", np.int32, 2 * W * n), ("counts", np.int32, 2 * W)])
    blk = gh.make_block(m, n, N, K=K, pos=pos, rule="mdl")
    blk.set_integration(alpha)
    for p in range(2):
        if p:
            blk.reset_integration()
        ang, bins, cnt = [], [], []
        for w0 in range(0, W, chunk):
            h = gh.host_call(blk, x[w0:w0 + chunk])
            ang.append(h["angles"])
            bins.append(h["bins"])
            cnt.append(h["counts"])
        sl = slice(p * W * n, (p + 1) * W * n)
        assert np.array_equal(out["angles"][sl], np.concatenate(ang).ravel())
        assert np.array_equal(out["bins"][sl], np.concatenate(bins).ravel())
        assert np.array_equal(out["counts"][p * W:(p + 1) * W], np.concatenate(cnt))
    blk.close()
