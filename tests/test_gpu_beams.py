"""GPU: beamformed source signals (music_b200_set_beamformer, music_b200_process_*_beams) against their fp64 definition
(tests/beams_oracle.py), through every entry point.

The oracle runs on the GPU's own covariance (process_device_ex with d_R on the same windows) and the GPU's own angles and
bins, so what is compared is the weight solver and the apply pass themselves."""
import math
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, synth
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import beams_oracle as bo
import helpers
import refine_oracle as ro
import test_dml_oracle as td
from test_gpu_root_music import LAM, dev_call, ula

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = -7
RULES = {"das": (bo.DAS, 0.0), "mvdr": (bo.MVDR, 0.01), "mvdr0": (bo.MVDR, 0.0), "lcmv": (bo.LCMV, 0.0)}
W_RTOL = 1e-9


# ---- fixtures --------------------------------------------------------------------------------------------------------
def geo_windows(pos, plan, seed, snaps, coherent=False):
    """complex64 windows [W][snaps * M] of the element positions pos (metres): plan[w] = (angles in degrees, snr_db);
    unit noise, independent unit-power sources (one shared signal when coherent)"""
    rng = np.random.default_rng(seed)
    m = len(pos)
    xs = []
    for degs, snr in plan:
        X = (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
        s = (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps)) / np.sqrt(2.0)
        for j, t in enumerate(degs):
            if j and not coherent:
                s = (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps)) / np.sqrt(2.0)
            X += 10.0 ** (snr / 20.0) * ro.steering(pos, LAM, math.radians(t))[0][:, None] * s[None, :]
        xs.append(X.T.reshape(-1))
    return np.ascontiguousarray(np.array(xs).astype(np.complex64))


def mixed_plan(rng, W=6):
    return [(rng.uniform(0.0, 360.0, S), snr) for S, snr in ((1, 30.0), (2, 20.0), (3, 20.0), (2, 10.0), (1, 0.0), (0, 0.0))][:W]


def handle(m, n, snaps, K, table=None, pos=None, mode="top_bins", rule="fixed", est=("music", 0.0), refine=False, devices=None):
    blk = music_doa(m, n, m * snaps, np.ones((K, m), np.complex64) if table is None else table, K, devices=devices)
    if pos is not None:
        blk.set_array_geometry(pos, LAM)
    blk.set_estimator(*est)
    blk.set_source_rule(rule)
    blk.set_peak_mode(mode, 0)
    if refine:
        blk.set_refine(True)
    return blk


def beams_call(blk, x, n, K, weights=True, beams=True, spectrum=False, bins=True, counts=True):
    """one process_device_beams call; returns (outputs, kernel launches)"""
    dev = torch.device("cuda:0")
    Wn, m, N = x.shape[0], blk.m, blk.nsamples // blk.m
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)
    o = {"angles": torch.full((Wn, n), SENTINEL, dtype=torch.float32, device=dev),
         "levels": torch.full((Wn, n), SENTINEL, dtype=torch.float32, device=dev)}
    if bins:
        o["bins"] = torch.full((Wn, n), SENTINEL, dtype=torch.int32, device=dev)
    if spectrum:
        o["spectrum"] = torch.full((Wn, K), SENTINEL, dtype=torch.float32, device=dev)
    if counts:
        o["counts"] = torch.full((Wn,), SENTINEL, dtype=torch.int32, device=dev)
    if weights:
        o["weights"] = torch.full((Wn, n, m, 2), SENTINEL, dtype=torch.float64, device=dev)
    if beams:
        o["beams"] = torch.full((Wn, n, N, 2), SENTINEL, dtype=torch.float32, device=dev)
    p = lambda k: o[k].data_ptr() if k in o else None
    l0 = blk.launch_count()
    blk.process_device_beams(d_in.data_ptr(), Wn, p("angles"), p("levels"), p("spectrum"), p("bins"), p("counts"), p("weights"),
                             p("beams"), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    for k in ("weights", "beams"):
        if k in out:
            out[k] = np.ascontiguousarray(out[k]).view(np.float64 if k == "weights" else np.float32)
            out[k] = out[k][..., 0] + 1j * out[k][..., 1]
    if "beams" in out:
        out["beams"] = out["beams"].astype(np.complex64)
    return out, blk.launch_count() - l0


def host_beams(blk, x, n, K, spectrum=False):
    W = x.shape[0]
    ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    outs = [ang, lvl] + ([np.zeros((W, K), np.float32)] if spectrum else [])
    assert blk.work(W, [x], outs) == W
    return {"angles": ang, "levels": lvl, "bins": blk.last_bins(), "counts": blk.last_counts(), "weights": blk.last_weights(),
            "beams": blk.last_beams(), **({"spectrum": outs[2]} if spectrum else {})}


def gram_cond(R, ang, bins, loading, table, pos):
    """condition number of the LCMV Gram of one window (1 when fewer than two slots are filled)"""
    A = bo.steering_vectors(ang, bins, table, pos, LAM)
    if len(A) < 2:
        return 1.0
    M = R.shape[0]
    RL = R + loading * np.trace(R).real / M * np.eye(M)
    Ys = [np.linalg.solve(np.linalg.cholesky(RL), A[i]) for i in sorted(A)]
    Y = np.array(Ys).T
    return float(np.linalg.cond(Y.conj().T @ Y))


def check_weights(got, ref_R, out, rule, loading, table, pos, ctx):
    """the GPU's weights against the oracle's on the GPU's R, angles and bins"""
    for w in range(len(ref_R)):
        ref = bo.weights(ref_R[w], out["angles"][w], out["bins"][w], rule, loading, table=table, pos=pos, lam=LAM)
        g = got[w]
        assert np.array_equal(g == 0, ref == 0), (ctx, w, g, ref)
        if not np.any(ref):
            continue
        tol = W_RTOL
        if rule == bo.LCMV:
            tol *= max(1.0, gram_cond(ref_R[w], out["angles"][w], out["bins"][w], loading, table, pos))
        for i in range(ref.shape[0]):
            s = np.max(np.abs(ref[i]))
            if s:
                assert np.max(np.abs(g[i] - ref[i])) <= tol * s, (ctx, w, i, g[i], ref[i], tol)


def check_beams(x, got_w, got_b):
    """beams within one float32 rounding of numpy applying the GPU's weights (+ fp64 accumulation order)"""
    Wn, n, M = got_w.shape
    X = x.astype(np.complex128).reshape(Wn, -1, M)  # [W][N][M]
    ref = np.einsum("wtm,wim->wit", X, np.conj(got_w))
    bound = np.einsum("wtm,wim->wit", np.abs(X), np.abs(got_w))
    dead = ~np.any(got_w != 0, axis=2)
    ref[dead] = 0
    bound[dead] = 0
    err = np.abs(got_b.astype(np.complex128) - ref)
    assert np.all(err <= 2.0 ** -24 * np.abs(ref) + 1e-12 * bound), np.max(err - 2.0 ** -24 * np.abs(ref))


def tables(m, K):
    """(name, table or None, positions or None): geometric x-axis ULA and UCA, random planar and calibrated tables"""
    uca = td.array("uca", m)
    return [("ula", None, ula(m, "x")), ("uca", None, uca), ("planar", helpers.planar_table(m, K, 50 + m), None),
            ("calibrated", helpers.calibrated_table(td.table(uca, K), 60 + m), None)]


def configs(name):
    """(peak mode, source rule, estimator, refine) per table kind"""
    c = [("top_bins", "fixed", ("music", 0.0), False), ("local_maxima", "mdl", ("mvdr", 0.01), False), ("dml", "fixed", ("music", 0.0), False)]
    if name in ("ula", "uca"):
        c.append(("local_maxima", "fixed", ("music", 0.0), True))
    if name == "ula":
        c += [("roots", "mdl", ("music", 0.0), False), ("esprit", "fixed", ("music", 0.0), False)]
    return c


# ---- parity with the oracle ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2, 3, 4, 8, 12, 16])
def test_weights_and_beams_parity(m):
    K, snaps = 360, 256
    for ti, (name, tab, pos) in enumerate(tables(m, K)):
        rng = np.random.default_rng(100 * m + ti)
        if pos is None:
            vecs = [[tab[k] for k in rng.choice(K, S, replace=False)] for S in (1, 2, 3, 2, 0, 1)]
            x = helpers.source_windows(rng, vecs, m, snaps, amp=10.0)
        else:
            x = geo_windows(pos, mixed_plan(rng), 7 * m + ti, snaps)
        for n in (1, 2, 3):
            if n >= m:
                continue
            for mode, rule, est, refine in configs(name):
                blk = handle(m, n, snaps, K, tab, pos, mode, rule, est, refine)
                ref, _ = dev_call(blk, x, n, K, R=True)
                for bname, (brule, loading) in RULES.items():
                    ctx = (m, name, n, mode, rule, est, refine, bname)
                    blk.set_beamformer(bname.rstrip("0"), loading)
                    out, _ = beams_call(blk, x, n, K)
                    for k in ("angles", "levels", "bins"):
                        assert np.array_equal(out[k], ref[k]), (ctx, k)
                    check_weights(out["weights"], ref["R"], out, brule, loading, tab, pos, ctx)
                    check_beams(x, out["weights"], out["beams"])
                blk.close()


# ---- invariants ------------------------------------------------------------------------------------------------------
def test_peak_outputs_match_ex_with_R():
    """angles, levels, spectrum, bins and counts are byte-identical to process_device_ex(d_R) / _counts"""
    m, n, snaps, K = 8, 2, 512, 720
    pos = td.array("uca", m)
    x = geo_windows(pos, mixed_plan(np.random.default_rng(1)) * 3, 2, snaps)
    for mode, rule in (("top_bins", "fixed"), ("local_maxima", "mdl"), ("dml", "fixed")):
        blk = handle(m, n, snaps, K, pos=pos, mode=mode, rule=rule)
        ref, _ = dev_call(blk, x, n, K, spectrum=True, R=True)
        cnt, _ = dev_call(blk, x, n, K, counts=True)
        for kind in ("das", "lcmv"):
            blk.set_beamformer(kind, 0.0)
            out, _ = beams_call(blk, x, n, K, spectrum=True)
            for k in ("angles", "levels", "bins", "spectrum"):
                assert np.array_equal(out[k], ref[k]), (mode, kind, k)
            assert np.array_equal(out["counts"], cnt["counts"])
        blk.close()


@pytest.mark.parametrize("k", [-40, 40])
def test_power_of_two_input_scaling(k):
    """input x 2^k: bit-identical weights, beams scaled by exactly 2^k"""
    m, n, snaps, K = 8, 2, 256, 360
    pos = td.array("uca", m)
    x = geo_windows(pos, [((40.0, 170.0), 20.0)] * 4, 3, snaps)
    xs = (x.astype(np.complex128) * 2.0 ** k).astype(np.complex64)
    for kind, loading in (("das", 0.0), ("mvdr", 0.0), ("mvdr", 0.1), ("lcmv", 0.0)):
        blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima")
        blk.set_beamformer(kind, loading)
        a, _ = beams_call(blk, x, n, K)
        b, _ = beams_call(blk, xs, n, K)
        blk.close()
        assert np.array_equal(a["bins"], b["bins"]) and np.array_equal(a["angles"], b["angles"])
        assert np.any(a["weights"] != 0)
        assert np.array_equal(a["weights"], b["weights"]), kind
        assert np.array_equal((a["beams"].astype(np.complex128) * 2.0 ** k).astype(np.complex64), b["beams"]), kind


def test_zeros():
    """unfilled slots and a NaN window give zero weights and beams; so does a dead-antenna window under MVDR and LCMV with
    loading 0 (its R_L has a zero pivot), while DAS still steers at the slots the peak stage filled there"""
    m, n, snaps, K = 4, 3, 256, 360
    pos = td.array("uca", m)
    x = geo_windows(pos, [((50.0,), 20.0)] * 4, 4, snaps)
    x[1, 5] = np.nan
    x[2].reshape(snaps, m)[:, 2] = 0  # antenna 2 dead
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima", rule="mdl")
    for kind in ("das", "mvdr", "lcmv"):
        blk.set_beamformer(kind, 0.0)
        out, _ = beams_call(blk, x, n, K)
        for w in (0, 3):
            d = int(out["counts"][w])
            assert d >= 1 and np.all(out["bins"][w, d:] == -1)
            assert np.all(out["weights"][w, d:] == 0) and np.all(out["beams"][w, d:] == 0)
            assert np.all(out["weights"][w, :d] != 0)
        assert np.all(out["weights"][1] == 0) and np.all(out["beams"][1] == 0), kind
    blk.close()
    # FIXED rule: the peak stage fills every slot of the dead-antenna window (MDL would count 0 sources there)
    blk = handle(m, n, snaps, K, pos=pos, mode="top_bins")
    for kind in ("das", "mvdr", "lcmv"):
        blk.set_beamformer(kind, 0.0)
        out, _ = beams_call(blk, x, n, K)
        assert np.all(out["bins"][2] >= 0), out["bins"][2]
        if kind == "das":
            assert np.all(out["weights"][2] != 0) and np.any(out["beams"][2] != 0)
        else:
            assert np.all(out["weights"][2] == 0) and np.all(out["beams"][2] == 0), kind
            assert np.all(out["weights"][0] != 0), kind  # the healthy windows still get beams
    blk.close()


def test_mirror_pair_under_lcmv():
    """an x-axis ULA under LOCAL_MAXIMA reports a source and its mirror: LCMV zeroes the window, MVDR does not"""
    m, n, snaps, K = 6, 2, 256, 360
    pos = ula(m, "x")
    x = geo_windows(pos, [((60.0,), 30.0)] * 3, 5, snaps)
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima")
    blk.set_beamformer("lcmv", 0.0)
    out, _ = beams_call(blk, x, n, K)
    assert np.all(out["bins"] >= 0) and np.all(out["bins"].sum(axis=1) % 360 == 0), out["bins"]
    assert np.all(out["weights"] == 0) and np.all(out["beams"] == 0)
    blk.set_beamformer("mvdr", 0.0)
    out, _ = beams_call(blk, x, n, K)
    assert np.all(out["weights"] != 0)
    blk.close()


# ---- physics ---------------------------------------------------------------------------------------------------------
def test_single_source_waveform():
    """one source at 40 dB: the DAS and MVDR beams reproduce its waveform (|normalised correlation| at least the oracle's
    on the same windows minus 1e-6, and above 0.99).  The angles are refined off the grid: at this SNR an MVDR beam
    steered half a grid bin off the source suppresses it (the signal is in R)."""
    m, snaps, K, Wn = 8, 1024, 3600, 16
    pos = td.array("uca", m)
    rng = np.random.default_rng(21)
    th = rng.uniform(0.0, 360.0, Wn)
    sig = (rng.standard_normal((Wn, snaps)) + 1j * rng.standard_normal((Wn, snaps))) / np.sqrt(2.0)
    noise = (rng.standard_normal((Wn, m, snaps)) + 1j * rng.standard_normal((Wn, m, snaps))) / np.sqrt(2.0)
    X = noise + 100.0 * np.array([ro.steering(pos, LAM, math.radians(t))[0][:, None] * sig[w][None, :] for w, t in enumerate(th)])
    x = np.ascontiguousarray(X.transpose(0, 2, 1).reshape(Wn, -1).astype(np.complex64))
    corr = lambda y, s: abs(np.vdot(y, s)) / (np.linalg.norm(y) * np.linalg.norm(s))
    for kind in ("das", "mvdr"):
        blk = handle(m, 1, snaps, K, pos=pos, refine=True)
        ref, _ = dev_call(blk, x, 1, K, R=True)
        blk.set_beamformer(kind, 0.0)
        out, _ = beams_call(blk, x, 1, K)
        blk.close()
        for w in range(Wn):
            W_ref = bo.weights(ref["R"][w], out["angles"][w], out["bins"][w], RULES[kind][0], 0.0, pos=pos, lam=LAM)
            c_ref = corr(bo.beams(x[w], W_ref)[0].astype(np.complex128), sig[w])
            c = corr(out["beams"][w, 0].astype(np.complex128), sig[w])
            assert c >= c_ref - 1e-6 and c > 0.99, (kind, w, c, c_ref)


def sir_db(W, a_own, a_other):
    return 10.0 * math.log10(abs(np.vdot(W, a_own)) ** 2 / max(abs(np.vdot(W, a_other)) ** 2, 1e-300))


def test_two_sources_interference_rejection():
    """two uncorrelated sources at 20 dB on a UCA 8, 15 to 25 degrees apart, inside each other's DAS main lobe
    (LOCAL_MAXIMA n = 2, refined angles): in >= 95 % of the windows both slots are filled, one per source, and the MVDR
    and LCMV beams of both raise the output signal-to-interference ratio over the DAS beam's by >= 10 dB; and in at
    least as many windows as the oracle's weights do on the GPU's R and angles (less one).  (With sources far apart the
    interferer can sit in a natural null of the DAS beam, where DAS reaches 30-50 dB and a finite-sample MVDR null is no
    deeper: there is no gain to test.)"""
    m, n, snaps, K, Wn = 8, 2, 1024, 360, 60
    pos = td.array("uca", m)
    rng = np.random.default_rng(31)
    plan = []
    for _ in range(Wn):
        t0 = rng.uniform(0.0, 360.0)
        plan.append(((t0, (t0 + rng.choice([-1.0, 1.0]) * rng.uniform(15.0, 25.0)) % 360.0), 20.0))
    x = geo_windows(pos, plan, 32, snaps)
    steer = lambda t: ro.steering(pos, LAM, math.radians(t))[0]
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima", refine=True)
    ref, _ = dev_call(blk, x, n, K, R=True)
    sir = {}
    for kind in ("das", "mvdr", "lcmv"):
        blk.set_beamformer(kind, 0.0)
        out, _ = beams_call(blk, x, n, K)
        got, want = np.full((Wn, n), np.nan), np.full((Wn, n), np.nan)  # NaN: the window did not resolve both sources
        for w, (truth, _) in enumerate(plan):
            own = [int(np.argmin([td.circ(out["angles"][w, i], t) for t in truth])) for i in range(n)]
            if np.any(out["bins"][w] < 0) or sorted(own) != [0, 1]:
                continue
            W_ref = bo.weights(ref["R"][w], out["angles"][w], out["bins"][w], RULES[kind][0], 0.0, pos=pos, lam=LAM)
            for i in range(n):
                a, b = steer(truth[own[i]]), steer(truth[1 - own[i]])
                got[w, i] = sir_db(out["weights"][w, i], a, b)
                want[w, i] = sir_db(W_ref[i], a, b)
        sir[kind] = (got, want)
    blk.close()
    for kind in ("mvdr", "lcmv"):
        with np.errstate(invalid="ignore"):
            ok = np.all(sir[kind][0] - sir["das"][0] >= 10.0, axis=1)
            ok_ref = np.all(sir[kind][1] - sir["das"][1] >= 10.0, axis=1)
        assert np.mean(ok) >= 0.95, (kind, np.sort(np.nanmin(sir[kind][0] - sir["das"][0], axis=1))[:5])
        assert np.sum(ok) >= np.sum(ok_ref) - 1, kind


# ---- plumbing --------------------------------------------------------------------------------------------------------
def test_entry_points_agree():
    """device, host and multi-device host entries give byte-identical peaks, weights and beams; the Python block's
    work() goes through the host entry"""
    m, n, snaps, K, Wn = 8, 2, 512, 720, 40
    pos = td.array("uca", m)
    x = geo_windows(pos, mixed_plan(np.random.default_rng(41)) * 7, 42, snaps)[:Wn]
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima", rule="mdl")
    blk.set_beamformer("lcmv", 0.05)
    assert blk.beamformer() == ("lcmv", 0.05)
    ref, _ = beams_call(blk, x, n, K, spectrum=True)
    got = host_beams(blk, x, n, K, spectrum=True)
    for k in ("angles", "levels", "bins", "counts", "spectrum", "weights", "beams"):
        assert np.array_equal(got[k], ref[k]), k
    blk.set_beamformer("off")
    assert host_beams(blk, x, n, K)["beams"] is None
    blk.close()
    G = torch.cuda.device_count()
    for devices in ([0], list(range(G))) if G > 1 else ([0],):
        mb = handle(m, n, snaps, K, pos=pos, mode="local_maxima", rule="mdl", devices=devices)
        mb.set_beamformer("lcmv", 0.05)
        got = host_beams(mb, x, n, K)
        mb.close()
        for k in ("angles", "levels", "bins", "counts", "weights", "beams"):
            assert np.array_equal(got[k], ref[k]), (devices, k)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_device_host_entry():
    m, n, snaps, K, Wn = 4, 1, 256, 360, 33
    pos = td.array("uca", m)
    x = geo_windows(pos, [((t,), 20.0) for t in np.linspace(0, 350, Wn)], 43, snaps)
    one = handle(m, n, snaps, K, pos=pos)
    one.set_beamformer("mvdr", 0.0)
    ref = host_beams(one, x, n, K)
    one.close()
    mb = handle(m, n, snaps, K, pos=pos, devices=list(range(torch.cuda.device_count())))
    mb.set_beamformer("mvdr", 0.0)
    got = host_beams(mb, x, n, K)
    mb.close()
    for k in ("angles", "bins", "weights", "beams"):
        assert np.array_equal(got[k], ref[k]), k


def test_launch_counts_and_sub_batches():
    """the ex(R) plan plus 2 launches per sub-batch (1 without beams); a call of several sub-batches equals its halves"""
    m, n, snaps = 4, 2, 256
    pos = td.array("uca", m)
    x = geo_windows(pos, [((40.0, 200.0), 20.0)] * 3, 51, snaps)
    blk = handle(m, n, snaps, 360, pos=pos, mode="local_maxima")
    _, l_ex = dev_call(blk, x, n, 360, R=True)
    blk.set_beamformer("das")
    _, l_both = beams_call(blk, x, n, 360, counts=False)  # (counts under FIXED add a fill launch)
    _, l_w = beams_call(blk, x, n, 360, beams=False, counts=False)
    _, l_b = beams_call(blk, x, n, 360, weights=False, bins=False, counts=False)
    blk.close()
    assert (l_both, l_w, l_b) == (l_ex + 2, l_ex + 1, l_ex + 2), (l_ex, l_both, l_w, l_b)
    Kb, Wb, Nb = 36000, 3000, 64
    xb = geo_windows(pos, [((40.0, 200.0), 20.0)] * Wb, 52, Nb)
    blk = handle(m, n, Nb, Kb, pos=pos, mode="local_maxima")
    _, l_ex = dev_call(blk, xb, n, Kb, R=True)
    blk.set_beamformer("mvdr", 0.0)
    whole, launches = beams_call(blk, xb, n, Kb, counts=False)
    assert (launches - l_ex) % 2 == 0 and (launches - l_ex) // 2 >= 2, (launches, l_ex)
    first, _ = beams_call(blk, xb[: Wb // 2], n, Kb, counts=False)
    second, _ = beams_call(blk, xb[Wb // 2:], n, Kb, counts=False)
    for k in ("angles", "levels", "bins", "weights", "beams"):
        assert np.array_equal(whole[k], np.concatenate([first[k], second[k]])), k
    blk.close()


def test_plain_calls_ignore_the_beamformer():
    """process_device on a handle with a beamformer set is byte-identical to one without, with the same launches"""
    cfg = synth.config(2)
    x = synth.gen_windows_numpy(cfg, 12, 0, 64)
    tab = helpers.table_for(cfg)
    K = cfg["resolution"]
    fresh = music_doa(4, 1, cfg["nsamples"], tab, K)
    ref, l_ref = dev_call(fresh, x, 1, K)
    fresh.set_beamformer("mvdr", 0.1)
    got, l_got = dev_call(fresh, x, 1, K)
    fresh.close()
    assert l_ref == l_got == 1
    assert all(np.array_equal(got[k], ref[k]) for k in ("angles", "levels", "bins"))


def test_invalid_arguments():
    m, n, K, snaps = 4, 1, 360, 64
    L = _capi.load()
    EINVAL, OK = _capi.EINVAL, _capi.OK
    blk = handle(m, n, snaps, K, pos=td.array("uca", m))
    h = blk._h
    for rule, loading in ((4, 0.0), (-1, 0.0), (2, float("nan")), (2, float("inf")), (3, -1.0), (0, 0.5), (1, 0.5)):
        assert L.music_b200_set_beamformer(h, rule, loading) == EINVAL, (rule, loading)
    assert blk.beamformer() == ("off", 0.0)
    with pytest.raises(ValueError):
        blk.set_beamformer("capon")
    x = geo_windows(td.array("uca", m), [((30.0,), 20.0)] * 2, 61, snaps)
    with pytest.raises(_capi.MusicB200Error):  # rule OFF
        beams_call(blk, x, n, K)
    blk.set_beamformer("das")
    with pytest.raises(_capi.MusicB200Error):  # neither weights nor beams
        beams_call(blk, x, n, K, weights=False, beams=False)
    dev = torch.device("cuda:0")
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)
    ang = torch.zeros((2, n), dtype=torch.float32, device=dev)
    wb = torch.zeros(2 * n * m * 2 + 2, dtype=torch.float64, device=dev)
    bb = torch.zeros(2 * n * snaps * 2 + 2, dtype=torch.float32, device=dev)
    call = lambda wp, bp: L.music_b200_process_device_beams(h, d_in.data_ptr(), 2, ang.data_ptr(), None, None, None, None, wp, bp, None)
    assert call(wb.data_ptr() + 8, None) == EINVAL  # weights 8-byte aligned only
    assert call(None, bb.data_ptr() + 4) == EINVAL  # beams 4-byte aligned only
    assert call(wb.data_ptr() + 16, bb.data_ptr() + 8) == OK
    torch.cuda.synchronize()
    blk.close()
    # N <= m: MVDR and LCMV need loading
    small = handle(m, n, m, K, pos=td.array("uca", m))
    for rule in (2, 3):
        assert L.music_b200_set_beamformer(small._h, rule, 0.0) == EINVAL
        assert L.music_b200_set_beamformer(small._h, rule, 0.1) == OK
    assert L.music_b200_set_beamformer(small._h, 1, 0.0) == OK
    small.close()
    az = music_doa_azel(m, n, m * snaps, 36, 3, (0.0, 30.0), np.c_[td.array("x", m), np.zeros(m)], LAM)
    assert L.music_b200_set_beamformer(az._h, 1, 0.0) == EINVAL
    az.close()


def test_cpp_block():
    """the C++ block's set_beamformer() and last_beams() equal the Python block's"""
    exe = os.path.join(ROOT, "lib", "_build", "test_block_beams")
    m, n, K, snaps, Wn = 8, 2, 720, 256, 16
    pos = td.array("uca", m)
    rng = np.random.default_rng(71)
    x = geo_windows(pos, [((t, (t + 120.0) % 360.0), 20.0) for t in rng.uniform(0, 360, Wn)], 72, snaps)
    N = snaps
    with tempfile.TemporaryDirectory() as tdir:
        fin, fout = os.path.join(tdir, "in.bin"), os.path.join(tdir, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("<7I", m, n, m * snaps, K, Wn, 1, 3))
            f.write(struct.pack("<2d", 0.01, LAM))
            f.write(np.ascontiguousarray(pos, np.float64).tobytes())
            f.write(x.view(np.float32).tobytes())
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        raw = open(fout, "rb").read()
    o = 0
    take = lambda cnt, dt, sz=4: np.frombuffer(raw[o:o + sz * cnt], dt)
    ca = take(Wn * n, np.float32); o += 4 * Wn * n
    cl = take(Wn * n, np.float32); o += 4 * Wn * n
    cs = take(Wn * K, np.float32); o += 4 * Wn * K
    cb = take(Wn * n, np.int32); o += 4 * Wn * n
    cbeams = take(Wn * n * N, np.complex64, 8)
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima")
    blk.set_beamformer("lcmv", 0.01)
    got = host_beams(blk, x, n, K, spectrum=True)
    blk.close()
    assert np.array_equal(ca, got["angles"].ravel()) and np.array_equal(cl, got["levels"].ravel())
    assert np.array_equal(cs, got["spectrum"].ravel()) and np.array_equal(cb, got["bins"].ravel())
    assert np.array_equal(cbeams, got["beams"].ravel())
    assert np.any(cbeams != 0)
