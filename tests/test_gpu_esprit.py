"""GPU: the ESPRIT peak mode (MUSIC_B200_PEAKS_ESPRIT) against its fp64 definition (tests/esprit_oracle.py,
np.linalg.solve and np.linalg.eigvals on LAPACK eigenvectors), through every entry point, and the other peak modes
unchanged.

The oracle runs on the GPU's own covariance (d_R), so what is compared is the ESPRIT stage itself."""
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, synth
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import esprit_oracle as eo
import gpu_harness as gh
from helpers import LAM, PLAN, axis_deg, circ, near_half, plan_windows as windows, two_source_windows, ula

pytestmark = pytest.mark.gpu

ESPRIT = 3
FLIP = 1e-9     # orderings or subspaces the oracle sees this close to flipping may go either way
L_RTOL = 1e-5
PEAKS = ("levels", "bins")


def handle(m, n, K, pos, snaps, mode="esprit", rule="fixed", devices=None):
    return gh.make_block(m, n, snaps, K, pos=pos, rule=rule, mode=mode, devices=devices)


# ---- parity with the oracle ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2, 3, 4, 5, 8, 12, 16])
def test_parity_with_oracle(m):
    """angles within 2 float32 ulps, levels within 1e-5, bins equal (except at half-bin ties), counts equal to a
    TOP_BINS handle's under MDL; noiseless windows within 1e-3 degrees of the truth"""
    snaps = 512
    edge = total = 0
    for n in (1, 2, 3):
        if n >= m:
            continue
        for gi, kind in enumerate(("x", "y", "oblique", "reversed")):
            pos = ula(m, kind)
            plan = [(min(S, m - 1), snr) for S, snr in PLAN]
            x, truth = windows(pos, plan, 2000 * m + 10 * n + gi, snaps)
            for rule in ("fixed", "mdl"):
                K = 3600 if (gi + n) % 2 else 360
                blk = handle(m, n, K, pos, snaps, rule=rule)
                out, _ = gh.device_call(blk, x, PEAKS + ("R",))
                counts = None
                if rule == "mdl":
                    cnt, _ = gh.device_call(blk, x, PEAKS + ("counts",))
                    top = handle(m, n, K, pos, snaps, mode="top_bins", rule=rule)
                    tc, _ = gh.device_call(top, x, PEAKS + ("counts",))
                    top.close()
                    assert np.array_equal(cnt["counts"], tc["counts"]), (m, n, kind)
                    assert np.array_equal(cnt["angles"], out["angles"]) and np.array_equal(cnt["bins"], out["bins"])
                    counts = tc["counts"]
                blk.close()
                for w in range(len(x)):
                    ctx = (m, n, kind, rule, K, w, plan[w])
                    d = n if counts is None else int(counts[w])
                    ref = eo.work_R(out["R"][w], pos, LAM, K, n, d=d)
                    ga, gl, gb = out["angles"][w], out["levels"][w], out["bins"][w]
                    assert np.all(gb[d:] == -1) and np.all(ga[d:] == 0.0) and np.all(gl[d:] == 0.0), ctx
                    if plan[w][1] is None:
                        if d != len(truth[w]):
                            continue  # a signal subspace reaching into the null space of R is not unique
                        want = sorted(min(t % 360.0, (2.0 * axis_deg(pos) - t) % 360.0) for t in truth[w])
                        got = sorted(float(a) for a in ga[:d])
                        assert max(circ(g, t) for g, t in zip(got, want)) <= 1e-3, (ctx, got, want)
                        continue
                    total += d
                    if ref["margin"] <= FLIP and not (np.array_equal(gb, ref["bins"]) and np.array_equal(ga, ref["angles"])):
                        edge += d
                        continue
                    assert np.array_equal(gb < 0, ref["bins"] < 0), (ctx, gb, ref["bins"])
                    for i in range(d):
                        if ref["bins"][i] < 0:
                            continue
                        ra = ref["angles"][i]
                        tol = 2.0 * float(np.spacing(np.float32(max(abs(float(ra)), abs(float(ga[i])), 1e-3))))
                        assert circ(ga[i], ra) <= tol, (ctx, i, ga, ref["angles"])
                        assert abs(float(gl[i]) - float(ref["levels"][i])) <= L_RTOL * abs(float(ref["levels"][i])), (ctx, i, gl, ref["levels"])
                        if gb[i] != ref["bins"][i]:
                            assert near_half(float(ra), K), (ctx, i, gb, ref["bins"])
    assert edge <= 0.01 * max(total, 1), (edge, total)


def test_degenerate_windows():
    """NaN and all-zero windows report (0, 0, -1); MDL with d = 0 reports no peak"""
    m, n, K, snaps = 4, 2, 360, 256
    pos = ula(m, "x")
    x, _ = windows(pos, [(2, 20.0), (2, 20.0), (0, 0.0), (2, 20.0)], 5, snaps)
    x[0] = 0
    x[1, 17] = np.nan
    for rule in ("fixed", "mdl"):
        blk = handle(m, n, K, pos, snaps, rule=rule)
        out, _ = gh.device_call(blk, x, PEAKS)
        empty = [0, 1] if rule == "fixed" else [0, 1, 2]
        for w in empty:
            assert np.all(out["bins"][w] == -1) and np.all(out["angles"][w] == 0.0) and np.all(out["levels"][w] == 0.0), (rule, w, out)
        assert np.all(out["bins"][3] >= 0) and np.all(out["levels"][3] > 0.0)
        blk.close()


# ---- entry points ------------------------------------------------------------------------------------------------------
def test_entries_agree():
    """host, device, _ex, _counts and planar (at the fused-eligible M = 4 / n = 1 shape) agree byte for byte, and so do
    multi-device handles and sharded calls; with the spectrum port the spectrum and P64 are a LOCAL_MAXIMA handle's"""
    m, n, K, snaps, Wn = 4, 1, 3600, 1024, 24
    pos = ula(m, "x")
    x, _ = windows(pos, [(1, 20.0)] * Wn, 41, snaps)
    blk = handle(m, n, K, pos, snaps)
    ref, _ = gh.device_call(blk, x, PEAKS)
    assert np.all(ref["bins"] >= 0)
    ex, _ = gh.device_call(blk, x, PEAKS + ("spectrum", "P64", "R"))
    cn, _ = gh.device_call(blk, x, PEAKS + ("counts",))
    for o in (ex, cn):
        assert all(np.array_equal(o[k], ref[k]) for k in ("angles", "levels", "bins"))
    assert np.all(cn["counts"] == n)
    loc = handle(m, n, K, pos, snaps, mode="local_maxima")
    lo, _ = gh.device_call(loc, x, PEAKS + ("spectrum", "P64"))
    loc.close()
    assert np.array_equal(lo["spectrum"], ex["spectrum"]) and np.array_equal(lo["P64"], ex["P64"])
    blk.close()
    e = gh.entry_outputs(lambda devices=None: handle(m, n, K, pos, snaps, devices=devices), x, spectrum=True)
    h = e["host"]
    assert np.array_equal(h["angles"], ref["angles"]) and np.array_equal(h["levels"], ref["levels"]) and np.array_equal(h["bins"], ref["bins"])
    assert np.array_equal(h["spectrum"], ex["spectrum"])
    ph = e["planar_host"]
    assert np.array_equal(ph["angles"], ref["angles"]) and np.array_equal(ph["levels"], ref["levels"]) and np.array_equal(ph["bins"], ref["bins"])
    assert e["planar_launches"] == 3  # the planar covariance, eig, ESPRIT: never the fused kernel
    assert np.array_equal(e["planar_device"]["angles"], ref["angles"])
    G = torch.cuda.device_count()
    for devices in ([0], list(range(G))):
        a2 = e["multi_host%s" % devices]
        assert np.array_equal(a2["angles"], ref["angles"]) and np.array_equal(a2["levels"], ref["levels"]), devices
        g = e["multi_device%s" % devices]
        assert np.array_equal(g["angles"], ref["angles"]) and np.array_equal(g["bins"], ref["bins"]), devices
    if G < 2:
        return
    for g, sh in enumerate(e["sharded"]):
        assert np.array_equal(sh["angles"], ref["angles"][g::G]), g
        assert np.array_equal(sh["bins"], ref["bins"]), g


def test_launch_counts_and_sub_batches():
    """per sub-batch: covariance + eig + ESPRIT, +1 source count under MDL, +1 scan with the spectrum"""
    m, n, K, snaps = 4, 1, 3600, 256
    pos = ula(m, "x")
    x, _ = windows(pos, [(1, 20.0)], 3, snaps)
    for rule, spectrum, want in (("fixed", False, 3), ("mdl", False, 4), ("fixed", True, 4), ("mdl", True, 5)):
        blk = handle(m, n, K, pos, snaps, rule=rule)
        _, launches = gh.device_call(blk, x, PEAKS + (("spectrum",) if spectrum else ()))
        assert launches == want, (rule, spectrum, launches)
        blk.close()
    # several sub-batches (the internal fp64 spectrum of K bins per window bounds one); the whole call equals its halves
    Kb, Wb, Nb = 36000, 3000, 64
    xb, _ = windows(pos, [(1, 20.0)] * Wb, 809, Nb)
    blk = handle(m, n, Kb, pos, Nb)
    whole, launches = gh.device_call(blk, xb, PEAKS + ("spectrum",))
    assert launches % 4 == 0 and launches // 4 >= 2, launches
    first, _ = gh.device_call(blk, xb[: Wb // 2], PEAKS + ("spectrum",))
    second, _ = gh.device_call(blk, xb[Wb // 2:], PEAKS + ("spectrum",))
    for k in ("angles", "levels", "bins", "spectrum"):
        assert np.array_equal(whole[k], np.concatenate([first[k], second[k]])), k
    blk.close()


def test_switching_back_to_top_bins():
    """TOP_BINS after ESPRIT is byte-identical to a fresh handle and runs the fused kernel once per call at the C2 shape"""
    cfg = synth.config(2, snapshots=4096)
    x = synth.gen_windows_numpy(cfg, 12, 0, 64)
    pos = ula(4, "x")
    fresh = handle(4, 1, cfg["resolution"], pos, cfg["snapshots"], mode="top_bins")
    ref, l_ref = gh.device_call(fresh, x, PEAKS)
    fresh.close()
    blk = handle(4, 1, cfg["resolution"], pos, cfg["snapshots"])
    _, l_esprit = gh.device_call(blk, x, PEAKS)
    assert l_esprit == 3
    blk.set_peak_mode("top_bins", 0)
    got, l_top = gh.device_call(blk, x, PEAKS)
    assert l_ref == l_top == 1
    assert all(np.array_equal(got[k], ref[k]) for k in ("angles", "levels", "bins"))
    blk.close()


# ---- what the mode is for ----------------------------------------------------------------------------------------------
def test_mirror_case():
    """M = 4 x-axis ULA, sources at 40 and 110 degrees at 20 dB: ESPRIT reports both in every window"""
    m, n, K, snaps, Wn = 4, 2, 3600, 4096, 100
    pos = ula(m, "x")
    x = two_source_windows(pos, (40.0, 110.0), 20.0, snaps, Wn, 40)
    blk = handle(m, n, K, pos, snaps)
    out, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    got = np.sort(out["angles"], axis=1)
    assert np.all(np.abs(got[:, 0] - 40.0) < 1.0) and np.all(np.abs(got[:, 1] - 110.0) < 1.0), got


@pytest.mark.parametrize("m,th", [(4, (70.0, 78.0)), (8, (30.0, 36.0))])
def test_resolution(m, th):
    """0 dB, 1024 snapshots: both sources within half their separation in at least 90 % of windows"""
    n, K, snaps, Wn = 2, 3600, 1024, 200
    pos = ula(m, "x")
    x = two_source_windows(pos, th, 0.0, snaps, Wn, 7 * m)
    blk = handle(m, n, K, pos, snaps)
    out, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    got = np.sort(out["angles"], axis=1)
    ok = np.all(np.abs(got - np.array(th)[None, :]) < (th[1] - th[0]) / 2.0, axis=1)
    assert ok.mean() >= 0.9, ok.mean()


# ---- invalid combinations ----------------------------------------------------------------------------------------------
def test_invalid_combinations():
    m, n, K, snaps = 4, 1, 360, 64
    pos = ula(m, "x")
    L = _capi.load()
    blk = music_doa(m, n, m * snaps, np.ones((K, m), np.complex64), K)
    EINVAL = _capi.EINVAL
    # a set_table() table has no geometry
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
    blk.set_array_geometry(pos, LAM)
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 1) == EINVAL  # exclusion_bins must be 0
    # MVDR / Bartlett / NEWTON, in either order
    for kind, loading in (("mvdr", 0.01), ("bartlett", 0.0)):
        blk.set_estimator(kind, loading)
        assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
        blk.set_estimator("music", 0.0)
    blk.set_refine(True)
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
    blk.set_refine(False)
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == _capi.OK
    assert L.music_b200_set_estimator(blk._h, 1, 0.01) == EINVAL
    assert L.music_b200_set_estimator(blk._h, 2, 0.0) == EINVAL
    assert L.music_b200_set_refine(blk._h, 1) == EINVAL
    assert L.music_b200_set_estimator(blk._h, 0, 0.0) == _capi.OK
    # non-ULA geometries: a UCA, one element off the line, 0.6 lambda spacing
    uca = np.asarray([[0.5 * math.cos(2 * math.pi * i / m), 0.5 * math.sin(2 * math.pi * i / m)] for i in range(m)])
    bent = ula(m, "x")
    bent[2, 1] += 1e-5 * 0.5
    x, _ = windows(pos, [(1, 20.0)], 2, snaps)
    for bad in (uca, bent, ula(m, "x") * 1.2):
        blk.set_array_geometry(bad, LAM)  # set_geometry() itself keeps its behaviour
        with pytest.raises(_capi.MusicB200Error):
            gh.device_call(blk, x, PEAKS)
        assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
        blk.set_array_geometry(pos, LAM)
        assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == _capi.OK
    # set_table() after set_peak_mode(ESPRIT): the call fails, no fall-back to grid peaks
    blk.set_array_response(np.ones((K, m), np.complex64))
    with pytest.raises(_capi.MusicB200Error):
        gh.device_call(blk, x, PEAKS)
    ang = np.zeros((1, n), np.float32)
    with pytest.raises(_capi.MusicB200Error):
        blk.work(1, [x], [ang])
    with pytest.raises(ValueError):
        blk.set_peak_mode("ESPRIT")
    blk.close()
    # az-el handles
    az = music_doa_azel(m, n, m * snaps, 36, 3, (0.0, 30.0), np.c_[pos, np.zeros(m)], LAM)
    assert L.music_b200_set_peak_mode(az._h, ESPRIT, 0) == EINVAL
    with pytest.raises(_capi.MusicB200Error):
        az.set_peak_mode("esprit")
    az.close()


def test_cpp_block():
    """the C++ block through set_estimator(0) and set_peak_mode(3, 0) equals the Python block"""
    m, n, K, snaps, Wn = 8, 2, 720, 256, 16
    pos = ula(m, "oblique")
    x, _ = windows(pos, [(2, 20.0)] * Wn, 78, snaps)
    c = gh.run_cpp_block("test_block_estimator", struct.pack("<10I", m, n, m * snaps, K, Wn, 0, ESPRIT, 0, 1, 0) +
                         struct.pack("<2d", 0.0, LAM), [np.ascontiguousarray(pos, np.float64), x],
                         [("a", np.float32, Wn * n), ("l", np.float32, Wn * n), ("s", np.float32, Wn * K),
                          ("b", np.int32, Wn * n), ("c", np.int32, Wn)])
    ca, cl, cs, cb, cc = c["a"], c["l"], c["s"], c["b"], c["c"]
    blk = handle(m, n, K, pos, snaps, rule="mdl")
    ang, lvl, spec = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32), np.zeros((Wn, K), np.float32)
    blk.work(Wn, [x], [ang, lvl, spec])
    assert np.array_equal(ca, ang.ravel()) and np.array_equal(cl, lvl.ravel()) and np.array_equal(cs, spec.ravel())
    assert np.array_equal(cb, blk.last_bins().ravel()) and np.array_equal(cc, blk.last_counts())
    assert np.all(cc == 2) and np.all(cb >= 0)
    blk.close()
