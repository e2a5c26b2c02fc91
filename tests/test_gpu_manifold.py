"""GPU: the manifold-separation root-MUSIC peak mode (MUSIC_B200_PEAKS_MANIFOLD) on uniform circular and random planar
arrays against its fp64 definition (tests/manifold_oracle.py: the FFT of the direct MUSIC denominator and
numpy.roots), through every entry point and mode combination, and its refusals.

The oracle runs on the GPU's own covariance (d_R), so what is compared is the manifold stage itself."""
import math

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import gpu_harness as gh
import manifold_oracle as mf
from helpers import LAM, PLAN, circ, near_half, plan_windows as windows, random_gains, corrupt

pytestmark = pytest.mark.gpu

FLIP = 1e-9     # selections the oracle sees this close to flipping may go either way
L_RTOL = 1e-5
PEAKS = ("levels", "bins")


def uca(m, spacing_wl=0.5):
    return mf.uca(m, spacing_wl, LAM)


def planar(m, seed, aperture_wl=2.5):
    rng = np.random.default_rng(seed)
    r = 0.5 * aperture_wl * LAM * np.sqrt(rng.uniform(0.0, 1.0, m))
    a = rng.uniform(0.0, 2 * math.pi, m)
    return np.c_[r * np.cos(a), r * np.sin(a)]


def handle(m, n, K, pos, snaps, mode="manifold", rule="fixed", devices=None, **kw):
    return gh.make_block(m, n, snaps, K, pos=pos, rule=rule, mode=mode, devices=devices, **kw)


def check_window(ga, gl, gb, ref, d, K, ctx):
    """one window against the oracle: True when compared, False when the selection is at a flip margin"""
    assert np.all(gb[d:] == -1) and np.all(ga[d:] == 0.0) and np.all(gl[d:] == 0.0), ctx
    if ref["margin"] <= FLIP and not np.array_equal(gb, ref["bins"]):
        return False
    assert np.all(gb[:d] >= 0), (ctx, gb)  # every root converged
    for i in range(d):
        ra = ref["angles"][i]
        tol = 2.0 * float(np.spacing(np.float32(max(abs(float(ra)), abs(float(ga[i])), 1e-3))))
        assert circ(ga[i], ra) <= tol, (ctx, i, ga, ref["angles"])
        assert abs(float(gl[i]) - float(ref["levels"][i])) <= L_RTOL * abs(float(ref["levels"][i])), (ctx, i, gl, ref["levels"])
        if gb[i] != ref["bins"][i]:
            assert near_half(float(ra), K), (ctx, i, gb, ref["bins"])
    return True


# ---- parity with the oracle ------------------------------------------------------------------------------------------
GEOMETRIES = [("uca", m) for m in (3, 4, 5, 8, 12, 16)] + [("planar", 5), ("planar", 8), ("planar", 12)]


@pytest.mark.parametrize("kind,m", GEOMETRIES)
def test_parity_with_oracle(kind, m):
    """angles within 2 float32 ulps, levels within 1e-5, bins equal (except at half-bin ties), every slot of a
    non-degenerate window filled, counts equal to a TOP_BINS handle's under MDL; noiseless windows within 5e-4
    degrees of the truth"""
    snaps = 512
    pos = uca(m) if kind == "uca" else planar(m, 40 + m)
    edge = total = 0
    for n in (1, 2, 3):
        if n >= m:
            continue
        plan = [(min(S, m - 1), snr) for S, snr in PLAN]
        x, truth = windows(pos, plan, 2000 * m + 10 * n + len(kind), snaps)
        for rule in ("fixed", "mdl"):
            K = 3600 if (n + len(kind)) % 2 else 360
            blk = handle(m, n, K, pos, snaps, rule=rule)
            out, _ = gh.device_call(blk, x, PEAKS + ("R",))
            counts = None
            if rule == "mdl":
                cnt, _ = gh.device_call(blk, x, PEAKS + ("counts",))
                top = handle(m, n, K, pos, snaps, mode="top_bins", rule=rule)
                tc, _ = gh.device_call(top, x, PEAKS + ("counts",))
                top.close()
                assert np.array_equal(cnt["counts"], tc["counts"]), (kind, m, n)
                assert np.array_equal(cnt["angles"], out["angles"]) and np.array_equal(cnt["bins"], out["bins"])
                counts = tc["counts"]
            blk.close()
            for w in range(len(x)):
                ctx = (kind, m, n, rule, K, w, plan[w])
                d = n if counts is None else int(counts[w])
                ga, gl, gb = out["angles"][w], out["levels"][w], out["bins"][w]
                if plan[w][1] is None:
                    # noiseless: a noise subspace inside the null space of R is unique only for d = the source count,
                    # and with a single noise vector D can have zeros besides the sources
                    if d != len(truth[w]) or m - d < 2:
                        continue
                    got = sorted(float(a) for a in ga[:d])
                    want = sorted(float(t) % 360.0 for t in truth[w])
                    assert max(circ(g, t) for g, t in zip(got, want)) <= 5e-4, (ctx, got, want)
                    continue
                ref = mf.work_R(out["R"][w], pos, LAM, K, n, d=d)
                total += d
                if not check_window(ga, gl, gb, ref, d, K, ctx):
                    edge += d
    assert edge <= 0.01 * max(total, 1), (edge, total)


def test_convergence_on_seeded_windows():
    """no non-converged window: every slot of 2000 seeded noisy UCA 16 windows (1 to 3 sources, 0 to 40 dB) is filled"""
    m, n, K, snaps = 16, 3, 3600, 256
    pos = uca(m)
    rng = np.random.default_rng(9)
    plan = [(int(rng.integers(1, 4)), float(rng.choice([0.0, 10.0, 20.0, 40.0]))) for _ in range(2000)]
    x, _ = windows(pos, plan, 99, snaps)
    blk = handle(m, n, K, pos, snaps)
    out, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    assert np.all(out["bins"] >= 0) and np.all(out["levels"] > 0.0)


def test_degenerate_windows():
    """NaN and all-zero windows report (0, 0, -1); MDL with d = 0 reports no peak; every element at one point
    (P = 0) reports no peak"""
    m, n, K, snaps = 5, 2, 360, 256
    pos = uca(m)
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
    blk = handle(m, n, K, np.zeros((m, 2)), snaps)
    out, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    assert np.all(out["bins"] == -1) and np.all(out["angles"] == 0.0) and np.all(out["levels"] == 0.0)


# ---- entry points ------------------------------------------------------------------------------------------------------
def test_entries_agree_and_launches():
    """host, device, _ex, _counts, planar, multi-device and sharded agree byte for byte; with the spectrum port the
    spectrum and P64 are a LOCAL_MAXIMA handle's, byte for byte; a call runs covariance, eigensolver and the manifold
    kernel (+ the source count under MDL, + the scan for the spectrum)"""
    m, n, K, snaps, Wn = 8, 2, 3600, 1024, 24
    pos = uca(m)
    x, _ = windows(pos, [(2, 20.0)] * Wn, 31, snaps)
    blk = handle(m, n, K, pos, snaps)
    ref, launches = gh.device_call(blk, x, PEAKS)
    assert launches == 3
    assert np.all(ref["bins"] >= 0)
    ex, launches = gh.device_call(blk, x, PEAKS + ("spectrum", "P64", "R"))
    assert launches == 4
    cn, _ = gh.device_call(blk, x, PEAKS + ("counts",))
    for o in (ex, cn):
        assert all(np.array_equal(o[k], ref[k]) for k in ("angles", "levels", "bins"))
    assert np.all(cn["counts"] == n)
    loc = handle(m, n, K, pos, snaps, mode="local_maxima")
    lo, _ = gh.device_call(loc, x, PEAKS + ("spectrum", "P64"))
    loc.close()
    assert np.array_equal(lo["spectrum"], ex["spectrum"]) and np.array_equal(lo["P64"], ex["P64"])
    blk.close()
    for rule, spectrum, want in (("mdl", False, 4), ("mdl", True, 5)):
        b = handle(m, n, K, pos, snaps, rule=rule)
        _, launches = gh.device_call(b, x, PEAKS + (("spectrum",) if spectrum else ()))
        b.close()
        assert launches == want, (rule, spectrum, launches)
    e = gh.entry_outputs(lambda devices=None: handle(m, n, K, pos, snaps, devices=devices), x, spectrum=True)
    h = e["host"]
    assert np.array_equal(h["angles"], ref["angles"]) and np.array_equal(h["levels"], ref["levels"]) and np.array_equal(h["bins"], ref["bins"])
    assert np.array_equal(h["spectrum"], ex["spectrum"])
    ph = e["planar_host"]
    assert np.array_equal(ph["angles"], ref["angles"]) and np.array_equal(ph["levels"], ref["levels"]) and np.array_equal(ph["bins"], ref["bins"])
    assert e["planar_launches"] == 4  # the planar covariance (two launches at M = 8), eig, manifold: never a fused kernel
    assert np.array_equal(e["planar_device"]["angles"], ref["angles"])
    G = torch.cuda.device_count()
    for devices in ([0], list(range(G))):
        a2 = e["multi_host%s" % devices]
        assert np.array_equal(a2["angles"], ref["angles"]) and np.array_equal(a2["levels"], ref["levels"]), devices
        g = e["multi_device%s" % devices]
        assert np.array_equal(g["angles"], ref["angles"]) and np.array_equal(g["bins"], ref["bins"]), devices
    if G > 1:
        for g, sh in enumerate(e["sharded"]):
            assert np.array_equal(sh["angles"], ref["angles"][g::G]), g
            assert np.array_equal(sh["bins"], ref["bins"]), g


# ---- combinations -----------------------------------------------------------------------------------------------------
def test_calibration_and_beams():
    """with calibration set the outputs are the oracle's on the corrected R; the beams entry's peak outputs are
    process_device_ex's byte for byte"""
    m, n, K, snaps, Wn = 8, 2, 3600, 512, 16
    pos = uca(m)
    g = random_gains(np.random.default_rng(4), m)
    x, _ = windows(pos, [(2, 20.0)] * Wn, 41, snaps)
    blk = handle(m, n, K, pos, snaps, calibration=g)
    out, _ = gh.device_call(blk, corrupt(x, g), PEAKS + ("R",))
    blk.close()
    for w in range(Wn):
        ref = mf.work_R(out["R"][w], pos, LAM, K, n)
        check_window(out["angles"][w], out["levels"][w], out["bins"][w], ref, n, K, ("calib", w))
    blk = handle(m, n, K, pos, snaps, beamformer=("das", 0.0))
    plain, _ = gh.device_call(blk, x, PEAKS)
    bm, _ = gh.device_call(blk, x, PEAKS + ("weights", "beams"))
    blk.close()
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(plain[k], bm[k]), k
    assert np.all(plain["bins"] >= 0)


def test_coherent_channel_handle():
    """a COHERENT music_doa_channels handle equals the oracle on the focused covariance it returns, with the reference
    channel's geometry and wavelength"""
    import channels_oracle as ch
    import focus_oracle as fo
    from test_gpu_focus import FC, FS, device_call, make, path_windows

    m, n, K, F, J, first, C, W = 8, 2, 360, 16, 8, 12, 8, 8
    lam_ref = ch.wavelengths(F, first, C, FC, FS)[fo.ref_channel(C)]
    pos = mf.uca(m, 0.5, lam_ref)
    blk = make(m, n, F * J, K, F, first, C, pos)
    blk.set_peak_mode("manifold", 0)
    x = path_windows(W, pos, F * J, 905, degs=(35.0, 120.0))
    got, _ = device_call(blk, x, ("levels", "bins", "R"))
    blk.close()
    compared = 0
    for w in range(W):
        ref = mf.work_R(got["R"][w], pos, lam_ref, K, n)
        compared += check_window(got["angles"][0, w], got["levels"][0, w], got["bins"][0, w], ref, n, K, ("coherent", w))
    assert compared >= W // 2, compared


# ---- retune and switching --------------------------------------------------------------------------------------------
def test_retune_and_switch_back():
    """set_geometry() to another UCA radius between calls gives the new geometry's answers (a fresh handle's, byte for
    byte, and the oracle's); TOP_BINS afterwards gives a fresh handle's outputs byte for byte"""
    m, n, K, snaps, Wn = 8, 2, 3600, 512, 12
    a, b = uca(m), uca(m, 0.35)
    x, _ = windows(b, [(2, 20.0)] * Wn, 61, snaps)
    blk = handle(m, n, K, a, snaps)
    gh.device_call(blk, x, PEAKS)
    blk.set_array_geometry(b, LAM)
    got, _ = gh.device_call(blk, x, PEAKS + ("R",))
    fresh = handle(m, n, K, b, snaps)
    want, _ = gh.device_call(fresh, x, PEAKS)
    fresh.close()
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(got[k], want[k]), k
    for w in range(Wn):
        ref = mf.work_R(got["R"][w], b, LAM, K, n)
        check_window(got["angles"][w], got["levels"][w], got["bins"][w], ref, n, K, ("retune", w))
    blk.set_peak_mode("top_bins", 0)
    top, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    fresh = handle(m, n, K, b, snaps, mode="top_bins")
    want, _ = gh.device_call(fresh, x, PEAKS)
    fresh.close()
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(top[k], want[k]), k


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_refusals():
    """exclusion_bins != 0, MVDR / Bartlett, NEWTON, a set_table() table, an aperture above the order cap, az-el and
    SEPARATE / INCOHERENT channel handles: EINVAL, in either order"""
    m, n, K, snaps = 8, 1, 360, 64
    pos = uca(m)
    L = _capi.load()
    EINVAL, MF = _capi.EINVAL, 5
    blk = music_doa(m, n, m * snaps, np.ones((K, m), np.complex64), K)
    assert L.music_b200_set_peak_mode(blk._h, MF, 0) == EINVAL  # a set_table() table has no geometry
    blk.set_array_geometry(pos, LAM)
    assert L.music_b200_set_peak_mode(blk._h, MF, 1) == EINVAL
    for kind, loading in (("mvdr", 0.01), ("bartlett", 0.0)):
        blk.set_estimator(kind, loading)
        assert L.music_b200_set_peak_mode(blk._h, MF, 0) == EINVAL
        blk.set_estimator("music", 0.0)
    blk.set_refine(True)
    assert L.music_b200_set_peak_mode(blk._h, MF, 0) == EINVAL
    blk.set_refine(False)
    assert L.music_b200_set_peak_mode(blk._h, MF, 0) == _capi.OK
    assert L.music_b200_set_estimator(blk._h, 1, 0.01) == EINVAL
    assert L.music_b200_set_estimator(blk._h, 2, 0.0) == EINVAL
    assert L.music_b200_set_refine(blk._h, 1) == EINVAL
    x, _ = windows(pos, [(1, 20.0)], 2, snaps)
    # an aperture above the cap: set_geometry() keeps its behaviour, the mode refuses the table
    wide = pos * 4.0
    blk.set_array_geometry(wide, LAM)
    with pytest.raises(_capi.MusicB200Error, match="wavelengths"):
        gh.device_call(blk, x, PEAKS)
    assert L.music_b200_set_peak_mode(blk._h, MF, 0) == EINVAL
    blk.set_array_geometry(pos, LAM)
    assert L.music_b200_set_peak_mode(blk._h, MF, 0) == _capi.OK
    gh.device_call(blk, x, PEAKS)
    # set_table() after set_peak_mode(MANIFOLD): the call fails, no fall-back to grid peaks
    blk.set_array_response(np.ones((K, m), np.complex64))
    with pytest.raises(_capi.MusicB200Error):
        gh.device_call(blk, x, PEAKS)
    with pytest.raises(_capi.MusicB200Error):
        blk.work(1, [x], [np.zeros((1, n), np.float32)])
    blk.close()
    az = music_doa_azel(m, n, m * snaps, 36, 3, (0.0, 30.0), np.c_[pos, np.zeros(m)], LAM)
    assert L.music_b200_set_peak_mode(az._h, MF, 0) == EINVAL
    az.close()
    from test_gpu_focus import make
    for combine in ("separate", "incoherent"):
        ch = make(4, 1, 16 * 8, 360, 16, 12, 4, mf.uca(4, 0.5, 0.7), combine=combine)
        assert L.music_b200_set_peak_mode(ch._h, MF, 0) == EINVAL, combine
        ch.close()
