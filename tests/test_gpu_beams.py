"""GPU: beamformed source signals (music_b200_set_beamformer, music_b200_process_*_beams) against their fp64 definition
(tests/beams_oracle.py), through every entry point.

The oracle runs on the GPU's own covariance (process_device_ex with d_R on the same windows) and the GPU's own angles and
bins, so what is compared is the weight solver and the apply pass themselves."""
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, synth
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import beams_oracle as bo
import gpu_harness as gh
import helpers
import refine_oracle as ro
from helpers import LAM, array_wl, check_beams, check_weights, circ, table_wl, ula

pytestmark = pytest.mark.gpu

RULES = {"das": (bo.DAS, 0.0), "mvdr": (bo.MVDR, 0.01), "mvdr0": (bo.MVDR, 0.0), "lcmv": (bo.LCMV, 0.0)}
PEAKS = ("levels", "bins")
BEAMS = PEAKS + ("counts", "weights", "beams")


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
    return gh.make_block(m, n, snaps, K, table=table, pos=pos, est=est, rule=rule, mode=mode, refine=refine, devices=devices)


def tables(m, K):
    """(name, table or None, positions or None): geometric x-axis ULA and UCA, random planar and calibrated tables"""
    uca = array_wl("uca", m)
    return [("ula", None, ula(m, "x")), ("uca", None, uca), ("planar", helpers.planar_table(m, K, 50 + m), None),
            ("calibrated", helpers.calibrated_table(table_wl(uca, K), 60 + m), None)]


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
                ref, _ = gh.device_call(blk, x, PEAKS + ("R",))
                for bname, (brule, loading) in RULES.items():
                    ctx = (m, name, n, mode, rule, est, refine, bname)
                    blk.set_beamformer(bname.rstrip("0"), loading)
                    out, _ = gh.device_call(blk, x, BEAMS)
                    for k in ("angles", "levels", "bins"):
                        assert np.array_equal(out[k], ref[k]), (ctx, k)
                    check_weights(out["weights"], ref["R"], out, brule, loading, tab, pos, ctx)
                    check_beams(x, out["weights"], out["beams"])
                blk.close()


# ---- invariants ------------------------------------------------------------------------------------------------------
def test_peak_outputs_match_ex_with_R():
    """angles, levels, spectrum, bins and counts are byte-identical to process_device_ex(d_R) / _counts"""
    m, n, snaps, K = 8, 2, 512, 720
    pos = array_wl("uca", m)
    x = geo_windows(pos, mixed_plan(np.random.default_rng(1)) * 3, 2, snaps)
    for mode, rule in (("top_bins", "fixed"), ("local_maxima", "mdl"), ("dml", "fixed")):
        blk = handle(m, n, snaps, K, pos=pos, mode=mode, rule=rule)
        ref, _ = gh.device_call(blk, x, PEAKS + ("spectrum", "R"))
        cnt, _ = gh.device_call(blk, x, PEAKS + ("counts",))
        for kind in ("das", "lcmv"):
            blk.set_beamformer(kind, 0.0)
            out, _ = gh.device_call(blk, x, BEAMS + ("spectrum",))
            for k in ("angles", "levels", "bins", "spectrum"):
                assert np.array_equal(out[k], ref[k]), (mode, kind, k)
            assert np.array_equal(out["counts"], cnt["counts"])
        blk.close()


@pytest.mark.parametrize("k", [-40, 40])
def test_power_of_two_input_scaling(k):
    """input x 2^k: bit-identical weights, beams scaled by exactly 2^k"""
    m, n, snaps, K = 8, 2, 256, 360
    pos = array_wl("uca", m)
    x = geo_windows(pos, [((40.0, 170.0), 20.0)] * 4, 3, snaps)
    xs = (x.astype(np.complex128) * 2.0 ** k).astype(np.complex64)
    for kind, loading in (("das", 0.0), ("mvdr", 0.0), ("mvdr", 0.1), ("lcmv", 0.0)):
        blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima")
        blk.set_beamformer(kind, loading)
        a, _ = gh.device_call(blk, x, BEAMS)
        b, _ = gh.device_call(blk, xs, BEAMS)
        blk.close()
        assert np.array_equal(a["bins"], b["bins"]) and np.array_equal(a["angles"], b["angles"])
        assert np.any(a["weights"] != 0)
        assert np.array_equal(a["weights"], b["weights"]), kind
        assert np.array_equal((a["beams"].astype(np.complex128) * 2.0 ** k).astype(np.complex64), b["beams"]), kind


def test_zeros():
    """unfilled slots and a NaN window give zero weights and beams; so does a dead-antenna window under MVDR and LCMV with
    loading 0 (its R_L has a zero pivot), while DAS still steers at the slots the peak stage filled there"""
    m, n, snaps, K = 4, 3, 256, 360
    pos = array_wl("uca", m)
    x = geo_windows(pos, [((50.0,), 20.0)] * 4, 4, snaps)
    x[1, 5] = np.nan
    x[2].reshape(snaps, m)[:, 2] = 0  # antenna 2 dead
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima", rule="mdl")
    for kind in ("das", "mvdr", "lcmv"):
        blk.set_beamformer(kind, 0.0)
        out, _ = gh.device_call(blk, x, BEAMS)
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
        out, _ = gh.device_call(blk, x, BEAMS)
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
    out, _ = gh.device_call(blk, x, BEAMS)
    assert np.all(out["bins"] >= 0) and np.all(out["bins"].sum(axis=1) % 360 == 0), out["bins"]
    assert np.all(out["weights"] == 0) and np.all(out["beams"] == 0)
    blk.set_beamformer("mvdr", 0.0)
    out, _ = gh.device_call(blk, x, BEAMS)
    assert np.all(out["weights"] != 0)
    blk.close()


# ---- physics ---------------------------------------------------------------------------------------------------------
def test_single_source_waveform():
    """one source at 40 dB: the DAS and MVDR beams reproduce its waveform (|normalised correlation| at least the oracle's
    on the same windows minus 1e-6, and above 0.99).  The angles are refined off the grid: at this SNR an MVDR beam
    steered half a grid bin off the source suppresses it (the signal is in R)."""
    m, snaps, K, Wn = 8, 1024, 3600, 16
    pos = array_wl("uca", m)
    rng = np.random.default_rng(21)
    th = rng.uniform(0.0, 360.0, Wn)
    sig = (rng.standard_normal((Wn, snaps)) + 1j * rng.standard_normal((Wn, snaps))) / np.sqrt(2.0)
    noise = (rng.standard_normal((Wn, m, snaps)) + 1j * rng.standard_normal((Wn, m, snaps))) / np.sqrt(2.0)
    X = noise + 100.0 * np.array([ro.steering(pos, LAM, math.radians(t))[0][:, None] * sig[w][None, :] for w, t in enumerate(th)])
    x = np.ascontiguousarray(X.transpose(0, 2, 1).reshape(Wn, -1).astype(np.complex64))
    corr = lambda y, s: abs(np.vdot(y, s)) / (np.linalg.norm(y) * np.linalg.norm(s))
    for kind in ("das", "mvdr"):
        blk = handle(m, 1, snaps, K, pos=pos, refine=True)
        ref, _ = gh.device_call(blk, x, PEAKS + ("R",))
        blk.set_beamformer(kind, 0.0)
        out, _ = gh.device_call(blk, x, BEAMS)
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
    pos = array_wl("uca", m)
    rng = np.random.default_rng(31)
    plan = []
    for _ in range(Wn):
        t0 = rng.uniform(0.0, 360.0)
        plan.append(((t0, (t0 + rng.choice([-1.0, 1.0]) * rng.uniform(15.0, 25.0)) % 360.0), 20.0))
    x = geo_windows(pos, plan, 32, snaps)
    steer = lambda t: ro.steering(pos, LAM, math.radians(t))[0]
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima", refine=True)
    ref, _ = gh.device_call(blk, x, PEAKS + ("R",))
    sir = {}
    for kind in ("das", "mvdr", "lcmv"):
        blk.set_beamformer(kind, 0.0)
        out, _ = gh.device_call(blk, x, BEAMS)
        got, want = np.full((Wn, n), np.nan), np.full((Wn, n), np.nan)  # NaN: the window did not resolve both sources
        for w, (truth, _) in enumerate(plan):
            own = [int(np.argmin([circ(out["angles"][w, i], t) for t in truth])) for i in range(n)]
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
    pos = array_wl("uca", m)
    x = geo_windows(pos, mixed_plan(np.random.default_rng(41)) * 7, 42, snaps)[:Wn]
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima", rule="mdl")
    blk.set_beamformer("lcmv", 0.05)
    assert blk.beamformer() == ("lcmv", 0.05)
    ref, _ = gh.device_call(blk, x, BEAMS + ("spectrum",))
    got = gh.host_call(blk, x, spectrum=True)
    for k in ("angles", "levels", "bins", "counts", "spectrum", "weights", "beams"):
        assert np.array_equal(got[k], ref[k]), k
    blk.set_beamformer("off")
    assert gh.host_call(blk, x)["beams"] is None
    blk.close()
    G = torch.cuda.device_count()
    for devices in ([0], list(range(G))) if G > 1 else ([0],):
        mb = handle(m, n, snaps, K, pos=pos, mode="local_maxima", rule="mdl", devices=devices)
        mb.set_beamformer("lcmv", 0.05)
        got = gh.host_call(mb, x)
        mb.close()
        for k in ("angles", "levels", "bins", "counts", "weights", "beams"):
            assert np.array_equal(got[k], ref[k]), (devices, k)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_device_host_entry():
    m, n, snaps, K, Wn = 4, 1, 256, 360, 33
    pos = array_wl("uca", m)
    x = geo_windows(pos, [((t,), 20.0) for t in np.linspace(0, 350, Wn)], 43, snaps)
    one = handle(m, n, snaps, K, pos=pos)
    one.set_beamformer("mvdr", 0.0)
    ref = gh.host_call(one, x)
    one.close()
    mb = handle(m, n, snaps, K, pos=pos, devices=list(range(torch.cuda.device_count())))
    mb.set_beamformer("mvdr", 0.0)
    got = gh.host_call(mb, x)
    mb.close()
    for k in ("angles", "bins", "weights", "beams"):
        assert np.array_equal(got[k], ref[k]), k


def test_launch_counts_and_sub_batches():
    """the ex(R) plan plus 2 launches per sub-batch (1 without beams); a call of several sub-batches equals its halves"""
    m, n, snaps = 4, 2, 256
    pos = array_wl("uca", m)
    x = geo_windows(pos, [((40.0, 200.0), 20.0)] * 3, 51, snaps)
    blk = handle(m, n, snaps, 360, pos=pos, mode="local_maxima")
    _, l_ex = gh.device_call(blk, x, PEAKS + ("R",))
    blk.set_beamformer("das")
    _, l_both = gh.device_call(blk, x, PEAKS + ("weights", "beams"))  # (counts under FIXED add a fill launch)
    _, l_w = gh.device_call(blk, x, PEAKS + ("weights",))
    _, l_b = gh.device_call(blk, x, ("levels", "beams"))
    blk.close()
    assert (l_both, l_w, l_b) == (l_ex + 2, l_ex + 1, l_ex + 2), (l_ex, l_both, l_w, l_b)
    Kb, Wb, Nb = 36000, 3000, 64
    xb = geo_windows(pos, [((40.0, 200.0), 20.0)] * Wb, 52, Nb)
    blk = handle(m, n, Nb, Kb, pos=pos, mode="local_maxima")
    _, l_ex = gh.device_call(blk, xb, PEAKS + ("R",))
    blk.set_beamformer("mvdr", 0.0)
    whole, launches = gh.device_call(blk, xb, PEAKS + ("weights", "beams"))
    assert (launches - l_ex) % 2 == 0 and (launches - l_ex) // 2 >= 2, (launches, l_ex)
    first, _ = gh.device_call(blk, xb[: Wb // 2], PEAKS + ("weights", "beams"))
    second, _ = gh.device_call(blk, xb[Wb // 2:], PEAKS + ("weights", "beams"))
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
    ref, l_ref = gh.device_call(fresh, x, PEAKS)
    fresh.set_beamformer("mvdr", 0.1)
    got, l_got = gh.device_call(fresh, x, PEAKS)
    fresh.close()
    assert l_ref == l_got == 1
    assert all(np.array_equal(got[k], ref[k]) for k in ("angles", "levels", "bins"))


def test_invalid_arguments():
    m, n, K, snaps = 4, 1, 360, 64
    L = _capi.load()
    EINVAL, OK = _capi.EINVAL, _capi.OK
    blk = handle(m, n, snaps, K, pos=array_wl("uca", m))
    h = blk._h
    for rule, loading in ((4, 0.0), (-1, 0.0), (2, float("nan")), (2, float("inf")), (3, -1.0), (0, 0.5), (1, 0.5)):
        assert L.music_b200_set_beamformer(h, rule, loading) == EINVAL, (rule, loading)
    assert blk.beamformer() == ("off", 0.0)
    with pytest.raises(ValueError):
        blk.set_beamformer("capon")
    x = geo_windows(array_wl("uca", m), [((30.0,), 20.0)] * 2, 61, snaps)
    with pytest.raises(_capi.MusicB200Error):  # rule OFF
        gh.device_call(blk, x, BEAMS)
    blk.set_beamformer("das")
    dev = torch.device("cuda:0")
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)
    ang = torch.zeros((2, n), dtype=torch.float32, device=dev)
    with pytest.raises(_capi.MusicB200Error):  # neither weights nor beams
        blk.process_device_beams(d_in.data_ptr(), 2, ang.data_ptr(), stream=gh.stream())
    wb = torch.zeros(2 * n * m * 2 + 2, dtype=torch.float64, device=dev)
    bb = torch.zeros(2 * n * snaps * 2 + 2, dtype=torch.float32, device=dev)
    call = lambda wp, bp: L.music_b200_process_device_beams(h, d_in.data_ptr(), 2, ang.data_ptr(), None, None, None, None, wp, bp, None)
    assert call(wb.data_ptr() + 8, None) == EINVAL  # weights 8-byte aligned only
    assert call(None, bb.data_ptr() + 4) == EINVAL  # beams 4-byte aligned only
    assert call(wb.data_ptr() + 16, bb.data_ptr() + 8) == OK
    torch.cuda.synchronize()
    blk.close()
    # N <= m: MVDR and LCMV need loading
    small = handle(m, n, m, K, pos=array_wl("uca", m))
    for rule in (2, 3):
        assert L.music_b200_set_beamformer(small._h, rule, 0.0) == EINVAL
        assert L.music_b200_set_beamformer(small._h, rule, 0.1) == OK
    assert L.music_b200_set_beamformer(small._h, 1, 0.0) == OK
    small.close()
    az = music_doa_azel(m, n, m * snaps, 36, 3, (0.0, 30.0), np.c_[array_wl("x", m), np.zeros(m)], LAM)
    assert L.music_b200_set_beamformer(az._h, 1, 0.0) == EINVAL
    az.close()


def test_cpp_block():
    """the C++ block's set_beamformer() and last_beams() equal the Python block's"""
    m, n, K, snaps, Wn = 8, 2, 720, 256, 16
    pos = array_wl("uca", m)
    rng = np.random.default_rng(71)
    x = geo_windows(pos, [((t, (t + 120.0) % 360.0), 20.0) for t in rng.uniform(0, 360, Wn)], 72, snaps)
    N = snaps
    c = gh.run_cpp_block("test_block_beams", struct.pack("<7I", m, n, m * snaps, K, Wn, 1, 3) + struct.pack("<2d", 0.01, LAM),
                         [np.ascontiguousarray(pos, np.float64), x],
                         [("a", np.float32, Wn * n), ("l", np.float32, Wn * n), ("s", np.float32, Wn * K), ("b", np.int32, Wn * n),
                          ("beams", np.complex64, Wn * n * N)])
    ca, cl, cs, cb, cbeams = c["a"], c["l"], c["s"], c["b"], c["beams"]
    blk = handle(m, n, snaps, K, pos=pos, mode="local_maxima")
    blk.set_beamformer("lcmv", 0.01)
    got = gh.host_call(blk, x, spectrum=True)
    blk.close()
    assert np.array_equal(ca, got["angles"].ravel()) and np.array_equal(cl, got["levels"].ravel())
    assert np.array_equal(cs, got["spectrum"].ravel()) and np.array_equal(cb, got["bins"].ravel())
    assert np.array_equal(cbeams, got["beams"].ravel())
    assert np.any(cbeams != 0)
