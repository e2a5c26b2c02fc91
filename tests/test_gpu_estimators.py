"""GPU: the MVDR and Bartlett spectra (music_b200_set_estimator) against their fp64 definition (tests/estimator_oracle.py),
through every branch of the pipeline, and the default MUSIC path unchanged.

Every GPU result is compared with the oracle evaluated on the GPU's own covariance (d_R) and table (get_table), so what
is compared is the estimator itself."""
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, synth
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel
from gr_baz_b200.music_doa_helper import music_doa_helper
from oracle import music_oracle as mo

import azel_oracle as ao
import estimator_oracle as eo
import gpu_harness as gh
import refine_oracle as ro
from helpers import LAM, offgrid_windows as windows, positions

pytestmark = pytest.mark.gpu

P_RTOL = 1e-9
EXCL = 3
PEAKS = ("levels", "bins")
ALL = PEAKS + ("spectrum", "P64", "R")


def handle(m, n, K, pos, snaps, kind="music", loading=0.0, devices=None):
    return gh.make_block(m, n, snaps, K, pos=pos, est=(kind, loading), devices=devices)


def assert_bins_match(got, P, ref_bins, ctx):
    """equal to the oracle's bins, except where the oracle's P at the two bins agree to P_RTOL"""
    for g, r in zip(got, ref_bins):
        if g != r:
            assert g >= 0 and r >= 0 and abs(P[g] - P[r]) <= P_RTOL * abs(P[r]), (ctx, got, ref_bins)


def kinds_loadings():
    return [("mvdr", 0.0), ("mvdr", 0.01), ("bartlett", 0.0)]


# ---- P64, bins and launches ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2, 3, 4, 5, 8, 12, 16])
def test_p64_and_bins_against_oracle(m):
    """P64 within 1e-9 of the oracle on the GPU's own R, bins equal up to P ties, levels the float of P at the bin,
    and the launches of the pipeline: Bartlett runs no eigensolver, MVDR runs its preparation in its place"""
    K, snaps, W = 300, 64, 5  # K not a multiple of the 256-bin tile
    n = 1 if m == 2 else 2
    for gi, geometry in enumerate(("ula_x", "uca")):
        pos = positions(geometry, m)
        x, _ = windows(pos, [n] * W, 100 * m + gi, snaps)
        music = handle(m, n, K, pos, snaps)
        _, l_music = gh.device_call(music, x, ALL)
        table = music.array_response_c64()
        music.close()
        for kind, loading in kinds_loadings():
            ctx = (m, geometry, kind, loading)
            blk = handle(m, n, K, pos, snaps, kind, loading)
            out, launches = gh.device_call(blk, x, ALL)
            assert launches == l_music - (1 if kind == "bartlett" else 0), (ctx, launches, l_music)
            for w in range(W):
                P = eo.spectrum(out["R"][w], table, kind, loading)
                assert np.max(np.abs(out["P64"][w] - P) / np.abs(P)) <= P_RTOL, ctx
                assert np.array_equal(out["spectrum"][w], P.astype(np.float32)) or \
                    np.max(np.abs(out["spectrum"][w] - P) / np.abs(P)) <= 1e-6, ctx
                _, _, rb = eo.picks(P, n, K)
                assert_bins_match(out["bins"][w], P, rb, (ctx, w))
                for i in range(n):
                    b = out["bins"][w, i]
                    assert out["levels"][w, i] == np.float32(out["P64"][w, b]), (ctx, w, i)
                    assert out["angles"][w, i] == np.float32(b * 360.0 / K), (ctx, w, i)
            blk.close()


# ---- branches ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,loading", kinds_loadings())
@pytest.mark.parametrize("m", [4, 8, 16])
def test_branches(kind, loading, m):
    """argmax n = 1 (peak only, and with the spectrum), TOP_BINS and LOCAL_MAXIMA with exclusion, MDL (d slots
    filled), process_host and planar input, each against the oracle on the GPU's own R"""
    K, snaps, W = 720, 128, 12
    pos = positions("uca", m)
    for n in (1, 2):
        n_of = [w % (n + 1) for w in range(W)]
        x, _ = windows(pos, n_of, 7 * m + n, snaps)
        blk = handle(m, n, K, pos, snaps, kind, loading)
        table = blk.array_response_c64()
        ref, _ = gh.device_call(blk, x, ALL)
        Ps = [eo.spectrum(ref["R"][w], table, kind, loading) for w in range(W)]
        for rule in ("fixed", "mdl"):
            blk.set_source_rule(rule)
            for peak in ("top", "local"):
                ctx = (kind, loading, m, n, rule, peak)
                blk.set_peak_mode("top_bins" if peak == "top" else "local_maxima", EXCL)
                for spectrum in (False, True):
                    out, launches = gh.device_call(blk, x, PEAKS + (("spectrum",) if spectrum else ()))
                    eig = 1 if rule == "mdl" else 0  # the eigensolver runs only to count
                    cnt = 1 if rule == "mdl" else 0
                    prep = 1 if kind == "mvdr" else 0
                    topn = 0 if (n == 1 and peak == "top") else 1
                    cov = launches - eig - cnt - prep - 1 - topn
                    assert cov in (1, 2), (ctx, launches)
                    for w in range(W):
                        d = n
                        if rule == "mdl":
                            import source_count_oracle as so
                            d = so.estimate_source_count(np.linalg.eigvalsh(ref["R"][w]), snaps, n, "mdl")[0]
                        _, _, rb = eo.picks(Ps[w], n, K, peak, EXCL, d)
                        assert_bins_match(out["bins"][w], Ps[w], rb, (ctx, w))
                        assert np.all(out["bins"][w, d:] == -1), (ctx, w)
                        if spectrum:
                            assert np.max(np.abs(out["spectrum"][w] - Ps[w]) / np.abs(Ps[w])) <= 1e-6, ctx
                    # the host entry and the device entry agree byte for byte
                    ang = np.zeros((W, n), np.float32)
                    lvl = np.zeros((W, n), np.float32)
                    blk.work(W, [x], [ang, lvl])
                    assert np.array_equal(blk.last_bins(), out["bins"]), ctx
                    assert np.array_equal(ang, out["angles"]) and np.array_equal(lvl, out["levels"]), ctx
        # planar input: the same windows as m antenna streams (hop = N); R is summed in another order for m > 4
        blk.set_source_rule("fixed")
        blk.set_peak_mode("top_bins", 0)
        streams = [np.ascontiguousarray(x.reshape(W, snaps, m)[:, :, r].reshape(-1)) for r in range(m)]
        ang = np.zeros((W, n), np.float32)
        lvl = np.zeros((W, n), np.float32)
        blk.work_planar(W, streams, [ang, lvl])
        for w in range(W):
            _, _, rb = eo.picks(Ps[w], n, K)
            assert_bins_match(blk.last_bins()[w], Ps[w], rb, (kind, m, n, "planar", w))
        blk.close()


# ---- refinement --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,loading", kinds_loadings())
@pytest.mark.parametrize("m", [3, 8, 16])
def test_refine_1d(kind, loading, m):
    """refined angles and levels against the oracle's refinement of the GPU's own bins and R"""
    K, snaps, W, n = 360, 256, 8, 2
    pos = positions("uca", m)
    x, truth = windows(pos, [n] * W, 31 * m, snaps)
    blk = handle(m, n, K, pos, snaps, kind, loading)
    blk.set_peak_mode("local_maxima", EXCL)
    off, _ = gh.device_call(blk, x, ALL)
    blk.set_refine(True)
    on, _ = gh.device_call(blk, x, ALL)
    for k in ("bins", "spectrum", "P64"):
        assert np.array_equal(on[k], off[k]), k
    moved = 0
    for w in range(W):
        for i in range(n):
            b = int(on["bins"][w, i])
            if b < 0:
                continue
            r = eo.refine_slot(on["R"][w], kind, loading, pos, LAM, b, K)
            moved += not r["kept"]
            d = abs(float(on["angles"][w, i]) - float(r["angle"]))
            assert min(d, 360.0 - d) <= 1e-4, (kind, m, w, i, on["angles"][w, i], r)
            assert abs(float(on["levels"][w, i]) - float(r["level"])) <= 1e-5 * abs(float(r["level"])), (kind, m, w, i)
    assert moved > 0
    blk.close()


@pytest.mark.parametrize("kind,loading", kinds_loadings())
def test_refine_azel(kind, loading):
    m, n, W, snaps = 8, 1, 6, 512
    pos = ao.uca_xyz(m, LAM, alternate_z=True)
    grid = ao.Grid(72, 19, 0.0, 90.0)
    x, _ = ao.windows(pos, LAM, [1] * W, 5, snaps)
    blk = music_doa_azel(m, n, m * snaps, grid.n_az, grid.n_el, (grid.el_lo, grid.el_hi), pos, LAM)
    blk.set_estimator(kind, loading)
    out = [np.zeros((W, n), np.float32) for _ in range(3)]
    blk.work(W, [x], out)
    bins0 = blk.last_bins().copy()
    blk.set_refine(True)
    l0 = blk.launch_count()
    ref = [np.zeros((W, n), np.float32) for _ in range(3)]
    blk.work(W, [x], ref)
    assert blk.launch_count() > l0
    assert np.array_equal(blk.last_bins(), bins0)
    table = blk.array_response_c64()
    for w in range(W):
        R = mo.covariance(x[w], m)
        P = eo.spectrum(R, table, kind, loading)
        assert bins0[w, 0] == int(np.nanargmax(P)) or abs(P[bins0[w, 0]] - np.nanmax(P)) <= 1e-9 * np.nanmax(P)
        r = eo.refine_slot_azel(R, kind, loading, pos, LAM, int(bins0[w, 0]), grid)
        assert abs(float(ref[0][w, 0]) - float(r["azimuth"])) <= 1e-3, (kind, w, ref[0][w], r)
        assert abs(float(ref[1][w, 0]) - float(r["elevation"])) <= 1e-3, (kind, w, ref[1][w], r)
        assert abs(float(ref[2][w, 0]) - float(r["level"])) <= 1e-5 * abs(float(r["level"])), (kind, w)
    blk.close()


# ---- non-positive-definite windows ----------------------------------------------------------------------------------
def test_mvdr_non_pd_windows():
    m, n, K = 4, 1, 360
    pos = positions("uca", m)
    small = handle(m, n, K, pos, snaps=m)  # N = m snapshots: R is singular
    with pytest.raises(_capi.MusicB200Error) as e:
        small.set_estimator("mvdr", 0.0)
    assert e.value.code == _capi.EINVAL
    small.set_estimator("mvdr", 0.01)  # loading makes R_L positive definite
    small.close()
    snaps = 64
    blk = handle(m, n, K, pos, snaps, "mvdr", 0.0)
    x, _ = windows(pos, [1, 1, 1], 3, snaps)
    x[0, 5] = np.complex64(np.nan)
    x[1] = 0
    for spectrum in (False, True):
        out, _ = gh.device_call(blk, x, PEAKS + (("spectrum", "P64") if spectrum else ()))
        for w in (0, 1):
            assert out["bins"][w, 0] == -1 and out["angles"][w, 0] == 0.0 and out["levels"][w, 0] == 0.0
            if spectrum:
                assert np.all(np.isnan(out["spectrum"][w])) and np.all(np.isnan(out["P64"][w]))
        assert out["bins"][2, 0] >= 0
    blk.close()


# ---- resolution and level ----------------------------------------------------------------------------------------------
SEP = 14.0  # degrees: two sources closer than the Bartlett beamwidth (~45 degrees) of this 8-element UCA


def test_resolution():
    """M = 8 UCA, 20 dB, 1024 snapshots, two sources SEP apart, LOCAL_MAXIMA with n = 2: MVDR and MUSIC resolve the
    pair (both slots within 1 degree of the truth) in >= 90 % of the windows, Bartlett in <= 10 %"""
    m, n, K, snaps, W = 8, 2, 3600, 1024, 60
    pos = positions("uca", m)
    x, truth = windows(pos, [2] * W, 4242, snaps, sep=SEP)
    frac = {}
    for kind in ("music", "mvdr", "bartlett"):
        blk = handle(m, n, K, pos, snaps, kind)
        blk.set_peak_mode("local_maxima", 0)
        ang = np.zeros((W, n), np.float32)
        blk.work(W, [x], [ang])
        ok = 0
        for w in range(W):
            e = [min(abs((float(a) - t + 180.0) % 360.0 - 180.0) for a in ang[w]) for t in truth[w]]
            ok += max(e) <= 1.0
        frac[kind] = ok / W
        blk.close()
    assert frac["music"] >= 0.9 and frac["mvdr"] >= 0.9 and frac["bartlett"] <= 0.1, frac


@pytest.mark.parametrize("kind", ["mvdr", "bartlett"])
def test_level_is_power(kind):
    """one unit-power source per window on a grid angle, 4096 snapshots, 20 dB: the mean grid level is within 1 % of
    p + s2 / M"""
    m, n, K, snaps, W = 8, 1, 360, 4096, 40
    pos = positions("uca", m)
    rng = np.random.default_rng(77)
    noise = 0.1
    xs = []
    for w in range(W):
        t = float(rng.integers(0, K)) * 360.0 / K
        a = ro.steering(pos, LAM, np.deg2rad(t))[0]
        X = noise * (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
        X += a[:, None] * np.exp(2j * np.pi * rng.uniform(0.0, 1.0, snaps))[None, :]
        xs.append(X.T.reshape(-1))
    x = np.ascontiguousarray(np.array(xs).astype(np.complex64))
    blk = handle(m, n, K, pos, snaps, kind)
    ang = np.zeros((W, n), np.float32)
    lvl = np.zeros((W, n), np.float32)
    blk.work(W, [x], [ang, lvl])
    expect = 1.0 + noise ** 2 / m
    assert abs(float(np.mean(lvl)) - expect) <= 0.01 * expect, (float(np.mean(lvl)), expect)
    blk.close()


# ---- the default stays MUSIC, byte for byte ------------------------------------------------------------------------------
@pytest.mark.parametrize("base", [2, 5])
def test_music_restored_byte_identical(base):
    """a handle switched MUSIC -> MVDR -> MUSIC gives the outputs and launches per call of a fresh handle"""
    cfg = synth.config(base)
    W = 64
    x = synth.gen_windows_numpy(cfg, synth.BASE_SEED + 3, 0, W)
    m, n, K = cfg["m"], cfg["n"], cfg["resolution"]
    table = mo.steering_table_c64(mo.scaled_antenna_array(synth.SPACING, cfg["antenna_array"]), K, LAM)
    res = []
    for switch in (False, True):
        blk = music_doa(m, n, cfg["nsamples"], table, K)
        if switch:
            blk.set_estimator("mvdr", 0.01)
            gh.device_call(blk, x, PEAKS)
            blk.set_estimator("music")
        out, launches = gh.device_call(blk, x, PEAKS)
        res.append((out, launches))
        blk.close()
    (a, la), (b, lb) = res
    assert la == lb
    if base == 2:
        assert la == 1  # the fused M = 4 kernel
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


# ---- errors -----------------------------------------------------------------------------------------------------------
def test_errors():
    m, n, K, snaps = 4, 1, 90, 64
    pos = positions("uca", m)
    blk = handle(m, n, K, pos, snaps)
    lib = _capi.load()
    for est, loading in ((3, 0.0), (-1, 0.0), (1, -0.5), (1, float("nan")), (1, float("inf")), (0, 0.1), (2, 0.1)):
        assert lib.music_b200_set_estimator(blk._h, est, loading) == _capi.EINVAL, (est, loading)
    with pytest.raises(ValueError):
        blk.set_estimator("capon")
    assert blk.estimator == ("music", 0.0)
    # refinement needs a geometric table, for every estimator
    blk.set_estimator("bartlett")
    blk.set_array_response(np.ones((K, m), np.complex64))
    with pytest.raises(_capi.MusicB200Error) as e:
        blk.set_refine(True)
    assert e.value.code == _capi.EINVAL
    blk.close()


def test_helper_estimator_argument():
    cfg = synth.config(1)
    W = 8
    x = synth.gen_windows_numpy(cfg, synth.BASE_SEED + 5, 0, W)
    outs = {}
    for est in ("music", "bartlett"):
        h = music_doa_helper(cfg["m"], cfg["n"], cfg["nsamples"], cfg["resolution"], synth.FREQUENCY, synth.SPACING,
                             cfg["antenna_array"], estimator=est)
        ang = np.zeros((W, cfg["n"]), np.float32)
        lvl = np.zeros((W, cfg["n"]), np.float32)
        h.work(W, [x], [ang, lvl])
        outs[est] = (ang, lvl)
        assert h.impl.estimator[0] == est
    assert not np.array_equal(outs["music"][1], outs["bartlett"][1])


# ---- multi-device -----------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_multi_device_and_sharded_gather():
    m, n, K, snaps, W = 8, 1, 360, 256, 20
    pos = positions("uca", m)
    x, _ = windows(pos, [1] * W, 11, snaps)
    single = handle(m, n, K, pos, snaps, "mvdr", 0.01)
    a1, l1 = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    single.work(W, [x], [a1, l1])
    multi = handle(m, n, K, pos, snaps, "mvdr", 0.01, devices=[0, 1])
    a2, l2 = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    multi.work(W, [x], [a2, l2])
    assert np.array_equal(a1, a2) and np.array_equal(l1, l2)
    assert np.array_equal(single.last_bins(), multi.last_bins())
    # sharded entry with the fused all-gather of the bins
    for sh in gh.sharded_call(multi, x):
        assert np.array_equal(sh["bins"], single.last_bins())
    single.close()
    multi.close()


# ---- the C++ block ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,loading,refine", [("mvdr", 0.01, 0), ("bartlett", 0.0, 1)])
def test_cpp_block_estimator(kind, loading, refine):
    m, n, K, snaps, Wn = 8, 2, 360, 128, 10
    pos = positions("uca", m)
    x, _ = windows(pos, [2] * Wn, 99, snaps)
    est = music_doa.ESTIMATORS[kind]
    got = gh.run_cpp_block("test_block_estimator", struct.pack("<10I", m, n, m * snaps, K, Wn, est, 1, EXCL, 0, refine) +
                           struct.pack("<2d", loading, LAM), [np.ascontiguousarray(pos), x],
                           [("angles", np.float32, Wn * n), ("levels", np.float32, Wn * n), ("spectrum", np.float32, Wn * K),
                            ("bins", np.float32, Wn * n), ("counts", np.float32, Wn)])
    blk = handle(m, n, K, pos, snaps, kind, loading)
    blk.set_peak_mode("local_maxima", EXCL)
    blk.set_refine(bool(refine))
    ang, lvl, spec = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32), np.zeros((Wn, K), np.float32)
    blk.work(Wn, [x], [ang, lvl, spec])
    assert np.array_equal(got["angles"], ang.ravel())
    assert np.array_equal(got["levels"], lvl.ravel())
    assert np.array_equal(got["spectrum"], spec.ravel())
    assert np.array_equal(got["bins"].view(np.int32), blk.last_bins().ravel())
    blk.close()
