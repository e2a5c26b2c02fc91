"""GPU: the DML peak mode (MUSIC_B200_PEAKS_DML) against its fp64 definition (tests/dml_oracle.py), through every entry
point, on geometric, planar, calibrated, scaled and zero-row tables, and the other peak modes unchanged.

The oracle runs on the GPU's own covariance (d_R), so what is compared is the DML stage itself.  A window whose oracle
trajectory passed through a search with a relative margin <= 1e-9 (a near-tie) may take the other branch."""
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, synth
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import dml_oracle as dm
import gpu_harness as gh
import helpers
from helpers import LAM, RESOLUTION, SNAPS, angle_windows, array_wl, resolution_case, resolved, table_wl

pytestmark = pytest.mark.gpu

DML = 4
FLIP = 1e-9
PEAKS = ("levels", "bins")


def handle(tab, n, snaps, rule="fixed", mode="dml", devices=None):
    return gh.make_block(tab.shape[1], n, snaps, table=tab, rule=rule, mode=mode, devices=devices)


def tables(m, K):
    """(name, [K][m] complex64): x-axis ULA, UCA, random planar array and a calibrated UCA"""
    uca = table_wl(array_wl("uca", m), K)
    return [("ula_x", table_wl(array_wl("x", m), K)), ("uca", uca), ("planar", helpers.planar_table(m, K, 50 + m)),
            ("calibrated", helpers.calibrated_table(uca, 60 + m))]


def mixed_windows(m, tab_pos, seed, snaps=256):
    """two coherent, two uncorrelated, one single-source, one noise-only window (20 dB)"""
    rng = np.random.default_rng(seed)
    out = []
    for coherent, S in ((True, 2), (True, 2), (False, 2), (False, 3), (False, 1), (False, 0)):
        th = [rng.uniform(0.0, 360.0, S)]
        if S == 0:
            out.append(angle_windows(tab_pos, [[]], False, 1, seed + len(out), snaps=snaps))
        else:
            out.append(angle_windows(tab_pos, th, coherent, 1, seed + len(out), snaps=snaps))
    return np.concatenate(out)


def level_ok(g, r, trR):
    """within one float32 ulp of the oracle's level (or within fp64 cancellation of tr R for a level near 0)"""
    return abs(float(g) - float(r)) <= max(float(np.spacing(np.abs(np.float32(r)))), 1e-10 * trR)


def check_parity(out, R, tab, n, counts=None, ctx=()):
    """bins equal to the oracle's on the GPU's R, except after near-ties; levels within one float32 ulp; returns the
    number of near-tie windows that differ"""
    edge = 0
    for w in range(len(R)):
        d = n if counts is None else int(counts[w])
        ref = dm.work_R(R[w], tab, n, d)
        gb, ga, gl = out["bins"][w], out["angles"][w], out["levels"][w]
        if not np.array_equal(gb, ref["bins"]):
            assert ref["margin"] <= FLIP, (ctx, w, gb, ref["bins"], ref["margin"])
            edge += 1
            continue
        assert np.array_equal(ga, ref["angles"]), (ctx, w, ga, ref["angles"])
        trR = float(np.trace(R[w]).real)
        assert all(level_ok(g, r, trR) for g, r in zip(gl, ref["levels"])), (ctx, w, gl, ref["levels"])
    return edge


# ---- parity with the oracle ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2, 3, 4, 5, 8, 12, 16])
def test_parity_with_oracle(m):
    K, snaps = 360, 256
    edge = total = 0
    for ti, (name, tab) in enumerate(tables(m, K)):
        pos = array_wl("uca", m) if name in ("uca", "calibrated") else array_wl("x", m) if name == "ula_x" else None
        if pos is None:  # the planar table's own positions are not kept: sources along random table rows
            rng = np.random.default_rng(m + 5)
            vecs = [[tab[k] for k in rng.choice(K, S, replace=False)] for S in (2, 2, 1, 3, 0, 2)]
            x = helpers.source_windows(rng, vecs, m, snaps, amp=10.0)
        else:
            x = mixed_windows(m, pos, 100 * m + ti, snaps)
        for n in (1, 2, 3):
            if n >= m:
                continue
            for rule in ("fixed", "mdl"):
                blk = handle(tab, n, snaps, rule)
                out, _ = gh.device_call(blk, x, PEAKS + ("R",))
                counts = None
                if rule == "mdl":
                    cnt, _ = gh.device_call(blk, x, PEAKS + ("counts",))
                    assert np.array_equal(cnt["bins"], out["bins"]) and np.array_equal(cnt["levels"], out["levels"])
                    counts = cnt["counts"]
                blk.close()
                edge += check_parity(out, out["R"], tab, n, counts, (m, name, n, rule))
                total += len(x)
    assert edge <= 0.02 * total, (edge, total)


def test_single_source_is_the_bartlett_bin():
    """bench.py's C2 windows, n = 1: the DML bin is the Bartlett TOP_BINS bin (up to oracle near-ties)"""
    cfg = synth.config(2)
    W, K = 64, cfg["resolution"]
    x = synth.gen_windows_numpy(cfg, synth.BASE_SEED + 2, 0, W)
    tab = helpers.table_for(cfg)
    blk = handle(tab, 1, cfg["snapshots"])
    out, launches = gh.device_call(blk, x, PEAKS + ("R",))
    blk.close()
    bart = music_doa(4, 1, cfg["nsamples"], tab, K)
    bart.set_estimator("bartlett", 0.0)
    bo, _ = gh.device_call(bart, x, PEAKS)
    bart.close()
    for w in range(W):
        if out["bins"][w, 0] != bo["bins"][w, 0]:
            assert dm.work_R(out["R"][w], tab, 1)["margin"] <= FLIP, (w, out["bins"][w], bo["bins"][w])
    assert np.mean(out["bins"][:, 0] == bo["bins"][:, 0]) >= 0.95


# ---- what the mode is for ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [("uca", 8, True, 20), ("uca", 16, True, 20), ("x", 8, True, 20)])
def test_coherent_resolution(case):
    """the seeded coherent rows of the oracle's resolution table: the GPU resolves the oracle's count (up to near-ties),
    MUSIC LOCAL_MAXIMA on the same windows far fewer"""
    kind, m, coherent, sep = case
    pos, tab, x, th = resolution_case(kind, m, coherent, sep)
    K = tab.shape[0]
    blk = handle(tab, 2, SNAPS)
    out, _ = gh.device_call(blk, x, PEAKS + ("R",))
    blk.close()
    edge = check_parity(out, out["R"], tab, 2, ctx=case)
    got = sum(resolved(out["angles"][w], th[w]) for w in range(len(x)))
    music_want, dml_want = RESOLUTION[case]
    assert abs(got - dml_want) <= edge, (got, dml_want, edge)
    loc = handle(tab, 2, SNAPS, mode="local_maxima")
    lo, _ = gh.device_call(loc, x, PEAKS)
    loc.close()
    got_music = sum(resolved([a for a, b in zip(lo["angles"][w], lo["bins"][w]) if b >= 0], th[w]) for w in range(len(x)))
    assert got_music <= music_want + 2 and got_music * 3 < got, (got_music, got)


# ---- entry points ------------------------------------------------------------------------------------------------------
def test_entries_agree():
    """host, device, _ex, _counts, planar host and planar device agree byte for byte, and so do multi-device handles and
    sharded calls; spectrum, P64, R, eigenvalues and counts are a TOP_BINS handle's"""
    m, n, snaps, Wn = 8, 2, 512, 24
    pos = array_wl("uca", m)
    tab = table_wl(pos, 720)
    K = tab.shape[0]
    rng = np.random.default_rng(4)
    x = angle_windows(pos, rng.uniform(0, 360, (Wn, 2)), True, Wn, 5, snaps=snaps)
    blk = handle(tab, n, snaps)
    ref, _ = gh.device_call(blk, x, PEAKS)
    assert np.all(ref["bins"] >= 0)
    ex, _ = gh.device_call(blk, x, PEAKS + ("spectrum", "P64", "R"))
    cn, _ = gh.device_call(blk, x, PEAKS + ("counts",))
    for o in (ex, cn):
        assert all(np.array_equal(o[k], ref[k]) for k in ("angles", "levels", "bins"))
    assert np.all(cn["counts"] == n)
    top = handle(tab, n, snaps, mode="top_bins")
    to, _ = gh.device_call(top, x, PEAKS + ("spectrum", "P64", "R"))
    tc, _ = gh.device_call(top, x, PEAKS + ("counts",))
    assert all(np.array_equal(to[k], ex[k]) for k in ("spectrum", "P64", "R"))
    assert np.array_equal(tc["counts"], cn["counts"])
    evs = [gh.device_call(b, x, ("eigvals",))[0]["eigvals"] for b in (blk, top)]
    assert np.array_equal(evs[0], evs[1])
    top.close()
    blk.close()
    e = gh.entry_outputs(lambda devices=None: handle(tab, n, snaps, devices=devices), x, spectrum=True, multi_device=False)
    h = e["host"]
    assert np.array_equal(h["angles"], ref["angles"]) and np.array_equal(h["levels"], ref["levels"]) and np.array_equal(h["bins"], ref["bins"])
    assert np.array_equal(h["spectrum"], ex["spectrum"])
    ph = e["planar_host"]
    assert np.array_equal(ph["angles"], ref["angles"]) and np.array_equal(ph["levels"], ref["levels"]) and np.array_equal(ph["bins"], ref["bins"])
    assert np.array_equal(e["planar_device"]["angles"], ref["angles"])
    G = torch.cuda.device_count()
    for devices in ([0], list(range(G))):
        a2 = e["multi_host%s" % devices]
        assert np.array_equal(a2["angles"], ref["angles"]) and np.array_equal(a2["levels"], ref["levels"]), devices
    if G < 2:
        return
    for g, sh in enumerate(e["sharded"]):
        assert np.array_equal(sh["angles"], ref["angles"][g::G]), g
        assert np.array_equal(sh["bins"], ref["bins"]), g


def test_launch_counts_and_sub_batches():
    """per sub-batch: covariance + DML; the eigensolver (+ source count) only under MDL or for the spectrum, + the scan
    with the spectrum; a call of several sub-batches equals its halves"""
    m, n, snaps = 4, 1, 256
    pos = array_wl("x", m)
    tab = table_wl(pos, 3600)
    x = angle_windows(pos, [(40.0,)] * 3, False, 3, 9, snaps=snaps)
    for rule, spectrum, want in (("fixed", False, 2), ("mdl", False, 4), ("fixed", True, 4), ("mdl", True, 5)):
        blk = handle(tab, n, snaps, rule)
        _, launches = gh.device_call(blk, x, PEAKS + (("spectrum",) if spectrum else ()))
        assert launches == want, (rule, spectrum, launches)
        blk.close()
    Kb, Wb, Nb = 36000, 3000, 64
    tb = table_wl(pos, Kb)
    xb = angle_windows(pos, [(40.0,)] * Wb, False, Wb, 10, snaps=Nb)
    blk = handle(tb, n, Nb)
    whole, launches = gh.device_call(blk, xb, PEAKS + ("spectrum",))
    assert launches % 4 == 0 and launches // 4 >= 2, launches
    first, _ = gh.device_call(blk, xb[: Wb // 2], PEAKS + ("spectrum",))
    second, _ = gh.device_call(blk, xb[Wb // 2:], PEAKS + ("spectrum",))
    for k in ("angles", "levels", "bins", "spectrum"):
        assert np.array_equal(whole[k], np.concatenate([first[k], second[k]])), k
    blk.close()


def test_switching_back_to_top_bins():
    """TOP_BINS after DML is byte-identical to a fresh handle and runs the fused kernel once per call at the C2 shape"""
    cfg = synth.config(2, snapshots=4096)
    x = synth.gen_windows_numpy(cfg, 12, 0, 64)
    tab = helpers.table_for(cfg)
    K = cfg["resolution"]
    fresh = handle(tab, 1, cfg["snapshots"], mode="top_bins")
    ref, l_ref = gh.device_call(fresh, x, PEAKS)
    fresh.close()
    blk = handle(tab, 1, cfg["snapshots"])
    _, l_dml = gh.device_call(blk, x, PEAKS)
    assert l_dml == 2
    blk.set_peak_mode("top_bins", 0)
    got, l_top = gh.device_call(blk, x, PEAKS)
    assert l_ref == l_top == 1
    assert all(np.array_equal(got[k], ref[k]) for k in ("angles", "levels", "bins"))
    blk.close()


# ---- tables ----------------------------------------------------------------------------------------------------------
def test_scaled_and_zero_row_tables():
    """a table scaled by 2^s: the same bins, levels times exactly 2^(-2 s) (every s here keeps them normal); zero rows,
    placed at the sources' own bins, are never picked"""
    m, n, snaps = 8, 2, 1024
    pos, tab, x, th = resolution_case("uca", m, True, 40, W=12)
    K = tab.shape[0]
    blk = handle(tab, n, snaps)
    ref, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    assert np.all(ref["bins"] >= 0) and np.all(np.abs(ref["levels"]) > 1e-3)
    for s in (-40, -20, -3, 4, 20, 40):
        st = (tab.astype(np.complex128) * 2.0 ** s).astype(np.complex64)
        blk = handle(st, n, snaps)
        got, _ = gh.device_call(blk, x, PEAKS)
        blk.close()
        assert np.array_equal(got["bins"], ref["bins"]), s
        assert np.array_equal(got["levels"], (ref["levels"].astype(np.float64) * 2.0 ** (-2 * s)).astype(np.float32)), s
    zero = sorted(set(np.round(th.ravel() * K / 360.0).astype(int) % K))
    zt = tab.copy()
    zt[zero] = 0
    blk = handle(zt, n, snaps)
    got, _ = gh.device_call(blk, x, PEAKS + ("R",))
    blk.close()
    assert np.all(got["bins"] >= 0) and not np.isin(got["bins"], zero).any()
    check_parity(got, got["R"], zt, n, ctx="zero rows")


def test_degenerate_windows():
    """NaN and all-zero windows report (0, 0, -1); MDL with d = 0 reports no peak"""
    m, n, snaps = 4, 2, 256
    pos = array_wl("x", m)
    tab = table_wl(pos)
    x = angle_windows(pos, [(40.0, 100.0)] * 4, False, 4, 3, snaps=snaps)
    x[2] = angle_windows(pos, [[]], False, 1, 4, snaps=snaps)[0]
    x[0] = 0
    x[1, 17] = np.nan
    for rule in ("fixed", "mdl"):
        blk = handle(tab, n, snaps, rule)
        out, _ = gh.device_call(blk, x, PEAKS)
        blk.close()
        for w in ([0, 1] if rule == "fixed" else [0, 1, 2]):
            assert np.all(out["bins"][w] == -1) and np.all(out["angles"][w] == 0.0) and np.all(out["levels"][w] == 0.0), (rule, w, out)
        assert np.all(out["bins"][3] >= 0) and np.all(out["levels"][3] > 0.0)


# ---- invalid combinations ----------------------------------------------------------------------------------------------
def test_invalid_combinations():
    m, n, K, snaps = 4, 1, 360, 64
    L = _capi.load()
    EINVAL = _capi.EINVAL
    tab = helpers.planar_table(m, K, 3)
    blk = music_doa(m, n, m * snaps, tab, K)
    assert L.music_b200_set_peak_mode(blk._h, DML, 1) == EINVAL  # exclusion_bins must be 0
    for kind, loading in (("mvdr", 0.01), ("bartlett", 0.0)):
        blk.set_estimator(kind, loading)
        assert L.music_b200_set_peak_mode(blk._h, DML, 0) == EINVAL
        blk.set_estimator("music", 0.0)
    blk.set_array_geometry(array_wl("uca", m), LAM)
    blk.set_refine(True)
    assert L.music_b200_set_peak_mode(blk._h, DML, 0) == EINVAL
    blk.set_refine(False)
    assert L.music_b200_set_peak_mode(blk._h, DML, 0) == _capi.OK  # a UCA from set_geometry()
    assert L.music_b200_set_estimator(blk._h, 1, 0.01) == EINVAL
    assert L.music_b200_set_estimator(blk._h, 2, 0.0) == EINVAL
    assert L.music_b200_set_refine(blk._h, 1) == EINVAL
    assert L.music_b200_set_peak_mode(blk._h, DML, 2) == EINVAL
    blk.set_array_response(tab)  # a set_table() table is accepted, unlike under ROOTS and ESPRIT
    x = angle_windows(array_wl("x", m), [(40.0,)], False, 1, 2, snaps=snaps)
    out, _ = gh.device_call(blk, x, PEAKS)
    assert out["bins"][0, 0] >= 0
    with pytest.raises(ValueError):
        blk.set_peak_mode("DML")
    blk.close()
    az = music_doa_azel(m, n, m * snaps, 36, 3, (0.0, 30.0), np.c_[array_wl("x", m), np.zeros(m)], LAM)
    assert L.music_b200_set_peak_mode(az._h, DML, 0) == EINVAL
    with pytest.raises(_capi.MusicB200Error):
        az.set_peak_mode("dml")
    az.close()


def test_cpp_block():
    """the C++ block through set_array_response() and set_peak_mode(4, 0) equals the Python block"""
    m, n, K, snaps, Wn = 8, 2, 720, 256, 16
    pos = array_wl("uca", m)
    tab = helpers.calibrated_table(table_wl(pos, K), 8)
    x = angle_windows(pos, np.random.default_rng(8).uniform(0, 360, (Wn, 2)), True, Wn, 78, snaps=snaps)
    c = gh.run_cpp_block("test_block_dml", struct.pack("<6I", m, n, m * snaps, K, Wn, 0), [tab, x],
                         [("a", np.float32, Wn * n), ("l", np.float32, Wn * n), ("s", np.float32, Wn * K),
                          ("b", np.int32, Wn * n), ("c", np.int32, Wn)])
    ca, cl, cs, cb, cc = c["a"], c["l"], c["s"], c["b"], c["c"]
    blk = handle(tab, n, snaps)
    ang, lvl, spec = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32), np.zeros((Wn, K), np.float32)
    blk.work(Wn, [x], [ang, lvl, spec])
    assert np.array_equal(ca, ang.ravel()) and np.array_equal(cl, lvl.ravel()) and np.array_equal(cs, spec.ravel())
    assert np.array_equal(cb, blk.last_bins().ravel()) and np.array_equal(cc, blk.last_counts())
    assert np.all(cc == 2) and np.all(cb >= 0)
    blk.close()
