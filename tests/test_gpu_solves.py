"""GPU: the Cholesky-based solvers (the MVDR preparation and scan, the MVDR and LCMV beam weights, the DML searches and
levels) against the mpmath reference, bounds and decision bands of tests/solve_oracle.py, on the GPU's own covariance
(d_R) and the table rows as installed, for M in {2, 3, 4, 5, 8, 12, 16}.

The mp reference evaluates D_k on every STRIDE-th bin of the K = 48 bin table plus the reported slots and the four
largest P64 of each window (solve_oracle.strided_bins); the DML searches are checked at the kernel's final slot set (each
slot against S(every other slot)).  Bins, slots and windows whose bound is too wide to compare are counted and printed
per family, with the occupancy of every decision band."""
import math

import numpy as np
import pytest

import azel_oracle as ao
import beams_oracle as bo
import estimator_oracle as est
import gpu_harness as gh
import helpers
import refine_oracle as ro
import solve_oracle as so
from helpers import LAM
from oracle import music_oracle as mo

pytestmark = pytest.mark.gpu

MS = [2, 3, 4, 5, 8, 12, 16]
K = 48
STRIDE = 6
PEAKS = ("levels", "bins")


def table(M):
    return helpers.table_wl(helpers.array_wl("uca", M), K)


def by_n(cases):
    groups = {}
    for c in cases:
        groups.setdefault(c[2].shape[0], []).append(c)
    return groups


def record(stats, fam, e, c, sk):
    w, cc, ss = stats.get(fam, (0.0, 0, 0))
    stats[fam] = (max(w, e), cc + c, ss + sk)


def report(kind, M, stats, bands):
    for fam, (w, c, sk) in sorted(stats.items()):
        print("%s M=%d %s: worst error %.3g of its bound, %d compared, %d skipped" % (kind, M, fam, w, c, sk))
    for key, v in sorted(bands.items()):
        print("%s M=%d band %s: %d" % (kind, M, key, v))


# ---- MVDR spectrum --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", MS)
def test_mvdr_spectrum(M):
    """every family at LOADINGS (the exact windows at their own loadings): P64 within the bound on every evaluated bin,
    the bins the top picks of P64 and never beaten by more than the bounds, the Cholesky band, and the launches of the
    MVDR pipeline (Bartlett's plus the preparation)"""
    tab = table(M)
    n = min(2, M - 1)
    stats, bands = {}, {}
    fams = so.mvdr_families(M, tab, 4000 + M)
    for N, group in sorted(by_n(fams).items()):
        x = np.stack([g[2].reshape(-1) for g in group])
        bart = gh.make_block(M, n, N, table=tab, est=("bartlett", 0.0))
        _, lb = gh.device_call(bart, x, PEAKS + ("spectrum",))
        bart.close()
        for loading in sorted({l for g in group for l in g[3]}):
            blk = gh.make_block(M, n, N, table=tab, est=("mvdr", loading))
            out, launches = gh.device_call(blk, x, PEAKS + ("spectrum", "P64", "R"))
            blk.close()
            assert launches == lb + 1, (M, N, loading, launches, lb)
            for w, (fam, name, _, loadings) in enumerate(group):
                if loading not in loadings:
                    continue
                P = out["P64"][w]
                ks = so.strided_bins(K, out["bins"][w], P, STRIDE)
                ref = so.mvdr_reference(out["R"][w], loading, tab, ks)
                e, c, sk, outcome, msg = so.check_mvdr(ref, P, out["bins"][w], out["levels"][w], out["angles"][w], M, K)
                assert msg is None, (M, fam, name, loading, msg)
                if outcome == "failed":
                    assert np.all(np.isnan(out["spectrum"][w])), (M, fam, name, loading)
                record(stats, fam, e, c, sk)
                key = (fam, ref["band"], outcome)
                bands[key] = bands.get(key, 0) + 1
    report("mvdr", M, stats, bands)
    for fam, (w, c, sk) in stats.items():
        assert c >= so.FLOOR.get(fam, 0.5) * (c + sk), (M, fam, c, sk)


# ---- beams ----------------------------------------------------------------------------------------------------------
def beam_cases(M, seed):
    """[(family, name, x, table, loadings)]: the LCMV close-pair sweep (one source at row 2j; TOP_BINS n = 2 reports rows
    2j and 2j + 1) and the MVDR families on the UCA table at loading 0 and the largest loading of each (so that a dead
    element is also compared where its weights exist)"""
    rng = np.random.default_rng(seed)
    out = []
    if M >= 3:
        lt, _, _ = so.lcmv_table(12, helpers.array_wl("uca", M))
        for j in range(12):
            out.append(("close pair", "j=%d" % j, so.sources(M, [lt[2 * j]], rng, so.N, 20.0), lt, (0.0,)))
    tab = table(M)
    for fam, name, x, loadings in so.mvdr_families(M, tab, seed):
        out.append((fam, name, x, tab, tuple(sorted({loadings[0], loadings[-1]}))))
    return out


@pytest.mark.parametrize("M", MS)
def test_beams(M):
    """MVDR and LCMV weights against the reference (LCMV's constraint residual included), both bands, zero weights and
    zero beams on a failed window, and the apply step (helpers.check_beams)"""
    n = min(2, M - 1)
    stats, bands = {}, {}
    cases = beam_cases(M, 5000 + M)
    groups = {}
    for c in cases:
        groups.setdefault((c[2].shape[0], id(c[3])), []).append(c)
    for (N, _), group in groups.items():
        tab = group[0][3]
        x = np.stack([g[2].reshape(-1) for g in group])
        for loading in sorted({l for g in group for l in g[4]}):
            blk = gh.make_block(M, n, N, table=tab)
            ref_out, _ = gh.device_call(blk, x, PEAKS + ("R",))
            for rule in ("mvdr", "lcmv"):
                blk.set_beamformer(rule, loading)
                out, _ = gh.device_call(blk, x, PEAKS + ("weights", "beams"))
                assert np.array_equal(out["bins"], ref_out["bins"]), (M, rule)
                helpers.check_beams(x, out["weights"], out["beams"])
                for w, (fam, name, _, _, loadings) in enumerate(group):
                    if loading not in loadings:
                        continue
                    rows = {i: tab[b].astype(np.complex128) for i, b in enumerate(out["bins"][w]) if b >= 0}
                    ref = so.beams_reference(ref_out["R"][w], rows, rule, loading)
                    e, c, sk, outcome, msg = so.check_weights(ref, out["weights"][w], rows, rule, M)
                    assert msg is None, (M, rule, fam, name, loading, msg)
                    if outcome == "failed":
                        assert not np.any(out["beams"][w]), (M, rule, fam, name)
                    record(stats, (rule, fam), e, c, sk)
                    key = (rule, fam, ref["band"], ref["pivot_band"] if rule == "lcmv" else "-", outcome)
                    bands[key] = bands.get(key, 0) + 1
            blk.close()
    report("beams", M, stats, bands)
    for (rule, fam), (w, c, sk) in stats.items():
        assert c >= so.FLOOR.get(fam, 0.5) * (c + sk), (M, rule, fam, c, sk)
    if M >= 3:
        piv = {k[3] for k in bands if k[0] == "lcmv" and k[1] == "close pair"}
        assert {"succeed", "fail"} <= piv, bands  # the sweep crosses 2^-20 on the device too


# ---- DML ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [3, 4, 5, 8, 12, 16])
def test_dml(M):
    """d = 2: every slot of the kernel's final set is an accepted S(every other slot); the levels within the level bound
    (plus their float32 rounding); slot order exact where the reference p values are separated by more than the bound"""
    stats = {}
    for fam, name, x, tab in so.dml_families(M, table(M), 6000 + M):
        blk = gh.make_block(M, 2, so.N, table=tab, mode="dml")
        out, _ = gh.device_call(blk, x.reshape(1, -1), PEAKS + ("R",))
        blk.close()
        R = out["R"][0]
        bins, lv = out["bins"][0], out["levels"][0]
        ctx = (M, fam, name)
        assert np.all(bins >= 0), (ctx, bins)
        slots = [int(b) for b in bins]
        for i in range(2):
            c, msg = so.check_search(R, tab, slots[:i] + slots[i + 1:], slots[i])
            assert msg is None, (ctx, msg)
            record(stats, fam + " search", 0.0, int(c), int(not c))
        p, s2, tinv2, kapA = so.levels_reference(R, tab, slots)
        b = so.level_bound(M, 2, float(np.trace(R).real), tinv2, kapA)
        if b > so.CHECKED * np.max(np.abs(p)):
            record(stats, fam, 0.0, 0, 1)
            continue
        e = np.abs(lv.astype(np.float64) - p) / (b + so.F32 * np.abs(p))
        assert np.all(e <= 1.0), (ctx, lv, p, b)
        record(stats, fam, float(np.max(e)), 1, 0)
        if abs(p[0] - p[1]) > 2 * b + so.F32 * np.max(np.abs(p)):
            assert p[0] > p[1], (ctx, p)  # slots come out in descending p
    report("dml", M, stats, {})
    for fam, (w, c, sk) in stats.items():
        assert c >= 0.5 * (c + sk), (M, fam, c, sk)


# ---- power-of-two scaling -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [4, 5, 8, 16])
def test_power_of_two_scaling(M):
    """windows rounded to multiples of 2^-9, then scaled by 2^-140 and 2^96 (exact in float32): R scales by 2^(2e), so
    L and P scale exactly.  P64 times 2^-2e, the bins, the MVDR / LCMV weights (scale-free) and the DML bins must be
    bit-identical to the unscaled run.  (The float32 levels over- or underflow at these scales and are not compared.)"""
    tab = table(M)
    rng = np.random.default_rng(70 + M)
    x = np.stack([so.sources(M, [tab[3], tab[20]], rng, so.N, snr).reshape(-1) for snr in (20, 80)])
    x = (np.round(x.astype(np.complex128) * 512.0) / 512.0).astype(np.complex64)
    n = min(2, M - 1)
    mv = gh.make_block(M, n, so.N, table=tab, est=("mvdr", 2.0 ** -20))
    bm = gh.make_block(M, n, so.N, table=tab)
    dml = gh.make_block(M, 2, so.N, table=tab, mode="dml") if M >= 3 else None
    base = gh.device_call(mv, x, PEAKS + ("P64",))[0]
    bw = {}
    for rule in ("mvdr", "lcmv"):
        bm.set_beamformer(rule, 0.0)
        bw[rule] = gh.device_call(bm, x, PEAKS + ("weights",))[0]
        assert np.any(bw[rule]["weights"] != 0), rule
    bd = gh.device_call(dml, x, PEAKS)[0] if dml else None
    for e in (-140, 96):
        xs = (x.astype(np.complex128) * 2.0 ** e).astype(np.complex64)
        assert np.array_equal(xs.astype(np.complex128) * 2.0 ** -e, x.astype(np.complex128))
        got = gh.device_call(mv, xs, PEAKS + ("P64",))[0]
        assert np.array_equal(got["P64"] * 2.0 ** (-2 * e), base["P64"]) and np.array_equal(got["bins"], base["bins"]), e
        for rule in ("mvdr", "lcmv"):
            bm.set_beamformer(rule, 0.0)
            g = gh.device_call(bm, xs, PEAKS + ("weights",))[0]
            assert np.array_equal(g["weights"], bw[rule]["weights"]) and np.array_equal(g["bins"], bw[rule]["bins"]), (e, rule)
        if dml:
            assert np.array_equal(gh.device_call(dml, xs, PEAKS)[0]["bins"], bd["bins"]), e
    for b in (mv, bm, dml):
        if b:
            b.close()


# ---- MVDR refinement ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [3, 4, 8, 12, 16])
def test_mvdr_refinement(M):
    """NEWTON on the high-SNR family (loading 0, LOCAL_MAXIMA on a geometric UCA): the refinement reads the prepared
    g_j at off-grid steering vectors.  Each refined level must be within the MVDR bound of the reference 1 / D at the
    reported angle t*, plus what the float32 rounding of t* moves D (|D'| h + |D''| h^2 / 2, h one float32 ulp of t* in
    radians) and one float32 rounding of the level; a failed factorisation must report nothing"""
    pos = helpers.positions("uca", M)
    n = min(2, M - 1)
    blk = gh.make_block(M, n, so.N, 360, pos=pos, est=("mvdr", 0.0), mode="local_maxima", excl=3, refine=True)
    tab = blk.array_response_c64()
    group = [f for f in so.mvdr_families(M, tab, 7000 + M) if f[0] == "high snr"]
    x = np.stack([g[2].reshape(-1) for g in group])
    out, _ = gh.device_call(blk, x, PEAKS + ("P64", "R"))
    blk.close()
    c = sk = 0
    worst = 0.0
    for w, (fam, name, _, _) in enumerate(group):
        ctx = (M, name)
        fac = so.factor(out["R"][w], 0.0)
        band = so.chol_band(fac, M)
        if np.all(np.isnan(out["P64"][w])):
            assert band != "succeed", ctx
            assert so.check_failed_clean(None, out["bins"][w], out["levels"][w], out["angles"][w]) is None, ctx
            continue
        assert band != "fail", ctx
        for i in range(n):
            if out["bins"][w, i] < 0:
                continue
            t = math.radians(float(out["angles"][w, i]))
            D, kap = so.mvdr_at(fac, ro.steering(pos, LAM, t)[0])
            b = so.mvdr_bound(M, kap)
            if b > so.CHECKED:
                sk += 1
                continue
            _, D1, D2 = est.objective(out["R"][w], "mvdr", 0.0, pos, LAM, t)
            h = math.radians(float(np.spacing(np.float32(abs(float(out["angles"][w, i])) + 1e-30))))
            tol = b + (abs(D1) * h + 0.5 * abs(D2) * h * h) / D + 2.0 * so.F32
            e = abs(float(out["levels"][w, i]) * D - 1.0) / tol
            assert e <= 1.0, (ctx, i, out["levels"][w, i], 1.0 / D, e)
            worst = max(worst, e)
            c += 1
    print("refine M=%d high snr: worst error %.3g of its bound, %d compared, %d skipped" % (M, worst, c, sk))
    assert c >= 1, (M, c, sk)


# ---- the other handles of the MVDR preparation -----------------------------------------------------------------------
@pytest.mark.parametrize("loading", [0.0, 2.0 ** -20, 0.01])
def test_channel_handle_row(loading):
    """one music_doa_channels handle (SEPARATE, MVDR, no P64 port): every channel's levels within the MVDR bound plus a
    float32 rounding on the device's own R_c and channel table, the bins not beaten by more than the bounds"""
    from test_gpu_channels import device_call, make, planar_pos, scene_windows

    m, n, K, F, J, first, C, W = 8, 2, 90, 16, 16, 0, 4, 4
    pos = planar_pos(m, 17)
    blk = make(m, n, F * J, K, F, first, C, "hann", "separate", pos, ("mvdr", loading))
    x = scene_windows(W, pos, F, F * J, first, C, 1700)
    got, _ = device_call(blk, x, ("levels", "bins", "spectrum", "R"))
    tabs = blk.array_response_c64()
    blk.close()
    c = sk = 0
    worst = 0.0
    for ci in range(C):
        for w in range(W):
            ks = so.strided_bins(K, got["bins"][ci, w], got["spectrum"][ci, w].astype(np.float64), STRIDE)
            ref = so.mvdr_reference(got["R"][ci, w], loading, tabs[ci], ks)
            e, cc, s, _, msg = so.check_levels(ref, got["spectrum"][ci, w], got["bins"][ci, w], got["levels"][ci, w], m)
            assert msg is None, (loading, ci, w, msg)
            worst, c, sk = max(worst, e), c + cc, sk + s
    print("channels loading %g: worst error %.3g of its bound, %d compared, %d skipped" % (loading, worst, c, sk))
    assert c >= 0.5 * (c + sk), (c, sk)


def test_azel_handle_row():
    """one az-el handle (MVDR, no R or P64 port) on the exact rank-deficient windows, whose R is exact in any summation
    order, so the host covariance is the device's: levels within the MVDR bound plus a float32 rounding, the bins not
    beaten by more than the bounds, across loadings 2^-10 .. 2^-40"""
    from gr_baz_b200.music_doa_azel import music_doa_azel

    m, n = 8, 2
    pos = ao.uca_xyz(m, LAM, alternate_z=True)
    grid = ao.Grid(36, 7, 0.0, 90.0)
    c = sk = 0
    worst = 0.0
    for loading in so.EXACT_LOADINGS:
        blk = music_doa_azel(m, n, m * so.EXACT_N, grid.n_az, grid.n_el, (grid.el_lo, grid.el_hi), pos, LAM)
        blk.set_estimator("mvdr", loading)
        tab = blk.array_response_c64().reshape(-1, m)  # row k = bin k (elevation-major)
        group = [f for f in so.mvdr_families(m, tab, 8000) if f[0] == "exact"]
        x = np.stack([g[2].reshape(-1) for g in group])
        got, _ = gh.device_call(blk, x, ("levels", "spectrum", "bins"))
        blk.close()
        K = len(tab)
        for w in range(len(group)):
            R = mo.covariance(x[w], m)
            X = x[w].reshape(-1, m).astype(np.complex128)
            assert np.array_equal(R, X.T @ X.conj() / X.shape[0])  # exact: the device's R is this R
            ks = so.strided_bins(K, got["bins"][w], got["spectrum"][w].astype(np.float64), 12)
            ref = so.mvdr_reference(R, loading, tab, ks)
            e, cc, s, _, msg = so.check_levels(ref, got["spectrum"][w], got["bins"][w], got["levels"][w], m)
            assert msg is None, (loading, w, msg)
            worst, c, sk = max(worst, e), c + cc, sk + s
    print("az-el exact: worst error %.3g of its bound, %d compared, %d skipped" % (worst, c, sk))
    assert c >= 0.5 * (c + sk), (c, sk)



# ---- geometric beams --------------------------------------------------------------------------------------------------
def test_geometric_close_pairs_local_maxima():
    """MVDR and LCMV weights steered at the reported float angles of a geometric UCA (beam_weights_kernel's sincos
    steering), two sources 0.5 .. 8 degrees apart at 60 dB under LOCAL_MAXIMA, against the reference at the same
    angles, with both bands and zero beams on a failed window"""
    M, n, K = 8, 2, 3600
    pos = helpers.array_wl("uca", M)
    rng = np.random.default_rng(8100)
    xs = []
    for th in (40.0, 130.0, 250.0):
        for sep in (0.5, 1.0, 2.0, 4.0, 8.0):
            vecs = [ro.steering(pos, LAM, math.radians(t))[0] for t in (th, th + sep)]
            xs.append(so.sources(M, vecs, rng, 256, 60.0).reshape(-1))
    x = np.stack(xs)
    blk = gh.make_block(M, n, 256, K, pos=pos, mode="local_maxima")
    ref_out, _ = gh.device_call(blk, x, PEAKS + ("R",))
    stats, bands = {}, {}
    for rule in ("mvdr", "lcmv"):
        blk.set_beamformer(rule, 0.0)
        out, _ = gh.device_call(blk, x, PEAKS + ("weights", "beams"))
        helpers.check_beams(x, out["weights"], out["beams"])
        for w in range(len(x)):
            rows = {i: bo.steering_geo(pos, LAM, out["angles"][w, i]) for i in range(n) if out["bins"][w, i] >= 0}
            ref = so.beams_reference(ref_out["R"][w], rows, rule, 0.0)
            e, c, sk, outcome, msg = so.check_weights(ref, out["weights"][w], rows, rule, M)
            assert msg is None, (rule, w, msg)
            if outcome == "failed":
                assert not np.any(out["beams"][w]), (rule, w)
            record(stats, (rule, "geometric close pair"), e, c, sk)
            key = (rule, ref["band"], ref["pivot_band"] if rule == "lcmv" else "-", outcome)
            bands[key] = bands.get(key, 0) + 1
    blk.close()
    report("beams geometric", M, stats, bands)
    for key, (w, c, sk) in stats.items():
        assert c >= 0.5 * (c + sk), (key, c, sk)
