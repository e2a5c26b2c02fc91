"""CPU: the gridless checker of tests/gridless_oracle.py.  The mpmath reference agrees with the fp64 oracles on benign
windows; the numpy restatements of roots_kernel and esprit_eigvals (tools/emulate_roots_warp.py,
tools/emulate_esprit_warp.py) reproduce the two failures the kernels had (QR stalling on a cyclic Psi, Horner
overflowing on a rounding-level outer coefficient) with the old rules, meet every bound with the current ones, and
planted defects fail the checker."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import emulate_esprit_warp as ee  # noqa: E402
import emulate_roots_warp as er  # noqa: E402

import esprit_oracle as eso  # noqa: E402
import gridless_oracle as go  # noqa: E402
import refine_oracle as ro  # noqa: E402
import root_music_oracle as rm  # noqa: E402
from helpers import LAM, ula  # noqa: E402
from oracle import music_oracle as mo  # noqa: E402

K = 3600


def cov(x):
    return mo.covariance(x.reshape(-1), x.shape[1])


def outputs(zs, G, d, n, pos, s):
    """(angles, levels, bins) of n slots from the slot roots / eigenvalues zs"""
    ang, lvl, bins = np.zeros(n, np.float32), np.zeros(n, np.float32), np.full(n, -1, np.int32)
    for i, z in enumerate(zs):
        t = rm.direction(complex(z), s, LAM)
        a = np.float32(t)
        ang[i] = 0.0 if a >= np.float32(360.0) else a
        lvl[i] = np.float32(1.0 / ro.objective(G, pos, LAM, math.radians(t))[0])
        bins[i] = int(math.floor(t * K / 360.0 + 0.5)) % K
    return ang, lvl, bins


def emulated(mode, R, d, pos, **kw):
    """(angles, levels, bins, ok) of the emulated kernel on LAPACK eigenvectors of R"""
    M = R.shape[0]
    _, _, s = rm.ula_geometry(pos, LAM)
    _, V = np.linalg.eigh(R)
    G = V[:, :M - d]
    if mode == "roots":
        o = er.roots_window(G, d, lambda z: rm.direction(complex(z), s, LAM), **kw)
        return outputs([z for _, z in o["slots"]], G, d, d, pos, s) + (o["ok"],)
    ev, _ = ee.esprit_window(V, d, **kw)
    zs = [] if ev is None else [e for e in ev if e != 0]
    return outputs(zs, G, d, d, pos, s) + (ev is not None,)


def sweep(mode, Ms=(4, 6, 8), **kw):
    """{family: (worst error / bound, checked, skipped, first failure)} of the emulated kernel over the families"""
    res = {}
    for M in Ms:
        pos = ula(M, "x")
        for fam, name, x, d, _ in go.families(M, 500 + M):
            R = cov(x)
            ref = (go.roots_reference if mode == "roots" else go.esprit_reference)(R, d, pos, LAM)
            a, l, b, _ = emulated(mode, R, d, pos, **kw)
            e, compared, msg = go.check(ref, a, l, b, d, d, pos, LAM, K)
            w, c, sk, f = res.get(fam, (0.0, 0, 0, None))
            if compared:
                res[fam] = (max(w, e), c + 1, sk, f or (msg and (M, name, msg)))
            else:
                res[fam] = (w, c, sk + 1, f)
    return res


def test_reference_agrees_with_the_fp64_oracles():
    rng = np.random.default_rng(5)
    for M in (4, 8):
        pos = ula(M, "x")
        for d in (1, 2, 3):
            x = go.random_sources(M, [go.z_of(t) for t in rng.uniform(10, 170, d)], rng, 20.0)
            R = cov(x)
            r = go.roots_reference(R, d, pos, LAM)
            o = rm.work_R(R, pos, LAM, K, d, d=d)
            assert np.allclose(sorted(s[0] for s in r["slots"]), np.sort(o["angles"]), atol=1e-4), (M, d)
            e = go.esprit_reference(R, d, pos, LAM)
            o = eso.work_R(R, pos, LAM, K, d, d=d)
            assert np.allclose(sorted(s[0] for s in e["slots"]), np.sort(o["angles"]), atol=1e-4), (M, d)


def test_comb_window_gives_a_block_covariance():
    """equal-power comb sources on their own snapshots: R is exactly zero off the residue classes mod d"""
    for M, d in ((6, 3), (8, 4), (12, 4)):
        x = go.exact_sources(go.comb(M, d, 1j), np.random.default_rng(M))
        R = cov(x)
        m = np.arange(M)
        off = (m[:, None] - m[None, :]) % d != 0
        assert np.all(R[off] == 0) and np.all(R[~off] != 0), (M, d)


def test_old_rules_reproduce_the_failures():
    # ESPRIT: Wilkinson shifts alone stall on the comb basis of a cyclic Psi
    # (the comb vectors with the random phases and order an eigensolver may return for the tied eigenvalues)
    M, d = 8, 4
    rng = np.random.default_rng(1)
    stalled = 0
    for _ in range(20):
        Es = np.stack([v / np.linalg.norm(v) * np.exp(2j * np.pi * rng.uniform()) for v in go.comb(M, d, 1)], 1)
        V = np.concatenate([np.zeros((M, M - d)), Es[:, rng.permutation(d)]], 1)
        stalled += ee.esprit_window(V, d, exceptional=False)[0] is None
        ev, _ = ee.esprit_window(V, d)
        want = np.exp(2j * np.pi * np.arange(d) / d)
        assert max(np.min(np.abs(want - e)) for e in ev) <= 1e-13 and max(np.min(np.abs(ev - w)) for w in want) <= 1e-13
    assert stalled >= 5, stalled
    # ROOTS: opposite spatial frequencies at M = 16, a rounding-level corner coefficient: Horner overflows
    x = go.exact_sources([go.steering(16, 1j), go.steering(16, -1j)], np.random.default_rng(1))
    _, V = np.linalg.eigh(cov(x))
    G = V[:, :14]
    old = er.roots_window(G, 2, lambda z: 0.0, circle=True, reversed_eval=False, conv_flag=False, backward=False)
    assert old["c"][15] != 0 and abs(old["c"][15]) < 1e-14
    assert not old["ok"]
    new = er.roots_window(G, 2, lambda z: -np.angle(z))
    assert new["ok"] and new["converged"] and np.allclose(sorted(a for a, _ in new["slots"]), [-math.pi / 2, math.pi / 2])
    # and at M = 8 the old iteration runs to its cap without converging
    x = go.exact_sources([go.steering(8, 1j), go.steering(8, -1j)], np.random.default_rng(2))
    _, V = np.linalg.eigh(cov(x))
    old = er.roots_window(V[:, :6], 2, lambda z: 0.0, circle=True, reversed_eval=False, conv_flag=False, backward=False)
    assert old["iterations"] == er.MAX_IT and not old["converged"]


@pytest.mark.parametrize("mode", ["roots", "esprit"])
def test_emulation_meets_the_bounds(mode):
    res = sweep(mode)
    for fam, (w, c, sk, f) in sorted(res.items()):
        print("%s %s: worst %.3g of the bound, %d checked, %d skipped" % (mode, fam, w, c, sk))
        assert w <= 1.0 and f is None, (fam, f)
        assert c >= go.floor(mode, fam) * (c + sk), (fam, c, sk)


DEFECTS = {
    "roots: Aberth capped at 5 iterations": ("roots", dict(max_it=5, conv_flag=False)),
    "roots: Newton without the Aberth sum": ("roots", dict(aberth_sum=False)),
    "esprit: QR with a zero shift": ("esprit", dict(zero_shift=True, exceptional=False)),
    "esprit: ESPRIT_MAX_IT = 3": ("esprit", dict(max_it=3)),
    "esprit: Sherman-Morrison without den": ("esprit", dict(den_on=False)),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_planted_defects_fail_the_checker(defect):
    mode, kw = DEFECTS[defect]
    res = sweep(mode, Ms=(4, 8), **kw)
    assert any(f is not None or w > 1.0 for w, _, _, f in res.values()), defect


def test_planted_merge_defect_fails_the_checker():
    """the merge decides the output when both approximants of a double root fall inside the unit circle (the modulus
    ranking then keeps both copies and drops another source).  The converged roots of the exact M = 16 opposite-frequency
    window (two double roots, a reference bound tight enough to compare) are moved just inside the circle, ~1e-9 apart:
    the kernel's selection with the merge passes the checker, without it fails.  (On the families themselves the
    kernel's approximants straddle the circle, so removing the merge changes no output there.)"""
    M, d = 16, 2
    pos = ula(M, "x")
    _, _, s = rm.ula_geometry(pos, LAM)
    x = go.exact_sources([go.steering(M, 1j), go.steering(M, -1j)], np.random.default_rng(1))
    R = cov(x)
    ref = go.roots_reference(R, d, pos, LAM)
    _, V = np.linalg.eigh(R)
    G = V[:, :M - d]
    o = er.roots_window(G, d, lambda z: 0.0)
    z = o["z"].copy()
    on = np.abs(np.abs(z) - 1.0) < 1e-6
    assert np.count_nonzero(on) == 4, np.abs(z)
    # every copy inside; both copies of the source at -j deeper inside than either copy of the one at +j
    for r in np.flatnonzero(on):
        deep = 3e-9 if z[r].imag < 0 else 1e-9
        z[r] = z[r] / abs(z[r]) * (1.0 - deep - 1e-9 * (r % 2))
    H = (len(z)) // 2
    direction = lambda zz: rm.direction(complex(zz), s, LAM)
    for merge_on, want in ((True, True), (False, False)):
        slots = er.select(z, H, d, direction, merge_on)
        a, l, b = outputs([zz for _, zz in slots], G, d, d, pos, s)
        e, compared, msg = go.check(ref, a, l, b, d, d, pos, LAM, K)
        assert compared, ref
        assert (msg is None and e <= 1.0) == want, (merge_on, e, msg, a)


@pytest.mark.parametrize("M", [12, 16])
def test_emulation_converges_at_large_M(M):
    """the current rules converge on every family at M = 12 and 16 (the reference comparison runs at M <= 8 on the CPU
    and at every M on the GPU); 40 steps at most, ROOTS_MAX_IT = 100"""
    pos = ula(M, "x")
    _, _, s = rm.ula_geometry(pos, LAM)
    worst = 0
    for fam, name, x, d, _ in go.families(M, 500 + M):
        _, V = np.linalg.eigh(cov(x))
        o = er.roots_window(V[:, :M - d], d, lambda z: rm.direction(complex(z), s, LAM))
        assert o["ok"] and o["converged"], (fam, name, o["iterations"])
        worst = max(worst, o["iterations"])
    assert worst <= 40, worst
