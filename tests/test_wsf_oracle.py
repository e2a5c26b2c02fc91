"""The WSF peak mode and the JOINT refinement as tests/wsf_oracle.py restates them (no GPU): X's invariances, the true
off-grid angles from exact covariances, JOINT against a bounded general-purpose minimiser, and DML + JOINT."""
import numpy as np
import pytest
from scipy.optimize import minimize

import dml_oracle as dm
import helpers
import wsf_oracle as wo

K = 360


def exact_R(pos, th, coherent, rng, noise=1.0):
    A = helpers.steering_wl(pos, th).T
    d = len(th)
    if coherent:
        g = np.exp(2j * np.pi * rng.uniform(size=d)) * rng.uniform(5.0, 10.0, d)
        S = np.outer(g, g.conj())
    else:
        S = np.diag(rng.uniform(25.0, 100.0, d))
    return A @ S @ A.conj().T + noise * np.eye(pos.shape[0])


def separated(rng, d, sep):
    while True:
        th = rng.uniform(0.0, 360.0, d)
        if d == 1 or np.min(helpers.circ(th[:, None], th[None, :]) + 1e3 * np.eye(d)) > sep:
            return th


def test_x_is_invariant_to_eigenvector_phase_and_degenerate_rotations():
    rng = np.random.default_rng(1)
    M, d = 8, 3
    Q, _ = np.linalg.qr(rng.standard_normal((M, M)) + 1j * rng.standard_normal((M, M)))
    l = np.array([1.0, 1.0, 1.1, 0.9, 1.05, 20.0, 20.0, 50.0])
    order = np.argsort(l)
    l, Q = l[order], Q[:, order]
    X = wo.wsf_matrix(l, Q, d)
    phased = Q * np.exp(2j * np.pi * rng.uniform(size=M))[None, :]
    assert np.allclose(wo.wsf_matrix(l, phased, d), X, rtol=0, atol=1e-12 * np.abs(X).max())
    U, _ = np.linalg.qr(rng.standard_normal((2, 2)) + 1j * rng.standard_normal((2, 2)))
    rot = Q.copy()
    rot[:, 5:7] = Q[:, 5:7] @ U  # the degenerate pair l = 20
    assert np.allclose(wo.wsf_matrix(l, rot, d), X, rtol=0, atol=1e-12 * np.abs(X).max())
    assert wo.wsf_matrix(l, Q, 0) is None
    assert wo.wsf_matrix(np.r_[0.0, l[1:]], Q, d) is None
    assert wo.wsf_matrix(np.r_[l[:-1], np.nan], Q, d) is None


# (geometry, M, d, coherent): exact R = A S A^H + I.  The fully coherent three-source rows are left out: their X has rank
# one, and the alternating-projection search (DML's, word for word) can stop in a local optimum there.
CASES = [(g, m, d, c) for g, m in (("uca", 8), ("uca", 16), ("random", 8)) for d in (1, 2, 3) for c in (False, True)
         if not (c and d == 3)]


@pytest.mark.parametrize("case", CASES)
def test_wsf_joint_returns_the_true_angles(case):
    """within 1e-9 degrees: V is evaluated as ||P_perp F||^2, which keeps its relative accuracy down to V = 0"""
    kind, m, d, coherent = case
    pos = helpers.array_wl(kind, m, seed=3)
    tab = helpers.table_wl(pos, K)
    rng = np.random.default_rng(CASES.index(case))
    checked = 0
    for _ in range(4):
        th = separated(rng, d, 25.0 if kind == "uca" else 40.0)
        R = exact_R(pos, th, coherent, rng)
        out = wo.window_R(R, tab, d, d, "wsf", pos, 1.0, True)
        if max(helpers.circ(np.sort(out["slots"]) * 360.0 / K, np.sort(th))) > 360.0 / K:
            continue  # a search that did not land within a bin of the truth (random planar ambiguities)
        got = np.sort(np.degrees(out["theta"]) % 360.0)
        assert np.max(helpers.circ(got, np.sort(th))) <= 1e-9, (case, th, got, out["info"])
        checked += 1
    assert checked >= 2, case


@pytest.mark.parametrize("m,d", [(8, 1), (8, 2), (16, 3)])
def test_dml_joint_returns_the_true_angles(m, d):
    """DML's V has a floor (M - d) s2 > 0, so its rounding limits the line search to about sqrt(eps) in relative V: the
    oracle measured up to 2.6e-8 degrees on these seeds; 1e-6 leaves room"""
    pos = helpers.array_wl("uca", m)
    tab = helpers.table_wl(pos, K)
    rng = np.random.default_rng(10 * m + d)
    for _ in range(4):
        th = separated(rng, d, 30.0)
        R = exact_R(pos, th, False, rng)
        out = wo.window_R(R, tab, d, d, "dml", pos, 1.0, True)
        got = np.sort(np.degrees(out["theta"]) % 360.0)
        assert np.max(helpers.circ(got, np.sort(th))) <= 1e-6, (th, got, out["info"])


def test_joint_is_no_worse_than_a_bounded_minimiser():
    """sample covariances: V(theta*) <= V of L-BFGS-B over the same box from the same start (+ 1e-12 relative)"""
    rng = np.random.default_rng(5)
    pos = helpers.array_wl("uca", 8)
    tab = helpers.table_wl(pos, K)
    for w in range(30):
        d = 1 + w % 3
        th = separated(rng, d, 30.0)
        x = helpers.angle_windows(pos, [th], w % 2 == 1 and d == 2, 1, 100 + w, snr_db=10.0, snaps=64)[0]
        out = wo.work(x, 8, d, tab, pos, 1.0, "wsf", True)
        if not out["slots"] or not out["info"]["moved"]:
            continue
        F = out["F"]
        bins = [int(b) for b in out["bins"] if b >= 0]
        tb = np.radians(np.array(bins) * 360.0 / K)
        delta = np.radians(360.0 / K)
        V = lambda t: wo.criterion(F, wo.steer(pos, 1.0, t)[0])
        ref = minimize(V, tb, method="L-BFGS-B", bounds=[(t - delta, t + delta) for t in tb],
                       options={"ftol": 1e-15, "gtol": 1e-13, "maxiter": 500})
        assert V(out["theta"]) <= ref.fun * (1.0 + 1e-12) + 1e-300, (w, V(out["theta"]), ref.fun)


def test_levels_are_least_squares_powers_at_the_refined_angles():
    rng = np.random.default_rng(8)
    pos = helpers.array_wl("uca", 8)
    tab = helpers.table_wl(pos, K)
    th = np.array([33.3, 101.7])
    R = exact_R(pos, th, False, rng)
    out = wo.window_R(R, tab, 2, 2, "wsf", pos, 1.0, True)
    A = helpers.steering_wl(pos, th).T
    S = np.linalg.pinv(A) @ (R - np.eye(8)) @ np.linalg.pinv(A).conj().T
    for i, b in enumerate(out["bins"]):
        k = int(np.argmin(helpers.circ(out["angles"][i], th)))
        assert abs(out["levels"][i] - S[k, k].real) <= 1e-5 * S[k, k].real


def test_wsf_matches_dml_search_on_x_and_takes_levels_from_r():
    rng = np.random.default_rng(2)
    pos = helpers.array_wl("uca", 8)
    tab = helpers.table_wl(pos, K)
    x = helpers.angle_windows(pos, [[20.0, 80.0]], True, 1, 3)[0]
    out = wo.work(x, 8, 2, tab)
    X = out["X"]
    ref = dm.work_R(X, tab, 2)
    assert sorted(ref["slots"]) == sorted(out["slots"])
    a, _ = dm.rows(tab, 8)
    p, _ = dm.levels(out["R"], a, out["slots"])
    assert np.allclose(sorted(p), sorted(out["levels"].astype(np.float64)), rtol=1e-6)
    assert helpers.resolved(out["angles"], [20.0, 80.0])
