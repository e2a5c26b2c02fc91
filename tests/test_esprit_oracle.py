"""CPU: the ESPRIT definition (tests/esprit_oracle.py) against the truth of noiseless windows, its invariance to the
basis of the signal subspace, the Sherman-Morrison form the kernel uses, the mirror-free output on a line array and the
unfilled-slot rules."""
import math

import numpy as np
import pytest

import esprit_oracle as eo
import refine_oracle as ro
import root_music_oracle as rm

LAM = 1.0


def ula(m, axis_deg=0.0, spacing=0.5, p0=(0.0, 0.0), reverse=False):
    a = math.radians(axis_deg)
    pos = np.array([[p0[0] + i * spacing * math.cos(a), p0[1] + i * spacing * math.sin(a)] for i in range(m)])
    return pos[::-1].copy() if reverse else pos


KINDS = {"x": dict(), "y": dict(axis_deg=90.0), "oblique": dict(axis_deg=30.0, p0=(0.7, -1.3)), "reversed": dict(reverse=True)}


def mirror_report(t, pos):
    """the angle a gridless ULA mode reports for a source at t degrees: the lower of t and its mirror across the axis"""
    _, _, s = rm.ula_geometry(pos, LAM)
    alpha = math.degrees(math.atan2(s[1], s[0]))
    return min(t % 360.0, (2.0 * alpha - t) % 360.0)


def circ(a, b):
    return abs((a - b + 180.0) % 360.0 - 180.0)


def separated_angles(rng, n, alpha, min_cos=0.05):
    """n angles over [0, 360), at least 2 degrees from end-fire, with distinct cos(t - alpha)"""
    while True:
        t = rng.uniform(0.0, 360.0, n)
        off = (t - alpha) % 180.0
        if np.any(np.minimum(off, 180.0 - off) < 2.0):
            continue
        cs = np.cos(np.radians(t - alpha))
        if n == 1 or np.min(np.abs(np.subtract.outer(cs, cs))[np.triu_indices(n, 1)]) >= min_cos:
            return t


def random_es(rng, m, d):
    Z = rng.standard_normal((m, m)) + 1j * rng.standard_normal((m, m))
    return np.linalg.qr(Z)[0][:, m - d:]


@pytest.mark.parametrize("m", list(range(2, 17)))
def test_noiseless_windows_give_the_truth(m):
    """R = A A^H with d = S sources: every angle within 1e-3 degrees of the source (or its mirror)"""
    rng = np.random.default_rng(200 + m)
    worst = 0.0
    for kind, kw in KINDS.items():
        pos = ula(m, **kw)
        _, _, s = rm.ula_geometry(pos, LAM)
        alpha = math.degrees(math.atan2(s[1], s[0]))
        for n in (1, 2, 3):
            if n >= m:
                continue
            for _ in range(10):
                th = separated_angles(rng, n, alpha)
                A = np.stack([ro.steering(pos, LAM, math.radians(t))[0] for t in th], axis=1)
                r = eo.work_R(A @ A.conj().T, pos, LAM, 3600, n)
                want = sorted(mirror_report(t, pos) for t in th)
                got = sorted(float(a) for a in r["angles"])
                err = max(circ(g, w) for g, w in zip(got, want))
                worst = max(worst, err)
                assert err <= 1e-3, (m, kind, th, got, want)
                assert np.all(r["bins"] >= 0) and np.all(r["levels"] > 0)
                assert list(r["levels"]) == sorted(r["levels"], reverse=True)
    print("m = %d: worst noiseless error %.2e deg" % (m, worst))


@pytest.mark.parametrize("m,d", [(4, 1), (4, 3), (8, 2), (16, 5), (16, 15)])
def test_eigenvalues_do_not_depend_on_the_basis(m, d):
    """E_s U for a random unitary U: Psi becomes U^-1 Psi U, with the same eigenvalues"""
    rng = np.random.default_rng(m * 31 + d)
    Es = random_es(rng, m, d)
    U = np.linalg.qr(rng.standard_normal((d, d)) + 1j * rng.standard_normal((d, d)))[0]
    a = np.sort_complex(np.linalg.eigvals(eo.psi_matrix(Es)))
    b = np.sort_complex(np.linalg.eigvals(eo.psi_matrix(Es @ U)))
    assert np.max(np.abs(a - b)) <= 1e-10 * max(1.0, np.max(np.abs(a))), (a, b)


@pytest.mark.parametrize("m", [2, 3, 4, 8, 12, 16])
def test_sherman_morrison_equals_solve(m):
    rng = np.random.default_rng(m)
    for d in range(1, m):
        Es = random_es(rng, m, d)
        P, S = eo.psi_matrix(Es), eo.psi_sherman_morrison(Es)
        assert np.max(np.abs(P - S)) <= 1e-12 * max(1.0, np.max(np.abs(P))), (m, d)


def test_no_mirror_on_an_x_axis_ula():
    """two sources on either side of broadside at 20 dB: each reported once, in [0, 180], never its mirror"""
    m, K, N = 4, 3600, 4096
    pos = ula(m)
    rng = np.random.default_rng(3)
    for th in ((40.0, 110.0), (20.0, 150.0), (70.0, 100.0)):
        A = np.stack([ro.steering(pos, LAM, math.radians(t))[0] for t in th], axis=1)
        S = (rng.standard_normal((2, N)) + 1j * rng.standard_normal((2, N))) / np.sqrt(2.0)
        X = 10.0 * (A @ S) + (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / np.sqrt(2.0)
        r = eo.work(X.T.reshape(-1).astype(np.complex64), m, 2, K, pos, LAM)
        got = sorted(float(a) for a in r["angles"])
        assert all(0.0 <= g <= 180.0 for g in got), got
        assert all(abs(g - t) < 0.5 for g, t in zip(got, th)), (th, got)


def test_unfilled_slots_and_degenerate_windows():
    m, n, K = 4, 3, 360
    pos = ula(m)
    empty = lambda r: np.all(r["bins"] == -1) and np.all(r["angles"] == 0.0) and np.all(r["levels"] == 0.0)
    # all-zero R: E_s holds the last unit vectors, |r| = 1, E1^H E1 is singular
    assert empty(eo.work_R(np.zeros((m, m), np.complex128), pos, LAM, K, n))
    # non-finite R, and d = 0
    R = np.eye(m, dtype=np.complex128)
    R[1, 2] = np.nan
    assert empty(eo.work_R(R, pos, LAM, K, n))
    A = ro.steering(pos, LAM, math.radians(60.0))[0][:, None]
    assert empty(eo.work_R(A @ A.conj().T + 0.01 * np.eye(m), pos, LAM, K, n, d=0))
    # one source, n = 3, d = 1: slots 1 and 2 unfilled
    r = eo.work_R(A @ A.conj().T + 0.01 * np.eye(m), pos, LAM, K, n, d=1)
    assert r["bins"][0] >= 0 and abs(float(r["angles"][0]) - 60.0) < 1e-3
    assert np.all(r["bins"][1:] == -1) and np.all(r["angles"][1:] == 0.0) and np.all(r["levels"][1:] == 0.0)
    # an eigenvalue exactly 0 has no direction: E_s = e_0 gives E1^H E2 = 0
    V = np.eye(m, dtype=np.complex128)[:, [1, 2, 3, 0]]
    a, lv, b, _ = eo.esprit_window(V, 1, pos, LAM, K, n)
    assert np.all(b == -1) and np.all(a == 0.0) and np.all(lv == 0.0)
    # |r| = 1: E1^H E1 not positive definite
    V = np.eye(m, dtype=np.complex128)
    assert eo.psi_matrix(V[:, m - 1:]) is None
    a, lv, b, _ = eo.esprit_window(V, 2, pos, LAM, K, n)
    assert np.all(b == -1)
