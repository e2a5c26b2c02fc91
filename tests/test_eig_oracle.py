"""CPU: the eigensolver checker of tests/eig_oracle.py.  The mpmath reference agrees with LAPACK, the exact windows give
the covariance and the eigenvalues they were built for bit for bit, the numpy restatements of the solvers
(tools/emulate_eig_coop_warp.py, tools/emulate_eig4_coop.py, tools/emulate_eig4_principal.py) pass the bounds on every
family, and planted defects - the ones a GPU test on the MUSIC outputs alone would let through - fail them."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import emulate_eig4_coop as e4c  # noqa: E402
import emulate_eig4_principal as e4p  # noqa: E402
import emulate_eig_coop_warp as ecw  # noqa: E402

import eig_oracle as eo  # noqa: E402
from oracle import music_oracle as mo  # noqa: E402


def covariance(x):
    return mo.covariance(x.reshape(-1), x.shape[1])


def matrices(M, n, seed):
    """(family, R) over the exact and the float32-rounded families (R = the fp64 covariance of the window)"""
    rng = np.random.default_rng(seed)
    out = [(name, R) for name, _, R, _ in eo.exact_family(M, n, rng)]
    Q = eo.unitary(M, rng)
    for name, lam in eo.prescribed_spectra(M, n):
        out.append((name, covariance(eo.spectrum_window(lam, Q, 64))))
    out.append(("imaginary", covariance(eo.imaginary_window(M, 64, rng))))
    out.append(("rank one f32", covariance(eo.rank_one_window(M, 64, rng))))
    return out


def worst(solve, M, n, seed):
    """largest (eigenvalue error / bound, projector error / bound) of `solve` over the families, and how many splits
    were too ill-conditioned to check"""
    we, wp, skipped = 0.0, 0.0, 0
    for name, R in matrices(M, n, seed):
        ref = eo.reference(R, n)
        w, Vt = solve(R)
        e, p = eo.check(M, n, ref, w, eo.noise_projector(Vt, n))
        we = max(we, e)
        if p is None:
            skipped += 1
        else:
            wp = max(wp, p)
    return we, wp, skipped


def test_reference_agrees_with_lapack():
    rng = np.random.default_rng(3)
    for M in (2, 4, 7, 16):
        X = rng.standard_normal((M, 2 * M)) + 1j * rng.standard_normal((M, 2 * M))
        R = X @ X.conj().T
        ref = eo.reference(R, 1)
        w, V = np.linalg.eigh(R)
        assert np.max(np.abs(ref["w"] - w)) <= 1e-13 * ref["norm"]
        G = V[:, :M - 1]
        assert eo.proj_err(G @ G.conj().T, ref["Pi"]) <= 1e-13 * ref["norm"] / ref["gap"]
        assert ref["norm"] == pytest.approx(np.linalg.norm(R, 2), rel=1e-14)


@pytest.mark.parametrize("M", range(2, 17))
def test_exact_windows_are_exact(M):
    """R of the float32 window, summed in fp64 in three different orders, is the intended R bit for bit; the mpmath
    eigenvalues are the closed-form ones"""
    n = max(1, M // 3)
    for diagonal in (False, True):
        for name, x, R, lam in eo.exact_family(M, n, np.random.default_rng(M), diagonal=diagonal):
            X = x.astype(np.complex128)
            assert np.array_equal(covariance(x), R), name
            assert np.array_equal(X[::-1].T @ X[::-1].conj() / len(X), R), name
            acc = np.zeros((M, M), np.complex128)
            for t in range(len(X)):
                acc += np.outer(X[t], X[t].conj())
            assert np.array_equal(acc / len(X), R), name
            ref = eo.reference(R, n)
            assert np.max(np.abs(ref["w"] - lam)) <= 1e-40 * lam.max(), name  # (zeros come back as ~1e-50 ||R||)
            if diagonal:
                assert np.count_nonzero(R - np.diag(np.diag(R))) == 0


def test_probe_readout_recovers_the_projector():
    rng = np.random.default_rng(8)
    for M in (2, 5, 16):
        R = covariance(eo.spectrum_window(np.linspace(1, 3, M), eo.unitary(M, rng), 32))
        ref = eo.reference(R, 1)
        P, _, _ = eo.strength_ref(ref, eo.probe_table(M))
        assert eo.proj_err(eo.projector_from_P(P, M), ref["Pi"]) <= 1e-14


@pytest.mark.parametrize("M", [8, 12, 16])
def test_coop_warp_emulation_meets_the_bounds(M):
    for n in (1, M // 2):
        we, wp, skipped = worst(lambda R: ecw.eig(R)[:2], M, n, 10 + M)
        assert we <= 1.0 and wp <= 1.0, (n, we, wp)
        assert skipped <= 3


DEFECTS = {
    "stop at off <= 1e-24 fro": dict(stop=1e-24, stagnation=False),
    "off by subtraction": dict(off_by_subtraction=True),
    "one sweep fewer": dict(sweeps_less=1),
}


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_planted_jacobi_defects_fail_the_bounds(defect):
    """each defect leaves eigenvalues and orthonormality nearly intact, yet puts the projector outside its bound on
    at least one of the families"""
    bad = 0.0
    for M in (8, 16):
        for n in (1, M // 2):
            we, wp, _ = worst(lambda R: ecw.eig(R, **DEFECTS[defect])[:2], M, n, 10 + M)
            bad = max(bad, we, wp)
    assert bad > 1.0, defect


def _eig4(R):
    Ar, Ai, Vr, Vi, _ = e4c.eig_coop(R)
    w = np.diag(Ar)
    order = np.argsort(w, kind="stable")
    return w[order], (Vr + 1j * Vi)[:, order].T


def test_eig4_emulations_meet_the_bounds():
    for n in (1, 2, 3):
        we, wp, _ = worst(_eig4, 4, n, 44)
        assert we <= 1.0 and wp <= 1.0, (n, we, wp)


def principal_windows(M, seed):
    """near-equal top pairs on both sides of the squaring / fallback boundary"""
    rng = np.random.default_rng(seed)
    Q = eo.unitary(M, rng)
    for r in eo.top_pair_ratios():
        yield r, covariance(eo.spectrum_window(eo.top_pair_spectrum(M, r), Q, 64))


def principal_worst(M):
    """(largest projector error / bound over the windows the solver accepts, solved, fell back)"""
    wp, solved, fell = 0.0, 0, 0
    for seed in range(4):
        for r, R in principal_windows(M, 60 + seed):
            Vt, _ = e4p.principal(R)
            if Vt is None:
                fell += 1
                continue
            solved += 1
            ref = eo.reference(R, 1)
            wp = max(wp, eo.proj_err(eo.noise_projector(Vt, 1), ref["Pi"]) / eo.proj_bound(M, ref["norm"], ref["gap"]))
    return wp, solved, fell


@pytest.mark.parametrize("M", [4, 8])
def test_principal_emulation_meets_the_bound_and_falls_back(M):
    wp, solved, fell = principal_worst(M)
    assert wp <= 1.0 and solved > 0 and fell > 0, (wp, solved, fell)
