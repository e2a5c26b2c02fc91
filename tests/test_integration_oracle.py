"""CPU checks of the covariance integration definition (tests/integration_oracle.py): the literal recurrence, N_eff,
the properties the header states, and the weak-source study that motivates the feature."""
import numpy as np
import pytest

import integration_oracle as io


def _random_R(rng, W, m):
    X = rng.standard_normal((W, 2 * m, m)) + 1j * rng.standard_normal((W, 2 * m, m))
    return np.einsum("wni,wnj->wij", X, X.conj()) / (2 * m)


def test_literal_recurrence():
    rng = np.random.default_rng(1)
    R = _random_R(rng, 6, 3)
    a = 0.7
    got, fac = io.integrate(R, a)
    for j in range(6):
        S = sum(a ** (j - i) * R[i] for i in range(j + 1))
        c = sum(a ** k for k in range(j + 1))
        q = sum(a ** (2 * k) for k in range(j + 1))
        assert np.allclose(got[j], S / c, rtol=1e-14, atol=0)
        assert fac[j] == pytest.approx(c * c / q, rel=1e-14)
    assert np.array_equal(got[0], R[0])  # the first window after a reset is its own R
    assert fac[0] == 1.0


def test_alpha_zero_is_identity_and_hermitian_kept():
    rng = np.random.default_rng(2)
    R = _random_R(rng, 5, 4)
    got, fac = io.integrate(R, 0.0)
    assert np.array_equal(got, R)
    assert np.array_equal(fac, np.ones(5))
    got, _ = io.integrate(R, 0.9)
    assert np.array_equal(got, np.conj(np.swapaxes(got, 1, 2)))


def test_constant_R_is_a_fixed_point():
    rng = np.random.default_rng(3)
    R = np.repeat(_random_R(rng, 1, 4), 50, axis=0)
    for a in (0.5, 0.9, 0.99):
        got, _ = io.integrate(R, a)
        assert np.max(io.rel_err(got, R)) <= 1e-14


@pytest.mark.parametrize("alpha", [0.5, 0.9, 0.99])
def test_n_eff(alpha):
    N = 32
    assert io.n_eff(N, alpha, 0) == N
    vals = [io.n_eff(N, alpha, j) for j in range(0, 5000, 50)]
    assert all(b >= a for a, b in zip(vals, vals[1:]))  # grows monotonically
    assert io.n_eff(N, alpha, 5000) == pytest.approx(io.n_eff_limit(N, alpha), rel=1e-12)
    # the oracle's per-window factor is the same number
    _, fac = io.integrate(np.ones((40, 1, 1)), alpha)
    assert N * fac[39] == pytest.approx(io.n_eff(N, alpha, 39), rel=1e-15)


def test_reset_and_split():
    rng = np.random.default_rng(4)
    R = _random_R(rng, 30, 3)
    whole, _ = io.integrate(R, 0.8)
    st = io.State(3)
    parts = np.concatenate([io.integrate(R[a:b], 0.8, st)[0] for a, b in ((0, 1), (1, 8), (8, 30))])
    assert np.array_equal(parts, whole)  # the carry makes the split invisible (same sequential order)
    fresh, _ = io.integrate(R[10:], 0.8)  # a reset: window 10 is its own R
    assert np.array_equal(fresh[0], R[10])
    assert not np.allclose(fresh[0], whole[10])


def test_weak_source_study():
    # -12 dB per element on a UCA-8 with 32 snapshots per window: one window alone rarely finds the source
    p0, m0 = io.study(0.0)
    p95, m95 = io.study(0.95)
    assert p0 <= 0.5 and m0 <= 0.1, (p0, m0)
    assert p95 >= 0.9 and m95 >= 0.9, (p95, m95)
