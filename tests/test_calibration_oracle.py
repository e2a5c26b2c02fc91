"""CPU: the receiver calibration model (tests/calibration_oracle.py) recovers the gains exactly on exact covariances,
where the principal eigenvector does not, and reports its failure cases."""
import math

import numpy as np
import pytest

import calibration_oracle as co

LAM = 1.0


def ula(m):
    return np.c_[np.arange(m) * 0.5, np.zeros(m)]


def uca(m):
    r = 0.5 / (2.0 * math.sin(math.pi / m))
    t = 2.0 * math.pi * np.arange(m) / m
    return np.c_[r * np.cos(t), r * np.sin(t)]


def random_gains(rng, m):
    """+-3 dB and a uniform phase per element"""
    return 10.0 ** (rng.uniform(-3.0, 3.0, m) / 20.0) * np.exp(1j * rng.uniform(-math.pi, math.pi, m))


def population(g, a0, p, s2):
    """R = G (p a0 a0^H + s2 I) G^H"""
    A = p * np.outer(a0, np.conj(a0)) + s2 * np.eye(len(a0))
    return (g[:, None] * A) * np.conj(g)[None, :]


ARRAYS = [("ula2", ula(2)), ("ula3", ula(3)), ("ula4", ula(4)), ("uca8", uca(8)), ("uca16", uca(16))]


@pytest.mark.parametrize("name,pos", ARRAYS)
def test_exact_on_population_covariance(name, pos):
    """on R = G(p a0 a0^H + s2 I)G^H the fit recovers g to 1e-11 for s2 from 0 to 10 p; the principal eigenvector does
    not once the noise is coloured by unequal gains"""
    m = len(pos)
    rng = np.random.default_rng(100 + m)
    kind = co.PHASE if m < 3 else co.GAIN_PHASE
    worst_eig = 0.0
    for trial in range(5):
        g = random_gains(rng, m)
        az = rng.uniform(0.0, 360.0)
        a0 = co.steering_1d(pos, LAM, az)
        want = co.normalised(g, kind)
        for s2 in (0.0, 0.1, 1.0, 10.0):
            got, rho, sweeps = co.solve(population(g, a0, 1.0, s2), a0, kind)
            assert np.max(np.abs(got - want)) <= 1e-11, (name, trial, s2, got, want)
            assert rho <= 1e-12 and 1 <= sweeps <= co.MAX_SWEEPS
            if s2 > 0:
                worst_eig = max(worst_eig, np.max(np.abs(co.principal(population(g, a0, 1.0, s2), a0, kind) - want)))
    if m >= 3:
        assert worst_eig > 1e-3, worst_eig


def test_phase_with_two_elements():
    """PHASE identifies the phase difference of a two-channel receiver; GAIN_PHASE is refused there"""
    pos = ula(2)
    g = np.array([0.7 * np.exp(0.4j), 1.9 * np.exp(-2.1j)])
    a0 = co.steering_1d(pos, LAM, 33.0)
    got, rho, _ = co.solve(population(g, a0, 2.0, 0.5), a0, co.PHASE)
    assert np.max(np.abs(got - co.normalised(g, co.PHASE))) <= 1e-12
    assert abs(got[0] - 1.0) <= 1e-15 and np.allclose(np.abs(got), 1.0, atol=1e-15)
    with pytest.raises(ValueError):
        co.solve(population(g, a0, 2.0, 0.5), a0, co.GAIN_PHASE)


def test_azel_steering_matches_1d_at_zero_elevation():
    pos = uca(8)
    a1 = co.steering_1d(pos, LAM, 71.0)
    a3 = co.steering_azel(np.c_[pos, np.zeros(8)], LAM, 71.0, 0.0)
    assert np.max(np.abs(a1 - a3)) <= 1e-14


def test_correct_inverts_the_gains():
    rng = np.random.default_rng(5)
    g = random_gains(rng, 6)
    R = population(np.ones(6), co.steering_1d(uca(6), LAM, 10.0), 1.0, 0.3)
    Rraw = (g[:, None] * R) * np.conj(g)[None, :]
    assert np.max(np.abs(co.correct(Rraw, g) - R)) <= 1e-14


def test_failures():
    pos = uca(4)
    a0 = co.steering_1d(pos, LAM, 0.0)
    with pytest.raises(ValueError):  # no power
        co.solve(np.zeros((4, 4), np.complex128), a0)
    R = population(np.ones(4), a0, 1.0, 0.1)
    bad = R.copy()
    bad[1, 2] = np.nan
    with pytest.raises(ValueError):  # not finite
        co.solve(bad, a0)
    dead = R.copy()
    dead[2, :] = 0
    dead[:, 2] = 0
    with pytest.raises(ValueError):  # a dead channel
        co.solve(dead, a0)
    with pytest.raises(ValueError):  # unknown kind
        co.solve(R, a0, 3)


def test_sample_covariance_accuracy():
    """16 windows of 1024 snapshots at 20 dB: phase within 0.5 degree, magnitude within 1 %"""
    rng = np.random.default_rng(9)
    pos = uca(8)
    m, N, W = 8, 1024, 16
    g = random_gains(rng, m)
    a0 = co.steering_1d(pos, LAM, 140.0)
    R = np.zeros((m, m), np.complex128)
    for _ in range(W):
        s = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / math.sqrt(2.0) * 10.0
        n = (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / math.sqrt(2.0)
        X = g[:, None] * (a0[:, None] * s[None, :] + n)
        R += X @ X.conj().T / N
    got, rho, sweeps = co.solve(R / W, a0)
    want = co.normalised(g, co.GAIN_PHASE)
    assert np.max(np.abs(np.angle(got / want))) <= math.radians(0.5)
    assert np.max(np.abs(np.abs(got) / np.abs(want) - 1.0)) <= 0.01
    assert rho < 0.05 and sweeps < co.MAX_SWEEPS
