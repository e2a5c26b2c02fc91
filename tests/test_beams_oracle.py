"""CPU: the beamformer oracle (tests/beams_oracle.py) against its definition's consequences: the distortionless and
LCMV constraints, MVDR's least output power among distortionless weights, LCMV = MVDR for one slot, exact power-of-two
scaling of R, the pivot rule on a mirror pair, failures and unfilled slots."""
import numpy as np
import pytest

import beams_oracle as bo

LAM = 1.0


def ula_x(m):
    return np.c_[0.5 * np.arange(m), np.zeros(m)]


def uca(m):
    r = 0.5 / (2.0 * np.sin(np.pi / m))
    t = 2.0 * np.pi * np.arange(m) / m
    return np.c_[r * np.cos(t), r * np.sin(t)]


def covariance(pos, degs, snaps=512, seed=0, snr_db=20.0):
    """sample covariance of uncorrelated sources at degs over unit noise"""
    rng = np.random.default_rng(seed)
    m = len(pos)
    X = (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
    for t in degs:
        s = (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps)) / np.sqrt(2.0)
        X += 10.0 ** (snr_db / 20.0) * bo.steering_geo(pos, LAM, t)[:, None] * s[None, :]
    return X @ X.conj().T / snaps


@pytest.mark.parametrize("rule", [bo.DAS, bo.MVDR, bo.LCMV])
@pytest.mark.parametrize("m", [3, 4, 8, 16])
def test_distortionless_and_lcmv_constraints(rule, m):
    pos = uca(m)
    degs = [30.0, 100.0, 250.0][: min(3, m - 1)]
    R = covariance(pos, degs, seed=m)
    ang = np.array(degs, np.float32)
    W = bo.weights(R, ang, np.arange(len(degs)), rule, 0.0 if rule == bo.DAS else 0.01, pos=pos, lam=LAM)
    A = np.array([bo.steering_geo(pos, LAM, t) for t in ang]).T  # [M][d]
    WhA = W.conj() @ A
    if rule == bo.LCMV:
        assert np.max(np.abs(WhA - np.eye(len(degs)))) <= 1e-12
    else:
        assert np.max(np.abs(np.diag(WhA) - 1.0)) <= 1e-12


@pytest.mark.parametrize("m", [4, 8])
def test_mvdr_has_least_output_power(m):
    """w^H R w of MVDR (loading 0) is below every distortionless perturbation w + v, v in the null space of a^H"""
    pos = uca(m)
    R = covariance(pos, [40.0, 200.0], seed=3)
    W = bo.weights(R, np.array([40.0, 200.0], np.float32), np.array([0, 1]), bo.MVDR, 0.0, pos=pos, lam=LAM)
    rng = np.random.default_rng(5)
    for i, t in enumerate((40.0, 200.0)):
        a = bo.steering_geo(pos, LAM, t)
        w = W[i]
        p0 = np.vdot(w, R @ w).real
        P = np.eye(m) - np.outer(a, a.conj()) / np.vdot(a, a).real  # projector onto the null space of a^H
        for _ in range(50):
            v = P @ (rng.standard_normal(m) + 1j * rng.standard_normal(m)) * 1e-3
            assert abs(np.vdot(w + v, a) - 1.0) <= 1e-12
            assert np.vdot(w + v, R @ (w + v)).real >= p0 * (1.0 - 1e-12)


def test_lcmv_with_one_slot_equals_mvdr():
    pos = uca(8)
    R = covariance(pos, [75.0], seed=7)
    for bins in ([3, -1], [-1, 3]):
        ang = np.array([75.0, 75.0], np.float32)
        wm = bo.weights(R, ang, np.array(bins), bo.MVDR, 0.1, pos=pos, lam=LAM)
        wl = bo.weights(R, ang, np.array(bins), bo.LCMV, 0.1, pos=pos, lam=LAM)
        assert np.max(np.abs(wm - wl)) <= 1e-12 * np.max(np.abs(wm))


@pytest.mark.parametrize("k", [-40, -3, 5, 40])
def test_power_of_two_scaling_of_R(k):
    pos = uca(8)
    R = covariance(pos, [10.0, 130.0, 260.0], seed=9)
    ang, bins = np.array([10.0, 130.0, 260.0], np.float32), np.array([0, 1, 2])
    for rule, loading in ((bo.MVDR, 0.0), (bo.MVDR, 0.05), (bo.LCMV, 0.0), (bo.LCMV, 0.05)):
        ref = bo.weights(R, ang, bins, rule, loading, pos=pos, lam=LAM)
        got = bo.weights(R * 2.0 ** (2 * k), ang, bins, rule, loading, pos=pos, lam=LAM)
        assert np.array_equal(got, ref), (rule, loading, k)


def test_pivot_rule_on_a_mirror_pair():
    """an x-axis ULA sees t and -t alike: LCMV on the mirror pair fails the pivot test and zeroes the window; MVDR and
    DAS are unaffected, and a pair apart passes"""
    pos = ula_x(6)
    R = covariance(pos, [60.0], seed=11)
    ang = np.array([60.0, 300.0], np.float32)
    assert np.all(bo.weights(R, ang, np.array([0, 1]), bo.LCMV, 0.0, pos=pos, lam=LAM) == 0)
    assert np.all(bo.weights(R, ang, np.array([0, 1]), bo.MVDR, 0.0, pos=pos, lam=LAM) != 0)
    assert np.all(bo.weights(R, ang, np.array([0, 1]), bo.DAS, 0.0, pos=pos, lam=LAM) != 0)
    apart = np.array([60.0, 120.0], np.float32)
    assert np.all(bo.weights(R, apart, np.array([0, 1]), bo.LCMV, 0.0, pos=pos, lam=LAM) != 0)


def test_failures_and_unfilled_slots():
    m = 4
    pos = uca(m)
    R = covariance(pos, [20.0], seed=13)
    ang = np.array([20.0, 0.0, 90.0], np.float32)
    bins = np.array([5, -1, 9])
    for rule in (bo.DAS, bo.MVDR, bo.LCMV):
        W = bo.weights(R, ang, bins, rule, 0.0, pos=pos, lam=LAM)
        assert np.all(W[1] == 0) and np.all(W[0] != 0) and np.all(W[2] != 0)
        x = (np.random.default_rng(1).standard_normal(64 * m) + 0j).astype(np.complex64)
        x[3] = np.nan
        y = bo.beams(x, W)
        assert np.all(y[1] == 0)
    dead = R.copy()
    dead[2, :] = dead[:, 2] = 0  # a dead antenna: R is singular without loading
    for rule in (bo.MVDR, bo.LCMV):
        assert np.all(bo.weights(dead, ang, bins, rule, 0.0, pos=pos, lam=LAM) == 0)
        assert np.all(bo.weights(dead, ang, bins, rule, 0.01, pos=pos, lam=LAM)[[0, 2]] != 0)
    nan = R.copy()
    nan[0, 1] = nan[1, 0] = np.nan
    assert np.all(bo.weights(nan, ang, bins, bo.MVDR, 0.0, pos=pos, lam=LAM) == 0)
    tab = np.ones((36, m), np.complex64)
    tab[9] = 0  # a zero table row: DAS's a^H a = 0, not finite
    assert np.all(bo.weights(None, ang, bins, bo.DAS, 0.0, table=tab) == 0)
    assert np.all(bo.weights(R, ang, np.array([-1, -1, -1]), bo.LCMV, 0.0, pos=pos, lam=LAM) == 0)
