"""CPU: the self-calibration model (tests/calib_blind_oracle.py) recovers the gains on exact covariances, meets its
accuracy on seeded statistical cases, and reports its refusals."""
import math

import numpy as np
import pytest

import calib_blind_oracle as cb


def uca(m):
    r = 0.5 / (2.0 * math.sin(math.pi / m))
    t = 2.0 * math.pi * np.arange(m) / m
    return np.c_[r * np.cos(t), r * np.sin(t)]


def steering(pos, deg):
    """exp(-j 2 pi (x cos + y sin)) of a geometry in wavelengths, [.., M]"""
    t = np.radians(np.asarray(deg, np.float64))[..., None]
    return np.exp(-2j * np.pi * (pos[:, 0] * np.cos(t) + pos[:, 1] * np.sin(t)))


def gains(rng, m):
    """magnitudes 0.8 - 1.2 and uniform +-180 degree phases"""
    return rng.uniform(0.8, 1.2, m) * np.exp(1j * rng.uniform(-math.pi, math.pi, m))


def population(m, K, d, S, seed, s2=0.1):
    """exact segment covariances G (A_s diag(p) A_s^H + s2 I) G^H with the d directions of segment s on grid bins,
    spread over the circle (segment s in sector s of S), against the fp64 table of K rows"""
    rng = np.random.default_rng(seed)
    pos = uca(m)
    table = steering(pos, np.arange(K) * 360.0 / K)
    g = gains(rng, m)
    Rs = []
    for s in range(S):
        k0 = s * K // S + rng.integers(0, K // S)
        ks = [(k0 + j * K // (d + 1) + rng.integers(0, K // (4 * (d + 1)))) % K for j in range(d)]
        A = table[ks].T
        R = A @ np.diag(rng.uniform(1.0, 3.0, d)) @ A.conj().T + s2 * np.eye(m)
        Rs.append((g[:, None] * R) * np.conj(g)[None, :])
    return np.array(Rs), table, g, pos


def statistical(m, d, S, seed, N=256, snr_db=10.0, K=3600):
    """one window of N snapshots per segment, d sources at uniform random directions, 10 dB each over unit noise, the
    complex64-rounded table and input"""
    rng = np.random.default_rng(seed)
    pos = uca(m)
    table = steering(pos, np.arange(K) * 360.0 / K).astype(np.complex64).astype(np.complex128)
    g = gains(rng, m)
    amp = 10.0 ** (snr_db / 20.0)
    Rs = []
    for _ in range(S):
        th = rng.uniform(0.0, 360.0, d)
        X = (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / math.sqrt(2.0)
        for t in th:
            s = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / math.sqrt(2.0)
            X += amp * steering(pos, t)[:, None] * s[None, :]
        X = (g[:, None] * X).astype(np.complex64).astype(np.complex128)
        Rs.append(X @ X.conj().T / N)
    return np.array(Rs), table, g, pos


POPULATION = [(m, d, S, seed) for m in (4, 8) for d in (1, 2) for S in (8, 16) for seed in range(10)]
# the one exact case the schedule misses: one bin off every direction (include/music_b200.h, "limits"); neither 128
# starts nor 48 iterations per start reach the exact fit
MISSED = {(8, 1, 8, 5)}


@pytest.mark.parametrize("m,d,S,seed", [pytest.param(*c, marks=pytest.mark.xfail(strict=True, reason="one-bin grid trap"))
                                        if c in MISSED else c for c in POPULATION])
def test_exact_on_population_covariances(m, d, S, seed):
    """magnitudes to 1e-9 relative and phases to 1e-7 degrees, a vanishing misfit; PHASE gives the same phases"""
    Rs, table, g, pos = population(m, 720, d, S, seed)
    got, angles, misfit, used, win = cb.solve(Rs, table, d, cb.GAIN_PHASE, 32, seed, pos)
    want = cb.normalised(g, cb.GAIN_PHASE)
    assert np.max(np.abs(np.abs(got) / np.abs(want) - 1.0)) <= 1e-9
    assert np.max(np.abs(np.degrees(np.angle(got / want)))) <= 1e-7
    assert misfit <= 1e-20 and 1 <= used <= cb.T2
    if seed == 0:
        ph, _, _, _, _ = cb.solve(Rs, table, d, cb.PHASE, 32, seed, pos)
        assert np.max(np.abs(ph - want / np.abs(want))) <= 1e-9


# (m, d, S) -> the largest phase RMS (degrees) over the seeds
STATISTICAL = {(4, 1, 16): 0.7, (8, 1, 16): 0.7, (4, 2, 8): 2.0, (8, 2, 8): 2.0}


@pytest.mark.parametrize("m,d,S", list(STATISTICAL))
def test_statistical_cases(m, d, S):
    """uniform +-180 degree phases, magnitudes 0.8 - 1.2, N = 256, 10 dB, 3600 rows, 32 starts: every seed within the
    phase RMS gate and magnitudes within 3 %"""
    for seed in range(4):
        Rs, table, g, pos = statistical(m, d, S, 100 + seed)
        got, angles, misfit, used, win = cb.solve(Rs, table, d, cb.GAIN_PHASE, 32, seed, pos)
        want = cb.normalised(g, cb.GAIN_PHASE)
        assert cb.phase_rms_deg(got, g) <= STATISTICAL[(m, d, S)], (seed, cb.phase_rms_deg(got, g))
        assert np.max(np.abs(np.abs(got) / np.abs(want) - 1.0)) <= 0.03
        assert angles.shape == (S, d)


def test_draw_is_counter_based():
    """the start phases depend on (seed, start, element) alone, lie in [-pi, pi), and start 0 is all ones"""
    phi = cb.start_phases(5, 4, 6)
    assert np.array_equal(phi[0], np.ones(6))
    assert np.array_equal(phi[:3], cb.start_phases(5, 3, 6)[:, :6])
    assert cb.draw(5, 2, 3) == cb.draw(5, 2, 3) != cb.draw(6, 2, 3)
    t = [cb.draw(s, p, e) for s in range(3) for p in range(1, 20) for e in range(16)]
    assert min(t) >= -math.pi and max(t) < math.pi and len(set(t)) == len(t)


def test_refusals():
    Rs, table, g, pos = population(4, 360, 1, 4, 0)
    ok = dict(d=1, kind=cb.GAIN_PHASE, starts=4)
    cb.solve(Rs, table, **ok, pos=pos)
    bad = [dict(ok, d=0), dict(ok, d=3), dict(ok, starts=0), dict(ok, starts=257), dict(ok, kind=3)]
    for kw in bad:
        with pytest.raises(ValueError):
            cb.solve(Rs, table, **kw, pos=pos)
    with pytest.raises(ValueError):
        cb.solve(Rs[:0], table, **ok, pos=pos)
    with pytest.raises(ValueError):
        cb.solve(Rs, table, **ok, pos=np.c_[np.arange(4) * 0.5, np.arange(4) * 0.25])  # collinear
    with pytest.raises(ValueError):
        cb.solve(Rs[:, :2, :2], table[:, :2], d=1, kind=cb.GAIN_PHASE, starts=4)  # m < 3
    nan = Rs.copy()
    nan[1, 2, 2] = np.nan
    with pytest.raises(ValueError):
        cb.solve(nan, table, **ok, pos=pos)
    assert cb.collinear(np.zeros((3, 2))) and not cb.collinear(uca(3))
