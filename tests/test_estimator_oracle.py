"""CPU: the MVDR / Bartlett oracle (tests/estimator_oracle.py) against closed forms, the beamformer view of both spectra,
finite differences and a 1000x finer grid."""
import math

import numpy as np
import pytest

from oracle import music_oracle as mo

import azel_oracle as ao
import estimator_oracle as eo
import refine_oracle as ro

LAM = 1.0
DEG = math.pi / 180.0


def uca(m, radius=0.5):
    t = 2.0 * np.pi * np.arange(m) / m
    return np.stack([radius * np.cos(t), radius * np.sin(t)], axis=1)


def random_hpd(m, rng):
    A = rng.standard_normal((m, 2 * m)) + 1j * rng.standard_normal((m, 2 * m))
    return A @ A.conj().T / (2 * m)


@pytest.mark.parametrize("kind,loading", [("mvdr", 0.0), ("mvdr", 0.1), ("bartlett", 0.0)])
@pytest.mark.parametrize("m", [2, 4, 8, 16])
def test_single_source_closed_form(kind, loading, m):
    """R = p a0 a0^H + s2 I with ||a0||^2 = M: P(theta0) = p + (s2 + delta) / M (delta = 0 for Bartlett)"""
    pos = uca(m)
    a0 = ro.steering(pos, LAM, 0.7)[0]
    p, s2 = 2.5, 0.3
    R = p * np.outer(a0, a0.conj()) + s2 * np.eye(m)
    P = eo.spectrum(R, a0[None, :], kind, loading)[0]
    delta = loading * np.trace(R).real / m if kind == "mvdr" else 0.0
    assert abs(P - (p + (s2 + delta) / m)) <= 1e-12 * P


@pytest.mark.parametrize("m", [2, 3, 5, 8, 16])
def test_beamformer_power(m):
    """MVDR is w^H R w for w = R^-1 a / (a^H R^-1 a); Bartlett is w^H R w for w = a / ||a||^2"""
    rng = np.random.default_rng(m)
    pos = uca(m)
    R = random_hpd(m, rng)
    table = np.array([ro.steering(pos, LAM, t)[0] for t in np.linspace(0.0, 2.0 * np.pi, 37)])
    Pm = eo.spectrum(R, table, "mvdr")
    Pb = eo.spectrum(R, table, "bartlett")
    for k, a in enumerate(table):
        y = np.linalg.solve(R, a)
        w = y / (a.conj() @ y)
        assert abs(Pm[k] - eo.beam_power(R, w)) <= 1e-10 * Pm[k]
        w = a / np.sum(np.abs(a) ** 2)
        assert abs(Pb[k] - eo.beam_power(R, w)) <= 1e-12 * Pb[k]


def test_mvdr_not_positive_definite_is_nan():
    m = 4
    R = np.zeros((m, m), complex)
    table = np.ones((5, m), np.complex64)
    assert np.all(np.isnan(eo.spectrum(R, table, "mvdr")))
    R[0, 0] = np.nan
    assert np.all(np.isnan(eo.spectrum(R, table, "mvdr", 0.01)))
    w = eo.picks(eo.spectrum(R, table, "mvdr"), 2, 5)
    assert list(w[2]) == [-1, -1] and list(w[0]) == [0.0, 0.0]


@pytest.mark.parametrize("kind", eo.KINDS)
def test_derivatives_central_differences(kind):
    rng = np.random.default_rng(5)
    m = 6
    pos = uca(m)
    R = random_hpd(m, rng)
    for t in (0.3, 1.9, 4.0):
        D, D1, D2 = eo.objective(R, kind, 0.05 if kind == "mvdr" else 0.0, pos, LAM, t)
        h = 1e-5
        Dp, D1p, _ = eo.objective(R, kind, 0.05 if kind == "mvdr" else 0.0, pos, LAM, t + h)
        Dm, D1m, _ = eo.objective(R, kind, 0.05 if kind == "mvdr" else 0.0, pos, LAM, t - h)
        assert abs((Dp - Dm) / (2 * h) - D1) <= 1e-6 * (abs(D1) + abs(D))
        assert abs((D1p - D1m) / (2 * h) - D2) <= 1e-6 * (abs(D2) + abs(D1))
    pos3 = np.concatenate([pos, rng.uniform(-0.3, 0.3, (m, 1))], axis=1)
    for ph, ep in ((0.4, 0.2), (2.5, -0.6)):
        ld = 0.05 if kind == "mvdr" else 0.0
        D, g, H = eo.objective_azel(R, kind, ld, pos3, LAM, ph, ep)
        h = 1e-5
        for u, (dp, de) in enumerate(((h, 0.0), (0.0, h))):
            fp = eo.objective_azel(R, kind, ld, pos3, LAM, ph + dp, ep + de)
            fm = eo.objective_azel(R, kind, ld, pos3, LAM, ph - dp, ep - de)
            assert abs((fp[0] - fm[0]) / (2 * h) - g[u]) <= 1e-6 * (np.max(np.abs(g)) + abs(D))
            assert np.max(np.abs((fp[1] - fm[1]) / (2 * h) - H[u])) <= 1e-6 * (np.max(np.abs(H)) + np.max(np.abs(g)))


def one_source_window(pos, truth_deg, snaps, seed, noise=0.1):
    rng = np.random.default_rng(seed)
    m = pos.shape[0]
    a = ro.steering(pos, LAM, truth_deg * DEG)[0]
    X = noise * (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
    X += a[:, None] * np.exp(2j * np.pi * rng.uniform(0.0, 1.0, snaps))[None, :]
    return X.T.reshape(-1).astype(np.complex64)


@pytest.mark.parametrize("kind", eo.KINDS)
@pytest.mark.parametrize("m", [4, 8])
def test_refinement_matches_fine_grid(kind, m):
    """the refined angle is the extremum of the objective on a 1000x finer grid around the grid bin"""
    pos = uca(m)
    K = 360
    table = mo.steering_table_c64(pos.tolist(), K, LAM)
    for seed, truth in ((1, 37.31), (2, 211.77)):
        x = one_source_window(pos, truth, 256, seed)
        loading = 0.01 if kind == "mvdr" else 0.0
        r = eo.work(x, m, 1, table, kind, loading)
        b = int(r["bins"][0])
        s = eo.refine_slot(r["R"], kind, loading, pos, LAM, b, K)
        assert not s["kept"]
        step = 1.0 / 1000.0
        grid = (b + np.arange(-1000, 1001) * step) * (360.0 / K) * DEG
        vals = [eo.objective(r["R"], kind, loading, pos, LAM, t)[0] for t in grid]
        best = grid[int(np.argmin(vals))]
        assert abs(s["theta"] - best) <= step * (360.0 / K) * DEG
        assert s["Dx"] <= min(vals) + 1e-12 * abs(min(vals))
        assert abs(float(s["angle"]) - truth) < 0.2


@pytest.mark.parametrize("kind", eo.KINDS)
def test_refinement_azel_matches_fine_grid(kind):
    m = 8
    pos = ao.uca_xyz(m, LAM, alternate_z=True)
    grid = ao.Grid(72, 19, 0.0, 90.0)
    rng = np.random.default_rng(9)
    az, el = 101.3, 33.7
    a = ao.steering(pos, LAM, az, el)
    X = 0.1 * (rng.standard_normal((m, 512)) + 1j * rng.standard_normal((m, 512))) / np.sqrt(2.0)
    X += a[:, None] * np.exp(2j * np.pi * rng.uniform(0.0, 1.0, 512))[None, :]
    R = mo.covariance(X.T.reshape(-1).astype(np.complex64), m)
    loading = 0.01 if kind == "mvdr" else 0.0
    P = eo.spectrum(R, ao.table(pos, LAM, grid).astype(np.complex64), kind, loading)
    b = int(np.nanargmax(P))
    s = eo.refine_slot_azel(R, kind, loading, pos, LAM, b, grid)
    assert not s["kept"]
    x0, x1 = s["x"]
    # a 1000x finer grid in each direction, locally around the refined point (one coarse step = 5 degrees)
    fine = 5.0 * DEG / 1000.0
    best = min(eo.objective_azel(R, kind, loading, pos, LAM, x0 + i * fine, x1 + j * fine)[0]
               for i in range(-3, 4) for j in range(-3, 4))
    assert s["Dx"] <= best + 1e-12 * abs(best)
    assert abs(float(s["azimuth"]) - az) < 0.5 and abs(float(s["elevation"]) - el) < 0.5
