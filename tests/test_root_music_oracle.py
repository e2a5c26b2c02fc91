"""CPU: the root-MUSIC definition (tests/root_music_oracle.py) against the direct MUSIC denominator, the truth of
noiseless windows, the reference's grid peak and the resolution it is there for."""
import math

import numpy as np
import pytest

from oracle import music_oracle as mo

import refine_oracle as ro
import root_music_oracle as rm

LAM = 1.0


def ula(m, axis_deg=0.0, spacing=0.5, p0=(0.0, 0.0), reverse=False):
    a = math.radians(axis_deg)
    pos = np.array([[p0[0] + i * spacing * math.cos(a), p0[1] + i * spacing * math.sin(a)] for i in range(m)])
    return pos[::-1].copy() if reverse else pos


def mirror_report(t, pos):
    """the angle the root mode reports for a source at t degrees: the lower of t and its mirror across the array axis"""
    _, _, s = rm.ula_geometry(pos, LAM)
    alpha = math.degrees(math.atan2(s[1], s[0]))
    return min(t % 360.0, (2.0 * alpha - t) % 360.0)


def circ(a, b):
    return abs((a - b + 180.0) % 360.0 - 180.0)


GEOMS = [ula(5), ula(5, 90.0), ula(5, 30.0, p0=(0.7, -1.3)), ula(5, 30.0, p0=(0.7, -1.3), reverse=True),
         ula(5, 0.0, 0.25, p0=(-2.0, 0.4), reverse=True)]


@pytest.mark.parametrize("gi", range(len(GEOMS)))
def test_laurent_polynomial_is_the_music_denominator(gi):
    pos = GEOMS[gi]
    m = pos.shape[0]
    ok, _, s = rm.ula_geometry(pos, LAM)
    assert ok
    rng = np.random.default_rng(gi)
    for p in range(1, m):
        Z = rng.standard_normal((m, m)) + 1j * rng.standard_normal((m, m))
        G = np.linalg.qr(Z)[0][:, :p]
        c = rm.coefficients(G)
        assert np.allclose(c, np.conj(c[::-1]), rtol=0, atol=1e-14)
        for t in rng.uniform(0.0, 2.0 * math.pi, 20):
            D = ro.objective(G, pos, LAM, t)[0]
            L = rm.laurent(c, rm.z0_of(s, LAM, t))
            assert abs(L.imag) <= 1e-12 * D and abs(L.real - D) <= 1e-12 * D, (gi, p, t, L, D)


def separated_angles(rng, n, alpha, min_cos=0.05):
    """n angles over [0, 360), at least 2 degrees from end-fire, with distinct cos(t - alpha) (distinct roots)"""
    while True:
        t = rng.uniform(0.0, 360.0, n)
        off = np.abs(((t - alpha) % 180.0))
        if np.any(np.minimum(off, 180.0 - off) < 2.0):
            continue
        cs = np.cos(np.radians(t - alpha))
        if n == 1 or np.min(np.abs(np.subtract.outer(cs, cs))[np.triu_indices(n, 1)]) >= min_cos:
            return t


@pytest.mark.parametrize("m", [2, 3, 4, 8, 12, 16])
def test_noiseless_roots_sit_at_the_sources(m):
    """exact double roots on the circle: fp64 rooting is good to about sqrt(eps), well inside 5e-4 degrees"""
    rng = np.random.default_rng(100 + m)
    worst = 0.0
    for n in (1, 2):
        if n >= m:
            continue
        for gi, axis in enumerate((0.0, 30.0)):
            pos = ula(m, axis, p0=(0.3 * gi, -0.2 * gi), reverse=bool(gi))
            _, _, s = rm.ula_geometry(pos, LAM)
            alpha = math.degrees(math.atan2(s[1], s[0]))
            for _ in range(100):
                th = separated_angles(rng, n, alpha)
                A = np.stack([ro.steering(pos, LAM, math.radians(t))[0] for t in th], axis=1)
                R = A @ A.conj().T
                r = rm.work_R(R, pos, LAM, 3600, n)
                want = sorted(mirror_report(t, pos) for t in th)
                got = sorted(float(a) for a in r["angles"])
                err = max(circ(g, w) for g, w in zip(got, want))
                worst = max(worst, err)
                assert err <= 5e-4, (m, n, axis, th, got, want)
                assert np.all(r["bins"] >= 0) and np.all(r["levels"] > 0)
    print("m = %d: worst noiseless error %.2e deg" % (m, worst))


def test_single_source_matches_the_grid_peak():
    """20 dB, one source every 7 degrees on the x-axis ULA (mirror rows bit-identical): the root angle is within one
    bin of the reference rule's n = 1 pick at K = 3600"""
    m, K, N = 4, 3600, 4096
    pos = ula(m)
    table = mo.steering_table_c64(pos.tolist(), K, LAM)
    rng = np.random.default_rng(7)
    for t in np.arange(3.0, 360.0, 7.0):
        off = t % 180.0
        if min(off, 180.0 - off) < 2.0:
            continue
        a = ro.steering(pos, LAM, math.radians(t))[0]
        X = a[:, None] * np.exp(2j * np.pi * rng.uniform(0, 1, N))[None, :]
        X += 0.1 * (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / np.sqrt(2.0)
        x = X.T.reshape(-1).astype(np.complex64)
        grid = mo.work(x, m, 1, table)
        r = rm.work(x, m, 1, K, pos, LAM)
        assert circ(float(r["angles"][0]), float(grid["angles"][0])) <= 360.0 / K + 1e-9, (t, r["angles"], grid["angles"])
        assert circ(float(r["angles"][0]), mirror_report(t, pos)) < 0.5


def test_ula_condition():
    assert rm.ula_geometry(ula(4), LAM)[0]
    assert rm.ula_geometry(ula(8, 0.0, 0.25), LAM)[0]
    assert rm.ula_geometry(ula(6, 123.0, p0=(5.0, -3.0), reverse=True), LAM)[0]
    uca = np.array([[math.cos(2 * math.pi * i / 6), math.sin(2 * math.pi * i / 6)] for i in range(6)]) * 0.5
    assert not rm.ula_geometry(uca, LAM)[0]
    bent = ula(5)
    bent[2, 1] += 1e-5 * 0.5
    assert not rm.ula_geometry(bent, LAM)[0]
    assert not rm.ula_geometry(ula(4, 0.0, 0.6), LAM)[0]
    assert not rm.ula_geometry(np.zeros((4, 2)), LAM)[0]


def two_source_window(rng, pos, th, N, snr_db):
    m = pos.shape[0]
    A = np.stack([ro.steering(pos, LAM, math.radians(t))[0] for t in th], axis=1)
    S = (rng.standard_normal((len(th), N)) + 1j * rng.standard_normal((len(th), N))) / np.sqrt(2.0)
    X = 10.0 ** (snr_db / 20.0) * (A @ S) + (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / np.sqrt(2.0)
    return X.T.reshape(-1).astype(np.complex64)


@pytest.mark.parametrize("m,th", [(4, (70.0, 78.0)), (8, (30.0, 36.0))])
def test_resolution(m, th):
    """0 dB, 1024 snapshots, 100 windows: both sources within half their separation in at least 90 % of windows"""
    rng = np.random.default_rng(1)
    pos = ula(m)
    ok = 0
    for _ in range(100):
        x = two_source_window(rng, pos, th, 1024, 0.0)
        r = rm.work(x, m, 2, 3600, pos, LAM)
        got = sorted(float(a) for a in r["angles"])
        ok += all(abs(g - t) < (th[1] - th[0]) / 2 for g, t in zip(got, th))
    assert ok >= 90, ok
