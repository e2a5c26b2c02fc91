"""CPU: the (azimuth, elevation) oracle (tests/azel_oracle.py) against hand-made spectra, brute-force minima and the
1-D helper's table."""
import math

import numpy as np
import pytest

from gr_baz_b200 import synth
from oracle import music_oracle as mo

import azel_oracle as ao

LAM = 1.0


def test_local_max_azimuth_wrap_and_edge_rows():
    g = ao.Grid(8, 4, 0.0, 90.0)
    P = np.full(g.K, 1.0)
    P[1 * 8 + 0] = 5.0   # row 1, k = 0: its left neighbour is k = 7 of rows 0..2
    P[1 * 8 + 7] = 4.0   # beaten across the wrap
    P[0 * 8 + 4] = 3.0   # bottom row: no row below it
    P[3 * 8 + 2] = 2.0   # top row: no row above it
    assert ao.pick_local_maxima_2d(P, 4, g) == [8, 4, 26, -1]
    assert not ao.is_local_max(P, 15, g)


def test_constant_zenith_row_has_one_maximum():
    g = ao.Grid(36, 10, 0.0, 90.0)
    P = np.zeros(g.K)
    for i in range(g.n_el):
        P[i * g.n_az:(i + 1) * g.n_az] = 1.0 + i  # rises to a constant zenith row
    cand = [b for b in range(g.K) if ao.is_local_max(P, b, g)]
    assert cand == [9 * 36]
    assert ao.pick_local_maxima_2d(P, 3, g) == [9 * 36, -1, -1]


def test_exclusion_is_chebyshev_and_circular():
    g = ao.Grid(10, 6, 0.0, 50.0)
    P = np.full(g.K, 0.5)
    peaks = {2 * 10 + 1: 9.0, 4 * 10 + 9: 8.0, 2 * 10 + 4: 7.0, 5 * 10 + 5: 6.0}
    for b, v in peaks.items():
        P[b] = v
    # (4, 9) is 2 azimuth steps (across the wrap) and 2 rows from (2, 1); (2, 4) is 3 azimuth steps away
    assert ao.chebyshev(21, 49, g) == 2 and ao.chebyshev(21, 24, g) == 3
    assert ao.pick_local_maxima_2d(P, 4, g, 0) == [21, 49, 24, 55]
    assert ao.pick_local_maxima_2d(P, 4, g, 2) == [21, 24, 55, -1]
    assert ao.pick_local_maxima_2d(P, 4, g, 3) == [21, 55, -1, -1]


def test_nan_and_nonpositive_are_never_maxima():
    g = ao.Grid(6, 3, 0.0, 60.0)
    P = np.full(g.K, 1.0)
    P[7] = np.nan   # (i, k) = (1, 1)
    P[8] = 3.0      # (1, 2): its NaN neighbour fails the comparison
    P[16] = 2.0     # (2, 4)
    assert not ao.is_local_max(P, 7, g) and not ao.is_local_max(P, 8, g)
    assert ao.pick_local_maxima_2d(P, 3, g) == [16, -1, -1]
    assert ao.pick_local_maxima_2d(np.zeros(g.K), 2, g) == [-1, -1]


def test_vectorised_mask_matches_the_literal_rule():
    rng = np.random.default_rng(1)
    for n_az, n_el in ((1, 5), (2, 4), (7, 1), (12, 6)):
        g = ao.Grid(n_az, n_el, 0.0, 60.0)
        P = rng.integers(0, 4, g.K).astype(np.float64)  # many ties
        P[rng.integers(0, g.K)] = np.nan
        assert list(ao.local_max_mask(P, g)) == [ao.is_local_max(P, b, g) for b in range(g.K)]


def test_derivatives_against_central_differences():
    rng = np.random.default_rng(3)
    pos = ao.uca_xyz(8, LAM, alternate_z=True)
    A = np.column_stack([ao.steering(pos, LAM, 40.0, 20.0), ao.steering(pos, LAM, 200.0, -35.0)])
    R = A @ A.conj().T + 0.01 * np.eye(8)
    G = np.linalg.eigh(R)[1][:, :6]
    for _ in range(5):
        ph, ep = rng.uniform(0, 2 * math.pi), rng.uniform(-1.2, 1.2)
        D, g, H = ao.objective(G, pos, LAM, ph, ep)
        h = 1e-5
        for u, d in enumerate(((h, 0.0), (0.0, h))):
            Dp, gp, _ = ao.objective(G, pos, LAM, ph + d[0], ep + d[1])
            Dm, gm, _ = ao.objective(G, pos, LAM, ph - d[0], ep - d[1])
            assert abs((Dp - Dm) / (2 * h) - g[u]) <= 1e-6 * max(1.0, abs(g[u]))
            assert np.allclose((gp - gm) / (2 * h), H[:, u], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("geometry", ["uca_z", "ura"])
def test_refinement_lands_on_the_box_minimum(geometry):
    """noise-free covariance: the refined point is the minimum of D over a 201 x 201 grid of the box to 1/100 of a
    step, unless that minimum lies on the box edge"""
    pos = ao.uca_xyz(8, LAM, alternate_z=True) if geometry == "uca_z" else ao.ura_xyz(4, 4, LAM)
    el_range = (-90.0, 90.0) if geometry == "uca_z" else (0.0, 90.0)
    g = ao.Grid(36, 10, *el_range)
    T = ao.table(pos, LAM, g).reshape(g.K, -1).astype(np.complex64)
    rng = np.random.default_rng(11 if geometry == "ura" else 12)
    checked = 0
    for _ in range(8):
        az, el = rng.uniform(0, 360), rng.uniform(el_range[0] + 5, el_range[1] - 5)
        a = ao.steering(pos, LAM, az, el)
        R = np.outer(a, a.conj())
        G = np.linalg.eigh(R)[1][:, : pos.shape[0] - 1]
        P = ao.spectrum(G, T)
        b = int(np.argmax(P))
        r = ao.refine_slot(G, pos, LAM, b, g)
        plo, phi, elo, ehi = ao.box(b, g)
        P0 = np.linspace(plo, phi, 201)
        P1 = np.linspace(elo, ehi, 201)
        Dg = np.array([[ao.objective(G, pos, LAM, x, y)[0] for y in P1] for x in P0])
        ia, ie = np.unravel_index(np.argmin(Dg), Dg.shape)
        if ia in (0, 200) or (ie in (0, 200) and ehi > elo):
            continue
        checked += 1
        step_az = (phi - plo) / 2.0
        step_el = math.radians((g.el_hi - g.el_lo) / (g.n_el - 1))
        assert abs(r["x"][0] - P0[ia]) <= 0.01 * step_az, (az, el, r["x"], P0[ia])
        assert abs(r["x"][1] - P1[ie]) <= 0.01 * step_el, (az, el, r["x"], P1[ie])
        assert r["Dx"] <= Dg[ia, ie] + 1e-12
    assert checked >= 3


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("geometry", ["ula_x", "uca"])
def test_horizon_row_matches_the_1d_helper(geometry):
    m, K = 8, 360
    pos2 = mo.scaled_antenna_array(synth.SPACING, synth.antenna_array(geometry, m))
    pos3 = np.array([[x, y, 0.0] for x, y in pos2])
    t1 = mo.steering_table_c64(pos2, K, LAM)
    t2 = ao.table(pos3, LAM, ao.Grid(K, 1, 0.0, 0.0)).reshape(K, m).astype(np.complex64)
    # at a zero crossing of cos / sin the value is the fp64 rounding error of the phase itself (|phase| 2^-53, below
    # 1e-14 here), and the two formulations round the phase differently: there the comparison is absolute
    for a, b in ((t1.real, t2.real), (t1.imag, t2.imag)):
        ok = (_ulps(a, b) <= 1) | (np.maximum(np.abs(a), np.abs(b)) <= 1e-14)
        assert ok.all(), np.argwhere(~ok)[:5]
