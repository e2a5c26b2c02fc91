"""The IAA oracle (tests/iaa_oracle.py) on the CPU: its start is Bartlett, its covariance form is the per-snapshot
weighted-least-squares form of Yardibi et al., its invariances and failure rules, and the seeded cases that show what it
is for (coherent paths on an az-el URA and a ULA, fewer snapshots than antennas) and where MUSIC stays better (closely
spaced uncorrelated sources)."""
import numpy as np
import pytest

from oracle import music_oracle as mo

import azel_oracle as ao
import estimator_oracle as eo
import helpers
import iaa_oracle as io


def random_R(rng, m, N):
    X = (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / np.sqrt(2.0)
    return X @ X.conj().T / N


def test_zero_iterations_is_bartlett():
    rng = np.random.default_rng(1)
    for m in (2, 4, 7, 16):
        tab = helpers.planar_table(m, 360, m)
        R = random_R(rng, m, 3 * m)
        assert np.array_equal(io.spectrum(R, tab, 0), eo.spectrum(R, tab, "bartlett"))


@pytest.mark.parametrize("m,N", [(4, 64), (8, 8), (16, 8)])
def test_covariance_form_is_the_snapshot_form(m, N):
    rng = np.random.default_rng(m + N)
    tab = helpers.planar_table(m, 360, m)
    X = (rng.standard_normal((N, m)) + 1j * rng.standard_normal((N, m))) / np.sqrt(2.0)
    X[:, :] += 3.0 * np.exp(-2j * np.pi * rng.uniform(size=m))[None, :] * rng.standard_normal((N, 1))
    R = X.T @ X.conj() / N
    for it in (1, 5, 15):
        got, ref = io.spectrum(R, tab, it), io.spectrum_snapshots(X, tab, it)
        assert np.max(np.abs(got - ref) / np.abs(ref)) <= 1e-12, it


def test_invariances():
    rng = np.random.default_rng(3)
    m, K = 8, 360
    tab = helpers.planar_table(m, K, 5).astype(np.complex128)
    R = random_R(rng, m, 32)
    P = io.spectrum(R, tab, 15, 0.01)
    # a row multiplied by a phase
    ph = tab * np.exp(1j * rng.uniform(0.0, 2.0 * np.pi, K))[:, None]
    assert np.max(np.abs(io.spectrum(R, ph, 15, 0.01) - P)) <= 1e-12 * np.max(P)
    # the antennas permuted in both R and the table
    perm = rng.permutation(m)
    Pp = io.spectrum(R[np.ix_(perm, perm)], tab[:, perm], 15, 0.01)
    assert np.max(np.abs(Pp - P)) <= 1e-12 * np.max(P)
    # R -> c R gives P -> c P (exactly for a power of two)
    assert np.array_equal(io.spectrum(4.0 * R, tab, 15, 0.01), 4.0 * P)
    assert np.max(np.abs(io.spectrum(3.0 * R, tab, 15, 0.01) - 3.0 * P)) <= 1e-12 * 3.0 * np.max(P)


def test_zero_and_duplicate_rows():
    rng = np.random.default_rng(4)
    m, K = 8, 360
    tab = helpers.calibrated_table(helpers.table_wl(helpers.array_wl("uca", m), K), 9)
    tab[[5, 77, 300]] = 0
    tab[200] = tab[100]
    R = random_R(rng, m, 64)
    P = io.spectrum(R, tab, 15)
    assert np.all(np.isfinite(P))
    assert np.all(P[[5, 77, 300]] == 0.0)
    assert P[200] == P[100]
    # a zero row adds nothing: the spectrum of the other rows is that of the table without it
    keep = np.ones(K, bool)
    keep[[5, 77, 300]] = False
    assert np.max(np.abs(io.spectrum(R, tab[keep], 15) - P[keep])) <= 1e-12 * np.max(P)


def test_failure_windows():
    tab = helpers.planar_table(4, 90, 1)
    R = random_R(np.random.default_rng(5), 4, 16)
    bad = R.copy()
    bad[1, 2] = np.nan
    for r in (bad, np.zeros((4, 4), complex), -R):
        assert np.all(np.isnan(io.spectrum(r, tab, 15)))
    w = io.window(np.zeros((4, 4), complex), tab, 2)
    assert list(w["bins"]) == [-1, -1] and not np.any(w["levels"])


def test_fewer_snapshots_than_antennas_with_loading_zero():
    rng = np.random.default_rng(6)
    tab = helpers.table_wl(helpers.array_wl("uca", 16), 360)
    R = random_R(rng, 16, 4)  # rank 4
    assert np.all(np.isfinite(io.spectrum(R, tab, 15, 0.0)))


# ---- what IAA is for, on seeded windows --------------------------------------------------------------------------------
def music_local_2d(R, tab, grid, n):
    ev, V = np.linalg.eigh(R)
    return ao.pick_local_maxima_2d(ao.spectrum(V[:, : R.shape[0] - n], tab), n, grid)


@pytest.mark.parametrize("N,need", [(256, 12), (8, 11)])
def test_coherent_azel_ura(N, need):
    """two coherent paths on a 4 x 4 URA.  Observed on these seeded windows: IAA finds both in 12 of 12 at N = 256 and
    in 11 of 12 at N = 8 < m, az-el MUSIC with LOCAL_MAXIMA in 1 and 0.  Held: IAA in at least the observed count
    (`need`), MUSIC in at most one."""
    pos, grid, tab, x = io.azel_case(N)
    iaa = music = 0
    levels = []
    truth = io.azel_truth_bins(grid)
    for w in range(len(x)):
        R = mo.covariance(x[w], 16)
        P = io.spectrum(R, tab, 15)
        iaa += io.azel_found(ao.pick_local_maxima_2d(P, 2, grid), grid)
        levels.append(P[truth])
        music += io.azel_found(music_local_2d(R, tab, grid, 2), grid)
    assert iaa >= need and music <= 1, (iaa, music)
    if N == 256:
        # the levels are the paths' powers (1 and 0.64): the means are 0.97 and 0.62
        lv = np.mean(levels, axis=0)
        assert 0.85 <= lv[0] <= 1.15 and 0.5 <= lv[1] <= 0.75, lv


def test_coherent_ula_pair():
    """an equal-power coherent pair 15 degrees apart on an 8-element ULA.  Observed on these seeded windows: IAA resolves
    it in 60 of 60, MUSIC in 4, MVDR (loading 0.01) in 12.  Held: IAA in all 60, MUSIC in at most 8 and MVDR in at most
    15, so that the case discriminates with a margin for other LAPACK builds."""
    tab, x, truth = io.ula_case("coherent")
    iaa = music = mvdr = 0
    for w in range(len(x)):
        R = mo.covariance(x[w], 8)
        iaa += io.ula_resolved(io.window(R, tab, 2, peak="local")["bins"], truth)
        ev, V = np.linalg.eigh(R)
        music += io.ula_resolved(eo.picks(ao.spectrum(V[:, :6], tab), 2, 180, "local")[2], truth)
        mvdr += io.ula_resolved(eo.picks(eo.spectrum(R, tab, "mvdr", 0.01), 2, 180, "local")[2], truth)
    assert iaa == 60 and music <= 8 and mvdr <= 15, (iaa, music, mvdr)


def test_uncorrelated_close_pair_is_the_weakness():
    """two uncorrelated sources 6 degrees apart (10 dB, N = 64).  Observed on these seeded windows: MUSIC resolves them in
    60 of 60, IAA in none.  Held: MUSIC in all 60, IAA in at most 3."""
    tab, x, truth = io.ula_case("uncorrelated")
    iaa = music = 0
    for w in range(len(x)):
        R = mo.covariance(x[w], 8)
        iaa += io.ula_resolved(io.window(R, tab, 2, peak="local")["bins"], truth)
        ev, V = np.linalg.eigh(R)
        music += io.ula_resolved(eo.picks(ao.spectrum(V[:, :6], tab), 2, 180, "local")[2], truth)
    assert music == 60 and iaa <= 3, (iaa, music)


def test_permuted_spread_bounds_a_third_order():
    """The GPU tests bound each window by SPREAD_FACTOR times the oracle's spread between the natural order and one
    other rounding order (permuted elements, reversed rows).  On these windows a second such order stays within that
    bound."""
    rng = np.random.default_rng(8)
    worst = 0.0
    for m in (4, 8, 16):
        tab = helpers.table_wl(helpers.array_wl("uca", m), 360)
        for w in range(6):
            R = random_R(rng, m, 2 * m if w % 2 else m // 2 + 1)
            P = io.spectrum(R, tab, 15)
            s1 = io.spread(R, tab, 15, 0.0, rng.permutation(m), P)
            s2 = io.spread(R, tab, 15, 0.0, rng.permutation(m), P)
            worst = max(worst, s2 / max(s1, io.floor(P)))
    assert worst <= io.SPREAD_FACTOR, worst
