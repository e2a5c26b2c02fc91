"""CPU: the DML oracle (tests/dml_oracle.py) against its definition's consequences: the Bartlett bin for one source,
true bins on noiseless windows of every array kind, coherent-source resolution where MUSIC fails, a non-decreasing
objective, mirror rows never taken twice, exact least-squares levels, exact power-of-two table scaling and the
degenerate windows.  The windows of the resolution rows (tests/helpers.py) are shared with tests/test_gpu_dml.py."""
import numpy as np
import pytest

from oracle import music_oracle as mo

import dml_oracle as dm
import estimator_oracle as eo
from helpers import RESOLUTION, resolution_case, resolved
from helpers import angle_windows as source_windows, array_wl as array, table_wl as table

K = 360


def music_local(R, tab, n):
    """MUSIC LOCAL_MAXIMA angles of one window (fp64 spectrum of the n-source noise subspace)"""
    m = R.shape[0]
    _, V = np.linalg.eigh(R)
    G = V[:, : m - n]
    a = tab.astype(np.complex128)
    P = 1.0 / np.sum(np.abs(a.conj() @ G) ** 2, axis=1)
    return [q[0] for q in mo.pick_local_maxima(P, n, tab.shape[0]) if q[2] >= 0]


# ---- definition --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,m", [("uca", 8), ("x", 4), ("random", 5)])
def test_one_source_is_the_bartlett_bin(kind, m):
    """d = 1: the argmax of a^H R a / ||a||^2, which on a unit-modulus table is the Bartlett bin"""
    pos = array(kind, m, seed=3)
    tab = table(pos)
    x = source_windows(pos, [(37.3, 200.0)] * 6, False, 6, 11, snaps=256)
    a, na = dm.rows(tab, m)
    for w in range(6):
        R = mo.covariance(x[w], m)
        out = dm.work_R(R, tab, 1)
        f = np.einsum("ki,ij,kj->k", a.conj(), R, a).real / na
        assert out["bins"][0] == int(np.argmax(f))
        P = eo.spectrum(R, tab, "bartlett")
        assert out["bins"][0] == eo.picks(P, 1, K)[2][0]
        assert out["sweeps"] == 0


@pytest.mark.parametrize("kind,m", [("uca", 8), ("uca", 16), ("x", 6), ("y", 6), ("random", 7)])
@pytest.mark.parametrize("coherent", [False, True])
def test_noiseless_sources_on_grid_bins(kind, m, coherent):
    """R = A S A^H from table rows: DML returns the true bins (coherent: two sources, S = s s^H of rank one;
    uncorrelated: S diagonal, three sources on the planar arrays)"""
    pos = array(kind, m, seed=5)
    tab = table(pos)
    true = {"x": (40, 110), "y": (20, 75)}.get(kind, (30, 100) if coherent else (30, 100, 250))
    A = tab[list(true)].astype(np.complex128).T
    rng = np.random.default_rng(len(true) + m)
    if coherent:
        s = np.exp(2j * np.pi * rng.uniform(size=len(true))) * np.linspace(1.0, 2.0, len(true))
        S = np.outer(s, s.conj())
    else:
        S = np.diag(np.linspace(1.0, 2.0, len(true)))
    out = dm.work_R(A @ S @ A.conj().T, tab, len(true))
    assert sorted(out["bins"].tolist()) == sorted(true), (out["bins"], true)


@pytest.mark.parametrize("case", sorted(RESOLUTION))
def test_coherent_resolution(case):
    """seeded 20 dB windows, 1024 snapshots, K = 360: DML resolves what MUSIC LOCAL_MAXIMA (n = 2) cannot"""
    kind, m, coherent, sep = case
    pos, tab, x, th = resolution_case(kind, m, coherent, sep)
    got_music = got_dml = 0
    for w in range(len(x)):
        R = mo.covariance(x[w], m)
        out = dm.work_R(R, tab, 2)
        got_dml += resolved(out["angles"], th[w])
        got_music += resolved(music_local(R, tab, 2), th[w])
        assert np.all(np.diff(out["trajectory"]) >= -1e-12 * out["trajectory"][0]), out["trajectory"]
        assert out["sweeps"] <= dm.MAX_SWEEPS
    assert (got_music, got_dml) == RESOLUTION[case]


def test_mirror_row_is_never_a_candidate():
    """x-axis ULA: once a source's bin is in B, its mirror row (bit-identical) and the bin itself are not candidates"""
    m = 8
    pos = array("x", m)
    tab = table(pos)
    a, na = dm.rows(tab, m)
    x = source_windows(pos, [(50.0, 80.0)], False, 1, 3)
    R = mo.covariance(x[0], m)
    for b in (10, 50, 123):
        mirror = (K - b) % K
        assert np.array_equal(tab[b], tab[mirror])
        _, _, cand, _ = dm.search(R, a, na, [b])
        assert not cand[b] and not cand[mirror]
        assert cand.sum() >= K - 4
    out = dm.work_R(R, tab, 2)
    assert (K - out["bins"][0]) % K != out["bins"][1]


@pytest.mark.parametrize("kind,m", [("uca", 8), ("random", 6)])
def test_exact_model_levels(kind, m):
    """R = A diag(p) A^H + s2 I exactly: p-hat = p and s2-hat = s2 to 1e-9"""
    pos = array(kind, m, seed=9)
    tab = table(pos)
    true = [35, 160, 290]
    p = np.array([3.0, 1.5, 0.25])
    A = tab[true].astype(np.complex128).T
    R = A @ np.diag(p) @ A.conj().T + 0.125 * np.eye(m)
    out = dm.work_R(R, tab, 3)
    assert sorted(out["slots"]) == true
    got = dict(zip(out["slots"], out["p"]))
    assert all(abs(got[b] - q) <= 1e-9 * q for b, q in zip(true, p)), got
    assert abs(out["s2"] - 0.125) <= 1e-9
    assert np.array_equal(out["bins"], np.array(true, np.int32))
    assert np.array_equal(out["levels"], p.astype(np.float32))


@pytest.mark.parametrize("s", [-40, -7, 5, 30])
def test_power_of_two_table_scaling(s):
    """a table scaled by 2^s: the same bins, every fp64 level times exactly 2^(-2 s)"""
    m = 8
    pos = array("uca", m)
    tab = table(pos)
    pos_, _, x, th = resolution_case("uca", m, True, 20, W=4)
    for w in range(4):
        R = mo.covariance(x[w], m)
        ref = dm.work_R(R, tab, 2)
        got = dm.work_R(R, (tab.astype(np.complex128) * 2.0 ** s).astype(np.complex64), 2)
        assert np.array_equal(got["bins"], ref["bins"])
        assert np.array_equal(got["p"], ref["p"] * 2.0 ** (-2 * s))


def test_degenerate_windows():
    """zero R, a NaN in R, d = 0 and a table without candidates (all rows zero) report no peaks"""
    m, n = 4, 2
    pos = array("x", m)
    tab = table(pos)
    R = mo.covariance(source_windows(pos, [(40.0, 100.0)], False, 1, 2)[0], m)
    bad = R.copy()
    bad[1, 2] = np.nan
    for out in (dm.work_R(np.zeros((m, m)), tab, n), dm.work_R(bad, tab, n), dm.work_R(R, tab, n, d=0),
                dm.work_R(R, np.zeros_like(tab), n)):
        assert np.all(out["bins"] == -1) and np.all(out["angles"] == 0) and np.all(out["levels"] == 0)
    one = dm.work_R(R, tab, n, d=1)
    assert one["bins"][0] >= 0 and one["bins"][1] == -1 and one["levels"][1] == 0.0
