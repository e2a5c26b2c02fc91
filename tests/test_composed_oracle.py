"""CPU: the composed oracle (tests/composed_oracle.py) reduces to each feature oracle when every other setting is at its
default, and a calibration with gains of 1 is the identity."""
import math

import numpy as np
import pytest

from gr_baz_b200 import synth
from oracle import music_oracle as mo

import calibration_oracle as co
import composed_oracle as cmp
import dml_oracle as dm
import esprit_oracle as es
import estimator_oracle as eo
import refine_oracle as ro
import root_music_oracle as rm
import source_count_oracle as so

LAM = synth.C_LIGHT / synth.FREQUENCY
N = 64
K = 360


def uca_case(m, seed):
    """(table, windows, positions) of so.mixed_windows: 0 to 3 sources per window on a UCA"""
    table, x, _ = so.mixed_windows(m, N, K, seed, per=2)
    pos = np.asarray(mo.scaled_antenna_array(synth.SPACING, synth.antenna_array("uca", m)), np.float64)
    return table, x, pos


def ula_case(m, seed):
    """(table, windows, positions): an x-axis ULA lambda / 2 apart, 0 to 3 sources per window at 20 dB"""
    rng = np.random.default_rng(seed)
    pos = np.array([[0.5 * LAM * i, 0.0] for i in range(m)])
    table = np.array([ro.steering(pos, LAM, math.radians(k * 360.0 / K))[0] for k in range(K)]).astype(np.complex64)
    xs = []
    for S in (0, 1, 2, 3, 1, 2):
        X = (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / math.sqrt(2.0)
        for t in rng.uniform(10.0, 170.0, min(S, m - 1)):
            X += 10.0 * ro.steering(pos, LAM, math.radians(t))[0][:, None] * rng.standard_normal(N)[None, :]
        xs.append(X.T.reshape(-1))
    return table, np.array(xs).astype(np.complex64), pos


def same(a, b, ctx):
    assert np.array_equal(a, b), (ctx, a, b)


@pytest.mark.parametrize("m,n", [(4, 1), (8, 3)])
@pytest.mark.parametrize("rule", ["fixed", "mdl", "aic"])
@pytest.mark.parametrize("peak,excl", [("top", 0), ("local", 3)])
def test_music_grid_is_the_source_count_oracle(m, n, rule, peak, excl):
    """MUSIC on the grid: FIXED is oracle/music_oracle.py's work(), MDL / AIC source_count_oracle.work()"""
    table, x, _ = uca_case(m, 10 * m + n)
    for w in range(len(x)):
        R = mo.covariance(x[w], m)
        got = cmp.work_R(R, cmp.modes(peak, excl, rule=rule), table, None, n, N)
        if rule == "fixed":
            ref = mo.work(x[w], m, n, table)
            if peak == "local":
                q = mo.pick_local_maxima(ref["P"], n, K, excl)
                ref = {"P": ref["P"], "bins": [p[2] for p in q], "angles": [p[0] for p in q], "levels": [p[1] for p in q]}
            d = n
        else:
            ref = so.work(x[w], m, n, table, rule, peak, excl)
            d = ref["count"]
        assert got["count"] == d and (rule != "fixed" or got["margin"] == math.inf)
        assert np.max(np.abs(got["P"] - ref["P"]) / ref["P"]) <= 1e-12, (m, n, rule, peak, w)
        same(got["bins"], np.asarray(ref["bins"], np.int32), (m, n, rule, peak, w))
        same(got["angles"], np.asarray(ref["angles"], np.float32), (m, n, rule, peak, w))
        filled = got["bins"] >= 0
        assert np.all(np.abs(got["levels"][filled] - np.asarray(ref["levels"], np.float32)[filled])
                      <= 1e-12 * np.abs(got["levels"][filled]) + np.spacing(got["levels"][filled]))
        assert np.all(got["levels"][~filled] == 0) and np.all(got["angles"][~filled] == 0)


@pytest.mark.parametrize("kind,loading", [("mvdr", 0.0), ("mvdr", 0.01), ("bartlett", 0.0)])
@pytest.mark.parametrize("rule", ["fixed", "mdl"])
@pytest.mark.parametrize("peak,excl", [("top", 0), ("local", 3)])
def test_mvdr_bartlett_is_the_estimator_oracle(kind, loading, rule, peak, excl):
    m, n = 7, 2
    table, x, _ = uca_case(m, 71)
    for w in range(len(x)):
        R = mo.covariance(x[w], m)
        got = cmp.work_R(R, cmp.modes(peak, excl, kind, loading, rule), table, None, n, N)
        ref = eo.work(x[w], m, n, table, kind, loading, peak, excl, None if rule == "fixed" else rule)
        assert got["count"] == ref["count"]
        for k in ("P", "bins", "angles", "levels"):
            same(got[k], ref[k], (kind, rule, peak, w, k))


@pytest.mark.parametrize("rule", ["fixed", "mdl", "aic"])
@pytest.mark.parametrize("mode", ["roots", "esprit"])
def test_gridless_is_the_root_and_esprit_oracles(rule, mode):
    m, n = 8, 3
    table, x, pos = ula_case(m, 81)
    for w in range(len(x)):
        R = mo.covariance(x[w], m)
        got = cmp.work_R(R, cmp.modes(mode, rule=rule), table, (pos, LAM), n, N)
        orc = rm if mode == "roots" else es
        ref = orc.work_R(R, pos, LAM, K, n, N, None if rule == "fixed" else rule)
        assert got["count"] == ref["count"]
        for k in ("bins", "angles", "levels"):
            same(got[k], ref[k], (mode, rule, w, k))
        assert np.all(got["flip"] == ref["margin"])


@pytest.mark.parametrize("rule", ["fixed", "mdl", "aic"])
def test_dml_is_the_dml_oracle(rule):
    m, n = 4, 2
    table, x, _ = uca_case(m, 91)
    for w in range(len(x)):
        got = cmp.work_R(mo.covariance(x[w], m), cmp.modes("dml", rule=rule), table, None, n, N)
        ref = dm.work(x[w], m, n, table, None if rule == "fixed" else rule)
        assert got["count"] == ref["count"]
        for k in ("bins", "angles", "levels"):
            same(got[k], ref[k], (rule, w, k))


@pytest.mark.parametrize("rule", ["fixed", "mdl"])
@pytest.mark.parametrize("peak,excl", [("top", 0), ("local", 3)])
def test_music_refinement_is_the_refine_oracle(rule, peak, excl):
    m, n = 8, 2
    table, x, pos = uca_case(m, 101)
    for w in range(len(x)):
        got = cmp.work_R(mo.covariance(x[w], m), cmp.modes(peak, excl, rule=rule, refine=True), table, (pos, LAM), n, N)
        ref = ro.work(x[w], m, n, table, pos, LAM, peak, excl, None if rule == "fixed" else rule)
        assert got["count"] == ref["count"]
        for k in ("bins", "angles", "levels"):
            same(got[k], ref[k], (rule, peak, w, k))


@pytest.mark.parametrize("kind,loading", [("mvdr", 0.01), ("bartlett", 0.0)])
def test_estimator_refinement_is_the_estimator_oracle(kind, loading):
    m, n = 5, 2
    table, x, pos = uca_case(m, 111)
    for w in range(len(x)):
        R = mo.covariance(x[w], m)
        got = cmp.work_R(R, cmp.modes("local", 3, kind, loading, refine=True), table, (pos, LAM), n, N)
        grid = cmp.work_R(R, cmp.modes("local", 3, kind, loading), table, (pos, LAM), n, N)
        same(got["bins"], grid["bins"], (kind, w))
        for i, b in enumerate(got["bins"]):
            if b < 0:
                assert got["angles"][i] == 0 and got["levels"][i] == 0
                continue
            r = eo.refine_slot(R, kind, loading, pos, LAM, int(b), K)
            assert got["angles"][i] == r["angle"] and got["levels"][i] == r["level"], (kind, w, i)
            assert got["flip"][i] == ro.flip_margin(r)


@pytest.mark.parametrize("m", [2, 5, 16])
def test_unit_gains_are_the_identity(m):
    table, x, _ = uca_case(m, 121) if m > 2 else ula_case(m, 121)
    R = cmp.covariance(x, m)
    same(R, co.covariance(x, m), m)
    same(cmp.covariance(x, m, np.ones(m)), R, m)
    same(cmp.covariance(x, m, np.ones(m, np.complex128)), R, m)


def test_power_of_two_gains_undo_exactly():
    """gains +-2^k are exact in complex64 and fp64: the corrected covariance of the corrupted windows is the clean one,
    and so is every later stage"""
    m, n = 8, 2
    table, x, pos = uca_case(m, 131)
    g = np.random.default_rng(132).choice([-1.0, 1.0], m) * 2.0 ** np.random.default_rng(133).integers(-2, 3, m)
    xr = (x.astype(np.complex128).reshape(len(x), -1, m) * g).reshape(len(x), -1).astype(np.complex64)
    Rc, R = cmp.covariance(xr, m, g), cmp.covariance(x, m)
    same(Rc, R, "R")
    md = cmp.modes("local", 3, "mvdr", 0.01, "mdl", True)
    for w in range(len(x)):
        a, b = cmp.work_R(Rc[w], md, table, (pos, LAM), n, N), cmp.work_R(R[w], md, table, (pos, LAM), n, N)
        for k in ("count", "bins", "angles", "levels", "P"):
            same(a[k], b[k], (w, k))
