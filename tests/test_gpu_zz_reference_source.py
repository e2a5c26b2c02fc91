"""GPU (runs last): the CUDA path against the reference's OWN work() - gr-baz's lib/baz_music_doa.cc compiled unmodified
against stand-in GNU Radio / Armadillo headers (see oracle/Makefile and tests/test_ref_shim.py), whose outputs on these
inputs are stored in tests/golden/reference/work.npz (angles and levels in full, spectra at the stored columns)."""
import numpy as np
import pytest

from gr_baz_b200.music_doa import music_doa

import helpers

pytestmark = pytest.mark.gpu

P_RTOL = 1e-5


@pytest.mark.parametrize("base,over,W", helpers.GPU_CASES)
def test_cuda_path_matches_the_reference_source(base, over, W):
    i = helpers.GPU_CASES.index((base, over, W))
    cfg, table, x = helpers.case_windows(base, over, W, helpers.GPU_SEED)
    K, n = cfg["resolution"], cfg["n"]
    ref = helpers.reference_outputs(helpers.case_key("gpu", i), x)
    blk = music_doa(cfg["m"], n, cfg["nsamples"], table.tolist(), K)
    ang = np.full((W, n), -7, np.float32)
    lvl = np.full((W, n), -7, np.float32)
    spec = np.zeros((W, K), np.float32)
    assert blk.work(W, [x], [ang, lvl, spec]) == W
    assert np.array_equal(ang, ref["angles"])  # = peak bins bit-exact (angle = (float)(k * 360 / K) is injective)
    assert helpers.rel_err(lvl, ref["levels"]) <= P_RTOL
    assert helpers.rel_err(spec[:, ref["bins"]], ref["spectrum"]) <= P_RTOL
    # peak-only call (the fused kernel for M = 4, n = 1)
    ang2 = np.zeros_like(ang)
    assert blk.work(W, [x], [ang2]) == W and np.array_equal(ang2, ref["angles"])


@pytest.mark.parametrize("kind,shapes,min_checked", [("random", helpers.random_small_shapes, 15),
                                                     ("wide", helpers.random_wide_shapes, 84)])
def test_cuda_path_matches_the_reference_source_on_random_shapes(kind, shapes, min_checked):
    """the sweeps of tests/test_ref_shim.py (m 2..9 / m 10..16, every n, grids of 7..721 bins, strong / weak / no
    signal) through work(): spectrum port connected, then peak outputs only - every covariance, eigensolver and scan
    instantiation of the unfused path, and the fused kernels where the shape allows"""
    checked = 0
    for trial, m, n, snaps, K, table, x in shapes():
        ref = helpers.reference_outputs(helpers.case_key(kind, trial), x)
        if not ref["finite"] or snaps < m:
            continue  # rank-deficient R: exact eigenvalue ties, LAPACK- and Jacobi-dependent (as tests/test_ref_shim.py)
        W = x.shape[0]
        ctx = (kind, trial, m, n, snaps, K)
        filled = ref["levels"] > 0  # n > K leaves the initial (0, 0) pairs in the last slots
        blk = music_doa(m, n, snaps * m, table.tolist(), K)
        ang = np.full((W, n), -7, np.float32)
        lvl = np.full((W, n), -7, np.float32)
        spec = np.full((W, K), -7, np.float32)
        assert blk.work(W, [x], [ang, lvl, spec]) == W
        assert np.array_equal(ang, ref["angles"]), ctx
        assert np.array_equal(lvl[~filled], ref["levels"][~filled]), ctx
        assert helpers.rel_err(lvl[filled], ref["levels"][filled]) <= 2e-6, ctx
        assert helpers.rel_err(spec[:, ref["bins"]], ref["spectrum"]) <= 2e-6, ctx
        ang2 = np.full((W, n), -7, np.float32)
        lvl2 = np.full((W, n), -7, np.float32)
        assert blk.work(W, [x], [ang2, lvl2]) == W
        assert np.array_equal(ang2, ref["angles"]), ctx
        assert np.array_equal(lvl2[~filled], ref["levels"][~filled]), ctx
        assert helpers.rel_err(lvl2[filled], ref["levels"][filled]) <= 2e-6, ctx
        blk.close()
        checked += 1
    assert checked >= min_checked
