"""CPU tests of the co-array definition (tests/coarray_oracle.py): the hole-free extent, lag table and virtual size of
the standard sparse arrays, R_ss on exact covariances, the gridless solvers on R_ss recovering more sources than
antennas, and the create checks of the library, which come before any device check."""
import ctypes

import numpy as np
import pytest
import torch

import coarray_oracle as co
from gr_baz_b200 import _capi, build

MRA4 = [0, 1, 4, 6]
NESTED6 = [0, 1, 2, 3, 7, 11]
NESTED8 = [0, 1, 2, 3, 4, 9, 14, 19]
COPRIME = [0, 2, 3, 4, 6, 9]  # extended coprime (M, N) = (2, 3): lag 8 is a hole
ULA5 = [0, 1, 2, 3, 4]
LAM, STEP = 1.0, (0.5, 0.0)


@pytest.mark.parametrize("p, U, mv", [(MRA4, 7, 7), (NESTED6, 12, 12), (NESTED8, 20, 16), (COPRIME, 8, 8), (ULA5, 5, 5)])
def test_extent_and_virtual_size(p, U, mv):
    assert co.hole_free_extent(p) == U
    assert co.resolve_mv(p) == mv
    assert co.resolve_mv(p, 2) == 2 and co.resolve_mv(p, mv) == mv
    assert co.resolve_mv(p, mv + 1) is None and co.resolve_mv(p, 1) is None


def test_lag_tables():
    assert co.lag_table(MRA4, 7) == [[(0, 0), (1, 1), (2, 2), (3, 3)], [(1, 0)], [(3, 2)], [(2, 1)], [(2, 0)], [(3, 1)],
                                     [(3, 0)]]
    t = co.lag_table(NESTED6, 12)
    assert [len(x) for x in t] == [6, 3, 2, 1, 2, 1, 1, 1, 1, 1, 1, 1]
    assert t[4] == [(4, 3), (5, 4)]
    for p in (NESTED8, COPRIME):
        mv = co.resolve_mv(p)
        for l, pairs in enumerate(co.lag_table(p, mv)):
            assert pairs and all(p[i] - p[j] == l for i, j in pairs)
            assert [i for i, _ in pairs] == sorted(i for i, _ in pairs)


@pytest.mark.parametrize("p", [MRA4, NESTED6, NESTED8, COPRIME, ULA5])
def test_exact_covariance_is_the_squared_virtual_covariance(p):
    rng = np.random.default_rng(len(p))
    mv = co.resolve_mv(p)
    deg = rng.uniform(10.0, 170.0, mv - 1)
    powers = rng.uniform(0.5, 2.0, mv - 1)
    R = co.exact_covariance(co.physical_positions(p, STEP), LAM, deg, powers, 0.3)
    Rv = co.exact_covariance(co.virtual_positions(STEP, mv), LAM, deg, powers, 0.3)
    Rss = co.smoothed(R, p, mv)
    ref = Rv @ Rv / mv
    assert np.max(np.abs(Rss - ref)) <= 1e-12 * np.max(np.abs(ref))
    assert np.max(np.abs(co.smoothed_batch(R[None], p, mv)[0] - Rss)) <= 1e-13 * np.max(np.abs(ref))
    assert np.array_equal(Rss, Rss.conj().T) and np.all(np.diag(Rss).imag == 0.0)
    assert np.min(np.linalg.eigvalsh(Rss)) > -1e-12 * np.max(np.abs(ref))


@pytest.mark.parametrize("p, d", [(MRA4, 6), (NESTED6, 9)])
@pytest.mark.parametrize("solver", ["esprit", "roots"])
def test_gridless_solvers_recover_more_sources_than_antennas(p, d, solver):
    rng = np.random.default_rng(100 + d)
    mv = co.resolve_mv(p)
    for _ in range(5):
        deg = np.sort(rng.uniform(15.0, 165.0, d))
        while np.min(np.diff(deg)) < 8.0:
            deg = np.sort(rng.uniform(15.0, 165.0, d))
        R = co.exact_covariance(co.physical_positions(p, STEP), LAM, deg, rng.uniform(0.5, 2.0, d), 0.1)
        Rss = co.smoothed(R, p, mv)
        out = getattr(co, solver)(Rss, STEP, LAM, 3600, d)
        assert out["count"] == d
        assert co.worst_error(out["angles"].astype(np.float64), deg) <= 2e-5  # float32 angles
        # the fp64 direction itself, before the float32 output rounding
        ang = [float(a) for a in out["angles"]]
        assert len(ang) == d and d > len(p)
    assert d >= len(p)


@pytest.mark.parametrize("p, d", [(MRA4, 6), (NESTED6, 9)])
def test_esprit_fp64_directions_to_1e9_degrees(p, d):
    # the fp64 directions ESPRIT computes on exact R_ss, before the float32 output: within 1e-9 degrees of the truth
    import esprit_oracle as eo
    from root_music_oracle import direction, ula_geometry

    rng = np.random.default_rng(7 + d)
    mv = co.resolve_mv(p)
    deg = np.linspace(20.0, 160.0, d) + rng.uniform(-2.0, 2.0, d)
    R = co.exact_covariance(co.physical_positions(p, STEP), LAM, deg, rng.uniform(0.5, 2.0, d), 0.1)
    Rss = co.smoothed(R, p, mv)
    V = np.linalg.eigh(Rss)[1]
    vpos = co.virtual_positions(STEP, mv)
    _, _, s = ula_geometry(vpos, LAM)
    phis = np.linalg.eigvals(eo.psi_matrix(V[:, mv - d:]))
    got = np.sort([direction(complex(f), s, LAM) for f in phis])
    assert np.max(np.abs(got - np.sort(deg))) <= 1e-9


def test_roots_fp64_directions_to_1e9_degrees():
    from root_music_oracle import coefficients, direction, ula_geometry

    for p, d in ((MRA4, 6), (NESTED6, 9)):
        rng = np.random.default_rng(11 + d)
        mv = co.resolve_mv(p)
        deg = np.linspace(20.0, 160.0, d) + rng.uniform(-2.0, 2.0, d)
        R = co.exact_covariance(co.physical_positions(p, STEP), LAM, deg, rng.uniform(0.5, 2.0, d), 0.1)
        V = np.linalg.eigh(co.smoothed(R, p, mv))[1]
        _, _, s = ula_geometry(co.virtual_positions(STEP, mv), LAM)
        r = np.roots(coefficients(V[:, : mv - d])[::-1])  # Q(z), highest power first
        r = r[np.argsort(np.abs(np.abs(r) - 1.0))][: 2 * d]  # the d double roots on the unit circle
        # each double root comes back as a pair split by about sqrt(eps): its midpoint direction
        got = np.sort([direction(complex(z), s, LAM) for z in r]).reshape(d, 2).mean(axis=1)
        assert np.max(np.abs(got - np.sort(deg))) <= 1e-9


@pytest.fixture(scope="module")
def lib():
    build.build_cuda()
    return _capi.load()


BAD = [
    dict(m=1), dict(m=17, positions=list(range(17)), nsamples=17 * 64), dict(positions=[1, 2, 5, 7]),
    dict(positions=[0, 1, 1, 6]), dict(positions=[0, 4, 1, 6]), dict(nsamples=0), dict(nsamples=1022), dict(resolution=0),
    dict(step=(0.5000001, 0.0)), dict(step=(0.0, 0.0)), dict(step=(float("nan"), 0.0)), dict(lam=0.0),
    dict(lam=float("inf")), dict(mv=8), dict(mv=1), dict(n=0), dict(n=7), dict(positions=[0, 2, 3, 4], mv=0),
]


@pytest.mark.parametrize("bad", BAD, ids=[",".join("%s=%s" % kv for kv in b.items()) for b in BAD])
def test_create_checks_come_before_the_device(lib, bad):
    a = dict(m=4, n=5, nsamples=1024, resolution=360, positions=MRA4, step=STEP, lam=LAM, mv=0)
    a.update(bad)
    if "m" in bad and "positions" not in bad:
        a["positions"] = list(range(max(a["m"], 1)))
    assert co.check_create(a["m"], a["n"], a["nsamples"], a["resolution"], a["positions"], a["step"], a["lam"], a["mv"]) == co.EINVAL
    pos = np.ascontiguousarray(a["positions"], np.int32)
    step = np.ascontiguousarray(a["step"], np.float64)
    h = ctypes.c_void_p()
    rc = lib.music_b200_create_coarray(ctypes.byref(h), a["m"], a["n"], a["nsamples"], a["resolution"], pos.ctypes.data,
                                       step.ctypes.data, a["lam"], a["mv"], 0)
    assert rc == _capi.EINVAL and not h
    assert lib.music_b200_last_error(None)


def test_create_null_arguments(lib):
    h = ctypes.c_void_p()
    step = np.array(STEP)
    pos = np.array(MRA4, np.int32)
    assert lib.music_b200_create_coarray(ctypes.byref(h), 4, 5, 1024, 360, None, step.ctypes.data, LAM, 0, 0) == _capi.EINVAL
    assert lib.music_b200_create_coarray(ctypes.byref(h), 4, 5, 1024, 360, pos.ctypes.data, None, LAM, 0, 0) == _capi.EINVAL
    assert lib.music_b200_create_coarray(None, 4, 5, 1024, 360, pos.ctypes.data, step.ctypes.data, LAM, 0, 0) == _capi.EINVAL


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_valid_create_reaches_the_device_check(lib):
    # n = 6 > m = 4 is valid on a co-array handle: the call gets past every argument check to ENODEVICE
    for p, n, mv in ((MRA4, 6, 0), (NESTED8, 15, 0), ([0, 1, 3], 3, 0), ([0, 1, 2, 5, 8], 7, 8)):
        assert co.check_create(len(p), n, 64 * len(p), 360, p, STEP, LAM, mv) == 0
        pos = np.ascontiguousarray(p, np.int32)
        h = ctypes.c_void_p()
        rc = lib.music_b200_create_coarray(ctypes.byref(h), len(p), n, 64 * len(p), 360, pos.ctypes.data,
                                           np.array(STEP).ctypes.data, LAM, mv, 0)
        assert rc == _capi.ENODEVICE and not h
