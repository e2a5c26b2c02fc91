"""CPU checks of tests/crb_oracle.py, the restatement of the stochastic CRB the *_crb entry points report: at the model
covariance it is the textbook Slepian-Bangs bound, it scales as a variance should, and on sampled windows the
estimators' spread sits at the bound.  The statistical bounds chosen here are the ones tests/test_gpu_crb.py uses."""
import numpy as np
import pytest

import crb_oracle as co

# empirical std / median reported std at 20 dB (ULA-8, sources at 60 and 80 degrees, N = 256, 300 windows): over seeds
# 11-13 root-MUSIC gave 0.95-1.03 and LS-ESPRIT, which is not efficient, 1.08-1.21; the band leaves room for the
# sampling noise of 300 windows (about 4 %)
RATIO_LO, RATIO_HI = 0.85, 1.35
# neighbouring windows of an alpha = 0.9 integration share most of their covariance, so fewer windows are independent
RATIO_LO_INTEG, RATIO_HI_INTEG = 0.7, 1.6


def _random_psd(rng, d, rank=None):
    rank = d if rank is None else rank
    X = rng.standard_normal((d, rank)) + 1j * rng.standard_normal((d, rank))
    return X @ X.conj().T / rank + (0.0 if rank < d else 0.1) * np.eye(d)


def _columns_1d(pos, thetas_deg):
    cols = [co.steer_1d(pos, 1.0, np.radians(t)) for t in thetas_deg]
    return np.stack([c[0] for c in cols], 1), np.stack([c[1] for c in cols], 1)


def _columns_azel(pos, pairs_deg):
    cols = [co.steer_azel(pos, 1.0, np.radians(a), np.radians(e)) for a, e in pairs_deg]
    A = np.stack([c[0] for c in cols], 1)
    D = np.stack([v for c in cols for v in (c[1], c[2])], 1)
    return A, D


def _window(pos, R, A, D, N):
    return co.crb_window(R, A, D, N, co.deriv_scale(pos, 1.0))


def _literal(pos, A, D, P, s2, N):
    R = A @ P @ A.conj().T + s2 * np.eye(A.shape[0])
    r = _window(pos, R, A, D, N)
    assert r["ok"]
    return r["C"]


GEOMS_1D = {
    "ula8": co.ula_x(8),
    "uca8": co.uca(8, 0.6),
    "planar7": np.random.default_rng(3).uniform(-0.8, 0.8, (7, 2)),
}


@pytest.mark.parametrize("geom", sorted(GEOMS_1D))
@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_literal_equals_slepian_bangs_1d(geom, d):
    rng = np.random.default_rng(10 * d + len(geom))
    pos = GEOMS_1D[geom]
    thetas = [20.0 + 37.0 * k + rng.uniform(0, 5) for k in range(d)]  # inside (0, 180): no ULA mirror pair
    A, D = _columns_1d(pos, thetas)
    P = _random_psd(rng, d)
    C = _literal(pos, A, D, P, 0.3, 200)
    ref = co.slepian_bangs_crb(A, D, P, 0.3, 200)
    assert np.max(np.abs(C - ref)) <= 1e-10 * np.max(np.abs(ref))


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_literal_equals_slepian_bangs_azel(d):
    rng = np.random.default_rng(40 + d)
    pos = rng.uniform(-0.7, 0.7, (9, 3))
    pairs = [(30.0 + 70.0 * k, 10.0 + 12.0 * k) for k in range(d)]
    A, D = _columns_azel(pos, pairs)
    P = _random_psd(rng, d)
    C = _literal(pos, A, D, P, 0.5, 128)
    ref = co.slepian_bangs_crb(A, D, P, 0.5, 128)
    assert np.max(np.abs(C - ref)) <= 1e-10 * np.max(np.abs(ref))


def test_literal_equals_slepian_bangs_ura():
    # a 4 x 4 uniform rectangular array at el != 0 (the 2-D ESPRIT geometry)
    g = np.arange(4) * 0.5
    pos = np.array([[x, y, 0.0] for y in g for x in g])
    A, D = _columns_azel(pos, [(40.0, 35.0), (150.0, 55.0)])
    P = _random_psd(np.random.default_rng(5), 2)
    C = _literal(pos, A, D, P, 0.2, 64)
    ref = co.slepian_bangs_crb(A, D, P, 0.2, 64)
    assert np.max(np.abs(C - ref)) <= 1e-10 * np.max(np.abs(ref))


def test_coherent_pair_rank_one_source_covariance():
    # a path and its reflection: P has rank one, which the definition never inverts
    pos = co.uca(8, 0.6)
    A, D = _columns_1d(pos, [50.0, 140.0])
    P = _random_psd(np.random.default_rng(6), 2, rank=1)
    assert np.linalg.matrix_rank(P) == 1
    C = _literal(pos, A, D, P, 0.1, 256)
    ref = co.slepian_bangs_crb(A, D, P, 0.1, 256)
    assert np.all(np.isfinite(C))
    assert np.max(np.abs(C - ref)) <= 1e-10 * np.max(np.abs(ref))


def test_scale_and_snapshot_invariances():
    rng = np.random.default_rng(8)
    pos = co.uca(8, 0.6)
    A, D = _columns_1d(pos, [30.0, 100.0, 250.0])
    R = A @ _random_psd(rng, 3) @ A.conj().T + 0.4 * np.eye(8)
    base = _window(pos, R, A, D, 100)["C"]
    assert np.allclose(_window(pos, 7.5 * R, A, D, 100)["C"], base, rtol=1e-12, atol=0)
    assert np.allclose(np.sqrt(np.diag(_window(pos, R, A, D, 400)["C"])), 0.5 * np.sqrt(np.diag(base)), rtol=1e-12, atol=0)


def test_single_source_ula_closed_form():
    # d = 1 on an x-axis ULA with half-wavelength spacing, noise power 1:
    # CRB(t) = (1 + M snr) / (2 N M snr^2 ||P_perp d||^2),  ||P_perp d||^2 = (pi sin t)^2 sum (k - kbar)^2
    M, N, snr, t = 8, 256, 0.7, np.radians(70.0)
    pos = co.ula_x(M)
    A, D = _columns_1d(pos, [70.0])
    C = _literal(pos, A, D, np.array([[snr]]), 1.0, N)
    k = np.arange(M)
    dperp2 = (np.pi * np.sin(t)) ** 2 * np.sum((k - k.mean()) ** 2)
    closed = (1.0 + M * snr) / (2.0 * N * snr ** 2 * M * dperp2)
    assert abs(C[0, 0] - closed) <= 1e-12 * closed


def test_failures():
    pos = co.ula_x(8)
    # the mirror slot of a line array: the same steering vector twice
    A, D = _columns_1d(pos, [60.0, 300.0])
    R = A[:, :1] @ A[:, :1].conj().T + 0.1 * np.eye(8)
    assert not _window(pos, R, A, D, 100)["ok"]
    # end-fire on a ULA: psi = 0
    A, D = _columns_1d(pos, [0.0])
    assert not _window(pos, A @ A.conj().T + 0.1 * np.eye(8), A, D, 100)["ok"]
    # a planar array at el = 0: da/del = 0
    g = np.arange(3) * 0.5
    pl = np.array([[x, y, 0.0] for y in g for x in g])
    A, D = _columns_azel(pl, [(40.0, 0.0)])
    assert not _window(pl, A @ A.conj().T + 0.1 * np.eye(9), A, D, 100)["ok"]
    # a covariance that is not finite: s2 is NaN
    A, D = _columns_1d(pos, [60.0])
    R = A @ A.conj().T + 0.1 * np.eye(8)
    R[2, 3] = np.nan
    assert not _window(pos, R, A, D, 100)["ok"]


def _monte_carlo(estimator, W=300, seed=11, snr_db=20.0):
    rng = np.random.default_rng(seed)
    M, N, truth = 8, 256, np.array([60.0, 80.0])
    pos = co.ula_x(M)
    A, D = _columns_1d(pos, truth)
    P = 10 ** (snr_db / 10) * np.eye(2)
    R = co.sample_cov(co.sample_windows(rng, A, P, 1.0, N, W))
    est = np.array([np.sort(estimator(R[w], 2)) for w in range(W)])
    bins = np.zeros((W, 2), np.int32)
    std, _ = co.crb_outputs(R, est.astype(np.float32), bins, N, pos, 1.0)
    return np.std(est - truth, axis=0) / np.median(std, axis=0)


@pytest.mark.parametrize("name", ["root_music", "esprit"])
def test_monte_carlo_ratio(name):
    est = {"root_music": co.root_music_ula, "esprit": co.esprit_ula}[name]
    ratio = _monte_carlo(est)
    assert np.all(ratio >= RATIO_LO) and np.all(ratio <= RATIO_HI), ratio


@pytest.mark.parametrize("theta", [0.0, 180.0])
def test_ula_end_fire_fails_on_both_sides(theta):
    # at 180 degrees sin(pi) is 1.2e-16 in fp64, not 0: the relative pivot test of F alone would pass that 1 x 1 matrix
    # and report about 5e14 degrees; the derivative-scale test of step 4 fails it, as at 0 degrees
    pos = co.ula_x(8)
    A, D = _columns_1d(pos, [float(np.float32(theta))])
    r = _window(pos, A @ A.conj().T + 0.1 * np.eye(8), A, D, 256)
    assert not r["ok"] and r["margin"] < 1e-6
    std, _ = co.crb_outputs((A @ A.conj().T + 0.1 * np.eye(8))[None], np.array([[theta]], np.float32), np.zeros((1, 1), np.int32),
                            256, pos, 1.0)
    assert np.isnan(std[0, 0])


def test_near_end_fire_and_near_zenith_stay_finite():
    # one degree away the angle is observable again: a large but finite bound
    pos = co.ula_x(8)
    A, D = _columns_1d(pos, [179.0])
    r = _window(pos, A @ A.conj().T + 0.1 * np.eye(8), A, D, 256)
    assert r["ok"] and np.all(np.isfinite(r["C"]))
    g = np.arange(3) * 0.5
    pl = np.array([[x, y, 0.0] for y in g for x in g])
    A, D = _columns_azel(pl, [(40.0, 89.0)])
    assert _window(pl, A @ A.conj().T + 0.1 * np.eye(9), A, D, 256)["ok"]
    # at the zenith the azimuth is unobservable (cos(pi / 2) is 6e-17 in fp64)
    A, D = _columns_azel(pl, [(40.0, 90.0)])
    assert not _window(pl, A @ A.conj().T + 0.1 * np.eye(9), A, D, 256)["ok"]


@pytest.mark.parametrize("geom", ["ula8", "uca8"])
def test_top_bins_neighbours_are_finite_and_meaningless(geom):
    # n = 2 under TOP_BINS on one source at 60.3 degrees: the slots are the neighbouring bins 60 and 61.  The definition
    # evaluates the bound of two sources one bin apart; the window does not fail (the header says so), and the values
    # are far above the bound of the one slot that describes the data
    rng = np.random.default_rng(12)
    pos = GEOMS_1D[geom]
    a0 = co.steer_1d(pos, 1.0, np.radians(60.3))[0][:, None]
    R = co.sample_cov(co.sample_windows(rng, a0, 1000.0 * np.eye(1), 1.0, 256, 20))
    two, info = co.crb_outputs(R, np.tile(np.float32([60.0, 61.0]), (20, 1)), np.zeros((20, 2), np.int32), 256, pos, 1.0)
    one, _ = co.crb_outputs(R, np.tile(np.float32([60.3]), (20, 1)), np.zeros((20, 1), np.int32), 256, pos, 1.0)
    assert all(r["ok"] for r in info)
    assert np.all(np.isfinite(two))
    assert np.all(two > 10.0 * one)
