"""CPU: the manifold-separation peak mode's definition.  The library's host hook (music_b200_manifold_coeffs_host: the
order L and the Bessel coefficient table the GPU path uploads) against the order rule and against FFTs of the
pair responses, and the numpy oracle (tests/manifold_oracle.py) against the truth and against a fine-grid rule."""
import ctypes
import itertools
import math

import numpy as np
import pytest

from gr_baz_b200 import _capi

import manifold_oracle as mf


def hook(pos, lam, want_beta=True):
    """(rc, L, beta [pairs][L + 1] complex or None)"""
    L = _capi.load()
    pos = np.ascontiguousarray(pos, np.float64)
    m = pos.shape[0]
    Lo = ctypes.c_uint32(0)
    rc = L.music_b200_manifold_coeffs_host(pos.ctypes.data, m, lam, ctypes.byref(Lo), None)
    if rc != _capi.OK or not want_beta:
        return rc, Lo.value, None
    beta = np.zeros((m * (m - 1) // 2, Lo.value + 1, 2), np.float64)
    assert L.music_b200_manifold_coeffs_host(pos.ctypes.data, m, lam, ctypes.byref(Lo), beta.ctypes.data) == _capi.OK
    return rc, Lo.value, beta[..., 0] + 1j * beta[..., 1]


def random_planar(rng, m, aperture_wl):
    """m positions (wavelengths = metres at lam 1) inside a disc of diameter aperture_wl"""
    r = 0.5 * aperture_wl * np.sqrt(rng.uniform(0.0, 1.0, m))
    a = rng.uniform(0.0, 2 * math.pi, m)
    return np.c_[r * np.cos(a), r * np.sin(a)]


def coeffs_from_beta(C, beta, L):
    """c [2L + 1] from the hook's table by the definition's formula"""
    M = C.shape[0]
    c = np.zeros(L + 1, np.complex128)
    c[0] = np.trace(C).real
    for q, (i, j) in enumerate(itertools.combinations(range(M), 2)):
        f = np.where(np.arange(L + 1) % 2 == 0, 2.0 * C[i, j].real, 2j * C[i, j].imag)
        c += beta[q] * f
    return np.r_[np.conj(c[:0:-1]), c]


def noise_projector(rng, m, p):
    Q, _ = np.linalg.qr(rng.standard_normal((m, p)) + 1j * rng.standard_normal((m, p)))
    return Q @ Q.conj().T


# ---- the order and the table ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,L", [(3, 21), (4, 24), (5, 26), (8, 32), (12, 39), (16, 46)])
def test_order_of_half_wavelength_ucas(m, L):
    assert mf.order(mf.uca(m), 1.0)[0] == L
    rc, got, _ = hook(mf.uca(m), 1.0, want_beta=False)
    assert rc == _capi.OK and got == L


def test_order_rule_edges_and_cap():
    rng = np.random.default_rng(5)
    # every element at one point: x = 0, L = 1 and only beta_0 = 1
    rc, L, beta = hook(np.tile([[0.3, -0.2]], (4, 1)), 0.5)
    assert rc == _capi.OK and L == 1
    assert np.array_equal(beta[:, 0], np.ones(6)) and np.array_equal(beta[:, 1], np.zeros(6))
    for trial in range(200):
        m = int(rng.integers(2, 17))
        pos = random_planar(rng, m, rng.uniform(0.01, 6.0))
        lam = rng.uniform(0.2, 3.0)
        rc, L, _ = hook(pos * lam, lam, want_beta=False)
        want = mf.order(pos * lam, lam)[0]
        assert L == want, (trial, L, want)
        assert (rc == _capi.OK) == (want <= mf.MAX_L), (trial, rc, want)
    # the cap: L = 64 is accepted, L = 65 refused after writing L
    for ap in np.linspace(4.0, 5.0, 201):
        pos = np.array([[0.0, 0.0], [ap, 0.0], [0.3, 0.4]])
        want = mf.order(pos, 1.0)[0]
        rc, L, _ = hook(pos, 1.0, want_beta=False)
        assert L == want and (rc == _capi.OK) == (want <= 64), (ap, L, rc)
    assert any(mf.order(np.array([[0.0, 0.0], [ap, 0.0]]), 1.0)[0] == 64 for ap in np.linspace(4.0, 5.0, 201))
    assert hook(np.array([[0.0, 0.0], [1e9, 0.0]]), 1.0)[0] == _capi.EINVAL
    assert hook(np.zeros((4, 2)), 0.0)[0] == _capi.EINVAL


def test_beta_matches_fft_of_pair_responses():
    """beta_ij,l = the l-th Fourier coefficient of exp(-j x_ij cos(t - theta_ij)), to 1e-14 absolute"""
    rng = np.random.default_rng(11)
    Tf = 1024
    t = 2 * math.pi * np.arange(Tf) / Tf
    worst = 0.0
    for trial in range(40):
        m = int(rng.integers(2, 17))
        pos = random_planar(rng, m, rng.uniform(0.05, 4.3))
        rc, L, beta = hook(pos, 1.0)
        if rc != _capi.OK:
            continue
        for q, (i, j) in enumerate(itertools.combinations(range(m), 2)):
            dx, dy = pos[j] - pos[i]
            x, th = 2 * math.pi * math.hypot(dx, dy), math.atan2(dy, dx)
            f = np.fft.fft(np.exp(-1j * x * np.cos(t - th))) / Tf
            worst = max(worst, float(np.max(np.abs(beta[q] - f[: L + 1]))))
    assert worst <= 1e-14, worst


def test_trig_polynomial_equals_direct_form():
    """sum_l c_l e^{j l t} from the hook's table equals a^H C a within the truncation bound plus rounding"""
    rng = np.random.default_rng(12)
    t = np.linspace(0.0, 2 * math.pi, 997)
    for trial in range(60):
        m = int(rng.integers(2, 17))
        pos = random_planar(rng, m, rng.uniform(0.1, 4.3)) if trial % 2 else mf.uca(m)
        rc, L, beta = hook(pos, 1.0)
        if rc != _capi.OK:
            continue
        C = noise_projector(rng, m, int(rng.integers(1, m + 1))) * 10.0 ** rng.uniform(-5, 5)
        c = coeffs_from_beta(C, beta, L)
        err = np.max(np.abs(mf.trig(c, t) - mf.direct_D(C, pos, 1.0, t)))
        bound = np.sum(np.abs(C)) * mf.EPS + 4.0 * (2 * L + 1) * m * m * mf.EPS * np.max(np.abs(C))
        assert err <= bound, (trial, m, L, err, bound)
        # the FFT coefficients of the oracle are the same polynomial
        assert np.max(np.abs(mf.coefficients(C, pos, 1.0, L) - c)) <= bound, trial


# ---- the oracle ---------------------------------------------------------------------------------------------------------
def source_R(pos, angles_deg, noise=0.0, rng=None, N=None, amp=1.0):
    A = mf.steering(pos, 1.0, np.radians(angles_deg)).T  # (M, d)
    if rng is None:
        return A @ A.conj().T
    M, d = A.shape
    S = amp * (rng.standard_normal((d, N)) + 1j * rng.standard_normal((d, N))) / math.sqrt(2)
    X = A @ S + noise * (rng.standard_normal((M, N)) + 1j * rng.standard_normal((M, N))) / math.sqrt(2)
    return X @ X.conj().T / N


def circ(a, b):
    d = abs(a - b) % 360.0
    return min(d, 360.0 - d)


def match_err(got, truth):
    """the largest error of the best one-to-one matching, degrees"""
    return min(max(circ(g, t) for g, t in zip(p, truth)) for p in itertools.permutations(got))


def separated(rng, d, sep=15.0):
    while True:
        th = rng.uniform(0.0, 360.0, d)
        if d < 2 or min(circ(a, b) for a, b in itertools.combinations(th, 2)) >= sep:
            return th


@pytest.mark.parametrize("m", [3, 4, 5, 8, 12, 16])
def test_oracle_recovers_noiseless_truth(m):
    rng = np.random.default_rng(100 + m)
    d = 1 if m == 3 else 2 if m <= 5 else 3
    pos = mf.uca(m)
    for trial in range(10):
        th = separated(rng, d)
        r = mf.work_R(source_R(pos, th), pos, 1.0, 3600, d)
        got = [float(a) for a in r["angles"][:d]]
        assert np.all(r["bins"] >= 0), (trial, r)
        assert match_err(got, th) <= 5e-4, (trial, got, th)


@pytest.mark.parametrize("m,d,snr", [(8, 3, 0.0), (5, 2, 10.0), (4, 2, 30.0), (16, 3, 0.0)])
def test_failure_rate_matches_fine_grid_rule(m, d, snr):
    """the largest-modulus root selection fails (error > 0.05 rad) about as often as the d smallest local minima of D
    on a 36 000-point grid, over seeded windows of sources at least 20 degrees apart (failures are 1 / 1, 0 / 0,
    12 / 15 and 0 / 0 of 300; at UCA 4 both share the array's own ambiguities)"""
    rng = np.random.default_rng(7 * m + d)
    pos = mf.uca(m)
    trials, f_roots, f_grid = 300, 0, 0
    for _ in range(trials):
        th = separated(rng, d, 20.0)
        R = source_R(pos, th, noise=1.0, rng=rng, N=256, amp=10.0 ** (snr / 20.0))
        r = mf.work_R(R, pos, 1.0, 3600, d)
        lim = math.degrees(0.05)
        got = [float(a) for a in r["angles"][:d]]
        f_roots += not (np.all(r["bins"] >= 0) and match_err(got, th) <= lim)
        g = mf.grid_minima(r["G"], pos, 1.0, d)
        f_grid += not (len(g) == d and match_err(list(g), th) <= lim)
    assert abs(f_roots - f_grid) <= 0.02 * trials, (f_roots, f_grid)


def test_line_array_gives_mirror_pairs():
    """on an x-axis ULA D(t) = D(-t): the coefficients are real, the roots come in conjugate pairs and a single source
    fills two slots with t and 360 - t"""
    m = 6
    pos = np.c_[0.5 * np.arange(m), np.zeros(m)]
    rng = np.random.default_rng(3)
    R = source_R(pos, [40.0], noise=0.1, rng=rng, N=512)
    r = mf.work_R(R, pos, 1.0, 3600, 2, d=2)
    z = r["roots"]
    z = z[(np.abs(z) > 0.8) & (np.abs(z) < 1.25)]  # the well-conditioned roots near the circle
    assert len(z) >= 4 and np.max(np.min(np.abs(z[:, None] - np.conj(z)[None, :]), axis=1)) <= 1e-8
    a = sorted(float(v) for v in r["angles"])
    assert abs(a[0] - 40.0) < 1.0 and abs(a[1] - 320.0) < 1.0, a
    rc, L, beta = hook(pos, 1.0)
    C = r["G"] @ r["G"].conj().T
    assert np.max(np.abs(coeffs_from_beta(C, beta, L).imag)) <= 1e-13 * np.sum(np.abs(C))
