"""fp64 restatement of the IAA spectrum estimator (MUSIC_B200_ESTIMATOR_IAA, include/music_b200.h).  Test
infrastructure: the definition is written out literally, so that it can be read against the header; the product path
never imports this file.

    Rh = the window's covariance,  a_k = table row k widened to fp64,  nu_k = ||a_k||^2,  delta = loading tr(Rh) / M
    p0_k   = a_k^H Rh a_k / nu_k^2                                 (estimator_oracle's Bartlett)
    R_i    = sum_k p(i-1)_k a_k a_k^H + delta I,  R_i = L L^H,  S_i = R_i^-1
    p(i)_k = (a_k^H S_i Rh S_i a_k) / (a_k^H S_i a_k)^2,  the denominator as ||L^-1 a_k||^2,   i = 1 .. I
    P = p(I); rows with nu_k = 0 have p_k = 0.  Every P[k] is NaN when Rh has a non-finite entry or tr Rh <= 0, a
    Cholesky pivot is not > 0, or any p(i)_k is not finite.
"""
import numpy as np
import scipy.linalg as sl

import estimator_oracle as eo

DEFAULT_ITERATIONS = 15


def _cholesky(A):
    """the lower Cholesky factor of the Hermitian A, or None when a pivot is not > 0 (NaN included)"""
    M = A.shape[0]
    L = np.zeros_like(A)
    for k in range(M):
        d = (A[k, k] - np.sum(np.abs(L[k, :k]) ** 2)).real
        if not d > 0.0:
            return None
        L[k, k] = np.sqrt(d)
        for i in range(k + 1, M):
            L[i, k] = (A[i, k] - np.sum(L[i, :k] * L[k, :k].conj())) / L[k, k]
    return L


def spectrum(R, table_c64, iterations=DEFAULT_ITERATIONS, loading=0.0, history=False):
    """fp64 P[k] of the (K, m) complex64 table for one window's covariance R (with history: also every p(i))"""
    R = np.asarray(R, dtype=np.complex128)
    M = R.shape[0]
    a = np.asarray(table_c64).reshape(-1, M).astype(np.complex128)  # (K, M)
    K = a.shape[0]
    nan = np.full(K, np.nan)
    tr = float(np.trace(R).real) if np.all(np.isfinite(R)) else np.nan
    if not (np.all(np.isfinite(R)) and tr > 0.0):
        return (nan, []) if history else nan
    delta = loading * tr / float(M)
    nu = np.sum(np.abs(a) ** 2, axis=1)
    live = nu != 0.0
    p = np.zeros(K)
    with np.errstate(divide="ignore", invalid="ignore"):
        p[live] = eo.spectrum(R, table_c64, "bartlett")[live]
    steps = [p.copy()]
    if not np.all(np.isfinite(p)):
        return (nan, steps) if history else nan
    for _ in range(iterations):
        Ri = np.einsum("k,ki,kj->ij", p, a, a.conj()) + delta * np.eye(M)
        L = _cholesky(Ri)
        if L is None:
            return (nan, steps) if history else nan
        y = sl.solve_triangular(L, a[live].T, lower=True)       # L^-1 a_k   (M, K')
        z = sl.solve_triangular(L.conj().T, y, lower=False)      # S a_k
        den = np.sum(np.abs(y) ** 2, axis=0)
        num = np.einsum("ik,ij,jk->k", z.conj(), R, z).real
        p = np.zeros(K)
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            p[live] = num / (den * den)
        steps.append(p.copy())
        if not np.all(np.isfinite(p)):
            return (nan, steps) if history else nan
    return (p, steps) if history else p


def spectrum_snapshots(X, table_c64, iterations=DEFAULT_ITERATIONS):
    """The per-snapshot weighted-least-squares form of Yardibi et al. (loading 0): X (N, M) snapshots, Rh = X^H X / N,
    p_k = (1/N) sum_n |a_k^H R_i^-1 y_n|^2 / (a_k^H R_i^-1 a_k)^2 with R_i from the previous p, started at Bartlett."""
    X = np.asarray(X, dtype=np.complex128)
    N, M = X.shape
    R = X.T @ X.conj() / N  # Rh[i, j] = (1/N) sum_n y_n[i] conj(y_n[j])
    a = np.asarray(table_c64).reshape(-1, M).astype(np.complex128)
    p = np.einsum("ki,ij,kj->k", a.conj(), R, a).real / np.sum(np.abs(a) ** 2, axis=1) ** 2
    for _ in range(iterations):
        Ri = (a.T * p) @ a.conj()
        Si = np.linalg.inv(Ri)
        w = a.conj() @ Si                                    # (K, M): a_k^H S_i
        num = np.mean(np.abs(w @ X.T) ** 2, axis=1)          # (1/N) sum_n |a_k^H S_i y_n|^2
        den = np.einsum("km,mk->k", w, a.T).real
        p = num / den ** 2
    return p


def window(R, table_c64, n, iterations=DEFAULT_ITERATIONS, loading=0.0, peak="top", exclusion=0, count=None):
    """One window's IAA spectrum and peak pick: {"P", "angles", "levels", "bins"}"""
    P = spectrum(R, table_c64, iterations, loading)
    K = np.asarray(table_c64).reshape(-1, np.asarray(R).shape[0]).shape[0]
    ang, lvl, bins = eo.picks(P, n, K, peak, exclusion, count)
    return {"P": P, "angles": ang, "levels": lvl, "bins": bins}


# ---- the seeded capability cases (shared by the CPU and GPU tests) -----------------------------------------------------
def _windows(rng, A, amps, N, snr_db, coherent, W):
    """complex64 (W, N * M) windows: sources along the rows of A with amplitudes amps, one signal with a random phase
    between the paths when coherent (a path and its reflection), independent signals otherwise, and complex white noise
    snr_db below a unit-amplitude source"""
    M = A.shape[1]
    sig = 10.0 ** (-snr_db / 20.0)
    out = []
    for _ in range(W):
        s = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / np.sqrt(2.0)
        X = np.zeros((M, N), np.complex128)
        for j, (a, g) in enumerate(zip(A, amps)):
            if not coherent and j:
                s = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / np.sqrt(2.0)
            ph = np.exp(2j * np.pi * rng.uniform()) if coherent and j else 1.0
            X += g * ph * a[:, None] * s[None, :]
        X += sig * (rng.standard_normal((M, N)) + 1j * rng.standard_normal((M, N))) / np.sqrt(2.0)
        out.append(X.T.reshape(-1))
    return np.ascontiguousarray(np.array(out).astype(np.complex64))


AZEL_TRUTH = ((40.0, 20.0), (70.0, 36.0))


def azel_case(N, W=12, seed=7):
    """4 x 4 URA (lambda / 2), az-el grid 180 x 46 over el 0 .. 90 degrees, two coherent paths at AZEL_TRUTH with
    amplitudes 1 and 0.8, 20 dB: (pos [16][3] in wavelengths, grid, table (K, 16) complex64, windows)"""
    import azel_oracle as ao
    grid = ao.Grid(180, 46, 0.0, 90.0)
    pos = ao.ura_xyz(4, 4, 1.0)
    tab = ao.table(pos, 1.0, grid).reshape(-1, 16).astype(np.complex64)
    A = np.array([ao.steering(pos, 1.0, az, el) for az, el in AZEL_TRUTH])
    return pos, grid, tab, _windows(np.random.default_rng(seed), A, (1.0, 0.8), N, 20.0, True, W)


def azel_found(bins, grid):
    """whether every path of AZEL_TRUTH has a reported bin within one grid step in azimuth and in elevation"""
    step_az, step_el = 360.0 / grid.n_az, (grid.el_hi - grid.el_lo) / (grid.n_el - 1)
    for az, el in AZEL_TRUTH:
        hit = False
        for b in bins:
            if b < 0:
                continue
            i, k = grid.split(int(b))
            daz = abs((grid.az_deg(k) - az + 180.0) % 360.0 - 180.0)
            hit = hit or (daz <= step_az * (1 + 1e-9) and abs(grid.el_deg(i) - el) <= step_el * (1 + 1e-9))
        if not hit:
            return False
    return True


def azel_truth_bins(grid):
    return [int(round((el - grid.el_lo) / ((grid.el_hi - grid.el_lo) / (grid.n_el - 1)))) * grid.n_az +
            int(round(az / (360.0 / grid.n_az))) for az, el in AZEL_TRUTH]


ULA_CASES = {"coherent": ((90.0, 105.0), True, 20.0), "uncorrelated": ((90.0, 96.0), False, 10.0)}


def ula_case(kind, W=60, seed=11, N=64, m=8):
    """an m-element x-axis ULA (lambda / 2) on a 180-row table, row k at theta = k degrees (0 .. 179: one of each
    mirror pair), and two equal-power sources: "coherent" at 90 / 105 degrees, 20 dB, or "uncorrelated" at 90 / 96
    degrees, 10 dB: (table (180, m) complex64, windows, the true rows)"""
    th, coherent, snr = ULA_CASES[kind]
    x = 0.5 * np.arange(m)
    tab = np.exp(-2j * np.pi * np.outer(np.cos(np.radians(np.arange(180.0))), x)).astype(np.complex64)
    A = np.exp(-2j * np.pi * np.outer(np.cos(np.radians(th)), x))
    return tab, _windows(np.random.default_rng(seed), A, (1.0, 1.0), N, snr, coherent, W), [int(t) for t in th]


def ula_resolved(bins, truth):
    """whether every true row has a reported bin within one row"""
    return all(any(b >= 0 and abs(int(b) - t) <= 1 for b in bins) for t in truth)


# ---- the per-window bound of the GPU comparison ------------------------------------------------------------------------
SPREAD_FACTOR = 32.0  # a second rounding order stays within it on CPU (test_iaa_oracle.test_permuted_spread_bounds_a_third_order)
FLOOR_ULPS = 64.0


def floor(P):
    """the least bound: FLOOR_ULPS * 2^-52 * max P"""
    fin = np.asarray(P)[np.isfinite(P)]
    return FLOOR_ULPS * 2.0 ** -52 * (float(np.max(np.abs(fin))) if fin.size else 0.0)


def spread(R, table_c64, iterations, loading, perm, P=None):
    """max_k |P - P'| between the natural order and another rounding order: the elements of R and the table in the
    order perm, and the table rows (the order of every sum over k) reversed"""
    P = spectrum(R, table_c64, iterations, loading) if P is None else P
    t = np.asarray(table_c64).reshape(-1, R.shape[0])
    Pp = spectrum(np.asarray(R)[np.ix_(perm, perm)], np.ascontiguousarray(t[::-1][:, perm]), iterations, loading)[::-1]
    d = np.abs(P - Pp)
    return float(np.max(d[np.isfinite(d)])) if np.any(np.isfinite(d)) else 0.0


def bound(R, table_c64, iterations, loading, rng, P=None):
    """the per-window bound on max_k |P_device - P|: SPREAD_FACTOR times the permuted-order spread, floored"""
    P = spectrum(R, table_c64, iterations, loading) if P is None else P
    return max(SPREAD_FACTOR * spread(R, table_c64, iterations, loading, rng.permutation(R.shape[0]), P), floor(P))
