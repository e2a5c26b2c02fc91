"""fp64 numpy model of receiver calibration (music_b200_set_calibration, music_b200_calib_*), restating the definition
of include/music_b200.h literally.

Model: receiver noise enters ahead of the chain gain, x_raw(t) = G (A s(t) + n(t)), G = diag(g).  The correction is
x = C x_raw, C = diag(c), c_m = 1 / g_m, applied to R: R_ij <- (c_i R_ij) conj(c_j).  It makes the noise white again
(correcting the table instead, a -> g o a, would leave it coloured by |g_m|^2).

Estimate, from the mean raw covariance Rbar of windows of one dominant source at a known direction with steering vector
a0: h minimises the off-diagonal misfit sum_{i != j} |Rbar_ij - h_i conj(h_j)|^2 (noise and its colouring live on the
diagonal only, so on a population covariance the minimiser is g o a0 exactly at any noise level):
  start   r = argmax_i Rbar_ii (lowest index on ties), h_r = sqrt(Rbar_rr), h_i = Rbar_ir / sqrt(Rbar_rr);
  sweeps  Gauss-Seidel, i = 0 .. M-1 in turn: h_i <- (sum_{j != i} Rbar_ij h_j) / (sum_{j != i} |h_j|^2) with the updated
          entries; stop after the first sweep whose largest change is <= 2^-40 max_i |h_i|, or after 200 sweeps.
Then g = h / a0, rotated so that g_0 is real and positive, and
  GAIN_PHASE  scaled to sum |g_m|^2 = M (needs M >= 3),
  PHASE       g_m / |g_m| (any M >= 2).
Residual rho = sqrt(sum_{i != j} |Rbar_ij - h_i conj(h_j)|^2 / sum_{i != j} |Rbar_ij|^2).
Failures (ValueError): Rbar_rr <= 0, anything not finite, some h_m = 0 (a dead channel).
"""
import math

import numpy as np

PHASE, GAIN_PHASE = 1, 2
MAX_SWEEPS = 200
TOL = 2.0 ** -40


def steering_1d(pos, lam, az_deg):
    """the unrounded fp64 steering vector of element positions pos (M, 2) at az_deg (the refinement's convention)"""
    pos = np.asarray(pos, np.float64)
    t = az_deg * (math.pi / 180.0)
    phi = 2.0 * math.pi * ((pos[:, 1] * math.sin(t) + pos[:, 0] * math.cos(t)) / lam)
    return np.cos(phi) - 1j * np.sin(phi)


def steering_azel(pos, lam, az_deg, el_deg):
    """the same for element positions (M, 3) and the direction u = (cos el cos az, cos el sin az, sin el)"""
    pos = np.asarray(pos, np.float64)
    az, el = az_deg * (math.pi / 180.0), el_deg * (math.pi / 180.0)
    u = np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])
    phi = 2.0 * math.pi * ((pos @ u) / lam)
    return np.cos(phi) - 1j * np.sin(phi)


def inverse(g):
    """c = 1 / g = conj(g) / |g|^2, as the library computes it"""
    g = np.asarray(g, np.complex128)
    d = g.real * g.real + g.imag * g.imag
    return g.real / d - 1j * (g.imag / d)


def correct(R, g):
    """R [..., M, M] corrected for the gains g: (c_i R_ij) conj(c_j)"""
    c = inverse(g)
    return (c[:, None] * np.asarray(R, np.complex128)) * np.conj(c)[None, :]


def covariance(x, m):
    """fp64 covariance x x^H / N of each window of x (W, N * m) complex64"""
    X = np.asarray(x, np.complex64).astype(np.complex128).reshape(x.shape[0], -1, m)
    return np.einsum("wti,wtj->wij", X, np.conj(X)) / X.shape[1]


def fit(Rbar):
    """(h, sweeps) of the off-diagonal fit; raises ValueError on the failures above"""
    Rbar = np.asarray(Rbar, np.complex128)
    M = Rbar.shape[0]
    if not np.all(np.isfinite(Rbar)):
        raise ValueError("not finite")
    d = Rbar.real.diagonal()
    r = int(np.argmax(d))  # lowest index on ties
    if not d[r] > 0.0:
        raise ValueError("no power")
    s = math.sqrt(d[r])
    h = Rbar[:, r] / s
    h[r] = s
    sweeps = 0
    while sweeps < MAX_SWEEPS:
        sweeps += 1
        dmax = 0.0
        for i in range(M):
            j = np.arange(M) != i
            hn = np.sum(Rbar[i, j] * h[j]) / np.sum(np.abs(h[j]) ** 2)
            dmax = max(dmax, abs(hn - h[i]))
            h[i] = hn
        if not dmax > TOL * np.max(np.abs(h)):
            break
    if not np.all(np.isfinite(h)):
        raise ValueError("not finite")
    if np.any(h == 0):
        raise ValueError("dead channel")
    return h, sweeps


def residual(Rbar, h):
    Rbar = np.asarray(Rbar, np.complex128)
    off = ~np.eye(Rbar.shape[0], dtype=bool)
    E = Rbar - np.outer(h, np.conj(h))
    return math.sqrt(np.sum(np.abs(E[off]) ** 2) / np.sum(np.abs(Rbar[off]) ** 2))


def solve(Rbar, a0, kind=GAIN_PHASE):
    """(gains, residual, sweeps) of the mean raw covariance Rbar and the known source's steering vector a0"""
    M = Rbar.shape[0]
    if kind not in (PHASE, GAIN_PHASE):
        raise ValueError("unknown kind")
    if kind == GAIN_PHASE and M < 3:
        raise ValueError("GAIN_PHASE needs M >= 3")
    h, sweeps = fit(Rbar)
    g = h / np.asarray(a0, np.complex128)
    g = g * (np.conj(g[0]) / abs(g[0]))
    if kind == PHASE:
        g = g / np.abs(g)
    else:
        g = g * math.sqrt(M / np.sum(np.abs(g) ** 2))
    if not np.all(np.isfinite(g)):
        raise ValueError("not finite")
    return g, residual(Rbar, h), sweeps


def normalised(g, kind):
    """the true gains g as the estimate reports them: g_0 real positive, then the kind's normalisation"""
    g = np.asarray(g, np.complex128)
    g = g * (np.conj(g[0]) / abs(g[0]))
    return g / np.abs(g) if kind == PHASE else g * math.sqrt(len(g) / np.sum(np.abs(g) ** 2))


def principal(Rbar, a0, kind=GAIN_PHASE):
    """the naive estimate for comparison: the principal eigenvector of Rbar in place of h"""
    w, V = np.linalg.eigh(np.asarray(Rbar, np.complex128))
    return normalised(V[:, -1] / np.asarray(a0, np.complex128), kind)
