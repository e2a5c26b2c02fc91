"""Covariance integration across windows (music_b200_set_integration), restated literally from include/music_b200.h.

The windows j = 0, 1, 2, ... since the last reset give S_j = alpha S_{j-1} + R_j, c_j = alpha c_{j-1} + 1,
q_j = alpha^2 q_{j-1} + 1 (all starting at 0), the integrated covariance Rbar_j = S_j / c_j, and the source count's
N_eff,j = N c_j^2 / q_j.  Everything here is the sequential fp64 recurrence in numpy; the device evaluates it as a
parallel scan, held to max |Rbar_gpu - Rbar_ref| <= REL_BOUND * max |Rbar_ref| per window.

`study` is the weak-source case behind the feature: a UCA-8 (adjacent elements lambda / 2 apart), one source at 73
degrees, -12 dB per element, N = 32 snapshots per window, scored over windows 200-399 of a stream."""
import math

import numpy as np

import source_count_oracle as sco

REL_BOUND = 1e-13


class State:
    """the carry of one handle: S, c, q and the windows since the reset"""

    def __init__(self, m):
        self.S = np.zeros((m, m), np.complex128)
        self.c = 0.0
        self.q = 0.0
        self.count = 0


def integrate(R, alpha, state=None):
    """Rbar [W][m][m] and N_eff factor c^2 / q [W] of the raw covariances R [W][m][m] after `state` (a fresh one when
    None, which is updated in place), in window order"""
    R = np.asarray(R, np.complex128)
    st = State(R.shape[1]) if state is None else state
    out = np.empty_like(R)
    fac = np.empty(R.shape[0])
    for j in range(R.shape[0]):
        st.S = alpha * st.S + R[j]
        st.c = alpha * st.c + 1.0
        st.q = alpha * alpha * st.q + 1.0
        st.count += 1
        out[j] = st.S / st.c
        fac[j] = st.c * st.c / st.q
    return out, fac


def n_eff(N, alpha, j):
    """N_eff of window j since the reset, by the recurrence"""
    c = q = 0.0
    for _ in range(j + 1):
        c = alpha * c + 1.0
        q = alpha * alpha * q + 1.0
    return N * c * c / q


def n_eff_limit(N, alpha):
    return N * (1.0 + alpha) / (1.0 - alpha)


def rel_err(got, ref):
    """per window max_entry |got - ref| / max_entry |ref|"""
    got = np.asarray(got).reshape(len(got), -1)
    ref = np.asarray(ref).reshape(len(ref), -1)
    return np.max(np.abs(got - ref), axis=1) / np.max(np.abs(ref), axis=1)


# ---- the weak-source study ----
def uca_wl(m):
    """UCA of m elements in wavelengths, adjacent elements lambda / 2 apart, element 0 on the x axis"""
    r = 0.5 / (2.0 * math.sin(math.pi / m))
    t = 2.0 * math.pi * np.arange(m) / m
    return np.stack([r * np.cos(t), r * np.sin(t)], axis=1)


def steering(pos, deg):
    t = np.radians(np.asarray(deg, np.float64))[..., None]
    return np.exp(-2j * np.pi * (pos[:, 0] * np.cos(t) + pos[:, 1] * np.sin(t)))


def weak_source_windows(W, seed, m=8, N=32, theta=73.0, snr_db=-12.0):
    """x [W][N * m] complex64 (snapshot-major, element fastest): one source at theta, snr_db per element over unit noise"""
    rng = np.random.default_rng(seed)
    a = steering(uca_wl(m), theta)
    amp = 10.0 ** (snr_db / 20.0)
    s = amp * (rng.standard_normal((W, N)) + 1j * rng.standard_normal((W, N))) / math.sqrt(2.0)
    n = (rng.standard_normal((W, N, m)) + 1j * rng.standard_normal((W, N, m))) / math.sqrt(2.0)
    x = s[..., None] * a[None, None, :] + n
    return x.reshape(W, N * m).astype(np.complex64)


def covariances(x, m):
    X = x.astype(np.complex128).reshape(x.shape[0], -1, m)  # [W][N][m]
    return np.einsum("wni,wnj->wij", X, X.conj()) / X.shape[1]


def music_peak_deg(Rbar, pos, n=1, K=360):
    """the TOP_BINS peak angle (degrees) of the MUSIC spectrum of each window"""
    A = steering(pos, np.arange(K) * 360.0 / K)  # [K][m]
    out = np.empty(len(Rbar))
    for w, R in enumerate(Rbar):
        _, V = np.linalg.eigh(R)
        G = V[:, : R.shape[0] - n]
        D = np.sum(np.abs(A.conj() @ G) ** 2, axis=1)
        out[w] = np.argmin(D) * 360.0 / K
    return out


def mdl_counts(Rbar, fac, N, n_max):
    return np.array([sco.estimate_source_count(np.linalg.eigvalsh(R), N * f, n_max, "mdl")[0] for R, f in zip(Rbar, fac)])


def study(alpha, snr_db=-12.0, seed=2026, W=400, first=200, m=8, N=32, theta=73.0):
    """(fraction of windows first..W-1 whose MUSIC peak is within 2 degrees of theta, fraction whose MDL count is 1)"""
    x = weak_source_windows(W, seed, m, N, theta, snr_db)
    Rbar, fac = integrate(covariances(x, m), alpha)
    pk = music_peak_deg(Rbar[first:], uca_wl(m))
    err = np.abs((pk - theta + 180.0) % 360.0 - 180.0)
    cnt = mdl_counts(Rbar[first:], fac[first:], N, m - 1)
    return float(np.mean(err <= 2.0)), float(np.mean(cnt == 1))
