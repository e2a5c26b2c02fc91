"""fp64 oracle of the frequency-channelised modes (music_b200_create_channels), a literal restatement of the definition in
include/music_b200.h with numpy's FFT:

    segments     window w is cut into J = N / F consecutive segments of F snapshots
    filter bank  X_j[b] = sum_t h[t] x[jF + t] exp(-2 pi i b t / F), h = 1 (rect) or 1/2 - 1/2 cos(2 pi t / F) (hann)
    channels     channel c is bin b_c = (first + c) mod F at offset f_c = fs * (s(b_c) / F), s(b) = b for b < F / 2, else b - F
    covariance   R_c = sum_j X_j[b_c] X_j[b_c]^H / (J sum_t h[t]^2)
    tables       a_c(theta) for lambda_c = c0 / (f_centre + f_c)
    separate     each (window, channel) is composed_oracle.work_R on (R_c, table_c) with J snapshots (the tests call it)
    incoherent   P = 1 / sum_c (1 / P_c), P_c channel c's MUSIC spectrum on its own table, then the peak rule

Test infrastructure; the product path never imports this file."""
import math

import numpy as np

import composed_oracle as cmp
import estimator_oracle as eo

C0 = 299792458.0
TAPERS = ("rect", "hann")


def taper(F, kind):
    assert kind in TAPERS
    t = np.arange(F)
    return np.ones(F) if kind == "rect" else 0.5 - 0.5 * np.cos(2.0 * math.pi * t / F)


def bins_of(F, first, C):
    """FFT bin of each channel: (first + c) mod F"""
    return (first + np.arange(C)) % F


def offsets(F, first, C, fs):
    """frequency offset f_c of each channel in Hz"""
    b = bins_of(F, first, C)
    s = np.where(b < F // 2, b, b - F)
    return fs * (s.astype(np.float64) / float(F))


def wavelengths(F, first, C, fc, fs):
    return C0 / (fc + offsets(F, first, C, fs))


def filter_bank(x, m, F, kind):
    """x: one window, complex64 (N * m,), antennas sample-interleaved.  Returns X (J, F, m) complex128."""
    X = np.asarray(x).reshape(-1, m).astype(np.complex128)
    J = X.shape[0] // F
    assert J * F == X.shape[0]
    seg = X.reshape(J, F, m) * taper(F, kind)[None, :, None]
    return np.fft.fft(seg, axis=1)


def covariances(x, m, F, first, C, kind):
    """R_c of one window for every channel: (C, m, m) complex128"""
    X = filter_bank(x, m, F, kind)
    J = X.shape[0]
    denom = J * np.sum(taper(F, kind) ** 2)
    Xc = X[:, bins_of(F, first, C), :]                    # (J, C, m)
    return np.einsum("jci,jck->cik", Xc, Xc.conj()) / denom


def table(pos, lam, K):
    """the steering table of the 1-D handles, fp64 rounded to complex64: a[k][r] = exp(-j 2 pi <p_r, u(theta_k)> / lam)"""
    th = np.arange(K) * (2.0 * math.pi / K)
    u = np.stack([np.cos(th), np.sin(th)], axis=1)
    return np.exp(-2j * math.pi * (u @ np.asarray(pos, np.float64).T) / lam).astype(np.complex64)


def incoherent(R, tables, n, peak="top", exclusion=0):
    """R (C, m, m), tables (C, K, m).  Returns P (K,) and the picks (angles, levels, bins)."""
    K = tables[0].shape[0]
    D = np.zeros(K)
    for c in range(len(R)):
        D = D + 1.0 / cmp.spectrum(R[c], tables[c], "music", 0.0, n)
    P = 1.0 / D
    return P, eo.picks(P, n, K, peak, exclusion, n)


# ---- scenarios the CPU and the GPU tests share ----

def ula_pos(m, lam):
    """lambda / 2 line array on the x axis"""
    return np.stack([np.arange(m) * lam / 2.0, np.zeros(m)], axis=1)


def steer(pos, lam, deg):
    th = math.radians(deg)
    return np.exp(-2j * math.pi * (np.asarray(pos) @ np.array([math.cos(th), math.sin(th)])) / lam)


def interleave(X):
    """(N, m) complex -> one window, complex64 (N * m,)"""
    return np.ascontiguousarray(X.astype(np.complex64)).reshape(-1)


def two_emitters(rng, pos, fc, fs, F, N, chans, degs, amps=(1.0, 1.0), noise=0.05, walk=0.02):
    """two narrowband emitters, emitter i a tone at the centre of channel chans[i] (with a random phase walk of `walk` radians per sample,
    far narrower than a channel) from direction degs[i], each with the steering vector of its own frequency, plus white noise"""
    m = len(pos)
    t = np.arange(N)
    X = noise * (rng.standard_normal((N, m)) + 1j * rng.standard_normal((N, m))) / math.sqrt(2.0)
    for ch, deg, amp in zip(chans, degs, amps):
        s = ch if ch < F // 2 else ch - F
        f = fs * s / F
        phase = np.cumsum(rng.standard_normal(N)) * walk
        sig = amp * np.exp(1j * (2.0 * math.pi * (s / F) * t + phase + rng.uniform(0, 2 * math.pi)))
        X += sig[:, None] * steer(pos, C0 / (fc + f), deg)[None, :]
    return interleave(X)


def white_source(rng, pos, fc, fs, N, deg, noise=0.1):
    """one source white across the sampled band from direction deg: each frequency component arrives with the steering
    vector of its own frequency (built in the frequency domain over the N-point grid), plus white noise"""
    m = len(pos)
    S = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / math.sqrt(2.0)
    f = np.fft.fftfreq(N) * fs
    A = np.stack([steer(pos, C0 / (fc + fi), deg) for fi in f])        # (N, m)
    X = np.fft.ifft(S[:, None] * A, axis=0) * math.sqrt(N)
    X = X + noise * (rng.standard_normal((N, m)) + 1j * rng.standard_normal((N, m))) / math.sqrt(2.0)
    return interleave(X)
