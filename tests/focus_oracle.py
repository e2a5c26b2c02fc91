"""fp64 oracle of the COHERENT combine of a channel handle (music_b200_create_channels, include/music_b200.h), a literal
restatement of the definition with np.linalg.svd:

    reference    c_ref = C // 2
    sector       S = {(first + i) mod K : i < count}
    steering     a_c(theta_k)[r] = exp(-j 2 pi <p_r, u(theta_k)> / lambda_c), theta_k = (k * 360 / K) * (pi / 180), fp64
    focusing     B_c = sum_{k in S} a_ref a_c^H + beta |S| I, beta = 1e-3;  T_c = U V^H (B_c = U S V^H);  T_ref = I
    error        e_c = ||T_c A_c - A_ref||_F / ||A_ref||_F
    covariance   R_foc = (1 / C) sum_c T_c R_c T_c^H in channel order, the c_ref term R_ref itself
    problem      composed_oracle.work_R on (R_foc, reference table) with J * C looks (the tests call it)

Test infrastructure; the product path never imports this file."""
import math

import numpy as np

import channels_oracle as ch

BETA = 1e-3
SINGULAR = 1e-12


def ref_channel(C):
    return C // 2


def sector(K, first=0, count=None):
    return (first + np.arange(K if count is None else count)) % K


def steering(pos, lam, K, bins):
    """fp64 steering vectors (len(bins), m) of the grid bins `bins` at wavelength lam"""
    th = (np.asarray(bins, np.float64) * 360.0 / K) * (math.pi / 180.0)
    u = np.stack([np.cos(th), np.sin(th)], axis=1)
    return np.exp(-2j * math.pi * (u @ np.asarray(pos, np.float64).T) / lam)


def focusing(pos, lams, K, first=0, count=None):
    """(T (C, m, m) complex128, err (C,)) for the wavelengths lams of the C channels; raises ValueError on a singular B_c"""
    C, m = len(lams), len(pos)
    ref = ref_channel(C)
    S = sector(K, first, count)
    A_ref = steering(pos, lams[ref], K, S).T          # (m, |S|): columns a(theta_k)
    T = np.zeros((C, m, m), np.complex128)
    err = np.zeros(C)
    for c in range(C):
        if c == ref:
            T[c] = np.eye(m)
            continue
        A_c = steering(pos, lams[c], K, S).T
        B = A_ref @ A_c.conj().T + BETA * len(S) * np.eye(m)
        U, s, Vh = np.linalg.svd(B)
        if s[-1] <= SINGULAR * s[0]:
            raise ValueError("B_%d is singular" % c)
        T[c] = U @ Vh
        err[c] = np.linalg.norm(T[c] @ A_c - A_ref) / np.linalg.norm(A_ref)
    return T, err


def focus(R, T):
    """R (C, m, m), T (C, m, m) -> R_foc (m, m)"""
    C = len(R)
    ref = ref_channel(C)
    acc = np.zeros_like(R[0])
    for c in range(C):
        acc = acc + (R[c] if c == ref else T[c] @ R[c] @ T[c].conj().T)
    return acc / C


# ---- the two-path wideband scenario the CPU and the GPU tests share ----

FC, FS = 1e9, 200e6        # carrier and sample rate
F, C, J = 256, 192, 16     # 192 of 256 channels: +-7.5 % of the carrier
FIRST = F - C // 2         # the channels run from -C/2 to C/2 - 1 bins: c_ref is the carrier
K = 360
DEGS = (60.0, 85.0)
DELAY, AMP = 1, 0.9        # the second path: one sample late, at 0.9 of the first


def uca(m, lam):
    """m-element uniform circular array, lam / 2 between neighbours"""
    r = 0.5 * lam / (2.0 * math.sin(math.pi / m))
    a = 2.0 * math.pi * np.arange(m) / m
    return np.stack([r * np.cos(a), r * np.sin(a)], axis=1)


def two_paths(rng, pos, N, degs=DEGS, delay=DELAY, amp=AMP, noise=0.1, fc=FC, fs=FS):
    """one signal white across the sampled band arriving from degs[0] and, `delay` samples later at amplitude amp, from
    degs[1] (multipath: the two are coherent in every narrow channel), each frequency with its own steering vectors,
    plus white noise of `noise` per element.  One window, complex64 (N * m,)"""
    m = len(pos)
    S = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / math.sqrt(2.0)
    f = np.fft.fftfreq(N) * fs
    A = np.stack([ch.steer(pos, ch.C0 / (fc + fi), degs[0]) + amp * np.exp(-2j * math.pi * fi * delay / fs) *
                  ch.steer(pos, ch.C0 / (fc + fi), degs[1]) for fi in f])
    X = np.fft.ifft(S[:, None] * A, axis=0) * math.sqrt(N)
    X = X + noise * (rng.standard_normal((N, m)) + 1j * rng.standard_normal((N, m))) / math.sqrt(2.0)
    return ch.interleave(X)


def geometry(m=8):
    """(pos, wavelengths) of the two-path case: an m-element UCA and the C channels"""
    return uca(m, ch.C0 / FC), ch.wavelengths(F, FIRST, C, FC, FS)


def scenario(windows, seed, noise=0.1, m=8):
    """(pos, wavelengths, x (windows, F J m)) of the two-path case on an m-element UCA"""
    pos, _ = geometry(m)
    rng = np.random.default_rng(seed)
    x = np.stack([two_paths(rng, pos, F * J, noise=noise) for _ in range(windows)])
    return pos, ch.wavelengths(F, FIRST, C, FC, FS), x


def resolved(angles, degs=DEGS, tol=2.0):
    """both paths found, each within tol degrees by a distinct pick"""
    a = np.asarray(angles, np.float64)
    return len(a) == len(degs) and all(np.min(np.abs(a - d)) <= tol for d in degs) and \
        np.argmin(np.abs(a - degs[0])) != np.argmin(np.abs(a - degs[1]))
