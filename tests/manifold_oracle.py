"""fp64 restatement of the manifold-separation root-MUSIC peak mode (MUSIC_B200_PEAKS_MANIFOLD, include/music_b200.h)
on any planar array, independent of the Bessel functions the library uses: the coefficients come from an FFT of the
direct MUSIC denominator, the roots from numpy.roots.  Test infrastructure next to root_music_oracle.py; the product
path never imports this file.

    L: the smallest L >= 1 with L + 1 >= x and 4 tau_{L+1} <= 2^-52, x = 2 pi rho_max / lambda,
       tau_0 = 1, tau_l = tau_{l-1} (x / 2) / l
    C = G G^H,  D(t) = a(t)^H C a(t),  c_l = (1 / T) sum_k D(2 pi k / T) e^{-j l 2 pi k / T} (T = 256 >= 4L), c_{-l} = conj(c_l)
    Q(z) = sum_l c_l z^(l + L); ROOTS's merge and selection (keep the L roots of smallest modulus; slots take the d kept
    roots of largest modulus, exact ties to the lower angle)
    angle t* = arg z in [0, 360) degrees; level = 1 / D(t*) (direct form), bin = floor(t* K / 360 + 0.5) mod K
"""
import math

import numpy as np

import refine_oracle as ro
import source_count_oracle as so

T = 256
MAX_L = 64
EPS = 2.0 ** -52
MERGE = 1e-6


def order(pos, lam):
    """(L, x) of positions (M, 2) in metres at wavelength lam"""
    pos = np.asarray(pos, np.float64)
    rho = 0.0
    for i in range(len(pos)):
        for j in range(i + 1, len(pos)):
            rho = max(rho, math.hypot(pos[j, 0] - pos[i, 0], pos[j, 1] - pos[i, 1]))
    x = 2.0 * math.pi * rho / lam
    tau, L = x / 2.0, 1
    while True:
        tau = tau * (x / 2.0) / (L + 1)
        if L + 1.0 >= x and 4.0 * tau <= EPS:
            return L, x
        L += 1


def uca(m, spacing_wl=0.5, lam=1.0):
    """a UCA with adjacent elements spacing_wl wavelengths apart, element 0 on the x axis (metres at lam)"""
    r = spacing_wl * lam / (2.0 * math.sin(math.pi / m))
    return np.array([[r * math.cos(2 * math.pi * i / m), r * math.sin(2 * math.pi * i / m)] for i in range(m)])


def steering(pos, lam, t):
    """a(t) [.., M] for t radians (array): exp(-j 2 pi (x cos t + y sin t) / lambda)"""
    t = np.asarray(t, np.float64)[..., None]
    phi = 2.0 * math.pi * ((pos[:, 0] * np.cos(t) + pos[:, 1] * np.sin(t)) / lam)
    return np.cos(phi) - 1j * np.sin(phi)


def direct_D(C, pos, lam, t):
    """D(t) = a^H C a for t radians (array)"""
    A = steering(np.asarray(pos, np.float64), lam, t)
    return np.real(np.einsum("...i,ij,...j->...", A.conj(), C, A))


def coefficients(C, pos, lam, L):
    """c [2L + 1] with c[l + L] = c_l, from the FFT of D at T points"""
    D = direct_D(C, pos, lam, 2.0 * math.pi * np.arange(T) / T)
    f = np.fft.fft(D) / T
    c = np.zeros(2 * L + 1, np.complex128)
    for l in range(L + 1):
        c[L + l] = f[l]
        c[L - l] = np.conj(f[l])
    c[L] = c[L].real
    return c


def trig(c, t):
    """sum_l c_l e^{j l t}"""
    L = (len(c) - 1) // 2
    l = np.arange(-L, L + 1)
    return np.real(np.exp(1j * np.multiply.outer(np.asarray(t, np.float64), l)) @ c)


def angle_deg(z):
    a = math.atan2(z.imag, z.real) * (180.0 / math.pi)
    return a + 360.0 if a < 0.0 else a


def select(r, H, d):
    """ROOTS's merge and selection on the roots r (H kept): list of (t* degrees, modulus, root) for the filled slots,
    and the selection margin (relative gap between the H-th and (H+1)-th root moduli, and between the d-th and
    (d+1)-th candidate moduli)"""
    P = len(r)
    z = np.array(r, np.complex128)
    key = np.abs(z).astype(np.float64)
    dup = np.zeros(P, bool)
    if P > 1:
        dist = np.abs(z[:, None] - z[None, :])
        np.fill_diagonal(dist, np.inf)
        nn = np.argmin(dist, axis=1)
        zz = z.copy()
        for i in range(P):
            j = nn[i]
            if nn[j] == i and dist[i, j] <= MERGE * max(key[i], key[j]):
                zz[i] = 0.5 * (z[i] + z[j])
                dup[i] = i > j
        merged = zz != z
        z = zz
        key[merged] = 1.0
    order_ = sorted(range(P), key=lambda i: (key[i], dup[i], i))
    kept = order_[:H]
    cand = sorted(((key[i], angle_deg(z[i]), i) for i in kept), key=lambda q: (-q[0], q[1], q[2]))
    srt = np.sort(key)
    edge_keep = abs(srt[H] - srt[H - 1]) / max(srt[H], 1e-300) if 0 < H < P else math.inf
    edge_slot = abs(cand[d][0] - cand[d - 1][0]) / cand[d - 1][0] if 0 < d < len(cand) else math.inf
    picks = [(q[1], q[0], z[q[2]]) for q in cand[:min(d, H)] if z[q[2]] != 0]
    return picks, min(edge_keep, edge_slot)


def window(G, pos, lam, K, n, d):
    """One window from its noise eigenvectors G (M, M - d): angles, levels, bins (n slots), the selection margin and
    the roots"""
    pos = np.asarray(pos, np.float64)
    angles = np.zeros(n, np.float32)
    levels = np.zeros(n, np.float32)
    bins = np.full(n, -1, np.int32)
    L, x = order(pos, lam)
    assert L <= MAX_L
    C = G @ G.conj().T
    if d == 0 or x == 0.0 or not np.all(np.isfinite(C)):
        return angles, levels, bins, math.inf, np.zeros(0)
    c = coefficients(C, pos, lam, L)
    t = 0  # exactly zero outer pairs: each a root at 0 and one at infinity
    while t < L and c[t] == 0 and c[2 * L - t] == 0:
        t += 1
    H = L - t
    r = np.roots(c[t:2 * L + 1 - t][::-1]) if H else np.zeros(0)  # highest power first
    if H == 0 or not np.all(np.isfinite(r)):
        return angles, levels, bins, math.inf, r
    picks, margin = select(r, H, d)
    for i, (tdeg, _, _) in enumerate(picks):
        D = ro.objective(G, pos, lam, tdeg * (math.pi / 180.0))[0]
        ang = np.float32(tdeg)
        if ang >= np.float32(360.0) or ang == 0.0:
            ang = np.float32(0.0)
        angles[i], levels[i] = ang, np.float32(1.0 / D if D != 0.0 else math.inf)
        bins[i] = int(math.floor(tdeg * K / 360.0 + 0.5)) % K
    return angles, levels, bins, margin, r


def work_R(R, pos, lam, K, n, N=None, rule=None, d=None):
    """The manifold mode on one covariance R (M, M) with d sources: d = n (FIXED), the MDL / AIC estimate from N
    snapshots, or the count given.  Returns a dict."""
    M = R.shape[0]
    if not np.all(np.isfinite(R)):
        d = n if rule is None and d is None else 0
        G = np.full((M, M - d), np.nan, np.complex128)
    else:
        ev, V = np.linalg.eigh(R)
        if d is None:
            d = n if rule is None else so.estimate_source_count(ev, N, n, rule)[0]
        G = V[:, : M - d]
    a, l, b, margin, r = window(G, pos, lam, K, n, d)
    return {"angles": a, "levels": l, "bins": b, "count": d, "margin": margin, "G": G, "roots": r}


def grid_minima(G, pos, lam, d, Kg=36000):
    """The d smallest circular local minima of D on a Kg-point grid, in degrees (the fine-grid rule the root selection
    is compared with)"""
    t = 2.0 * math.pi * np.arange(Kg) / Kg
    D = direct_D(G @ G.conj().T, pos, lam, t)
    loc = np.nonzero((D < np.roll(D, 1)) & (D <= np.roll(D, -1)))[0]
    loc = loc[np.argsort(D[loc], kind="stable")][:d]
    return loc * 360.0 / Kg
