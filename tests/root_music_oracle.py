"""fp64 restatement of the root-MUSIC peak mode (MUSIC_B200_PEAKS_ROOTS, include/music_b200.h) for uniform linear
arrays, with numpy.roots on LAPACK eigenvectors.  Test infrastructure next to refine_oracle.py; the product path never
imports this file.

    s = (p_{M-1} - p_0) / (M - 1);  ULA iff |s| > 0, max ||p_m - (p_0 + m s)|| <= 1e-6 |s|, |s| <= (lambda / 2)(1 + 1e-12)
    C = G G^H,  c_l = sum_{j - i = l} C_ij,  Q(z) = sum_l c_l z^(l + M - 1),  D(t) = sum_l c_l z0^l,
    z0 = exp(-j 2 pi (s . u(t)) / lambda)
    roots: each exactly zero outer pair c_{+-l} is a root at 0 and one at infinity; two roots that are each other's
    nearest and closer than 1e-6 max(|z_a|, |z_b|) are one double root on the unit circle (midpoint, modulus 1, the
    copy of the higher index sorted after every other root of modulus 1)
    keep the M - 1 roots of smallest modulus; slots take the d kept roots of largest modulus (descending, exact ties to
    the lower angle); a kept root at 0 leaves its slot unfilled
    angle: cpsi = clamp(-arg(z) lambda / (2 pi |s|), -1, 1), t* = min over alpha +- acos(cpsi) wrapped into [0, 360)
    level = 1 / D(t*) (direct form), bin = floor(t* K / 360 + 0.5) mod K
"""
import math

import numpy as np

from oracle import music_oracle as mo

import refine_oracle as ro
import source_count_oracle as so

MERGE = 1e-6


def ula_geometry(pos, lam):
    """(is a ULA the root mode accepts, p_0, s) for positions (M, 2)"""
    pos = np.asarray(pos, np.float64)
    M = pos.shape[0]
    p0 = pos[0].copy()
    s = (pos[M - 1] - pos[0]) / (M - 1)
    sa = math.hypot(s[0], s[1])
    dev = max(math.hypot(pos[m, 0] - (p0[0] + m * s[0]), pos[m, 1] - (p0[1] + m * s[1])) for m in range(M))
    ok = sa > 0.0 and dev <= 1e-6 * sa and sa <= 0.5 * lam * (1.0 + 1e-12)
    return ok, p0, s


def coefficients(G):
    """c (2M - 1,) with c[l + M - 1] = c_l = sum_{j - i = l} (G G^H)_ij"""
    M = G.shape[0]
    C = G @ G.conj().T
    c = np.zeros(2 * M - 1, np.complex128)
    for l in range(-(M - 1), M):
        c[l + M - 1] = sum(C[i, i + l] for i in range(M) if 0 <= i + l < M)
    return c


def laurent(c, z0):
    """D = sum_l c_l z0^l"""
    M = (len(c) + 1) // 2
    return sum(c[l + M - 1] * z0 ** l for l in range(-(M - 1), M))


def z0_of(s, lam, t):
    """z0 = exp(-j 2 pi (s . u(t)) / lambda), t in radians"""
    return np.exp(-2j * math.pi * (s[0] * math.cos(t) + s[1] * math.sin(t)) / lam)


def all_roots(c):
    """(roots of the reduced polynomial, t): t exactly-zero outer pairs, each a root at 0 and at infinity"""
    M = (len(c) + 1) // 2
    t = 0
    while t < M - 1 and c[2 * M - 2 - t] == 0 and c[t] == 0:
        t += 1
    b = c[t:2 * M - 1 - t]  # coefficients of z^0 .. z^(2(M-1-t))
    r = np.roots(b[::-1]) if len(b) > 1 else np.zeros(0, np.complex128)
    return r, t


def direction(z, s, lam):
    """t* in degrees (the lower of alpha +- psi in [0, 360))"""
    sa = math.hypot(s[0], s[1])
    cpsi = min(1.0, max(-1.0, -math.atan2(z.imag, z.real) * lam / (2.0 * math.pi * sa)))
    psi, alpha = math.acos(cpsi), math.atan2(s[1], s[0])
    a1 = math.fmod((alpha + psi) * (180.0 / math.pi), 360.0)
    a2 = math.fmod((alpha - psi) * (180.0 / math.pi), 360.0)
    a1 += 360.0 if a1 < 0.0 else 0.0
    a2 += 360.0 if a2 < 0.0 else 0.0
    return min(a1, a2)


def select(r, t, M, d, s, lam):
    """The filled slots: list of (t* degrees, modulus key, root), plus the edge margins of the selection (relative gap
    between the (M-1)-th and M-th root moduli, and between the d-th and (d+1)-th candidate moduli)"""
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
    H = M - 1 - t
    order = sorted(range(P), key=lambda i: (key[i], dup[i], i))
    kept = order[:H]
    cand = sorted(((key[i], direction(z[i], s, lam), i) for i in kept), key=lambda q: (-q[0], q[1], q[2]))
    srt = np.sort(key)
    edge_keep = abs(srt[H] - srt[H - 1]) / max(srt[H], 1e-300) if 0 < H < P else math.inf
    edge_slot = abs(cand[d][0] - cand[d - 1][0]) / cand[d - 1][0] if 0 < d < len(cand) else math.inf
    return [(q[1], q[0], z[q[2]]) for q in cand[:min(d, H)]], min(edge_keep, edge_slot)


def roots_window(G, pos, lam, K, n, d):
    """One window from its noise eigenvectors G (M, M - d): angles, levels, bins (n slots) and the selection margin"""
    ok, _, s = ula_geometry(pos, lam)
    assert ok
    M = G.shape[0]
    angles = np.zeros(n, np.float32)
    levels = np.zeros(n, np.float32)
    bins = np.full(n, -1, np.int32)
    c = coefficients(G)
    if d == 0 or not np.all(np.isfinite(c)):
        return angles, levels, bins, math.inf
    r, t = all_roots(c)
    if not np.all(np.isfinite(r)):
        return angles, levels, bins, math.inf
    picks, margin = select(r, t, M, d, s, lam)
    for i, (tdeg, _, _) in enumerate(picks):
        D = ro.objective(G, pos, lam, tdeg * (math.pi / 180.0))[0]
        ang = np.float32(tdeg)
        if ang >= np.float32(360.0) or ang == 0.0:
            ang = np.float32(0.0)
        angles[i], levels[i] = ang, np.float32(1.0 / D if D != 0.0 else math.inf)
        bins[i] = int(math.floor(tdeg * K / 360.0 + 0.5)) % K
    return angles, levels, bins, margin


def work_R(R, pos, lam, K, n, N=None, rule=None, d=None):
    """The root mode on one covariance R (M, M) with d sources: d = n (FIXED), the MDL / AIC estimate from N snapshots,
    or the count given.  Returns a dict."""
    M = R.shape[0]
    if not np.all(np.isfinite(R)):  # non-finite C: no peak under any rule
        d = n if rule is None and d is None else 0
        G = np.full((M, M - d), np.nan, np.complex128)
    else:
        ev, V = np.linalg.eigh(R)
        if d is None:
            d = n if rule is None else so.estimate_source_count(ev, N, n, rule)[0]
        G = V[:, : M - d]
    a, l, b, margin = roots_window(G, pos, lam, K, n, d)
    return {"angles": a, "levels": l, "bins": b, "count": d, "margin": margin, "G": G}


def work(in_c64, m, n, K, pos, lam, rule=None):
    """One window of complex64 samples"""
    R = mo.covariance(np.ascontiguousarray(in_c64, dtype=np.complex64), m)
    return work_R(R, pos, lam, K, n, len(in_c64) // m, rule)
