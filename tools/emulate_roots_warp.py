#!/usr/bin/env python
"""CPU emulation (numpy fp64) of roots_kernel (gr-baz_b200/csrc/music_roots.cuh): the coefficients c_l in the kernel's
summation order, then its root finder roots_solve (shared with manifold_kernel): the outer-pair deflation, the
Newton-polygon starting points, the Aberth-Ehrlich loop over one thread per root with its reversed evaluation outside
the unit circle and its stopping rule, the double-root merge and the selection of the slot roots.  The threads (called
lanes here) are numpy vectors; every lane takes the kernel's decisions.  The keyword switches restore the behaviour
before the fixes (unit-circle starts, plain Horner everywhere, no convergence flag) and plant the defects that
tests/test_gridless_oracle.py shows the checker failing."""
import math

import numpy as np

MAX_IT = 100
EPS = 2.220446049250313e-16
STOP = 4.0 * EPS
BACK = 8.0  # a lane has converged once |Q(z)| <= BACK P eps sum_k |b_k| |z|^k (an exact root of a nearby polynomial)
MERGE = 1e-6


def coefficients(G):
    """c_l, l = 0 .. M-1, from the noise eigenvectors G (M, p) (columns), summed as the kernel's lane l does"""
    M, p = G.shape
    c = np.zeros(M, np.complex128)
    for l in range(M):
        s = 0j
        for j in range(p):
            for i in range(M - l):
                s += G[i, j] * np.conj(G[i + l, j])
        c[l] = s
    return c


def starts(b, P, circle=False):
    """the starting points of the P lanes: on the unit circle (circle=True, the former rule) or on the circles of the
    upper convex hull of (k, log|b_k|) (Bini), the roots of hull segment [k_i, k_i+1) at radius
    (|b_k_i| / |b_k_i+1|)^(1 / (k_i+1 - k_i)), angles 2 pi j / (k_i+1 - k_i) + 2 pi k_i / P + 0.5 / P * pi"""
    lane = np.arange(P)
    if circle:
        return np.exp(1j * math.pi * (2.0 * lane / P + 0.5 / P))
    lg = np.array([math.log2(abs(x)) if x != 0 else -math.inf for x in b])
    hull = [0]
    for k in range(1, P + 1):
        if lg[k] == -math.inf:
            continue
        while len(hull) >= 2:
            i, j = hull[-2], hull[-1]
            # j lies on or below the chord i -> k: drop it
            if (lg[j] - lg[i]) * (k - i) <= (lg[k] - lg[i]) * (j - i):
                hull.pop()
            else:
                break
        hull.append(k)
    z = np.zeros(P, np.complex128)
    for i, j in zip(hull, hull[1:]):
        n = j - i
        u = 2.0 ** ((lg[i] - lg[j]) / n)
        for r in range(i, j):
            z[r] = u * np.exp(1j * math.pi * (2.0 * (r - i) / n + 2.0 * i / P + 0.5 / P))
    return z


def aberth(b, P, max_it=MAX_IT, circle=False, reversed_eval=True, aberth_sum=True, backward=True):
    """Aberth-Ehrlich on sum_k b_k z^k: returns (z, iterations, every lane met the stopping rule).  A lane stops when its
    correction is within 4 ulps of |z| or (backward) its residual is at rounding level; a stopped lane stays put."""
    z = starts(b, P, circle)
    done = np.zeros(P, bool)
    ab = np.abs(b)
    for it in range(max_it):
        S = np.zeros(P, np.complex128)
        if aberth_sum:
            for s in range(P):
                dz = z - z[s]
                with np.errstate(divide="ignore", invalid="ignore"):
                    S += np.where(np.arange(P) != s, 1.0 / dz, 0.0)
        outside = (np.abs(z) > 1.0) if reversed_eval else np.zeros(P, bool)
        with np.errstate(all="ignore"):
            w = np.where(outside, 1.0 / z, z)
            # inside: Horner for Q and Q'; outside: for R(w) = sum_k b_k w^(P-k) and R'
            q = np.where(outside, b[0], b[P]).astype(np.complex128)
            dq = np.zeros(P, np.complex128)
            aw = np.abs(w)
            acc = np.where(outside, ab[0], ab[P])
            for k in range(1, P + 1):
                dq = dq * w + q
                q = q * w + np.where(outside, b[k], b[P - k])
                acc = acc * aw + np.where(outside, ab[k], ab[P - k])
            wc_in = q / (dq - q * S)
            num = z * q
            wc_out = num / (P * q - w * dq - num * S)
            wc = np.where(outside, wc_out, wc_in)
            if backward:
                done = done | (np.abs(q) <= BACK * P * EPS * acc)
            wc = np.where(done, 0.0, wc)
        z = z - wc
        with np.errstate(invalid="ignore", over="ignore"):
            done = done | (np.abs(wc) ** 2 <= STOP * STOP * np.abs(z) ** 2)
        if np.all(done):
            return z, it + 1, True
    return z, max_it, False


def merge(z, P, enabled=True):
    """(z, key, dup): two lanes that are each other's nearest and closer than MERGE max|z| become their midpoint with
    modulus key 1; dup marks the higher lane of the pair"""
    key = np.abs(z)
    dup = np.zeros(P, bool)
    merged = np.zeros(P, bool)
    if P < 2 or not enabled:
        return z, key, dup, merged
    dist = np.abs(z[:, None] - z[None, :])
    np.fill_diagonal(dist, np.inf)
    nn = np.argmin(dist, axis=1)  # the lowest lane among equal distances, as the kernel's strict '<'
    zz, kk = z.copy(), key.copy()
    for r in range(P):
        s = nn[r]
        if nn[s] == r and dist[r, s] <= MERGE * max(key[r], key[s]):
            zz[r] = 0.5 * (z[r] + z[s])
            kk[r] = 1.0
            dup[r] = r > s
            merged[r] = True
    return zz, kk, dup, merged


def roots_window(G, d, direction, max_it=MAX_IT, circle=False, reversed_eval=True, conv_flag=True, aberth_sum=True,
                 merge_on=True, backward=True):
    """One window: G (M, M - d) noise eigenvectors, d sources, direction(z) -> t* degrees.  Returns dict(ok, slots =
    [(t*, z)] in slot order, iterations, converged, z, t)."""
    M = G.shape[0]
    c = coefficients(G)
    out = {"ok": False, "slots": [], "iterations": 0, "converged": False, "t": None, "c": c}
    if not np.all(np.isfinite(c)):
        return out
    nzl = [l for l in range(M) if c[l] != 0]
    t = M - 1 - max(nzl) if nzl else M - 1
    P, H = 2 * (M - 1 - t), M - 1 - t
    out["t"] = t
    if d <= 0 or P <= 0:
        return out
    b = np.array([c[k - H] if k >= H else np.conj(c[H - k]) for k in range(P + 1)])
    z, its, conv = aberth(b, P, max_it, circle, reversed_eval, aberth_sum, backward)
    out.update(iterations=its, converged=conv, z=z)
    ok = bool(np.all(np.isfinite(z)))
    if conv_flag:
        ok = ok and conv
    if not ok:
        return out
    out.update(ok=True, slots=select(z, H, d, direction, merge_on))
    return out


def select(z, H, d, direction, merge_on=True):
    """the slot roots [(t*, z)] of the P = 2H converged lanes z: merge, keep the H smallest keys (a double root's
    second copy after every other root of key 1), slots in descending key, ties to the lower angle"""
    P = len(z)
    z, key, dup, _ = merge(z, P, merge_on)
    order = sorted(range(P), key=lambda r: (key[r], dup[r], r))
    kept = order[:H]
    td = {r: direction(z[r]) for r in kept}
    slots = sorted(kept, key=lambda r: (-key[r], td[r], r))[:min(d, H)]
    return [(td[r], z[r]) for r in slots]
