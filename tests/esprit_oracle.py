"""fp64 restatement of the ESPRIT peak mode (MUSIC_B200_PEAKS_ESPRIT, include/music_b200.h) for uniform linear arrays,
with np.linalg.solve and np.linalg.eigvals on LAPACK eigenvectors.  Test infrastructure next to root_music_oracle.py;
the product path never imports this file.

    E_s = the d eigenvectors of largest eigenvalue, E1 = rows 0 .. M-2, E2 = rows 1 .. M-1
    Psi = (E1^H E1)^-1 E1^H E2; no peaks unless E1^H E1 is positive definite (1 - |r|^2 > 0, r = last row of E_s) and
    Psi is finite
    each eigenvalue phi of Psi: t* = the root mode's direction of z = phi (an eigenvalue exactly 0: slot unfilled),
    level = 1 / D(t*) (direct form over the M - d noise eigenvectors), bin = floor(t* K / 360 + 0.5) mod K
    slots in descending fp64 level, exact ties to the lower t*, then the lower eigenvalue index
"""
import math

import numpy as np

from oracle import music_oracle as mo

import refine_oracle as ro
import source_count_oracle as so
from root_music_oracle import direction, ula_geometry


def psi_matrix(Es):
    """Psi = (E1^H E1)^-1 E1^H E2 by np.linalg.solve, or None when E1^H E1 is not positive definite"""
    r = Es[-1]
    if not 1.0 - float(np.sum(np.abs(r) ** 2)) > 0.0:
        return None
    E1, E2 = Es[:-1], Es[1:]
    return np.linalg.solve(E1.conj().T @ E1, E1.conj().T @ E2)


def psi_sherman_morrison(Es):
    """the same Psi through (E1^H E1)^-1 = I + r^H r / (1 - |r|^2), the form the kernel uses"""
    r = Es[-1][None, :]
    den = 1.0 - float(np.sum(np.abs(r) ** 2))
    B = Es[:-1].conj().T @ Es[1:]
    return B + r.conj().T @ (r @ B) / den


def esprit_window(V, d, pos, lam, K, n):
    """One window from its eigenvectors V (M, M, ascending eigenvalues) and source count d: angles, levels, bins (n
    slots) and the ordering margin (the smallest relative gap between adjacent filled levels)"""
    ok, _, s = ula_geometry(pos, lam)
    assert ok
    M = V.shape[0]
    angles = np.zeros(n, np.float32)
    levels = np.zeros(n, np.float32)
    bins = np.full(n, -1, np.int32)
    if d == 0 or not np.all(np.isfinite(V)):
        return angles, levels, bins, math.inf
    G, Es = V[:, : M - d], V[:, M - d:]
    Psi = psi_matrix(Es)
    if Psi is None or not np.all(np.isfinite(Psi)):
        return angles, levels, bins, math.inf
    cand = []
    for i, phi in enumerate(np.linalg.eigvals(Psi)):
        if phi == 0:
            continue
        tdeg = direction(complex(phi), s, lam)
        D = ro.objective(G, pos, lam, tdeg * (math.pi / 180.0))[0]
        cand.append((1.0 / D if D != 0.0 else math.inf, tdeg, i, D))
    cand.sort(key=lambda q: (-q[0], q[1], q[2]))
    for i, (_, tdeg, _, D) in enumerate(cand):
        ang = np.float32(tdeg)
        if ang >= np.float32(360.0) or ang == 0.0:
            ang = np.float32(0.0)
        angles[i], levels[i] = ang, np.float32(1.0 / D if D != 0.0 else math.inf)
        bins[i] = int(math.floor(tdeg * K / 360.0 + 0.5)) % K
    lv = [q[0] for q in cand]
    margin = min((abs(a - b) / max(abs(a), 1e-300) for a, b in zip(lv, lv[1:])), default=math.inf)
    return angles, levels, bins, margin


def work_R(R, pos, lam, K, n, N=None, rule=None, d=None):
    """ESPRIT on one covariance R (M, M) with d sources: d = n (FIXED), the MDL / AIC estimate from N snapshots, or the
    count given.  The margin also holds the relative eigenvalue gap at the subspace boundary."""
    M = R.shape[0]
    if not np.all(np.isfinite(R)):  # non-finite R: no peak under any rule
        d = n if rule is None and d is None else 0
        return {"angles": np.zeros(n, np.float32), "levels": np.zeros(n, np.float32), "bins": np.full(n, -1, np.int32),
                "count": d, "margin": math.inf}
    ev, V = np.linalg.eigh(R)
    if d is None:
        d = n if rule is None else so.estimate_source_count(ev, N, n, rule)[0]
    a, l, b, margin = esprit_window(V, d, pos, lam, K, n)
    if 0 < d < M:
        lo, hi = ev[M - d - 1], ev[M - d]
        margin = min(margin, abs(hi - lo) / max(abs(hi), 1e-300))
    return {"angles": a, "levels": l, "bins": b, "count": d, "margin": margin}


def work(in_c64, m, n, K, pos, lam, rule=None):
    """One window of complex64 samples"""
    R = mo.covariance(np.ascontiguousarray(in_c64, dtype=np.complex64), m)
    return work_R(R, pos, lam, K, n, len(in_c64) // m, rule)
