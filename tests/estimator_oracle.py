"""fp64 restatement of the MVDR (Capon) and Bartlett spectra (music_b200_set_estimator, include/music_b200.h), their peak
picks and both refinements (1-D and az-el).  Test infrastructure: the definition is written out literally, so that it can
be read against the header; the product path never imports this file.  MVDR is evaluated with np.linalg.solve, never
with a Cholesky factor, so that it checks the engine's factor route independently.

    R = the window's covariance,  a = a_k (table row k widened to fp64),  M = m
    BARTLETT  P[k] = (a^H R a) / (a^H a)^2
    MVDR      delta = loading tr(R) / M,  R_L = R + delta I,  P[k] = 1 / (a^H R_L^-1 a)   (NaN when R_L is not PD)
    refinement: MVDR minimises D = a(t)^H R_L^-1 a(t), level 1 / D;  BARTLETT minimises F = -B, B = a(t)^H R a(t),
                level B / M^2; the drivers are those of refine_oracle.py (1-D) and azel_oracle.py (az-el).
"""
import math

import numpy as np

from oracle import music_oracle as mo

import azel_oracle as ao
import refine_oracle as ro
import source_count_oracle as so

KINDS = ("mvdr", "bartlett")
MAX_IT = ro.MAX_IT
TOL = ro.TOL
T_MIN = ao.T_MIN
DEG = math.pi / 180.0


def loaded(R, loading):
    """R_L = R + delta I, delta = loading * tr(R) / M"""
    M = R.shape[0]
    delta = loading * float(np.trace(R).real) / float(M)
    return R + delta * np.eye(M)


def positive_definite(A):
    """whether the Hermitian A is positive definite (every eigenvalue > 0; any NaN / inf fails)"""
    if not np.all(np.isfinite(A)):
        return False
    return bool(np.min(np.linalg.eigvalsh(A)) > 0.0)


def spectrum(R, table_c64, kind, loading=0.0):
    """fp64 P[k] of the (K, m) complex64 table for one window's covariance R"""
    a = np.asarray(table_c64).reshape(-1, R.shape[0]).astype(np.complex128)  # (K, M)
    if kind == "bartlett":
        num = np.einsum("ki,ij,kj->k", a.conj(), R, a).real
        den = np.sum(np.abs(a) ** 2, axis=1) ** 2
        with np.errstate(divide="ignore", invalid="ignore"):
            return num / den
    if kind == "mvdr":
        RL = loaded(R, loading)
        if not positive_definite(RL):
            return np.full(a.shape[0], np.nan)
        y = np.linalg.solve(RL, a.T)  # (M, K) = R_L^-1 a_k
        return 1.0 / np.einsum("ik,ik->k", a.T.conj(), y).real
    raise ValueError(kind)


def beam_power(R, w):
    """w^H R w: the output power of the beamformer w"""
    return float((w.conj() @ R @ w).real)


def picks(P, n, K, peak="top", exclusion=0, count=None):
    """(angles, levels, bins) of the first `count` (default n) slots under the peak rule, the rest (0, 0, -1)"""
    count = n if count is None else count
    if count == 0:
        return np.zeros(n, np.float32), np.zeros(n, np.float32), np.full(n, -1, np.int32)
    if peak == "local":
        q = mo.pick_local_maxima(P, count, K, exclusion)
    else:
        q = mo.pick_top_n(P, count, K)
    ang = np.zeros(n, np.float32)
    lvl = np.zeros(n, np.float32)
    bins = np.full(n, -1, np.int32)
    for i, (a, l, b) in enumerate(q):
        ang[i], lvl[i], bins[i] = a, l, b
    return ang, lvl, bins


def work(in_c64, m, n, table_c64, kind, loading=0.0, peak="top", exclusion=0, rule=None):
    """One window: R, the estimator's spectrum, the source count (MDL / AIC: only to count) and the peak pick."""
    x = np.ascontiguousarray(in_c64, dtype=np.complex64)
    R = mo.covariance(x, m)
    K = np.asarray(table_c64).reshape(-1, m).shape[0]
    P = spectrum(R, table_c64, kind, loading)
    d = n
    if rule is not None:
        d = so.estimate_source_count(np.linalg.eigvalsh(R), x.shape[0] // m, n, rule)[0]
    ang, lvl, bins = picks(P, n, K, peak, exclusion, d)
    return {"R": R, "P": P, "angles": ang, "levels": lvl, "bins": bins, "count": d}


# ---- 1-D refinement ---------------------------------------------------------------------------------------------------
def objective(R, kind, loading, pos, lam, t):
    """(D, D', D'') of the objective the refinement minimises: MVDR a^H R_L^-1 a, BARTLETT -a^H R a"""
    a, phi, psi = ro.steering(pos, lam, t)
    a1 = -1j * psi * a
    a2 = (1j * phi - psi * psi) * a
    if kind == "mvdr":
        RL = loaded(R, loading)
        y, y1 = np.linalg.solve(RL, a), np.linalg.solve(RL, a1)
        sign = 1.0
    else:
        y, y1 = R @ a, R @ a1
        sign = -1.0
    D = float((a.conj() @ y).real)
    D1 = float(2.0 * (a1.conj() @ y).real)
    D2 = float(2.0 * ((a1.conj() @ y1).real + (a2.conj() @ y).real))
    return sign * D, sign * D1, sign * D2


def level_of(kind, D, M):
    return np.float32(-D / (float(M) * float(M))) if kind == "bartlett" else np.float32(1.0 / D)


def refine_slot(R, kind, loading, pos, lam, b, K):
    """refine_oracle.refine_slot on this estimator's objective"""
    M = R.shape[0]
    obj = lambda t: objective(R, kind, loading, pos, lam, t)
    deg_b = float(b) * 360.0 / float(K)
    tb = deg_b * DEG
    delta = (360.0 / float(K)) * DEG
    Db, f, df = obj(tb)
    lo, hi = tb - delta, tb + delta
    fl = obj(lo)[1]
    fh = obj(hi)[1]
    x = tb
    if fl < 0.0 and fh > 0.0:
        dxold = hi - lo
        dx = dxold
        for _ in range(MAX_IT):
            if f == 0.0:
                break
            if ((x - hi) * df - f) * ((x - lo) * df - f) > 0.0 or abs(2.0 * f) > abs(dxold * df):
                dxold = dx
                dx = 0.5 * (hi - lo)
                x = lo + dx
            else:
                dxold = dx
                dx = f / df
                x = x - dx
            if abs(dx) <= TOL:
                break
            _, f, df = obj(x)
            if f < 0.0:
                lo = x
            else:
                hi = x
    out = {"fl": fl, "fh": fh, "Db": Db, "Dx": Db, "kept": True, "theta": tb, "angle": np.float32(deg_b),
           "level": level_of(kind, Db, M)}
    if x != tb:
        Dx = obj(x)[0]
        out["Dx"] = Dx
        if Dx <= Db:
            a = math.fmod(x * (180.0 / math.pi), 360.0)
            if a < 0.0:
                a += 360.0
            ang = np.float32(a)
            if ang >= np.float32(360.0) or ang == 0.0:
                ang = np.float32(0.0)
            out.update(kept=False, theta=x, angle=ang, level=level_of(kind, Dx, M))
    return out


# ---- az-el refinement -------------------------------------------------------------------------------------------------
def objective_azel(R, kind, loading, pos, lam, ph, ep):
    """(D, gradient (2,), Hessian (2, 2)) of the az-el objective: MVDR a^H R_L^-1 a, BARTLETT -a^H R a"""
    pos = np.asarray(pos, dtype=np.float64)
    x, y, z = pos[:, 0], pos[:, 1], pos[:, 2]
    sp, cp, se, ce = math.sin(ph), math.cos(ph), math.sin(ep), math.cos(ep)
    h = x * cp + y * sp
    v = y * cp - x * sp
    c = 2.0 * math.pi / lam
    th = c * (ce * h + z * se)
    tp = c * (ce * v)
    te = c * (z * ce - se * h)
    tpp = -c * (ce * h)
    tpe = -c * (se * v)
    tee = -th
    a = np.cos(th) - 1j * np.sin(th)
    da = [-1j * tp * a, -1j * te * a]
    d2 = [[(-tp * tp - 1j * tpp) * a, (-tp * te - 1j * tpe) * a], [None, (-te * te - 1j * tee) * a]]
    d2[1][0] = d2[0][1]
    if kind == "mvdr":
        RL = loaded(R, loading)
        Q = lambda u: np.linalg.solve(RL, u)
        sign = 1.0
    else:
        Q = lambda u: R @ u
        sign = -1.0
    ya = Q(a)
    yu = [Q(da[0]), Q(da[1])]
    D = float((a.conj() @ ya).real)
    g = np.array([2.0 * (da[u].conj() @ ya).real for u in range(2)])
    H = np.empty((2, 2))
    for u in range(2):
        for w in range(2):
            H[u, w] = 2.0 * ((da[u].conj() @ yu[w]).real + (d2[u][w].conj() @ ya).real)
    return sign * D, sign * g, sign * H


def refine_slot_azel(R, kind, loading, pos, lam, b, grid):
    """azel_oracle.refine_slot on this estimator's objective"""
    M = R.shape[0]
    obj = lambda p, e: objective_azel(R, kind, loading, pos, lam, p, e)
    i, k = grid.split(b)
    ph_b = grid.az_deg(k) * DEG
    ep_b = grid.el_deg(i) * DEG
    dph = (360.0 / float(grid.n_az)) * DEG
    dep = ((grid.el_hi - grid.el_lo) / float(grid.n_el - 1)) * DEG if grid.n_el > 1 else 0.0
    plo, phi = ph_b - dph, ph_b + dph
    elo, ehi = max(ep_b - dep, grid.el_lo * DEG), min(ep_b + dep, grid.el_hi * DEG)
    D, g, H = obj(ph_b, ep_b)
    Db = D
    x0, x1 = ph_b, ep_b
    for _ in range(MAX_IT):
        if g[0] == 0.0 and g[1] == 0.0:
            break
        det = H[0, 0] * H[1, 1] - H[0, 1] * H[0, 1]
        if H[0, 0] > 0.0 and det > 0.0:
            s0 = -(H[1, 1] * g[0] - H[0, 1] * g[1]) / det
            s1 = -(H[0, 0] * g[1] - H[0, 1] * g[0]) / det
        else:
            gn = math.sqrt(g[0] * g[0] + g[1] * g[1])
            s0 = -g[0] * dph / gn
            s1 = -g[1] * dph / gn
        s0 = ao.clamp(x0 + s0, plo, phi) - x0
        s1 = ao.clamp(x1 + s1, elo, ehi) - x1
        t = 1.0
        found = None
        while t > T_MIN:
            y0, y1 = x0 + t * s0, x1 + t * s1
            f = obj(y0, y1)
            if f[0] <= D:
                found = f
                break
            t *= 0.5
        if found is None:
            break
        step = max(abs(t * s0), abs(t * s1))
        x0, x1 = y0, y1
        D, g, H = found
        if step <= TOL:
            break
    out = {"Db": Db, "Dx": D, "kept": True, "x": (ph_b, ep_b), "azimuth": np.float32(grid.az_deg(k)),
           "elevation": np.float32(grid.el_deg(i)), "level": level_of(kind, Db, M)}
    if (x0 != ph_b or x1 != ep_b) and D <= Db:
        a = math.fmod(x0 * (180.0 / math.pi), 360.0)
        if a < 0.0:
            a += 360.0
        az = np.float32(a)
        if az >= np.float32(360.0) or az == 0.0:
            az = np.float32(0.0)
        out.update(kept=False, x=(x0, x1), azimuth=az, elevation=np.float32(x1 * (180.0 / math.pi)), level=level_of(kind, D, M))
    return out
