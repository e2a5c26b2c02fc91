"""fp64 restatement of the WSF peak mode (MUSIC_B200_PEAKS_WSF) and of the joint refinement (MUSIC_B200_REFINE_JOINT)
of include/music_b200.h.  Test infrastructure: the definition is written out literally, so that it can be read against
the header; the product path never imports this file.

    WSF     l_0 <= .. <= l_{M-1}, e_i = np.linalg.eigh(R); s2 = mean(l_0 .. l_{M-d-1}); w_i = (l_i - s2)^2 / l_i for the
            d largest (0 unless l_i > s2); X = sum_i w_i e_i e_i^H; the DML search (dml_oracle) on X, levels from R.
    JOINT   V(t) = Re tr(P_perp X), P_perp = I - A (A^H A)^-1 A^H; g_i = -2 Re(A+ X P_perp D)_ii;
            H = 2 Re((D^H P_perp D) o (A+ X A+^H)^T); s = -H^-1 g by np.linalg.solve, projected onto the box
            |t_i - t_b,i| <= delta, accepted iff V strictly decreases, else halved (up to 30 times); at most 50 steps.
            Positive definiteness is read from the pivots of the leading minors (det ratios), never from a Cholesky.
"""
import math

import numpy as np

from oracle import music_oracle as mo

import dml_oracle as dm
import source_count_oracle as so

T_REL = 2.0 ** -30    # pivot l of A^H A must exceed this fraction of ||a_l||^2
H_REL = 2.0 ** -40    # pivot k of H must exceed this fraction of H_kk
MAX_STEPS = 50
MAX_HALVINGS = 30
STEP_TOL = 1e-12      # radians
DEG2RAD = math.pi / 180.0
RAD2DEG = 180.0 / math.pi


# ---- WSF ---------------------------------------------------------------------------------------------------------------
def wsf_factor(l, E, d):
    """F (M, c): the columns sqrt(w_i) e_i with w_i > 0 in ascending i, so that X = F F^H; None when the window fails"""
    l = np.asarray(l, np.float64)
    M = l.shape[0]
    if d == 0 or not np.all(np.isfinite(l)) or not l[0] > 0.0:
        return None
    s2 = float(np.sum(l[:M - d])) / float(M - d)
    cols = [math.sqrt((l[i] - s2) ** 2 / l[i]) * E[:, i] for i in range(M - d, M) if l[i] > s2]
    return np.stack(cols, 1) if cols else np.zeros((M, 0), np.complex128)


def wsf_matrix(l, E, d):
    """X (M, M) from ascending eigenvalues l (M,) and eigenvectors in the columns of E; None when the window fails"""
    F = wsf_factor(l, E, d)
    if F is None:
        return None
    X = F @ F.conj().T
    if not float(np.trace(X).real) > 0.0:
        return None
    return X


def wsf_R(R, table_c64, n, d=None):
    """One window from its covariance R: the DML search on X with DML's levels from R.  Returns dml_oracle's dict plus X."""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    d = n if d is None else int(d)
    out = dm.empty(n)
    out["X"] = out["F"] = None
    if not np.all(np.isfinite(R)):
        return out
    l, E = np.linalg.eigh(R)
    X = wsf_matrix(l, E, d)
    if X is None:
        return out
    s = dm.work_R(X, table_c64, n, d)
    s["X"], s["F"] = X, wsf_factor(l, E, d)
    if not s["slots"]:
        return s
    a, _ = dm.rows(table_c64, M)
    K = a.shape[0]
    slots = s["slots"]
    p, s2 = dm.levels(R, a, slots)
    order = sorted(range(d), key=lambda i: (-p[i], slots[i]))
    for r, i in enumerate(order):
        s["angles"][r] = np.float32(float(slots[i]) * 360.0 / float(K))
        s["levels"][r] = np.float32(p[i])
        s["bins"][r] = slots[i]
    s.update(p=p, s2=s2)
    return s


# ---- JOINT -------------------------------------------------------------------------------------------------------------
def steer(pos, lam, t):
    """A (M, d) and D = dA/dt (M, d) at the angles t (d,) radians: a_m = exp(-j phi_m), the refinement's convention"""
    pos = np.asarray(pos, np.float64)
    t = np.asarray(t, np.float64)
    st, ct = np.sin(t)[None, :], np.cos(t)[None, :]
    phi = 2.0 * np.pi * ((pos[:, 1:2] * st + pos[:, 0:1] * ct) / lam)
    psi = 2.0 * np.pi * ((pos[:, 1:2] * ct - pos[:, 0:1] * st) / lam)
    A = np.cos(phi) - 1j * np.sin(phi)
    return A, -1j * psi * A


def pivots(G):
    """the pivots of an LDL^H factorisation of G, as ratios of leading principal minors"""
    dets = [1.0] + [float(np.linalg.det(G[:k, :k]).real) for k in range(1, G.shape[0] + 1)]
    return [dets[k + 1] / dets[k] if dets[k] != 0.0 else -np.inf for k in range(G.shape[0])]


def gram_ok(A):
    G = A.conj().T @ A
    na = np.sum(np.abs(A) ** 2, axis=0)
    return all(p > T_REL * na[k] for k, p in enumerate(pivots(G)))


def criterion(F, A):
    """V = ||P_perp F||_F^2 = Re tr(P_perp X), or None when A^H A is not positive definite"""
    if not gram_ok(A):
        return None
    M = A.shape[0]
    P = np.eye(M) - A @ np.linalg.solve(A.conj().T @ A, A.conj().T)
    E = P @ F
    return float(np.sum(E.real * E.real + E.imag * E.imag))


def grad_hess(F, A, D):
    M = A.shape[0]
    X = F @ F.conj().T
    Ap = np.linalg.solve(A.conj().T @ A, A.conj().T)
    P = np.eye(M) - A @ Ap
    g = -2.0 * np.real(np.diag(Ap @ X @ P @ D))
    H = 2.0 * np.real((D.conj().T @ P @ D) * (Ap @ X @ Ap.conj().T).T)
    return g, H


def hess_ok(H):
    Hd = np.diag(H)
    return all(p > 0.0 and p > H_REL * Hd[k] for k, p in enumerate(pivots(H)))


def dml_factor(R):
    """F = L of R = L L^H (lower, real diagonal), or None when R is not positive definite"""
    try:
        return np.linalg.cholesky(np.asarray(R, np.complex128))
    except np.linalg.LinAlgError:
        return None


def joint(F, bins, K, pos, lam):
    """The refined angles theta* (radians, slot order) of the filled slots `bins`, and a dict of what happened: moved
    (False when A^H A is not positive definite at the grid angles), steps, V."""
    deg_b = np.array([float(b) * 360.0 / float(K) for b in bins])
    tb = deg_b * DEG2RAD
    delta = (360.0 / float(K)) * DEG2RAD
    lo, hi = tb - delta, tb + delta
    th = tb.copy()
    A, D = steer(pos, lam, th)
    V = criterion(F, A) if F is not None else None
    info = {"moved": V is not None, "steps": 0, "V": V, "stop": "start"}
    if V is None:
        return th, info
    for it in range(MAX_STEPS):
        g, H = grad_hess(F, A, D)
        if not hess_ok(H):
            info["stop"] = "hessian"
            break
        s = -np.linalg.solve(H, g)
        if not np.max(np.abs(s)) > STEP_TOL:
            info["stop"] = "step"
            break
        accepted = False
        for _ in range(MAX_HALVINGS + 1):
            trial = np.minimum(np.maximum(th + s, lo), hi)
            At, Dt = steer(pos, lam, trial)
            Vt = criterion(F, At)
            if Vt is not None and Vt < V:
                accepted = True
                break
            s = 0.5 * s
        if not accepted:
            info["stop"] = "line search"
            break
        th, A, D, V = trial, At, Dt, Vt
        info["steps"] = it + 1
    else:
        info["stop"] = "steps"
    info["V"] = V
    return th, info


def ls_levels(R, A):
    """DML's least-squares powers p = diag(A+ (R - s2 I) A+^H), s2 = Re tr(P_perp R) / (M - d)"""
    M, d = A.shape
    G = A.conj().T @ A
    Ap = np.linalg.solve(G, A.conj().T)
    P = np.eye(M) - A @ Ap
    s2 = float(np.trace(P @ R).real) / float(M - d)
    return np.real(np.diag(Ap @ (R - s2 * np.eye(M)) @ Ap.conj().T)), s2


def wrap_deg(t):
    """float32 degrees in [0, 360) of t radians, 360 -> 0 as under NEWTON"""
    a = math.fmod(t * RAD2DEG, 360.0)
    if a < 0.0:
        a += 360.0
    f = np.float32(a)
    return np.float32(0.0) if f >= np.float32(360.0) or f == 0.0 else f


def refine_window(F, R, out, K, pos, lam):
    """JOINT with the factor F (wsf_factor, or dml_factor(R) under DML) on one window's peak-stage outputs `out`
    (angles, levels, bins of n slots): a new dict with the refined angles and levels, theta (radians, filled slot
    order) and the JOINT info"""
    res = {k: np.array(out[k]) for k in ("angles", "levels", "bins")}
    S = [i for i in range(len(res["bins"])) if res["bins"][i] >= 0]
    res["theta"], res["info"] = None, None
    if not S:
        return res
    bins = [int(res["bins"][i]) for i in S]
    th, info = joint(F, bins, K, pos, lam)
    res["theta"], res["info"] = th, info
    if not info["moved"]:
        return res
    A, _ = steer(pos, lam, th)
    p, _ = ls_levels(np.asarray(R, np.complex128), A)
    for k, i in enumerate(S):
        deg_b = float(bins[k]) * 360.0 / float(K)
        res["angles"][i] = np.float32(deg_b) if th[k] == deg_b * DEG2RAD else wrap_deg(th[k])
        res["levels"][i] = np.float32(p[k])
    return res


# ---- one window from its samples ---------------------------------------------------------------------------------------
def window_R(R, table_c64, n, d=None, mode="wsf", pos=None, lam=None, joint_on=False):
    """One window from its covariance R under mode "wsf" or "dml", then JOINT when joint_on (pos, lam: the geometry)"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    out = wsf_R(R, table_c64, n, d) if mode == "wsf" else dm.work_R(R, table_c64, n, d)
    K = np.asarray(table_c64).reshape(-1, M).shape[0]
    F = out.get("F") if mode == "wsf" else dml_factor(R)
    if joint_on and out["slots"]:
        out.update(refine_window(F, R, out, K, pos, lam))
    return out


def work(in_c64, m, n, table_c64, pos=None, lam=None, mode="wsf", joint_on=False, rule=None):
    """One window from its samples: R, the source count (MDL / AIC, or n), the peak mode and JOINT"""
    x = np.ascontiguousarray(in_c64, dtype=np.complex64)
    R = mo.covariance(x, m)
    d = n
    if rule is not None:
        d = so.estimate_source_count(np.linalg.eigvalsh(R), x.shape[0] // m, n, rule)[0]
    out = window_R(R, table_c64, n, d, mode, pos, lam, joint_on)
    out["R"], out["count"] = R, d
    return out
