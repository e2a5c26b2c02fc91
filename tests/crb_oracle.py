"""numpy restatement of the stochastic CRB of include/music_b200.h (music_b200_process_*_crb, music_crb.cuh), step by
step as the header defines it, plus the textbook Slepian-Bangs Fisher matrix it must equal at the model covariance and
the small array-processing helpers the statistical tests use.

Everything is fp64.  Angles are taken as the float32 values the device reports, widened to fp64."""
import numpy as np

T_REL = 2.0 ** -30
PIVOT_REL = 2.0 ** -40
B_REL = 2.0 ** -40
RAD2DEG = 180.0 / np.pi


# ---- steering vectors and their derivatives (the refinement's conventions) ---------------------------------------------
def steer_1d(pos_xy, lam, theta_rad):
    """a (M,) and d = da/dtheta (M,) of a planar array at the angle theta (radians): a_m = exp(-j phi_m),
    phi_m = 2 pi (x cos t + y sin t) / lam, psi_m = dphi_m / dt, d = -j psi a"""
    pos = np.asarray(pos_xy, np.float64)
    st, ct = np.sin(theta_rad), np.cos(theta_rad)
    phi = 2.0 * np.pi * ((pos[:, 1] * st + pos[:, 0] * ct) / lam)
    psi = 2.0 * np.pi * ((pos[:, 1] * ct - pos[:, 0] * st) / lam)
    a = np.exp(-1j * phi)
    return a, -1j * psi * a


def steer_azel(pos_xyz, lam, az_rad, el_rad):
    """a (M,), da/daz and da/del of a 3-D array at (az, el) in radians: a_m = exp(-j theta_m),
    theta_m = 2 pi <p_m, u> / lam, u = (cos el cos az, cos el sin az, sin el)"""
    pos = np.asarray(pos_xyz, np.float64)
    x, y, z = pos[:, 0], pos[:, 1], pos[:, 2]
    sp, cp, se, ce = np.sin(az_rad), np.cos(az_rad), np.sin(el_rad), np.cos(el_rad)
    h, v = x * cp + y * sp, y * cp - x * sp
    th = 2.0 * np.pi * ((ce * h + z * se) / lam)
    tp = 2.0 * np.pi * ((ce * v) / lam)
    te = 2.0 * np.pi * ((z * ce - se * h) / lam)
    a = np.exp(-1j * th)
    return a, -1j * tp * a, -1j * te * a


def deriv_scale(pos, lam):
    """G = (2 pi / lam)^2 sum_m |p_m - centroid|^2, the largest |P_perp d|^2 of any direction (1-D or az-el)"""
    pos = np.asarray(pos, np.float64)
    return float(np.sum((pos - pos.mean(axis=0)) ** 2) * (2.0 * np.pi / lam) ** 2)


# ---- the literal definition ------------------------------------------------------------------------------------------------
def _mgs2(A):
    M, d = A.shape
    Q = np.zeros((M, d), complex)
    T = np.zeros((d, d), complex)
    for l in range(d):
        v = A[:, l].copy()
        for _ in range(2):
            for j in range(l):
                c = np.vdot(Q[:, j], v)
                v = v - c * Q[:, j]
                T[j, l] += c
        nrm = np.sqrt(np.real(np.vdot(v, v)))
        Q[:, l] = v / nrm
        T[l, l] = nrm
    return Q, T


def _cholesky(A, ok):
    """lower L with A = L L^H; ok(k, pivot) tests each pivot before its square root.  Returns (L or None, pivots)."""
    A = np.array(A, complex)
    n = A.shape[0]
    L = np.zeros_like(A)
    piv = []
    for k in range(n):
        p = np.real(A[k, k] - np.vdot(L[k, :k], L[k, :k]))
        piv.append(p)
        if not ok(k, p):
            return None, piv
        L[k, k] = np.sqrt(p)
        for i in range(k + 1, n):
            L[i, k] = (A[i, k] - np.dot(L[i, :k], np.conj(L[k, :k]))) / L[k, k]
    return L, piv


def crb_window(R, A, D, N, G):
    """The header's steps 1-5 for one window.  R (M, M); A (M, d) steering columns in slot order; D (M, p) derivative
    columns (p = d on a 1-D handle, 2 d on an az-el one: (az_0, el_0, az_1, ...)); N the snapshot count; G the array's
    derivative scale (deriv_scale).  Returns a dict:
    ok, C (p, p) or None, F, margin (the smallest ratio of a checked quantity to its threshold, < 1 where a check fails),
    cond_F."""
    R = np.asarray(R, complex)
    M, d = A.shape
    per = D.shape[1] // d
    out = {"ok": False, "C": None, "F": None, "margin": np.inf, "cond_F": np.inf}
    Q, T = _mgs2(A)
    na = np.sum(np.abs(A) ** 2, axis=0)
    tm = np.abs(np.diag(T)) ** 2 / (T_REL * na)
    out["margin"] = float(np.min(tm))
    if not np.all(tm > 1.0):
        return out
    C = Q.conj().T @ R @ Q
    s2 = (np.real(np.trace(R)) - np.real(np.trace(C))) / (M - d)
    if not (s2 > 0.0 and np.isfinite(s2)):
        out["margin"] = 0.0
        return out
    Ti = np.linalg.inv(np.triu(T))
    H = Ti @ C @ Ti.conj().T
    Gamma = Ti @ Ti.conj().T
    P = H - s2 * Gamma
    L, _ = _cholesky(H, lambda k, p: p > 0.0)
    if L is None:
        out["margin"] = 0.0
        return out
    U = P @ np.linalg.solve(L.conj().T, np.linalg.solve(L, P))
    # B = D^H P_perp D as the Gram matrix of the projected columns (P_perp is an idempotent projector), each projected
    # twice: D^H D - (Q^H D)^H (Q^H D) would cancel where the derivatives lie almost in span(A)
    E = D - Q @ (Q.conj().T @ D)
    E = E - Q @ (Q.conj().T @ E)
    B = E.conj().T @ E
    bm = np.real(np.diag(B)) / (B_REL * G)
    out["margin"] = float(min(out["margin"], np.min(bm)))
    if not np.all(bm > 1.0):
        return out
    idx = np.arange(D.shape[1]) // per
    F = (2.0 * N / s2) * np.real(B * U[idx][:, idx].T)
    out["F"] = F
    Fd = np.diag(F).copy()
    LF, piv = _cholesky(F, lambda k, p: p > PIVOT_REL * Fd[k])
    ratios = [p / (PIVOT_REL * Fd[k]) if Fd[k] > 0 else -np.inf for k, p in enumerate(piv)]
    out["margin"] = float(min(out["margin"], min(ratios)))
    if LF is None:
        return out
    Li = np.linalg.inv(np.real(LF))
    out["C"] = Li.T @ Li
    out["cond_F"] = float(np.linalg.cond(F))
    out["ok"] = True
    return out


def crb_outputs(R, angles, bins, N, pos, lam, elev=None):
    """The device's output for W windows.  R (W, M, M); angles / bins (W, n) (angles as float32); N scalar or (W,);
    pos (M, 2) with elev None, else (M, 3) with elev (W, n).  Returns (out, info): out (W, n) or (W, n, 3) float32
    (unfilled 0, failed NaN) and per window the crb_window dict."""
    W, n = np.asarray(bins).shape
    azel = elev is not None
    N = np.broadcast_to(np.asarray(N, np.float64), (W,))
    out = np.zeros((W, n, 3) if azel else (W, n), np.float32)
    info = []
    for w in range(W):
        S = [i for i in range(n) if bins[w][i] >= 0]
        if not S:
            info.append(None)
            continue
        cols, ders = [], []
        for i in S:
            t = np.float64(np.float32(angles[w][i])) * (np.pi / 180.0)
            if azel:
                e = np.float64(np.float32(elev[w][i])) * (np.pi / 180.0)
                a, da, de = steer_azel(pos, lam, t, e)
                ders += [da, de]
            else:
                a, da = steer_1d(pos, lam, t)
                ders.append(da)
            cols.append(a)
        r = crb_window(R[w], np.stack(cols, 1), np.stack(ders, 1), N[w], deriv_scale(pos, lam))
        info.append(r)
        for k, i in enumerate(S):
            if not r["ok"]:
                out[w, i] = np.nan
            elif azel:
                C = r["C"]
                caa, cee, cae = C[2 * k, 2 * k], C[2 * k + 1, 2 * k + 1], C[2 * k, 2 * k + 1]
                out[w, i] = (np.sqrt(caa) * RAD2DEG, np.sqrt(cee) * RAD2DEG, cae / np.sqrt(caa * cee))
            else:
                out[w, i] = np.sqrt(r["C"][k, k]) * RAD2DEG
    return out, info


# ---- the textbook bound: Slepian-Bangs with every nuisance parameter -------------------------------------------------
def slepian_bangs_crb(A, D, P, s2, N):
    """The stochastic CRB of the p angle parameters at R = A P A^H + s2 I: the full Fisher matrix over (angles, Re / Im of
    the Hermitian P, s2), FIM_kl = N tr(R^-1 R_k R^-1 R_l), reduced by the Schur complement of the nuisance block.
    Returns C (p, p) in radians^2."""
    M, d = A.shape
    p = D.shape[1]
    per = p // d
    R = A @ P @ A.conj().T + s2 * np.eye(M)
    derivs = []
    for c in range(p):
        i = c // per
        E = np.zeros((d, d))
        E[i, i] = 1.0
        Ad = np.zeros_like(A)
        Ad[:, i] = D[:, c]
        derivs.append(Ad @ P @ A.conj().T + A @ P @ Ad.conj().T)
    for i in range(d):
        for j in range(i, d):
            E = np.zeros((d, d), complex)
            if i == j:
                E[i, i] = 1.0
                derivs.append(A @ E @ A.conj().T)
            else:
                E[i, j] = E[j, i] = 1.0
                derivs.append(A @ E @ A.conj().T)
                E = np.zeros((d, d), complex)
                E[i, j], E[j, i] = 1j, -1j
                derivs.append(A @ E @ A.conj().T)
    derivs.append(np.eye(M, dtype=complex))
    Ri = np.linalg.inv(R)
    X = [Ri @ Dk for Dk in derivs]
    K = len(derivs)
    FIM = np.empty((K, K))
    for k in range(K):
        for l in range(K):
            FIM[k, l] = N * np.real(np.trace(X[k] @ X[l]))
    Faa, Fan, Fnn = FIM[:p, :p], FIM[:p, p:], FIM[p:, p:]
    return np.linalg.inv(Faa - Fan @ np.linalg.solve(Fnn, Fan.T))


# ---- helpers of the statistical tests ----------------------------------------------------------------------------------------
def ula_x(M, spacing=0.5):
    """element positions (M, 2) of an x-axis ULA with the given spacing in wavelengths (lam = 1)"""
    return np.stack([np.arange(M) * spacing, np.zeros(M)], 1)


def uca(M, radius):
    k = np.arange(M)
    return np.stack([radius * np.cos(2 * np.pi * k / M), radius * np.sin(2 * np.pi * k / M)], 1)


def sample_windows(rng, A, P, s2, N, W):
    """complex64 snapshots X (W, M, N) of Gaussian sources with covariance P through A in white noise s2"""
    M, d = A.shape
    Lp = np.linalg.cholesky(P + 1e-300 * np.eye(d)) if d else np.zeros((0, 0))
    s = Lp @ (rng.standard_normal((W, d, N)) + 1j * rng.standard_normal((W, d, N))) / np.sqrt(2.0)
    noise = np.sqrt(s2 / 2.0) * (rng.standard_normal((W, M, N)) + 1j * rng.standard_normal((W, M, N)))
    return (A @ s + noise).astype(np.complex64)


def sample_cov(X):
    X = X.astype(np.complex128)
    return X @ np.conj(np.swapaxes(X, -1, -2)) / X.shape[-1]


def root_music_ula(R, d, spacing=0.5):
    """root-MUSIC angles (degrees in [0, 180]) of an x-axis ULA, z = exp(-j 2 pi spacing cos t)"""
    M = R.shape[0]
    _, V = np.linalg.eigh(R)
    G = V[:, : M - d]
    C = G @ G.conj().T
    coef = np.array([np.trace(C, offset=-k) for k in range(M - 1, -M, -1)])  # z^k: sum of C[n + k][n]
    roots = np.roots(coef)
    roots = roots[np.abs(roots) < 1.0]
    roots = roots[np.argsort(np.abs(np.abs(roots) - 1.0))][:d]
    # a_m = exp(-j 2 pi spacing m cos t): the polynomial in z = exp(+j 2 pi spacing cos t)
    return np.degrees(np.arccos(np.clip(np.angle(roots) / (2 * np.pi * spacing), -1, 1)))


def esprit_ula(R, d, spacing=0.5):
    """LS-ESPRIT angles (degrees) of an x-axis ULA"""
    _, V = np.linalg.eigh(R)
    Es = V[:, -d:]
    Psi = np.linalg.lstsq(Es[:-1], Es[1:], rcond=None)[0]
    ev = np.linalg.eigvals(Psi)
    # a_(m+1) / a_m = exp(-j 2 pi spacing cos t)
    return np.degrees(np.arccos(np.clip(-np.angle(ev) / (2 * np.pi * spacing), -1, 1)))
