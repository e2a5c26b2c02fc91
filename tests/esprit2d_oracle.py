"""fp64 restatement of 2-D LS-ESPRIT on az-el handles (MUSIC_B200_PEAKS_ESPRIT on a planar lattice,
include/music_b200.h): the lattice condition, the doublets, Psi_j by Cholesky, the pairing through the eigenvectors of
Psi_c = Psi_1 + gamma Psi_2, the direction, level, bin and slot rules.  LAPACK does the linear algebra (eigh for E_s,
cholesky / solve for Psi_j, eig for the eigenvectors of Psi_c); the kernel's own sequence (Householder with Z, the
whole-row QR, back-substitution) is emulated by tools/emulate_esprit2d_warp.py.  Test infrastructure: the product path
never imports it.

The keyword switches of `psi_pair` plant the defects that tests/test_esprit2d_oracle.py shows the checker failing."""
import math

import numpy as np

import azel_oracle as ao

GAMMA = complex(0.37, 0.61)
PIVOT = 2.0 ** -40
DEG = math.pi / 180.0


def lattice(pos, lam):
    """(Mx, My, s1, s2) of positions (M, 3) under the lattice condition, or None"""
    pos = np.asarray(pos, np.float64)
    M = pos.shape[0]
    for mx in range(2, M // 2 + 1):
        if M % mx:
            continue
        my = M // mx
        s1, s2 = pos[1, :2] - pos[0, :2], pos[mx, :2] - pos[0, :2]
        a1, a2 = math.hypot(*s1), math.hypot(*s2)
        if not (a1 > 0.0 and a2 > 0.0):
            continue
        if not abs(s1[0] * s2[1] - s1[1] * s2[0]) > 1e-6 * a1 * a2:
            continue
        tol = 1e-6 * min(a1, a2)
        fit = True
        for m in range(M):
            k, i = divmod(m, mx)
            e = pos[0, :2] + i * s1 + k * s2
            fit = fit and math.hypot(*(pos[m, :2] - e)) <= tol and abs(pos[m, 2] - pos[0, 2]) <= tol
        if not fit:
            continue
        if not (a1 <= 0.5 * lam * (1.0 + 1e-12) and a2 <= 0.5 * lam * (1.0 + 1e-12)):
            continue
        return mx, my, s1.copy(), s2.copy()
    return None


def doublets(mx, my):
    """(P1, P2): lists of (first, second) element indices in ascending first index"""
    P1 = [(k * mx + i, k * mx + i + 1) for k in range(my) for i in range(mx - 1)]
    P2 = [(k * mx + i, (k + 1) * mx + i) for k in range(my - 1) for i in range(mx)]
    return P1, P2


def d_max(mx, my):
    return min((mx - 1) * my, mx * (my - 1))


def psi_pair(Es, mx, my, swap=False, no_conj=False):
    """(Psi_1, Psi_2) from the signal eigenvectors Es (M, d), or None where the mode reports no peaks.
    swap: doublets taken (second, first); no_conj: C_j = A_j^T B_j."""
    out = []
    for P in doublets(mx, my):
        f = [a for a, b in P]
        s = [b for a, b in P]
        if swap:
            f, s = s, f
        A, B = Es[f], Es[s]
        G = A.conj().T @ A
        C = (A.T if no_conj else A.conj().T) @ B
        piv = _cholesky_pivots(G)
        if piv is None or np.min(piv) <= PIVOT:
            return None
        Psi = np.linalg.solve(G, C)
        if not np.all(np.isfinite(Psi)):
            return None
        out.append(Psi)
    return out


def _cholesky_pivots(G):
    """the pivots of the Cholesky factorisation of G before their square roots (None at the first non-positive one)"""
    d = G.shape[0]
    A = np.array(G, np.complex128)
    piv = np.empty(d)
    for k in range(d):
        p = A[k, k].real
        if not p > PIVOT:
            piv[k] = p
            return piv[: k + 1]
        piv[k] = p
        l = A[k + 1:, k] / math.sqrt(p)
        A[k + 1:, k + 1:] -= np.outer(l, l.conj())
    return piv


def quotients(P1, P2, gamma=GAMMA):
    """(phi_1, phi_2, eigenvalues of Psi_c): Rayleigh quotients of the eigenvectors of Psi_c = Psi_1 + gamma Psi_2"""
    w, X = np.linalg.eig(P1 + gamma * P2)
    xn = np.sum(np.abs(X) ** 2, axis=0)
    f1 = np.einsum("ak,ab,bk->k", X.conj(), P1, X) / xn
    f2 = np.einsum("ak,ab,bk->k", X.conj(), P2, X) / xn
    return f1, f2, w


def direction(f1, f2, s1, s2, lam, el_hi):
    """(az, el) degrees of one source's phase pair, or None for a phase exactly 0 or not finite"""
    if not (np.isfinite(f1) and np.isfinite(f2)) or f1 == 0 or f2 == 0:
        return None
    w1 = -math.atan2(f1.imag, f1.real) * lam / (2.0 * math.pi)
    w2 = -math.atan2(f2.imag, f2.real) * lam / (2.0 * math.pi)
    det = s1[0] * s2[1] - s1[1] * s2[0]
    ux, uy = (w1 * s2[1] - w2 * s1[1]) / det, (w2 * s1[0] - w1 * s2[0]) / det
    az = math.fmod(math.degrees(math.atan2(uy, ux)), 360.0)
    if az < 0.0:
        az += 360.0
    el = math.degrees(math.acos(min(math.hypot(ux, uy), 1.0)))
    return az, (-el if el_hi <= 0.0 else el)


def bin_of(az, el, grid):
    k = int(math.floor(az * grid.n_az / 360.0 + 0.5)) % grid.n_az
    i = 0
    if grid.n_el > 1:
        i = int(math.floor((el - grid.el_lo) * (grid.n_el - 1) / (grid.el_hi - grid.el_lo) + 0.5))
        i = min(max(i, 0), grid.n_el - 1)
    return i * grid.n_az + k


def work_V(V, d, pos, lam, grid, n, gamma=GAMMA, swap=False, no_conj=False):
    """One window from the eigenvectors V (M, M, ascending eigenvalues, columns) and d: {az, el, levels, bins} (n slots,
    unfilled (0, 0, 0, -1)) and the unsorted fp64 'sources' [(level, az, el)]"""
    pos = np.asarray(pos, np.float64)
    M = V.shape[0]
    az_o, el_o = np.zeros(n, np.float32), np.zeros(n, np.float32)
    lv_o, b_o = np.zeros(n, np.float32), np.full(n, -1, np.int32)
    res = {"az": az_o, "el": el_o, "levels": lv_o, "bins": b_o, "sources": []}
    lat = lattice(pos, lam)
    if lat is None:
        raise ValueError("not a lattice")
    mx, my, s1, s2 = lat
    if d <= 0 or d > d_max(mx, my):
        return res
    Ps = psi_pair(V[:, M - d:], mx, my, swap, no_conj)
    if Ps is None:
        return res
    f1, f2, _ = quotients(Ps[0], Ps[1], gamma)
    G = V[:, : M - d]
    src = []
    for k in range(d):
        dr = direction(f1[k], f2[k], s1, s2, lam, grid.el_hi)
        if dr is None:
            continue
        a = ao.steering(pos, lam, dr[0], dr[1])
        D = float(np.sum(np.abs(G.conj().T @ a) ** 2))
        src.append((1.0 / D, dr[0], dr[1], k))
    if any(math.isnan(s[0]) for s in src):
        return res
    src.sort(key=lambda s: (-s[0], s[1], s[2], s[3]))
    res["sources"] = src
    for r, (lvl, az, el, _) in enumerate(src[:n]):
        fa = np.float32(az)
        az_o[r] = 0.0 if fa >= 360.0 or fa == 0.0 else fa
        el_o[r] = np.float32(el)
        lv_o[r] = np.float32(lvl)
        b_o[r] = bin_of(az, el, grid)
    return res


def work_R(R, d, pos, lam, grid, n, **kw):
    """work_V on the LAPACK eigenvectors of the covariance R"""
    _, V = np.linalg.eigh(np.asarray(R, np.complex128))
    return work_V(V, d, pos, lam, grid, n, **kw)


def noiseless_V(pos, lam, dirs):
    """eigenvectors (ascending, columns) of the noiseless covariance of unit-power uncorrelated sources at dirs"""
    A = np.stack([ao.steering(pos, lam, az, el) for az, el in dirs], axis=1)
    _, V = np.linalg.eigh(A @ A.conj().T)
    return V


def lattice_xyz(mx, my, s1, s2, p0=(0.0, 0.0, 0.0)):
    """positions (mx my, 3) of the lattice p_0 + i s1 + k s2, element k mx + i"""
    return np.array([[p0[0] + i * s1[0] + k * s2[0], p0[1] + i * s1[1] + k * s2[1], p0[2]] for k in range(my) for i in range(mx)],
                    np.float64)


# ---- accuracy model: what the GPU test's RMS thresholds rest on ------------------------------------------------------
RMS_FACTOR = 1.5  # ESPRIT's RMS may be at most this multiple of grid + NEWTON's (numpy model: 0.6)


def _rms(errs):
    return math.sqrt(float(np.mean(np.square(errs))))


def matched_errors(got, truth):
    """great-circle errors of the reported (az, el) pairs against the truth, each true source matched to its nearest
    unused report (a missing report counts as 90 degrees)"""
    errs, used = [], set()
    for t in truth:
        c = [(ao.direction_error(g[0], g[1], t[0], t[1]), j) for j, g in enumerate(got) if j not in used]
        if not c:
            errs.append(90.0)
            continue
        e, j = min(c)
        used.add(j)
        errs.append(e)
    return errs


def rms_model(pos, lam, grid, n, windows_, seed, snaps=512, noise=0.1, el_range=(5.0, 80.0)):
    """RMS direction errors in degrees of ESPRIT, TOP_BINS, LOCAL_MAXIMA and LOCAL_MAXIMA + NEWTON on the same windows
    (n sources of unit power, 20 dB per element at the default noise), all in fp64 numpy"""
    m = pos.shape[0]
    x, truth = ao.windows(pos, lam, [n] * windows_, seed, snaps, el_range=el_range, noise=noise)
    tab = ao.table(pos, lam, grid).reshape(-1, m).astype(np.complex64)
    e = {"esprit": [], "top_bins": [], "local_maxima": [], "newton": []}
    for w in range(windows_):
        from oracle import music_oracle as mo
        R = mo.covariance(np.ascontiguousarray(x[w]), m)
        res = work_R(R, n, pos, lam, grid, n)
        e["esprit"] += matched_errors(list(zip(res["az"], res["el"])), truth[w])
        top = ao.work(x[w], m, n, tab, grid, peak="top")
        e["top_bins"] += matched_errors(list(zip(top["azimuth"], top["elevation"])), truth[w])
        loc = ao.work(x[w], m, n, tab, grid, peak="local")
        e["local_maxima"] += matched_errors(list(zip(loc["azimuth"], loc["elevation"])), truth[w])
        ref = [ao.refine_slot(loc["G"], pos, lam, int(b), grid) for b in loc["bins"] if b >= 0]
        e["newton"] += matched_errors([(r["azimuth"], r["elevation"]) for r in ref], truth[w])
    return {k: _rms(v) for k, v in e.items()}
