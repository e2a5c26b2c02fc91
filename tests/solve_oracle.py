"""High-precision reference for the Cholesky-based solvers (the MVDR preparation and scan: mvdr_prep_kernel +
warp_cholesky + mvdr_form; the MVDR and LCMV beam weights: beam_weights_kernel; the DML searches and levels: dml_kernel),
the bounds a backward-stable solver meets, the decision bands where rounding may legitimately decide an outcome, and
the windows that stress them (not a test module; the same shape as eig_oracle.py and gridless_oracle.py).

Reference: mpmath at eig_oracle.REF_DPS digits on the fp64 covariance R as given (the GPU's own R wherever R is not
exact, so that the covariance's rounding is not charged to the solver) and on the table rows as stored (complex64,
widened).  It restates the definitions of include/music_b200.h, not the kernels' arithmetic: delta, R_L and its
Cholesky factor, D_k = a^H R_L^-1 a, the MVDR weights R_L^-1 a / D, the LCMV weights R_L^-1 A (A^H R_L^-1 A)^-1 and the
exact pivot ratios of G = A^H R_L^-1 A, the DML objective f(k) and the levels p = diag(A^+ (R - s2 I) A^+^H).
||R_L||_2, lambda_min(R_L) (as 1 / ||R_L^-1||_2 from the mp inverse), kappa(G) and kappa(A) are read off fp64
eigenvalues of mp-accurate matrices: they enter the bounds and bands only, where a relative error of M eps is moot.

Bounds (one named constant each; eps = 2^-53):
    MVDR       |D^_k - D_k| / D_k <= C_MVDR M eps kappa_k + C_SCAN M eps,  kappa_k = ||R_L|| a^H R_L^-2 a / a^H R_L^-1 a
               (a backward error E of R_L, ||E|| <= c M eps ||R_L||, moves D_k by a^H R_L^-1 E R_L^-1 a <= ||E|| ||R_L^-1 a||^2
               to first order; the scan's sum of squares adds C_SCAN M eps relative; 1 <= kappa_k <= kappa(R_L))
    weights    ||w^ - w|| <= C_W M eps kappa(R_L) ||w||   (the solve of a backward-stable factor, normalised by D)
    LCMV       ||w^ - w|| <= C_W M eps kappa(R_L) kappa(G) ||w||   (G's own solve multiplies the error by kappa(G))
    residual   |w^_i^H a_j - delta_ij| <= C_RES M eps kappa(R_L) kappa(G) ||w_i|| ||a_j||  (the weight bound through a_j)
    DML f      |f^ - f| <= C_F M eps kappa(A_B) (tr R + f) ||a||^2 / den   (num and den are formed to M eps tr R ||a||^2
               and M eps ||a||^2, P_B to eps kappa(A_B); den / ||a||^2 is the sine^2 of a_k to span(B))
    levels     |p^ - p| <= (C_LVL kappa(T) + C_S2 / (M - d)) M eps tr R ||T^-1||^2,  kappa(T) = kappa(A)
               (MGS2 is backward stable, A + dA = Q T with ||dA|| <= c M eps ||A||, and A^+ = T^-1 Q^H then moves by
               ||A^+||^2 ||dA|| = kappa(T) ||T^-1|| c M eps, so p = diag(A^+ (R - s2 I) A^+^H) moves by
               2 kappa(T) ||T^-1||^2 c M eps ||R||; C = Q^H R Q - s2 I is formed to M eps tr R and s2 = (tr R -
               tr Q^H R Q) / (M - d) cancels to M eps tr R / (M - d), both reaching p through ||row l of T^-1||^2 <=
               ||T^-1||^2 = 1 / sigma_min(A)^2.  Without kappa(T) the bound fails a correct kernel on nearly collinear
               slots: tests/test_solve_oracle.py's near-span rows)
A window, bin or slot whose bound exceeds CHECKED (relative) is counted, not compared.

Decision bands (inside a band either outcome is accepted, outside it the reference's is required):
    Cholesky of R_L  must succeed where lambda_min(R_L) > t, must fail where an exact zero or NaN pivot occurs (a
                     non-finite R, or an exactly zero diagonal entry of R_L, i.e. a dead element with delta = 0) or
                     where lambda_min(R_L) < -t, with t = C_PD M^2 (M + 1) eps max_i (R_L)_ii.  Derivation (Higham,
                     Accuracy and Stability, Thm 10.7 and 10.3): Cholesky runs to completion if M gamma_{M+1} kappa(H)
                     < 1 for the diagonally scaled H = D^-1/2 R_L D^-1/2, and kappa(H) <= M max_i (R_L)_ii / lambda_min
                     (lambda_max(H) <= tr H = M, lambda_min(H) >= lambda_min / max_i (R_L)_ii); a completed Cholesky
                     is exact for R_L + E with ||E|| <= M gamma_{M+1} max_i (R_L)_ii, so lambda_min >= -t.  C_PD
                     covers the 1 / (1 - (M + 1) eps) of gamma_{M+1}.  A failure must be clean: an all-NaN P64 row,
                     no peaks, zero weights and beams.  A success must give finite outputs.
    LCMV pivot rule  rho_k = g_k / G_kk (exact) against 2^-20; rho_k is sin^2 of y_k to span(y_<k), so an error e_y in
                     the whitened vectors y = L^-1 a moves it by 2 e_y sqrt(rho) + e_y^2, e_y = C_PIV M eps sqrt(kappa(R_L))
                     (the forward substitution on a backward-stable factor), plus C_PIV d eps for G's own rounding.
    DML candidates   den(k) > 2^-30 ||a_k||^2 by subtraction: the ratio is known to C_DEN M eps kappa(A_B).
    DML searches     a kernel's winner is accepted if its reference f is within the sum of the two f bounds of the
                     reference maximum over the certain candidates, and it is itself at least a possible candidate.
"""
import math

import mpmath as mp
import numpy as np

import eig_oracle as eo

EPS = eo.EPS
C_MVDR = 16.0    # backward error of the Cholesky factor and L^-1 by column substitution, through kappa_k
C_SCAN = 8.0     # mvdr_form's sum of M (M + 1) / 2 products and M squares
C_W = 16.0       # MVDR / LCMV weights
C_RES = 16.0     # LCMV constraint residual
C_PD = 1.01      # Cholesky band: t = C_PD M^2 (M + 1) eps max_i (R_L)_ii (Higham Thm 10.7)
C_PIV = 16.0     # LCMV pivot band
C_F = 16.0       # DML objective
C_DEN = 16.0     # DML candidate band
C_LVL = 16.0     # DML levels: the products Q^H R Q and the back substitution
C_S2 = 8.0       # DML levels: the cancellation in s2
CHECKED = 1e-3   # relative bounds above this are counted, not compared
PIVOT_REL = 2.0 ** -20
DEN_MIN = 2.0 ** -30
F32 = 2.0 ** -24  # the relative rounding of a float32 level


# ---- mp helpers -----------------------------------------------------------------------------------------------------
def _mpc(z):
    z = complex(z)
    return mp.mpc(z.real, z.imag)


def _mat(A):
    A = np.asarray(A, np.complex128)
    return mp.matrix([[_mpc(A[i, j]) for j in range(A.shape[1])] for i in range(A.shape[0])])


def _vec(a):
    return [_mpc(x) for x in np.asarray(a, np.complex128)]


def _np(A):
    return np.array([[complex(A[i, j]) for j in range(A.cols)] for i in range(A.rows)])


def mp_cholesky(A, tiny):
    """lower L (list of rows) with A = L L^H, or None at the first pivot <= tiny"""
    n = A.rows
    L = [[mp.mpc(0)] * n for _ in range(n)]
    for j in range(n):
        s = mp.re(A[j, j]) - mp.fsum(abs(L[j][q]) ** 2 for q in range(j))
        if not s > tiny:
            return None
        L[j][j] = mp.sqrt(s)
        for i in range(j + 1, n):
            L[i][j] = (A[i, j] - mp.fsum(L[i][q] * mp.conj(L[j][q]) for q in range(j))) / L[j][j]
    return L


def _fwd(L, b):
    y = []
    for k in range(len(b)):
        y.append((b[k] - mp.fsum(L[k][q] * y[q] for q in range(k))) / L[k][k])
    return y


def _bwd(L, y):
    n = len(y)
    z = [mp.mpc(0)] * n
    for k in range(n - 1, -1, -1):
        z[k] = (y[k] - mp.fsum(mp.conj(L[q][k]) * z[q] for q in range(k + 1, n))) / L[k][k]
    return z


def _n2(v):
    return mp.fsum(abs(x) ** 2 for x in v)


def loaded(R, loading):
    """(R_L as an mp matrix, delta): delta = loading tr(R) / M"""
    M = R.shape[0]
    Rm = _mat(R)
    delta = mp.mpf(loading) * mp.fsum(mp.re(Rm[i, i]) for i in range(M)) / M
    for i in range(M):
        Rm[i, i] += delta
    return Rm, delta


def factor(R, loading):
    """dict(L = mp Cholesky factor of R_L or None, norm = ||R_L||_2, lam_min = lambda_min(R_L), delta, zero_pivot)"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    out = {"L": None, "finite": bool(np.all(np.isfinite(R)))}
    if not out["finite"]:
        return dict(out, norm=math.nan, dmax=math.nan, lam_min=math.nan, delta=math.nan, zero_pivot=True)
    with mp.workdps(eo.REF_DPS):
        RL, delta = loaded(R, loading)
        RLf = _np(RL)
        norm = float(np.max(np.abs(np.linalg.eigvalsh(RLf)))) if np.any(RLf) else 0.0
        dmax = float(np.max(np.abs(np.diag(RLf).real)))
        zero = any(RL[i, i] == 0 for i in range(M))
        L = None if zero else mp_cholesky(RL, mp.mpf(10) ** (-(eo.REF_DPS - 10)) * max(norm, 1e-300))
        if L is None:
            lam = min(0.0, float(np.min(np.linalg.eigvalsh(RLf))))
        else:
            Li = [_fwd(L, [mp.mpc(1) if i == c else mp.mpc(0) for i in range(M)]) for c in range(M)]  # columns of L^-1
            Inv = np.array([[complex(mp.fsum(mp.conj(Li[i][q]) * Li[j][q] for q in range(M))) for j in range(M)]
                            for i in range(M)])  # R_L^-1 = L^-H L^-1
            lam = 1.0 / float(np.max(np.linalg.eigvalsh(Inv)))
    return dict(out, L=L, norm=norm, dmax=dmax, lam_min=lam, delta=float(delta), zero_pivot=zero)


def chol_band(fac, M):
    """"succeed", "either" or "fail" for the Cholesky of R_L"""
    if not fac["finite"] or fac["zero_pivot"]:
        return "fail"
    t = C_PD * M * M * (M + 1) * EPS * fac["dmax"]
    if fac["lam_min"] > t:
        return "succeed"
    return "fail" if fac["lam_min"] < -t else "either"


# ---- MVDR -----------------------------------------------------------------------------------------------------------
def mvdr_reference(R, loading, table, ks):
    """dict(fac, band, D = {k: D_k}, kappa = {k: kappa_k}) over the bins ks of the complex64 table"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    fac = factor(R, loading)
    out = {"fac": fac, "band": chol_band(fac, M), "D": {}, "kappa": {}}
    if fac["L"] is None:
        return out
    for k in ks:
        out["D"][k], out["kappa"][k] = mvdr_at(fac, table[k])
    return out


def mvdr_at(fac, a):
    """(D = a^H R_L^-1 a, kappa_k) for one steering vector a and a successful factor(R, loading)"""
    with mp.workdps(eo.REF_DPS):
        y = _fwd(fac["L"], _vec(a))
        D = _n2(y)
        return float(D), float(fac["norm"] * _n2(_bwd(fac["L"], y)) / D) if D > 0 else math.inf


def mvdr_bound(M, kappa):
    return C_MVDR * M * EPS * kappa + C_SCAN * M * EPS


def check_failed_clean(P64, bins, levels, angles):
    """None when a failed window is clean (all-NaN P64, no peaks), else the message"""
    if P64 is not None and not np.all(np.isnan(P64)):
        return "failed window with a non-NaN P64"
    if np.any(bins != -1) or np.any(levels != 0) or np.any(angles != 0):
        return "failed window reports peaks: %s %s %s" % (bins, levels, angles)
    return None


def check_mvdr(ref, P64, bins, levels, angles, M, K):
    """(worst relative error / bound over the compared bins, bins compared, bins skipped, outcome, message or None).
    outcome: "ok" or "failed".  The slots must be the top-n picks of the kernel's own P64 (TOP_BINS), each level the
    float of P64 at its bin, and no evaluated bin's reference P may beat a slot's by more than the two bounds."""
    failed = bool(np.all(np.isnan(P64)))
    band = ref["band"]
    if failed:
        if band == "succeed":
            return math.inf, 0, 0, "failed", "Cholesky failed where lambda_min %.3g > band (||R_L|| %.3g)" % (
                ref["fac"]["lam_min"], ref["fac"]["norm"])
        return 0.0, 0, 0, "failed", check_failed_clean(P64, bins, levels, angles)
    if band == "fail":
        return math.inf, 0, 0, "ok", "Cholesky succeeded on a window that must fail"
    if not np.all(np.isfinite(P64)) or not np.all(P64 > 0):
        return math.inf, 0, 0, "ok", "a successful factorisation gave a non-finite or non-positive P64"
    n = len(bins)
    order = sorted(range(K), key=lambda k: (-P64[k], k))
    if list(bins) != order[:n]:
        return math.inf, 0, 0, "ok", "bins %s are not the top picks %s of P64" % (bins, order[:n])
    for i in range(n):
        if levels[i] != np.float32(P64[bins[i]]) or angles[i] != np.float32(bins[i] * 360.0 / K):
            return math.inf, 0, 0, "ok", "slot %d: level / angle not those of its bin" % i
    worst, c, sk = 0.0, 0, 0
    tol = {}
    for k, D in ref["D"].items():
        b = mvdr_bound(M, ref["kappa"][k])
        if b > CHECKED:
            sk += 1
            continue
        tol[k] = b
        e = abs(1.0 / P64[k] - D) / D / b
        c += 1
        if e > 1.0:
            return e, c, sk, "ok", "bin %d: D off by %.3g of its bound (kappa_k %.3g)" % (k, e, ref["kappa"][k])
        worst = max(worst, e)
    for i, b in enumerate(bins):
        if b not in tol:
            continue
        Pb = 1.0 / ref["D"][b]
        for k in tol:
            if k not in bins[:i + 1] and 1.0 / ref["D"][k] > Pb * (1.0 + tol[b] + tol[k]) * (1.0 + 2.0 * EPS):
                return math.inf, c, sk, "ok", "slot %d at bin %d, the reference's P is larger at bin %d" % (i, b, k)
    return worst, c, sk, "ok", None


def check_levels(ref, spectrum, bins, levels, M):
    """(worst error / bound, slots compared, slots skipped, outcome, message or None) for a handle that reports no P64
    (a channel handle, an az-el handle): each level is float32(1 / D^) at its bin, so it must be within the MVDR bound
    plus one float32 rounding of the reference 1 / D_k, and no evaluated bin's reference P may beat a slot's by more
    than the two bounds plus two float32 roundings"""
    failed = bool(np.all(np.isnan(spectrum)))
    if failed:
        if ref["band"] == "succeed":
            return math.inf, 0, 0, "failed", "Cholesky failed inside the must-succeed band"
        return 0.0, 0, 0, "failed", check_failed_clean(None, bins, levels, levels * 0)
    if ref["band"] == "fail":
        return math.inf, 0, 0, "ok", "Cholesky succeeded on a window that must fail"
    if not np.all(np.isfinite(spectrum)) or np.any(bins < 0):
        return math.inf, 0, 0, "ok", "a successful factorisation gave a non-finite spectrum or an empty slot"
    worst, c, sk = 0.0, 0, 0
    tol = {k: mvdr_bound(M, ref["kappa"][k]) for k in ref["D"]}
    for i, b in enumerate(bins):
        if tol[b] > CHECKED:
            sk += 1
            continue
        P = 1.0 / ref["D"][b]
        e = abs(float(levels[i]) - P) / (P * (tol[b] + 2.0 * F32))
        worst = max(worst, e)
        c += 1
        if e > 1.0:
            return e, c, sk, "ok", "slot %d (bin %d): level %.9g, want %.9g (%.3g of the bound)" % (i, b, levels[i], P, e)
        for k in ref["D"]:
            if k not in bins[:i + 1] and tol[k] <= CHECKED and \
                    1.0 / ref["D"][k] > P * (1.0 + tol[b] + tol[k] + 4.0 * F32):
                return math.inf, c, sk, "ok", "slot %d at bin %d, the reference's P is larger at bin %d" % (i, b, k)
    return worst, c, sk, "ok", None


def strided_bins(K, bins, P64, stride):
    """the bins the mp reference evaluates: every stride-th, the reported slots and the four largest P64"""
    ks = set(range(0, K, stride)) | {int(b) for b in bins if b >= 0}
    if np.all(np.isfinite(P64)):
        ks |= set(int(k) for k in np.argsort(-P64, kind="stable")[:4])
    return sorted(ks)


# ---- beams ----------------------------------------------------------------------------------------------------------
def beams_reference(R, rows, rule, loading):
    """rows: {slot: a (complex128)} of the filled slots.  dict(fac, band, W = {slot: w}, kappa = kappa(R_L),
    kappa_G, rho = the exact pivot ratios g_k / G_kk (LCMV), pivot_band)"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    fac = factor(R, loading)
    out = {"fac": fac, "band": chol_band(fac, M), "W": {}, "kappa": math.inf, "kappa_G": 1.0, "rho": [],
           "pivot_band": "succeed"}
    if fac["L"] is None or not rows:
        return out
    S = sorted(rows)
    lam = fac["lam_min"]
    out["kappa"] = fac["norm"] / lam if lam > 0 else math.inf
    with mp.workdps(eo.REF_DPS):
        Y = {i: _fwd(fac["L"], _vec(rows[i])) for i in S}
        Z = {i: _bwd(fac["L"], Y[i]) for i in S}
        if rule == "mvdr" or len(S) == 1:
            for i in S:
                D = _n2(Y[i])
                out["W"][i] = np.array([complex(z / D) for z in Z[i]])
            if rule == "mvdr":
                return out
        d = len(S)
        G = mp.matrix(d, d)
        for r in range(d):
            for c in range(d):
                G[r, c] = mp.fsum(mp.conj(Y[S[r]][m]) * Y[S[c]][m] for m in range(M))
        C = mp_cholesky(G, mp.mpf(0))
        # the exact pivots: g_k = G_kk - sum |C_kq|^2 before the square root
        rho = []
        for k in range(d):
            if C is None:
                Gk = G[:k + 1, :k + 1]
                rho.append(float(1.0 / mp.re(mp.inverse(Gk)[k, k]) / mp.re(G[k, k])) if k else 1.0)
            else:
                rho.append(float(C[k][k] ** 2 / mp.re(G[k, k])))
        out["rho"] = rho
        Gf = _np(G)
        ev = np.linalg.eigvalsh(Gf)
        out["kappa_G"] = float(ev[-1] / ev[0]) if ev[0] > 0 else math.inf
        ey = C_PIV * M * EPS * math.sqrt(out["kappa"])
        band = "succeed"
        for r in rho[1:]:
            slack = 2.0 * ey * math.sqrt(max(r, 0.0)) + ey * ey + C_PIV * d * EPS
            if r < PIVOT_REL - slack:
                band = "fail"
                break
            if r <= PIVOT_REL + slack:
                band = "either"
        out["pivot_band"] = band
        if C is None or band == "fail":
            return out
        Gi = mp.inverse(G)
        for r, i in enumerate(S):
            out["W"][i] = np.array([complex(mp.fsum(Z[S[q]][m] * Gi[q, r] for q in range(d))) for m in range(M)])
    return out


def check_weights(ref, wts, rows, rule, M):
    """(worst error / bound over the compared slots, compared, skipped, outcome, message or None); wts [n][M]"""
    zero = not np.any(wts)
    chol, piv = ref["band"], ref["pivot_band"] if rule == "lcmv" else "succeed"
    if zero:
        if rows and chol == "succeed" and piv == "succeed":
            return math.inf, 0, 0, "failed", "zero weights on a window that must succeed (pivot ratios %s)" % ref["rho"]
        return 0.0, 0, 0, "failed", None
    if chol == "fail" or piv == "fail":
        return math.inf, 0, 0, "ok", "weights on a window that must fail (%s, %s, rho %s)" % (chol, piv, ref["rho"])
    if not np.all(np.isfinite(wts)):
        return math.inf, 0, 0, "ok", "non-finite weights"
    for i in range(len(wts)):
        if (i in rows) != bool(np.any(wts[i])):
            return math.inf, 0, 0, "ok", "slot %d: weights %s, filled %s" % (i, np.any(wts[i]), i in rows)
    kap = ref["kappa"] * (ref["kappa_G"] if rule == "lcmv" else 1.0)
    bw = C_W * M * EPS * kap
    br = C_RES * M * EPS * kap
    if bw > CHECKED or not ref["W"]:
        return 0.0, 0, len(rows), "ok", None
    worst, c = 0.0, 0
    for i in sorted(rows):
        w = ref["W"][i]
        e = np.linalg.norm(wts[i] - w) / (bw * np.linalg.norm(w))
        worst = max(worst, e)
        c += 1
        if e > 1.0:
            return e, c, 0, "ok", "slot %d: weights off by %.3g of the bound (kappa %.3g)" % (i, e, kap)
        for j in sorted(rows):
            if rule == "mvdr" and j != i:
                continue
            res = abs(np.vdot(wts[i], rows[j]) - (1.0 if i == j else 0.0))
            e = res / (br * np.linalg.norm(wts[i]) * np.linalg.norm(rows[j]))
            worst = max(worst, e)
            if e > 1.0:
                return e, c, 0, "ok", "slot %d: constraint residual on slot %d %.3g, %.3g of its bound" % (i, j, res, e)
    return worst, c, 0, "ok", None


# ---- DML ------------------------------------------------------------------------------------------------------------
def _gram(A):
    """mp: the Gram matrix A^H A of the columns A (list of mp vectors)"""
    r = len(A)
    G = mp.matrix(r, r)
    for i in range(r):
        for j in range(r):
            G[i, j] = mp.fsum(mp.conj(A[i][m]) * A[j][m] for m in range(len(A[0])))
    return G


def dml_f(Rm, table, B, ks):
    """mp f(k) and den(k) / ||a_k||^2 for the bins ks given the held rows B"""
    M = Rm.rows
    A = [_vec(table[b]) for b in B]
    Gi = mp.inverse(_gram(A)) if A else None
    out = {}
    for k in ks:
        a = _vec(table[k])
        na = _n2(a)
        if A:
            c = [mp.fsum(mp.conj(A[i][m]) * a[m] for m in range(M)) for i in range(len(A))]
            coef = [mp.fsum(Gi[i, j] * c[j] for j in range(len(A))) for i in range(len(A))]
            pa = [a[m] - mp.fsum(A[i][m] * coef[i] for i in range(len(A))) for m in range(M)]
        else:
            pa = a
        den = _n2(pa)
        num = mp.re(mp.fsum(mp.conj(pa[i]) * Rm[i, j] * pa[j] for i in range(M) for j in range(M)))
        out[k] = (float(num / den) if den > 0 else math.inf, float(den / na) if na > 0 else 0.0, float(na))
    return out


def _cond(table, B):
    if not B:
        return 1.0
    s = np.linalg.svd(np.asarray(table, np.complex128)[list(B)].T, compute_uv=False)
    return float(s[0] / s[-1]) if s[-1] > 0 else math.inf


def f_bound(M, kapB, trR, f, den_ratio):
    return C_F * M * EPS * kapB * (trR + abs(f)) / max(den_ratio, 1e-300)


def check_search(R, table, B, won):
    """(compared?, message or None) for one search S(B) whose kernel winner is `won`, with the mp f(k) of every bin"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    ks = range(len(table))
    trR = float(np.trace(R).real)
    kapB = _cond(table, B)
    with mp.workdps(eo.REF_DPS):
        ref = dml_f(_mat(R), table, B, ks)
    sl = C_DEN * M * EPS * kapB
    certain = {k: v for k, v in ref.items() if v[1] > DEN_MIN + sl}
    fw, rw, _ = ref[won]
    bw = f_bound(M, kapB, trR, fw, rw)
    if not certain or bw > CHECKED * max(abs(fw), 1e-300):
        return False, None
    if rw < DEN_MIN - sl:
        return True, "winner %d is not a candidate (den / ||a||^2 = %.3g)" % (won, rw)
    for k, (fk, rk, _) in certain.items():
        if fk > fw + bw + f_bound(M, kapB, trR, fk, rk):
            return True, "winner %d (f %.17g) loses to bin %d (f %.17g)" % (won, fw, k, fk)
    return True, None


def levels_reference(R, table, slots):
    """mp (p [d] in slot order, s2, ||T^-1||^2 = 1 / sigma_min(A)^2, kappa(A))"""
    R = np.asarray(R, np.complex128)
    M, d = R.shape[0], len(slots)
    with mp.workdps(eo.REF_DPS):
        Rm = _mat(R)
        A = [_vec(table[b]) for b in slots]
        Gi = mp.inverse(_gram(A))
        # A^+ = G^-1 A^H, rows l; P_A R trace via A^+
        Ap = [[mp.fsum(Gi[l, j] * mp.conj(A[j][m]) for j in range(d)) for m in range(M)] for l in range(d)]
        RA = [[mp.fsum(Rm[i, m] * A[l][m] for m in range(M)) for i in range(M)] for l in range(d)]  # R a_l
        trR = mp.fsum(mp.re(Rm[i, i]) for i in range(M))
        trC = mp.re(mp.fsum(Ap[l][i] * RA[l][i] for l in range(d) for i in range(M)))  # tr(A A^+ R) = tr(A^+ R A)
        s2 = (trR - trC) / (M - d)
        p = []
        for l in range(d):
            v = mp.fsum(Ap[l][i] * Rm[i, j] * mp.conj(Ap[l][j]) for i in range(M) for j in range(M))
            p.append(float(mp.re(v) - s2 * _n2(Ap[l])))
    s = np.linalg.svd(np.asarray(table, np.complex128)[list(slots)].T, compute_uv=False)
    if not s[-1] > 0:
        return np.array(p), float(s2), math.inf, math.inf
    return np.array(p), float(s2), float(1.0 / s[-1] ** 2), float(s[0] / s[-1])


# ---- how much of each family must be compared ----------------------------------------------------------------------
FLOOR = {"high snr": 0.3}  # per family (MVDR spectrum and beam weights), else half
# high snr: three of its five windows (120 dB, 160 dB, noiseless) have kappa(R_L) ~ 1e12 .. 1e16, so kappa_k puts most
# of their bins above CHECKED; the 40 and 80 dB windows and the bins away from the sources are compared (0.38 .. 0.49)


def level_bound(M, d, trR, tinv2, kapA):
    return (C_LVL * kapA + C_S2 / (M - d)) * M * EPS * trR * tinv2


# ---- windows --------------------------------------------------------------------------------------------------------
def sources(M, vectors, rng, N, snr_db=None):
    """x [N][M] complex64: independent unit complex Gaussian sources along `vectors`, plus noise at snr_db below them
    (None: noiseless)"""
    X = np.zeros((N, M), np.complex128)
    for v in vectors:
        X += np.outer(rng.standard_normal(N) + 1j * rng.standard_normal(N), np.asarray(v, np.complex128)) / math.sqrt(2.0)
    if snr_db is not None:
        X += 10.0 ** (-snr_db / 20.0) * (rng.standard_normal((N, M)) + 1j * rng.standard_normal((N, M))) / math.sqrt(2.0)
    return X.astype(np.complex64)


N = 64  # snapshots per window (the N = M + 1 family and the exact windows aside)
EXACT_N = eo.EXACT_N
LOADINGS = (0.0, 2.0 ** -40, 2.0 ** -20, 0.01)
EXACT_LOADINGS = (2.0 ** -10, 2.0 ** -20, 2.0 ** -30, 2.0 ** -40)


def mvdr_families(M, table, seed):
    """[(family, name, x [N'][M], loadings)]: the exact rank-deficient windows at their own loadings, the others at
    LOADINGS (a dead element and the high-SNR rows also at loading 0 only where the family says so)"""
    rng = np.random.default_rng(seed)
    K = len(table)
    out = []
    # exact: R = (1/N) sum S_k h_k h_k^H with half the S_k zero: kappa(R_L) = (lambda_max + delta) / delta
    L = 2 ** 36
    r = max(1, M // 2)
    x, _, _ = eo.exact_window(M, [0] * (M - r) + [L + 4096 * k for k in range(r)], rng)
    out.append(("exact", "rank %d" % r, x, EXACT_LOADINGS))
    x, _, _ = eo.exact_window(M, [0] * (M - 1) + [L], rng)
    out.append(("exact", "rank 1", x, EXACT_LOADINGS))
    d = min(2, M - 1)
    vecs = lambda: [table[k] for k in rng.choice(K, d, replace=False)]
    for snr in (40, 80, 120, 160):
        out.append(("high snr", "%d dB" % snr, sources(M, vecs(), rng, N, snr), (0.0,)))
    out.append(("high snr", "noiseless d=%d" % d, sources(M, vecs(), rng, N), (0.0,)))
    out.append(("N = M + 1", "20 dB", sources(M, vecs(), rng, M + 1, 20.0), LOADINGS))
    x = sources(M, vecs(), rng, N, 20.0)
    x[:, int(rng.integers(M))] = 0
    out.append(("dead element", "20 dB", x, LOADINGS))
    out.append(("benign", "20 dB", sources(M, vecs(), rng, N, 20.0), LOADINGS))
    return out


def exact_kappa(x, loading):
    """kappa(R_L) of an exact window in closed form: its R is diagonal in an exactly orthogonal basis"""
    X = x.astype(np.complex128)
    R = X.T @ X.conj() / X.shape[0]
    lam = np.linalg.eigvalsh(R)
    M = R.shape[0]
    delta = loading * float(np.trace(R).real) / M
    return (lam[-1] + delta) / delta


def lcmv_table(K2, geometric_pos):
    """(table [2 K2][M], thetas, eps): rows 2j, 2j + 1 = a(theta_j), a(theta_j + eps_j) with eps_j from 2^-4 to 2^-22
    radians' worth of angle: the exact pivot ratio of the pair sweeps ~2^-8 .. 2^-32, across LCMV's 2^-20"""
    th = np.arange(K2) * 360.0 / K2 + 7.0
    epsd = np.degrees(2.0 ** -np.linspace(4, 22, K2))
    t = np.empty(2 * K2)
    t[0::2], t[1::2] = th, th + epsd
    return np.exp(-2j * np.pi * (np.outer(np.cos(np.radians(t)), geometric_pos[:, 0]) +
                                 np.outer(np.sin(np.radians(t)), geometric_pos[:, 1]))).astype(np.complex64), th, epsd


def dml_families(M, table, seed):
    """[(family, name, x [N][M], table)] of the DML rows (d = 2): coherent and uncorrelated pairs of adjacent table rows
    at 20, 60 and 100 dB, and sources along rows 0 and 1 of near_span_table at 40 and 100 dB"""
    rng = np.random.default_rng(seed)
    K = len(table)
    out = []
    for snr in (20, 60, 100):
        k = int(rng.integers(K))
        vecs = [table[k], table[(k + 1) % K]]
        out.append(("close pair", "uncorrelated %d dB" % snr, sources(M, vecs, rng, N, snr), table))
        s = rng.standard_normal(N) + 1j * rng.standard_normal(N)
        X = np.outer(s, vecs[0].astype(np.complex128) + np.exp(1j * rng.uniform(0, 6.3)) * vecs[1]) / math.sqrt(2)
        X += 10.0 ** (-snr / 20) * (rng.standard_normal((N, M)) + 1j * rng.standard_normal((N, M)))
        out.append(("close pair", "coherent %d dB" % snr, X.astype(np.complex64), table))
    nt = near_span_table(M, K, seed)
    for snr in (40, 100):
        out.append(("near span", "%d dB" % snr, sources(M, [nt[0], 3.0 * nt[1]], rng, N, snr), nt))
    return out


def near_span_table(M, K, seed):
    """DML rows nearly in the span of a held slot: [K][M] with row 0 = a, row 1 = b (a second direction), rows 2.. =
    a + eta_j P_a^perp b with den / ||a||^2 from 2^-26 to 2^-34, the rest random directions.  A window with sources
    along a and b makes rows 1 and 2.. tie exactly in f once row 0 is held."""
    rng = np.random.default_rng(seed)
    a = np.exp(2j * np.pi * rng.uniform(size=M))
    b = np.exp(2j * np.pi * rng.uniform(size=M))
    u = b - a * np.vdot(a, b) / np.vdot(a, a)
    rows = [a, b]
    for e in np.linspace(-13, -17, 9):
        rows.append(a + 2.0 ** e * u * math.sqrt(M) / np.linalg.norm(u))
    while len(rows) < K:
        rows.append(np.exp(2j * np.pi * rng.uniform(size=M)))
    return np.array(rows).astype(np.complex64)
