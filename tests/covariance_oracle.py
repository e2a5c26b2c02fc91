"""Exact references and per-entry bounds for the covariance R = x x^H / N of every covariance kernel, and for the
integrated covariance Rbar_j = S_j / c_j of music_integrate.cuh.  eps = 2^-53 throughout.

Raw R.  A float32 is an integer times a power of two, so with one power of two per element (the finest ulp of that
element in the window) every product x_i(t) conj(x_j(t)) and every sum over snapshots is an integer at the common scale
2^(s_i + s_j).  `exact_sums` splits those integers into 12-bit digits, so every digit product is below 2^24 and every
digit Gram matrix (N <= 2^16 snapshots, two parts) below 2^41: float64 matrix products of the digits are exact whatever
their order, and Python ints put the digits back together.  R = S / N is then an exact rational.

Raw R bound, per entry and separately for the real and imaginary parts:
    |R^_ij - R_ij| <= eps |R_ij| + C_COV L_k eps A_ij,   A_ij = sum_t |x_i(t)| |x_j(t)| / N  (that part's two products)
(Higham, Accuracy and Stability, eq. 4.4: a sum computed with at most L roundings on any term's path is in error by at
most gamma_L = L eps / (1 - L eps) times the sum of the terms' magnitudes; the products of widened float32 values are
exact in fp64, and the final / N adds eps |R|).  L_k is the longest path of roundings of kernel k:
    kernel                                  per-lane snapshots      rounds per snapshot   reduction          L_k
    cov_tile_kernel<false / true>           ceil(N / 32)            2 (nested fma)        warp_sum, 5        2 ceil(N/32) + 5
    cov4_tma_kernel                         ceil(N / 32)            2                     warp_sum, 5        2 ceil(N/32) + 5
    covN_tma_kernel<8>, <16>                ceil(N / 32)            2                     butterfly, 5       2 ceil(N/32) + 5
    cov_planar_kernel<false / true>         ceil(N / 32)            2                     warp_sum, 5        2 ceil(N/32) + 5
    cov_generic_kernel (S = 256 / E slices) ceil(N / S)             2                     S - 1 serial adds  2 ceil(N/S) + S - 1
Every warp kernel takes snapshot t in lane t mod 32, in increasing t, and the transposing butterfly of covN_tma_kernel adds
the same pairs (lanes differing in bit 4, then 3, ... 0) as warp_sum, so all warp kernels compute the same bits;
`emulate_R` restates both summation orders in numpy (fma(a, b, c) of widened float32 a, b is a*b + c exactly, since a*b
is exact).  C_COV = 1.01 covers gamma_L / (L eps) and the (1 + eps) of the division at every L used here.

Integration.  `integrate_exact` runs S_j = alpha S_{j-1} + R_j, c_j, q_j and N_eff,j on the device's raw R_j at 60
decimal digits.  The device runs the recurrence as a three-kernel scan per sub-batch (music_integrate.cuh); every
rounding on the path of a term R_k into S_j multiplies something no larger than sum_k alpha^(j-k) |R_k| = c_j Abar_j, so
    |Rbar^_j - Rbar_j| <= eps |Rbar_j| + C_INT eps (L_int(W_b) Abar_j + carry_j / c_j)
with L_int the rounding depth inside one sub-batch of W_b windows (`integ_depth`, derived next to it) and eps carry_j
the bound on the error of the carry S that the sub-batch started from, propagated by alpha^(windows since) (E and carry
are counted in units of eps, which the bound applies once):
    E_b = alpha^(W_b) E_{b-1} + L_int(W_b) c_end Abar_end,   carry_j = alpha^(j - start_b + 1) E_{b-1}.
C_INT = 1.01, as C_COV.  N_eff,j's relative error is at most C_NEFF eps."""
import decimal
import math
from fractions import Fraction

import numpy as np

EPS = 2.0 ** -53
C_COV = 1.01
C_INT = 1.01
C_POW = 8       # relative error of integ_one_minus_pow / (1 - alpha), in eps: log1p or log (2), the product (1), expm1 (2),
                # the division and 1 - alpha (2), and the sensitivity of -expm1(y) to y, |y e^y / (1 - e^y)| <= 1
C_NEFF = 40     # N_eff = N c^2 / q: 2 C_POW through c^2, C_POW + 4 through q, 3 products and quotients, rounded up
INTEG_T = 32
INTEG_SCAN_THREADS = 256
DIGIT = 12
DPS = 60


# ---- which kernels a call runs (launch_cov and launch_cov_planar in music_b200.cu) ----
def cov_kernels(m, N, planar=False):
    """the covariance kernels one sub-batch launches, in order"""
    if planar:
        return ["cov_planar_kernel<false>"] + (["cov_planar_kernel<true>"] if m > 4 else [])
    if m == 4:
        return ["cov4_tma_kernel"]
    if m in (8, 16) and N >= 128 and N % (16 // m) == 0:
        return ["covN_tma_kernel<%d>" % m]
    if m % 4 == 0:
        return ["cov_tile_kernel<false>", "cov_tile_kernel<true>"]
    return ["cov_generic_kernel"]


def generic_slices(m):
    return 256 // (m * (m + 1) // 2)


def depth(kernel, m, N):
    """L_k, the longest path of roundings of one entry's sum in `kernel` (the table above)"""
    if kernel == "cov_generic_kernel":
        S = generic_slices(m)
        return 2 * -(-N // S) + S - 1
    return 2 * -(-N // 32) + 5


# ---- exact sums ----
def _columns(X):
    """per element (column of the complex64 window X [N][m]): its scale exponent s_i and its real and imaginary parts as
    integers times 2^s_i (float64 arrays, exact), with the number of bits they need"""
    re = X.real.astype(np.float64)
    im = X.imag.astype(np.float64)
    s, bits = [], 0
    for i in range(X.shape[1]):
        v = np.concatenate([re[:, i], im[:, i]])
        v = v[v != 0]
        if len(v) == 0:
            s.append(0)
            continue
        _, e = np.frexp(v)
        s.append(int(e.min()) - 24)  # every float32 is an integer multiple of 2^(its exponent - 24)
        bits = max(bits, int(e.max()) - s[-1])
    sc = np.ldexp(1.0, -np.array(s))
    return np.array(s), re * sc, im * sc, bits


def _digits(Z, D):
    """signed base-2^12 digits of the integer-valued float64 array Z [N][m] -> [N][m][D], least significant first"""
    a = np.abs(Z)
    out = np.empty(Z.shape + (D,))
    for d in range(D):
        q = np.floor(a / 2.0 ** DIGIT)
        out[..., d] = a - q * 2.0 ** DIGIT
        a = q
    assert not np.any(a), "more digits than planned"
    return out * np.sign(Z)[..., None]


def exact_sums(X):
    """S = sum_t x(t) x(t)^H of one window X (complex64 [N][m]) exactly: (Sre, Sim) [m][m] Python ints and the exponent
    matrix s_i + s_j, S_ij = (Sre_ij + i Sim_ij) 2^(s_i + s_j)"""
    N, m = X.shape
    assert N <= 1 << 16
    s, zr, zi, bits = _columns(X)
    D = max(1, -(-bits // DIGIT))
    dr = _digits(zr, D).reshape(N, m * D)
    di = _digits(zi, D).reshape(N, m * D)
    Grr, Gii, Gir, Gri = (np.rint(a.T @ b).astype(object) for a, b in ((dr, dr), (di, di), (di, dr), (dr, di)))
    w = [1 << (DIGIT * k) for k in range(2 * D - 1)]
    Sre = [[0] * m for _ in range(m)]
    Sim = [[0] * m for _ in range(m)]
    for i in range(m):
        for j in range(m):
            a = b = 0
            for p in range(D):
                for q in range(D):
                    u, v = i * D + p, j * D + q
                    a += int(Grr[u, v] + Gii[u, v]) * w[p + q]
                    b += int(Gir[u, v] - Gri[u, v]) * w[p + q]
            Sre[i][j], Sim[i][j] = a, b
    return Sre, Sim, s[:, None] + s[None, :]


def _frac(n, e, N):
    return Fraction(n * (1 << e), N) if e >= 0 else Fraction(n, N << -e)


def exact_R(X):
    """R = S / N of one window X (complex64 [N][m]) as two [m][m] object arrays of Fractions"""
    N, m = X.shape
    Sre, Sim, e = exact_sums(X)
    re = np.empty((m, m), object)
    im = np.empty((m, m), object)
    for i in range(m):
        for j in range(m):
            re[i, j] = _frac(Sre[i][j], int(e[i, j]), N)
            im[i, j] = _frac(Sim[i][j], int(e[i, j]), N)
    return re, im


def rounded(F):
    """the correctly rounded fp64 values of a Fraction array"""
    return np.vectorize(float, otypes=[np.float64])(F)


def abs_sums(X):
    """A = sum_t |x_i(t)| |x_j(t)| / N per part: (A_re, A_im) [m][m] (fp64; its own rounding, ~N eps relative, is far
    inside C_COV's slack)"""
    ar, ai = np.abs(X.real.astype(np.float64)), np.abs(X.imag.astype(np.float64))
    N = X.shape[0]
    return (ar.T @ ar + ai.T @ ai) / N, (ai.T @ ar + ar.T @ ai) / N


def raw_ratios(R_hat, X, L):
    """per part the worst |R^ - R| / (eps |R| + C_COV L eps A) of one window (R_hat complex128 [m][m]); an entry whose
    bound is 0 (all its terms 0) must be exact and counts as ratio 0 or inf"""
    re, im = exact_R(X)
    Are, Aim = abs_sums(X)
    worst = 0.0
    for F, got, A in ((re, R_hat.real, Are), (im, R_hat.imag, Aim)):
        err = np.vectorize(lambda f, g: float(abs(Fraction(g) - f)) if math.isfinite(g) else math.inf,
                           otypes=[np.float64])(F, got)
        bound = EPS * np.abs(rounded(F)) + C_COV * L * EPS * A
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
        worst = max(worst, float(np.max(r)))
    return worst


# ---- the summation orders, restated ----
def _fma_step(acc, ar, ai, br, bi):
    """fma(ar, br, fma(ai, bi, acc)) and fma(ai, br, fma(-ar, bi, acc)) of widened float32 values: the products are exact
    in fp64, so each fma is one rounded addition"""
    return ar * br + (ai * bi + acc[0]), ai * br + (-ar * bi + acc[1])


def emulate_R(X, kernel="warp", defect=None):
    """R of one window X (complex64 [N][m]) in the summation order of a warp kernel ("warp": lane t mod 32, increasing t,
    then the 5-level pairwise tree) or of cov_generic_kernel ("generic"), upper triangle mirrored.  `defect` plants a
    bug for the checker to catch: "f32_lane" (lane 0's partial sum kept in float32), "drop_tail" / "twice_tail" (the
    last snapshot dropped or counted twice), "recip" (* (1 / N) in place of / N), "no_conj" (the lower triangle mirrored
    without conjugation)."""
    N, m = X.shape
    Xd = X.astype(np.complex128)
    if defect == "drop_tail":
        Xd = Xd[:-1]
    elif defect == "twice_tail":
        Xd = np.concatenate([Xd, Xd[-1:]])
    n = Xd.shape[0]
    ar, ai = Xd.real[:, :, None], Xd.imag[:, :, None]
    br, bi = Xd.real[:, None, :], Xd.imag[:, None, :]
    S = 32 if kernel == "warp" else generic_slices(m)
    acc = [np.zeros((S, m, m)), np.zeros((S, m, m))]
    for c0 in range(0, n, S):
        k = min(S, n - c0)
        sl = slice(c0, c0 + k)
        re, im = _fma_step([acc[0][:k], acc[1][:k]], ar[sl], ai[sl], br[sl], bi[sl])
        if defect == "f32_lane":
            re[0], im[0] = np.float32(re[0]), np.float32(im[0])
        acc[0][:k], acc[1][:k] = re, im
    if kernel == "warp":
        lanes = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            acc = [a + a[lanes ^ o] for a in acc]
        sre, sim = acc[0][0], acc[1][0]
    else:
        sre, sim = np.zeros((m, m)), np.zeros((m, m))
        for q in range(S):
            sre, sim = sre + acc[0][q], sim + acc[1][q]
    R = sre * (1.0 / N) + 1j * sim * (1.0 / N) if defect == "recip" else sre / N + 1j * (sim / N)
    iu = np.triu_indices(m)
    out = np.zeros((m, m), np.complex128)
    out[iu] = R[iu]
    out[np.diag_indices(m)] = out.diagonal().real
    low = out.T if defect == "no_conj" else out.T.conj()
    return out + np.tril(low, -1)


# ---- input families ----
def family_e1(rng, W, N, m, k=0):
    """E1: Gaussian integers |re|, |im| <= 2^11, times 2^k: every partial sum is an integer below 2^53 (times 2^2k), so
    every summation order gives S exactly and R = fl(S / N) bit for bit"""
    x = rng.integers(-2048, 2049, (W, N, m, 2)).astype(np.float32)
    x = np.ldexp(x, k).astype(np.float32)
    assert np.all(np.ldexp(x.astype(np.float64), -k) == np.rint(np.ldexp(x.astype(np.float64), -k)))
    return (x[..., 0] + 1j * x[..., 1]).astype(np.complex64)


def e1_reference(x, k=0):
    """fl(S / N) of E1 windows x [W][N][m] (complex64, already scaled by 2^k): S at scale 2^-2k is an integer below 2^53
    (float64 Gram exact in any order), the scaling by 2^2k is exact, and IEEE division rounds correctly"""
    X = np.ldexp(x.astype(np.complex128).real, -k) + 1j * np.ldexp(x.astype(np.complex128).imag, -k)
    S = np.einsum("wti,wtj->wij", X, X.conj())
    assert np.all(np.abs(S.real) < 2.0 ** 53) and np.all(S.real == np.rint(S.real)) and np.all(S.imag == np.rint(S.imag))
    N = x.shape[1]
    return (np.ldexp(S.real, 2 * k) / N) + 1j * (np.ldexp(S.imag, 2 * k) / N)


def family_e2(rng, W, N, m, spread=60):
    """E2: element r scaled by 2^s_r, s_r spread over [-spread, spread], with random 24-bit mantissas and signs"""
    s = np.rint(np.linspace(-spread, spread, m)).astype(int)
    rng.shuffle(s)
    mant = rng.integers(1 << 23, 1 << 24, (W, N, m, 2)) * rng.choice([-1, 1], (W, N, m, 2))
    x = np.ldexp(mant.astype(np.float64), (s - 23)[None, None, :, None]).astype(np.float32)
    return (x[..., 0] + 1j * x[..., 1]).astype(np.complex64)


def family_e3(rng, W, N, m, common=0.0):
    """E3: the second half of the snapshots repeats the first with the elements of a random set negated, so every R_ij
    with i in the set and j not is exactly 0 while A_ij is not; `common` adds a large common component to every element
    of the first half (its cross terms cancel too).  Odd N: one zero snapshot at the end.  Returns (x, zero mask)."""
    h = N // 2
    base = rng.standard_normal((W, h, m)) + 1j * rng.standard_normal((W, h, m)) + common * (1 + 1j)
    base = base.astype(np.complex64)
    neg = rng.random(m) < 0.5
    neg[0], neg[-1] = True, False
    x = np.zeros((W, N, m), np.complex64)
    x[:, :h] = base
    x[:, h:2 * h] = base * np.where(neg, -1, 1).astype(np.float32)
    zero = neg[:, None] != neg[None, :]
    return x, zero


def family_e4(rng, W, N, m, value):
    """E4: E1 windows with `value` (NaN or +-Inf) in element r(w) of one snapshot t(w) of each window, and the same windows
    with that value 0.  Returns (x_bad, x_zero, r per window)."""
    x = family_e1(rng, W, N, m)
    r = rng.integers(0, m, W)
    t = rng.integers(0, N, W)
    part = rng.integers(0, 2, W)
    bad = x.copy()
    zero = x.copy()
    for w in range(W):
        v = complex(value, 0.0) if part[w] == 0 else complex(0.0, value)
        bad[w, t[w], r[w]] = v
        zero[w, t[w], r[w]] = 0
    return bad, zero, r


# ---- integration ----
def _ctx():
    c = decimal.Context(prec=DPS, Emin=-999999, Emax=999999)
    return c


def integrate_exact(R, alpha, N=None):
    """the recurrence S_j = alpha S_{j-1} + R_j, c_j = alpha c_{j-1} + 1, q_j = alpha^2 q_{j-1} + 1 over R [W][m][m]
    (complex128, one stream since a reset) at 60 digits: (Rbar [W][m][m] rounded to fp64, Rbar - fl(Rbar) [W][m][m]
    rounded to fp64 parts, c [W] as Decimal, N_eff [W] as float when N is given)"""
    ctx = _ctx()
    W, m = R.shape[0], R.shape[1]
    D = np.vectorize(decimal.Decimal, otypes=[object])
    a = decimal.Decimal(alpha)
    a2 = ctx.multiply(a, a)
    S = np.full(2 * m * m, decimal.Decimal(0), object)
    c = q = decimal.Decimal(0)
    hi = np.empty((W, 2 * m * m))
    lo = np.empty((W, 2 * m * m))
    cs, neff = [], np.empty(W)
    flat = np.stack([R.real, R.imag], axis=-1).reshape(W, -1)
    with decimal.localcontext(ctx):
        for j in range(W):
            S = a * S + D(flat[j])
            c = a * c + 1
            q = a2 * q + 1
            Rb = S / c
            h = np.array([float(v) for v in Rb])
            hi[j] = h
            lo[j] = [float(v - decimal.Decimal(f)) for v, f in zip(Rb, h)]
            cs.append(c)
            if N is not None:
                neff[j] = float(N * c * c / q)
    shape = (W, m, m, 2)
    hi, lo = hi.reshape(shape), lo.reshape(shape)
    return hi[..., 0] + 1j * hi[..., 1], lo[..., 0] + 1j * lo[..., 1], cs, neff


def integ_depth(W):
    """L_int: the longest path of roundings of a term R_k into Rbar_j inside one sub-batch of W windows.
       integ_tiles_kernel   Horner over the tile:                                      INTEG_T - 1
       integ_carry_kernel   thread Horner over its chunk of tiles (fma into B, product into A):   2 chunk
                            warp scan, 5 levels of (fma, product); composition of <= 7 earlier warps: 2 (5 + 7)
                            xA, xB and the carry-in fma:                                3
                            aT = pow(alpha, 32) on the host, within 1 ulp (<= 2 eps) per tile a term crosses:  2 ntiles
       integ_apply_kernel   Horner from the carry-in and the division by c:             INTEG_T + 1
                            c: the closed form (C_POW) and INTEG_T - 1 fma steps:       C_POW + INTEG_T - 1"""
    nt = -(-W // INTEG_T)
    chunk = -(-nt // INTEG_SCAN_THREADS)
    return (INTEG_T - 1) + 2 * chunk + 2 * (5 + 7) + 3 + 2 * nt + (INTEG_T + 1) + (C_POW + INTEG_T - 1)


def integ_bounds(R, alpha, calls):
    """the per-entry bound (without the eps |Rbar| term) of every window: R [W][m][m] the raw covariances since the
    reset, `calls` the sizes of the sub-batches they were integrated in (sum = W).  Returns [W][m][m] complex128, the
    real and imaginary parts' bounds in the two parts."""
    W = R.shape[0]
    assert sum(calls) == W
    absR = np.abs(R.real) + 1j * np.abs(R.imag)
    out = np.empty_like(absR)
    sabs = np.zeros_like(absR[0])
    c = 0.0
    E = np.zeros_like(absR[0])
    j = 0
    for Wb in calls:
        L = integ_depth(Wb)
        prop = 1.0
        for _ in range(Wb):
            sabs = alpha * sabs + absR[j]
            c = alpha * c + 1.0
            prop *= alpha
            out[j] = C_INT * EPS * (L * sabs + prop * E) / c
            j += 1
        E = prop * E + L * sabs  # in units of eps
    return out


def integ_ratios(got, hi, lo, bound):
    """per window the worst |Rbar^ - Rbar| / (eps |Rbar| + bound) over both parts (got, hi, lo, bound [W][m][m])"""
    r = []
    for part in (np.real, np.imag):
        err = np.abs((part(got) - part(hi)) - part(lo))  # got - hi is exact (Sterbenz) wherever it matters
        b = EPS * np.abs(part(hi)) + part(bound)
        r.append(np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err > 0, np.inf, 0.0)).reshape(len(got), -1))
    return np.max(np.concatenate(r, axis=1), axis=1)


def one_minus_pow(a, k):
    """integ_one_minus_pow of music_integrate.cuh"""
    return -math.expm1(k * (math.log1p(a - 1.0) if a >= 0.5 else math.log(a)))


def integ_c(alpha, n, closed_form=False):
    """integ_c of music_integrate.cuh; `closed_form`: the cancelling (1 - pow(alpha, n + 1)) / (1 - alpha)"""
    if n == 0:
        return 1.0
    if closed_form:
        return (1.0 - math.pow(alpha, n + 1.0)) / (1.0 - alpha)
    return one_minus_pow(alpha, n + 1.0) / (1.0 - alpha)


def integ_neff(alpha, n, N, naive_q=False):
    """integ_neff of music_integrate.cuh; `naive_q`: q with 1 - alpha * alpha"""
    if n == 0:
        return float(N)
    k = n + 1.0
    d = one_minus_pow(alpha, k)
    c = d / (1.0 - alpha)
    if naive_q:
        a2 = alpha * alpha
        q = (1.0 - math.pow(a2, k)) / (1.0 - a2)
    else:
        q = d * (2.0 - d) / ((1.0 - alpha) * (1.0 + alpha))
    return N * c * c / q


def exact_c_neff(alpha, n, N):
    """c_n and N_eff,n at 60 digits (closed forms of the recurrences, exact up to the 60-digit rounding)"""
    with decimal.localcontext(_ctx()):
        a = decimal.Decimal(alpha)
        one = decimal.Decimal(1)
        c = (one - a ** (n + 1)) / (one - a)
        q = (one - (a * a) ** (n + 1)) / (one - a * a)
        return c, N * c * c / q


def emulate_integration(R, alpha, closed_form=False):
    """the three-kernel scan of music_integrate.cuh on one sub-batch after a reset, in Python with correctly rounded fma
    (R [W][E] float64).  Returns Rbar [W][E]."""
    def fma(a, b, c):
        return float(Fraction(a) * Fraction(b) + Fraction(c))

    W, E = R.shape
    nt = -(-W // INTEG_T)
    aT = math.pow(alpha, INTEG_T)
    alast = math.pow(alpha, W - (nt - 1) * INTEG_T)
    chunk = -(-nt // INTEG_SCAN_THREADS)
    out = np.empty_like(R)
    for e in range(E):
        agg = []
        for t in range(nt):
            a = R[t * INTEG_T, e]
            for i in range(t * INTEG_T + 1, min(W, (t + 1) * INTEG_T)):
                a = fma(alpha, a, R[i, e])
            agg.append(a)
        maps = []
        for tid in range(INTEG_SCAN_THREADS):
            t0, t1 = min(nt, tid * chunk), min(nt, tid * chunk + chunk)
            A, B = 1.0, 0.0
            for t in range(t0, t1):
                a = alast if t == nt - 1 else aT
                B = fma(a, B, agg[t])
                A *= a
            maps.append((A, B, t0, t1))
        incl = []
        for w in range(INTEG_SCAN_THREADS // 32):
            lane = [(A, B) for A, B, _, _ in maps[32 * w:32 * w + 32]]
            off = 1
            while off < 32:
                lane = [(A * lane[l - off][0], fma(A, lane[l - off][1], B)) if l >= off else (A, B)
                        for l, (A, B) in enumerate(lane)]
                off *= 2
            incl.append(lane)
        cin = [None] * nt
        for tid, (_, _, t0, t1) in enumerate(maps):
            w, l = divmod(tid, 32)
            pA, pB = 1.0, 0.0
            for v in range(w):
                pB = fma(incl[v][31][0], pB, incl[v][31][1])
                pA *= incl[v][31][0]
            eA, eB = (1.0, 0.0) if l == 0 else incl[w][l - 1]
            xA, xB = eA * pA, fma(eA, pB, eB)
            x = fma(xA, 0.0, xB)
            for t in range(t0, t1):
                a = alast if t == nt - 1 else aT
                cin[t] = x
                x = fma(a, x, agg[t])
        for t in range(nt):
            x, c = cin[t], integ_c(alpha, t * INTEG_T, closed_form)
            for i in range(t * INTEG_T, min(W, (t + 1) * INTEG_T)):
                if i > t * INTEG_T:
                    c = fma(alpha, c, 1.0)
                x = R[i, e] if i == 0 else fma(alpha, x, R[i, e])
                out[i, e] = x / c
    return out


# ---- channels (music_channels.cuh) and focusing (music_focus.cuh) ----
# The filter bank's R_c = sum_j X_j[b] X_j[b]^H / (J sum_t h[t]^2) is built here at CHAN_DPS digits from the header's
# definition: the exact taper h and the exact twiddles exp(-2 pi i b t / F), not the host table.  Its bound is relative
# to each segment's energy, not to the channel's power: a radix-2 FFT with correctly rounded twiddles is in error by at
# most log2(F) eta sqrt(F) ||h x_j||_2 in every bin, eta = mu + gamma_4 (sqrt 2 + mu) <= 7 eps (Higham, Accuracy and
# Stability, thm 24.2), and the tapered input adds (1 + 2) eps sqrt(F) ||h x_j||_2 (one rounding of h x, the taper's own
# one rounding after a correctly rounded cosine).  With e = (C_FFT log2 F + 3) eps sqrt(F) ||h x_j|| per antenna and
# segment, the rank-one update and its accumulation (2 roundings per segment, two parts each bounded by |X_a| |X_b|):
#     |R^_ab - R_ab| <= (F + 4) eps |R_ab| + C_CH sum_j (e_a |X_b| + |X_a| e_b + e_a e_b + 2 J eps (|X_a| + e_a)(|X_b| + e_b))
#                                           / (J sum_t h^2)
# (F + 4: the denominator's own sum of F rounded squares and the division).  C_CH = 1.01 as C_COV.
C_FFT = 7
C_CH = 1.01
CHAN_DPS = 40


def channel_exact(x, m, F, bins, kind):
    """one window x (complex64 [N * m]): (R [C][m][m] of mpc, |X| [C][J][m] and ||h x_j|| [J][m] as floats,
    J sum h^2 as mpf) at CHAN_DPS digits"""
    import mpmath as mp
    bins = [int(b) for b in bins]
    with mp.workdps(CHAN_DPS):
        X = np.asarray(x).reshape(-1, m).astype(np.complex128)
        J = X.shape[0] // F
        h = [mp.mpf(1) if kind == "rect" else mp.mpf(1) / 2 - mp.cos(2 * mp.pi * t / F) / 2 for t in range(F)]
        denom = J * mp.fsum(v * v for v in h)
        tw = {(b, t): mp.expjpi(-mp.mpf(2 * ((b * t) % F)) / F) for b in bins for t in range(F)}
        Xc = np.empty((len(bins), J, m), object)
        norm = np.empty((J, m))
        for j in range(J):
            seg = [[h[t] * mp.mpc(float(v.real), float(v.imag)) for v in X[j * F + t]] for t in range(F)]
            for a in range(m):
                norm[j, a] = float(mp.sqrt(mp.fsum(abs(seg[t][a]) ** 2 for t in range(F))))
            for ci, b in enumerate(bins):
                for a in range(m):
                    Xc[ci, j, a] = mp.fsum(seg[t][a] * tw[(b, t)] for t in range(F))
        R = np.empty((len(bins), m, m), object)
        for ci in range(len(bins)):
            for a in range(m):
                for b in range(m):
                    R[ci, a, b] = mp.fsum(Xc[ci, j, a] * mp.conj(Xc[ci, j, b]) for j in range(J)) / denom
        absX = np.vectorize(lambda v: float(abs(v)), otypes=[np.float64])(Xc)
        return R, absX, norm, denom


def channel_ratios(R_hat, x, m, F, bins, kind):
    """per channel the worst |R^_c - R_c| / bound over the entries and parts of one window (R_hat [C][m][m])"""
    import mpmath as mp
    R, absX, norm, denom = channel_exact(x, m, F, bins, kind)
    J = norm.shape[0]
    e = (C_FFT * math.log2(F) + 3) * EPS * math.sqrt(F) * norm  # [J][m]
    out = []
    with mp.workdps(CHAN_DPS):
        for ci in range(len(bins)):
            Xa = absX[ci]  # [J][m]
            num = (e.T @ Xa + Xa.T @ e + e.T @ e + 2 * J * EPS * (Xa + e).T @ (Xa + e))
            worst = 0.0
            for a in range(m):
                for b in range(m):
                    ref = R[ci, a, b]
                    for got, exact in ((R_hat[ci, a, b].real, ref.real), (R_hat[ci, a, b].imag, ref.imag)):
                        err = float(abs(mp.mpf(got) - exact)) if math.isfinite(got) else math.inf
                        bound = (F + 4) * EPS * float(abs(exact)) + C_CH * num[a, b] / float(denom)
                        worst = max(worst, err / bound if bound > 0 else (math.inf if err > 0 else 0.0))
            out.append(worst)
    return out


def twiddles(F):
    """tw[k] = exp(-2 pi i k / F), k < F / 2, correctly rounded (the table chan_tables_host promises)"""
    import mpmath as mp
    with mp.workdps(50):
        return np.array([complex(float(mp.cospi(mp.mpf(2 * k) / F)), -float(mp.sinpi(mp.mpf(2 * k) / F)))
                         for k in range(F // 2)])


def emulate_channel_fft(seg, tw):
    """the radix-2 decimation-in-frequency transform of chan_cov_kernel (natural order in, bin order out) of the rows of
    seg [rows][F] complex128 with the twiddle table tw [F / 2]"""
    y = np.array(seg, np.complex128)
    F = y.shape[-1]
    half, s = F // 2, 0
    while half >= 1:
        for start in range(0, F, 2 * half):
            for k in range(half):
                a, b = y[:, start + k].copy(), y[:, start + k + half].copy()
                y[:, start + k] = a + b
                y[:, start + k + half] = (a - b) * tw[k << s]
        half //= 2
        s += 1
    logF = F.bit_length() - 1
    order = [int(format(i, "0%db" % logF)[::-1], 2) for i in range(F)]
    return y[:, order]


def emulate_channel_R(x, m, F, bins, kind, tw):
    """R_c of one window through emulate_channel_fft, accumulated segment after segment"""
    X = np.asarray(x).reshape(-1, m).astype(np.complex128)
    J = X.shape[0] // F
    t = np.arange(F)
    h = np.ones(F) if kind == "rect" else 0.5 - 0.5 * np.cos(2 * math.pi * t / F)
    R = np.zeros((len(bins), m, m), np.complex128)
    for j in range(J):
        Y = emulate_channel_fft((X[j * F:(j + 1) * F] * h[:, None]).T, tw)[:, bins].T  # [C][m]
        R += Y[:, :, None] * Y[:, None, :].conj()
    return R / (J * np.sum(h * h))


def channel_windows(rng, W, m, F, J, tone_bin, weak_bin):
    """a unit on-bin tone in bin tone_bin on every element, a tone 2^-30 weaker in weak_bin, noise at 2^-40"""
    t = np.arange(F * J)
    s = np.exp(2j * np.pi * tone_bin * t / F) + 2.0 ** -30 * np.exp(2j * np.pi * weak_bin * t / F)
    ph = np.exp(2j * np.pi * rng.random(m))
    x = s[None, :, None] * ph[None, None, :] + 2.0 ** -40 * (rng.standard_normal((W, F * J, m))
                                                              + 1j * rng.standard_normal((W, F * J, m)))
    return x.reshape(W, -1).astype(np.complex64)


C_FOC = 4


def focus_ratio(R_foc_hat, T, R_c):
    """the worst |R^_foc - R_foc| / (eps |R_foc| + (C_FOC M + C + 2) eps (1/C) sum_c (|T_c| |R_c| |T_c|^H)) of one
    window, R_foc = (1/C) sum_c T_c R_c T_c^H at CHAN_DPS digits on the device's own T_c and R_c"""
    import mpmath as mp
    C, m = R_c.shape[0], R_c.shape[1]
    with mp.workdps(CHAN_DPS):
        Tm = [mp.matrix([[mp.mpc(v) for v in row] for row in T[c]]) for c in range(C)]
        Rm = [mp.matrix([[mp.mpc(v) for v in row] for row in R_c[c]]) for c in range(C)]
        ref = sum((Tm[c] * Rm[c] * Tm[c].H for c in range(C)), mp.zeros(m, m)) / C
        A = sum(np.abs(T[c]) @ np.abs(R_c[c]) @ np.abs(T[c]).T for c in range(C)) / C
        worst = 0.0
        for a in range(m):
            for b in range(m):
                for got, ex in ((R_foc_hat[a, b].real, ref[a, b].real), (R_foc_hat[a, b].imag, ref[a, b].imag)):
                    err = float(abs(mp.mpf(got) - ex))
                    bound = EPS * float(abs(ex)) + (C_FOC * m + C + 2) * EPS * A[a, b]
                    worst = max(worst, err / bound if bound > 0 else (math.inf if err > 0 else 0.0))
    return worst
