"""High-precision reference for the Hermitian eigensolvers, the bounds a backward-stable solver meets, the windows that
stress them and the probe tables that read a noise projector back through the MUSIC scan (not a test module).

Reference: mpmath at REF_DPS digits on the fp64 matrix R as given (the GPU's own R wherever R is not exact, so that the
covariance's rounding is not charged to the eigensolver): ascending eigenvalues, the noise projector Pi = G G^H of the
M - n smallest, the boundary gap lambda_{M-n+1} - lambda_{M-n} and ||R||_2.

Bounds (one named constant each):
    eigenvalues   |w^ - w|          <= C_EIG  M eps ||R||_2
    projector     ||Pi^ - Pi||_2    <= C_PROJ M eps ||R||_2 / gap   (+ the scan's own readout error, C_SCAN M eps)
with eps = 2^-53.  A cyclic Jacobi run to its stopping rule stays about an order of magnitude inside both; a Jacobi that
stops one sweep early, at the stagnation threshold, or on an off-diagonal norm computed by subtraction does not
(tests/test_eig_oracle.py plants each of those defects and shows this checker failing them).

Windows (x: [N][M] complex64):
  * exact windows: snapshots c_t h_k, h_k the columns of an exactly orthogonal matrix with entries in {0, +-1, +-i}
    (Sylvester / DFT-4 tensor products and block-diagonal sums of them under a signed permutation), c_t Gaussian
    integers exact in float32.  Every product and partial sum of the covariance is an integer below 2^53 times a power
    of two, so R is exact in any summation order and lambda_k = b_k S_k / N in closed form (b_k = ||h_k||^2,
    S_k = sum |c_t|^2 over the snapshots of column k): exact ties, exact zeros, gaps down to 2^-36 relative;
  * prescribed spectra Q diag(lambda) Q^H, rounded to float32 (the reference then runs on the GPU's R);
  * edges: diagonal unsorted R with ties, all-zero, NaN and Inf windows, and the exact families scaled by 2^-140 / 2^96.
"""
import math

import mpmath as mp
import numpy as np

EPS = 2.0 ** -53
REF_DPS = 50
C_EIG = 16.0     # eigenvalue bound:  C_EIG M eps ||R||_2
C_PROJ = 16.0    # projector bound:   C_PROJ M eps ||R||_2 / gap
C_SCAN = 8.0     # the scan's readout of Pi^ through 1 / P64 (complement form included): C_SCAN M eps absolute
PROJ_CHECKED = 1e-3  # projector bounds above this are not checked (ill-conditioned split): counted, not compared
EXACT_N = 256    # snapshots per exact window (a power of two: the fused M = 8 path accepts it, 1 / N is exact)


# ---- reference ------------------------------------------------------------------------------------------------------
def reference(R, n):
    """mpmath eigen-decomposition of the Hermitian fp64 matrix R: dict(w = ascending eigenvalues, Pi = noise projector
    of the M - n smallest (complex128), gap = lambda_{M-n+1} - lambda_{M-n} (0.0 for n in {0, M}), norm = ||R||_2,
    V = all eigenvectors as columns, ascending)"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    with mp.workdps(REF_DPS):
        A = mp.matrix([[mp.mpc(R[i, j].real, R[i, j].imag) for j in range(M)] for i in range(M)])
        E, Q = mp.eighe(A)
        order = sorted(range(M), key=lambda i: E[i])
        w = [E[i] for i in order]
        Pi = mp.matrix(M, M)
        for k in order[:M - n]:
            for i in range(M):
                for j in range(M):
                    Pi[i, j] += Q[i, k] * mp.conj(Q[j, k])
        gap = float(w[M - n] - w[M - n - 1]) if 0 < n < M else 0.0
        V = np.array([[complex(Q[i, k]) for k in order] for i in range(M)])
        return {"w": np.array([float(x) for x in w]), "Pi": np.array([[complex(Pi[i, j]) for j in range(M)] for i in range(M)]),
                "gap": gap, "norm": float(max(abs(x) for x in w)), "V": V}


def eig_bound(M, norm):
    return C_EIG * M * EPS * norm


def proj_bound(M, norm, gap):
    """bound on ||Pi^ - Pi||_2 for a solver; inf when the split is not defined (gap <= 0)"""
    return C_PROJ * M * EPS * norm / gap if gap > 0 else math.inf


def proj_err(Pi_hat, Pi):
    E = Pi_hat - Pi
    return float(np.max(np.abs(np.linalg.eigvalsh((E + E.conj().T) / 2)))) if np.all(np.isfinite(E)) else math.inf


def check(M, n, ref, w_hat, Pi_hat, readout=0.0):
    """(eigenvalue error / bound, projector error / bound or None when the split is ill-conditioned); readout: the
    absolute error the projector's readout itself may add"""
    ew = float(np.max(np.abs(np.asarray(w_hat) - ref["w"]))) / eig_bound(M, ref["norm"]) if ref["norm"] > 0 else (
        0.0 if np.all(np.asarray(w_hat) == 0) else math.inf)
    pb = proj_bound(M, ref["norm"], ref["gap"])
    if not pb <= PROJ_CHECKED:
        return ew, None
    return ew, proj_err(Pi_hat, ref["Pi"]) / (pb + readout)


def noise_projector(Vt, n):
    """Pi = sum over the M - n smallest of e e^H, from a solver's Vt[rank][i] (eigenvector rank, component i)"""
    G = np.asarray(Vt)[: Vt.shape[0] - n].T
    return G @ G.conj().T


# ---- exact windows --------------------------------------------------------------------------------------------------
H2 = np.array([[1, 1], [1, -1]], np.complex128)
F4 = np.array([[1, 1, 1, 1], [1, -1j, -1, 1j], [1, -1, 1, -1], [1, 1j, -1, -1j]], np.complex128)
BLOCKS = {1: np.ones((1, 1), np.complex128), 2: H2, 4: F4, 8: np.kron(F4, H2), 16: np.kron(F4, F4)}


def orthogonal_columns(M, rng, diagonal=False):
    """an M x M matrix with entries in {0, +-1, +-i} and exactly orthogonal columns (||h_k||^2 = block size b_k), rows
    under a random signed permutation; returns (H, b).  diagonal: signed permutation of the identity."""
    sizes = [1] * M if diagonal else [s for s in (16, 8, 4, 2, 1) if M & s]
    H = np.zeros((M, M), np.complex128)
    o = 0
    for s in sizes:
        H[o:o + s, o:o + s] = BLOCKS[s]
        o += s
    b = np.concatenate([[s] * s for s in sizes]).astype(np.int64)
    perm = rng.permutation(M)
    signs = np.array([1, -1, 1j, -1j])[rng.integers(0, 4, M)]
    return H[perm] * signs[:, None], b


def sum_of_squares(S):
    """greedy: integers a_1 >= a_2 >= ... with sum a_i^2 = S (a few terms for S < 2^53)"""
    out = []
    while S > 0:
        a = math.isqrt(S)
        out.append(a)
        S -= a * a
    return out


def exact_window(M, S, rng, N=EXACT_N, diagonal=False):
    """x [N][M] complex64 with R = (1/N) sum_k S_k h_k h_k^H exactly; returns (x, R, ascending eigenvalues).  S: M
    non-negative integers, S_k < 2^44 (so |c_t| < 2^22 and every partial sum of R stays below 2^53)."""
    H, b = orthogonal_columns(M, rng, diagonal)
    S = [int(s) for s in S]
    assert len(S) == M and all(0 <= s < 2 ** 44 for s in S)
    snaps = []
    for k in range(M):
        a = sum_of_squares(S[k])
        a += [0] * (len(a) % 2)
        for t in range(0, len(a), 2):
            c = complex(a[t], a[t + 1]) * [1, -1, 1j, -1j][int(rng.integers(0, 4))]
            snaps.append(c * H[:, k])
    assert len(snaps) <= N, (M, len(snaps))
    x = np.zeros((N, M), np.complex128)
    x[:len(snaps)] = snaps
    x = x[rng.permutation(N)]
    assert np.array_equal(x.astype(np.complex64).astype(np.complex128), x)
    R = sum(S[k] * np.outer(H[:, k], H[:, k].conj()) for k in range(M)) / N
    lam = np.sort(np.array([b[k] * S[k] for k in range(M)], np.float64) / N)
    return x.astype(np.complex64), R, lam


def exact_spectra(M, n, rng):
    """(name, S) per exact family; the values are per unit block size (S_k = L_k * 16 / b_k keeps ties exact)"""
    L = 2 ** 36
    fam = []
    fam.append(("ties", [L] * (M - n) + [4 * L] * n))                           # exact repeated eigenvalues
    fam.append(("zero noise", [0] * (M - n) + [L + 16 * k for k in range(n)]))  # exact zeros, close signal values
    fam.append(("rank one", [0] * (M - 1) + [L]))
    fam.append(("gap 2^-28 at the boundary", [L] * (M - n) + [L + 2 ** 8] * n))
    fam.append(("gap 2^-36 at the boundary", [L] * (M - n) + [L + 1] * n))
    fam.append(("graded 2^-30", [2 ** (2 * k + 6) for k in range(M)]))
    fam.append(("cluster in noise", [L + k for k in range(M - n)] + [8 * L] * n))
    return fam


def exact_family(M, n, rng, diagonal=False):
    """[(name, x, R, lambda)] for the exact windows of size M (block sizes folded into S so that ties stay ties)"""
    out = []
    _, b = orthogonal_columns(M, np.random.default_rng(0), diagonal)
    for name, L in exact_spectra(M, n, rng):
        perm = rng.permutation(M)          # which column gets which value: the spectrum arrives unsorted
        S = [(L[perm[k]] * 16) // int(b[k]) for k in range(M)]
        x, R, lam = exact_window(M, S, np.random.default_rng(rng.integers(1 << 30)), diagonal=diagonal)
        out.append((name, x, R, lam))
    return out


# ---- prescribed spectra (rounded to float32) ------------------------------------------------------------------------
def unitary(M, rng):
    Q, _ = np.linalg.qr(rng.standard_normal((M, M)) + 1j * rng.standard_normal((M, M)))
    return Q


def spectrum_window(lam, Q, N):
    """x [N][M] complex64 with (1/N) X^H X = Q diag(lam) Q^H before the float32 rounding"""
    M = len(lam)
    x = np.zeros((N, M), np.complex128)
    x[:M] = (Q * np.sqrt(N * np.asarray(lam, np.float64))).T
    return x.astype(np.complex64)


def prescribed_spectra(M, n):
    """(name, ascending eigenvalues) of the prescribed families"""
    base = np.linspace(1.0, 2.0, M - n)
    out = [("noise cluster 1e-9", np.concatenate([1.0 + 1e-9 * np.arange(M - n), 10.0 + np.arange(n)]))]
    for r in (1e-6, 1e-9, 1e-13):
        out.append(("boundary cluster %g" % r, np.concatenate([base, 2.0 * (1 + r) + np.arange(n) * r])))
    out.append(("graded 1e-14", 10.0 ** np.linspace(-14, 0, M)))
    return out


def top_pair_ratios():
    """lambda_1 / lambda_2 of the near-equal top pair: both sides of the squaring / fallback boundary (~1.01)"""
    return (1.001, 1.005, 1.01, 1.02, 1.05)


def top_pair_spectrum(M, ratio):
    return np.concatenate([np.linspace(0.1, 0.5, M - 2), [1.0, ratio]])


def imaginary_window(M, N, rng):
    """R = D + i S with S real antisymmetric (purely imaginary off-diagonals), positive definite"""
    S = rng.standard_normal((M, M))
    S = (S - S.T) / 2
    D = np.diag(np.linspace(1.0, 3.0, M) + 2.0 * np.abs(S).sum(1))
    w, Q = np.linalg.eigh(D + 1j * S)
    return spectrum_window(w, Q, N)


def rank_one_window(M, N, rng):
    v = unitary(M, rng)[:, 0]
    x = np.zeros((N, M), np.complex128)
    x[0] = 3.0 * v
    return x.astype(np.complex64)


# ---- probe tables ---------------------------------------------------------------------------------------------------
def probe_table(M):
    """K = M^2 rows, exact in float32: e_i, then e_i + e_j and e_i + i e_j for i < j"""
    rows = [np.eye(M)[i] for i in range(M)]
    for i in range(M):
        for j in range(i + 1, M):
            rows.append(np.eye(M)[i] + np.eye(M)[j])
            rows.append(np.eye(M)[i] + 1j * np.eye(M)[j])
    return np.array(rows).astype(np.complex64)


def projector_from_P(P, M):
    """Pi^ from the MUSIC strengths P = 1 / (a^H Pi^ a) of the probe_table rows"""
    d = 1.0 / np.asarray(P, np.float64)
    Pi = np.zeros((M, M), np.complex128)
    Pi[np.diag_indices(M)] = d[:M]
    k = M
    for i in range(M):
        for j in range(i + 1, M):
            re = (d[k] - d[i] - d[j]) / 2
            im = -(d[k + 1] - d[i] - d[j]) / 2
            Pi[i, j] = complex(re, im)
            Pi[j, i] = complex(re, -im)
            k += 2
    return Pi


def sensitive_rows(ref, n, etas=(1e-3, 1e-4)):
    """rows a = u + eta v (u: principal eigenvector, v: the noise eigenvectors in turn), rounded to float32: d ~ eta^2,
    so an eigenvector error delta moves P by ~ 2 delta / eta relative"""
    V = ref["V"]
    M = V.shape[0]
    u = V[:, M - 1]
    rows = [u + eta * V[:, j] for eta in etas for j in range(M - n)]
    return np.array(rows).astype(np.complex64)


def strength_ref(ref, table):
    """reference MUSIC strength P = 1 / a^H Pi a per row of the float32 table (a taken as stored), with Pi at REF_DPS
    digits; returns (P, d = a^H Pi a, ||a||^2)"""
    a = table.astype(np.complex128)
    Pi = ref["Pi"]
    na = np.sum(np.abs(a) ** 2, axis=1)
    d = np.einsum("ki,ij,kj->k", a.conj(), Pi, a).real
    with np.errstate(divide="ignore"):
        return 1.0 / d, d, na


def strength_tol(ref, table, M):
    """relative tolerance of a fused kernel's float32 strength at each row of table: the float32 rounding plus what the
    projector bound lets through at that row (a^H E a <= 2 ||E|| |a_noise| ||a|| + ||E||^2 ||a||^2 for a projector
    error E of norm ||E||, a_noise = Pi a) and the scan's relative rounding"""
    B = proj_bound(M, ref["norm"], ref["gap"])
    a = table.astype(np.complex128)
    _, d, na = strength_ref(ref, table)
    an = np.sqrt(np.maximum(d, 0.0))
    return 2.0 ** -23 + (2 * B * an * np.sqrt(na) + B * B * na) / d + C_SCAN * M * EPS * na / d
