"""Literal numpy restatements of the Cholesky-based device solvers, in the kernels' operation order, for the CPU tests
of tests/solve_oracle.py (tests/test_solve_oracle.py):

    warp_cholesky        right-looking, the trailing update A[i][j] -= L[i][k] conj(L[j][k]) for k < j <= i
    mvdr_prep            delta = loading * tr / M (the diagonal summed in index order), the factor, then column c of
                         L^-1 by forward substitution; the scan form mvdr_form sums |g_j^H a|^2 over the conjugated rows
    beam_weights         y = L^-1 a and z = L^-H y per slot; MVDR w = z / ||y||^2; LCMV G = Y^H Y over the filled slots,
                         factored with the 2^-20 pivot rule against diag(G) before elimination, W = Z G^-1 per antenna
    dml_levels           MGS applied twice (Q_A, T), C = Q^H R Q, s2 by subtracting the traces, U = T^-1 by back
                         substitution column by column, p_l = sum_{a, b} U[l][a] C[a][b] conj(U[l][b])

Complex products are Python / numpy complex128 products (re = ar br - ai bi, im = ar bi + ai br, each rounded once);
the kernels' fma contractions change each rounding by at most one more ulp, which the bounds' constants cover.  The
mvdr_form accumulation keeps the kernel's order.  Keyword switches plant the defects the CPU tests show the checker
catching; with every switch at its default the emulation is the kernel.
"""
import numpy as np

PIVOT_REL = 2.0 ** -20


def warp_cholesky(A, pivot_ok, conj=True):
    """in-place right-looking Cholesky of the Hermitian A (lower triangle read); the lower L or None"""
    A = np.array(A, np.complex128)
    M = A.shape[0]
    for k in range(M):
        d = A[k, k].real
        if not pivot_ok(k, d):
            return None
        l = np.sqrt(d)
        A[k, k] = l
        A[k + 1:, k] = A[k + 1:, k] / l
        for i in range(k + 1, M):
            for j in range(k + 1, i + 1):
                b = np.conj(A[j, k]) if conj else A[j, k]
                A[i, j] -= A[i, k] * b
    return np.tril(A)


def delta_of(R, loading, div=None):
    tr = 0.0
    for i in range(R.shape[0]):
        tr += R[i, i].real
    return loading * tr / float(R.shape[0] if div is None else div)


def mvdr_prep(R, loading, f32_subst=False, conj=True, delta_div=None):
    """Vt [M][M]: conj(row j of L^-1), NaN everywhere when a pivot is not > 0"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    A = R.copy()
    delta = delta_of(R, loading, None if delta_div is None else delta_div(M))
    for i in range(M):
        A[i, i] += delta
    L = warp_cholesky(A, lambda k, d: d > 0.0, conj)
    if L is None:
        return np.full((M, M), np.nan + 1j * np.nan)
    I = np.zeros((M, M), np.complex128)
    acc = np.complex64 if f32_subst else np.complex128
    for c in range(M):
        I[c, c] = 1.0 / L[c, c].real
        for i in range(c + 1, M):
            s = acc(0)
            for q in range(c, i):
                s = acc(s + acc(L[i, q] * I[q, c]))
            I[i, c] = -complex(s) / L[i, i].real
    return np.conj(I)


def mvdr_form(G, table):
    """D_k = sum_j |g_j^H a_k|^2 over the rows of the complex64 table, in mvdr_form's order"""
    a = np.asarray(table, np.complex64).astype(np.complex128)
    M = G.shape[0]
    acc = np.zeros(a.shape[0])
    for j in range(M):
        c = np.zeros(a.shape[0], np.complex128)
        for i in range(j + 1):
            c = c + np.conj(G[j, i]) * a[:, i]
        acc = acc + (c.real * c.real + c.imag * c.imag)
    return acc


def mvdr_p64(R, loading, table, **defects):
    with np.errstate(all="ignore"):
        return 1.0 / mvdr_form(mvdr_prep(R, loading, **defects), table)


def _fwd(L, b):
    y = np.array(b, np.complex128)
    for k in range(len(y)):
        s = y[k]
        for q in range(k):
            s -= L[k, q] * y[q]
        y[k] = s / L[k, k].real
    return y


def _bwd(L, y):
    z = np.array(y, np.complex128)
    for k in range(len(z) - 1, -1, -1):
        s = y[k]
        for q in range(k + 1, len(z)):
            s -= np.conj(L[q, k]) * z[q]
        z[k] = s / L[k, k].real
    return z


def beam_weights(R, rows, n, rule, loading, gram_conj=True, running_pivot=False, conj=True):
    """wts [n][M] for the filled slots rows = {slot: a}; rule "mvdr" or "lcmv"; zeros on any failure"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    W = np.zeros((n, M), np.complex128)
    if not rows:
        return W
    A = R.copy()
    delta = delta_of(R, loading)
    for i in range(M):
        A[i, i] += delta
    L = warp_cholesky(A, lambda k, d: d > 0.0, conj)
    if L is None:
        return W
    S = sorted(rows)
    Y = {i: _fwd(L, rows[i]) for i in S}
    Z = {i: _bwd(L, Y[i]) for i in S}
    with np.errstate(all="ignore"):
        if rule == "mvdr":
            for i in S:
                nrm = 0.0
                for m in range(M):
                    nrm += Y[i][m].real * Y[i][m].real + Y[i][m].imag * Y[i][m].imag
                W[i] = Z[i] / nrm
        else:
            d = len(S)
            G = np.zeros((d, d), np.complex128)
            for r in range(d):
                for c in range(d):
                    s = 0j
                    for m in range(M):
                        s += (np.conj(Y[S[r]][m]) if gram_conj else Y[S[r]][m]) * Y[S[c]][m]
                    G[r, c] = s
            D = G.diagonal().real.copy()
            ok = (lambda k, p: p > PIVOT_REL * p) if running_pivot else (lambda k, p: p > PIVOT_REL * D[k])
            C = warp_cholesky(G, ok)
            if C is None:
                return W
            for m in range(M):
                u = _bwd(C, _fwd(C, np.array([np.conj(Z[i][m]) for i in S])))
                for r, i in enumerate(S):
                    W[i, m] = np.conj(u[r])
    if not np.all(np.isfinite(W)):
        return np.zeros((n, M), np.complex128)
    return W


def mgs(A, passes=2):
    """dml_mgs2: columns of A (M x r) in order, `passes` projection passes; (Q, T)"""
    M, r = A.shape
    Q = np.zeros((M, r), np.complex128)
    T = np.zeros((r, r), np.complex128)
    for l in range(r):
        v = A[:, l].astype(np.complex128).copy()
        for _ in range(passes):
            for j in range(l):
                c = np.sum(np.conj(Q[:, j]) * v)
                v = v - c * Q[:, j]
                T[j, l] += c
        nrm = np.sqrt(np.sum(v.real * v.real + v.imag * v.imag))
        Q[:, l] = v / nrm
        T[l, l] = nrm
    return Q, T


def dml_levels(R, table, slots, passes=2, s2_div=None, transpose_u=False):
    """(p [d] in slot order, s2) of the levels block"""
    R = np.asarray(R, np.complex128)
    M, d = R.shape[0], len(slots)
    Q, T = mgs(np.asarray(table, np.complex64).astype(np.complex128)[list(slots)].T, passes)
    C = np.zeros((d, d), np.complex128)
    for a in range(d):
        for b in range(d):
            y = R @ Q[:, b]
            C[a, b] = np.sum(np.conj(Q[:, a]) * y)
    trR = 0.0
    for i in range(M):
        trR += R[i, i].real
    trQ = 0.0
    for a in range(d):
        trQ += C[a, a].real
    s2 = (trR - trQ) / float(M - d if s2_div is None else s2_div(M, d))
    for a in range(d):
        C[a, a] -= s2
    U = np.zeros((d, d), np.complex128)
    for c in range(d):
        for i in range(d - 1, -1, -1):
            if i <= c:
                s = 1.0 + 0j if i == c else 0j
                for q in range(i + 1, c + 1):
                    s -= T[i, q] * U[q, c]
                U[i, c] = s / T[i, i].real
    if transpose_u:
        U = U.T.copy()
    p = np.zeros(d)
    for l in range(d):
        acc = 0.0
        for a in range(l, d) if not transpose_u else range(d):
            y = 0j
            for b in range(l, d) if not transpose_u else range(d):
                y += C[a, b] * np.conj(U[l, b])
            acc += (U[l, a] * y).real
        p[l] = acc
    return p, s2
