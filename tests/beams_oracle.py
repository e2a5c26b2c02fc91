"""fp64 oracle of the beamformed source signals (music_b200_set_beamformer, include/music_b200.h), restated literally:

For window w the filled slots are S = {i : bins[w][i] >= 0} as the call's peak stage reported them (not assumed to
form a prefix).  M = m, x(r, c) = in[c m + r].
  steering   a_i (fp64): a geometric table (set_geometry()): a_m = exp(-j phi_m), phi_m = 2 pi (p_x,m cos t + p_y,m sin t)
             / lambda, t = the reported float angle (double)angles[w][i] in radians; a set_table() table: row bins[w][i]
             widened to fp64.
  DAS        w_i = a_i / (a_i^H a_i).  It reads no R.
  MVDR       R_L = R + delta I, delta = loading * tr(R) / M; R_L = L L^H (a pivot that is not > 0 fails);
             y_i = L^-1 a_i, z_i = L^-H y_i, w_i = z_i / ||y_i||^2.
  LCMV       Y = [y_i], Z = [z_i] over i in S, G = Y^H Y (d x d), G = C C^H where every pivot g_k (before its square root)
             must satisfy g_k > 2^-20 G_kk (the diagonal entry before elimination); W = Z G^-1, column i is w_i, and
             w_i^H a_j = delta_ij.  With d = 1, LCMV equals MVDR.
  failure    every weight and beam of the window is 0 when the Cholesky of R_L fails (MVDR, LCMV), when LCMV's pivot test
             fails, or when any weight is not finite.  Unfilled slots always get zero weights and zero beams.
  outputs    weights[w][i][m] = w_i (complex128); beams[w][i][t] = (complex64)(sum_m conj(w_im) x_m(t)), t < N,
             accumulated in fp64, re and im each rounded once.
"""
import math

import numpy as np

DAS, MVDR, LCMV = 1, 2, 3
PIVOT_REL = 2.0 ** -20


def steering_geo(pos, lam, deg):
    """a(t) for the element positions pos [M][x, y] (metres) at the float angle deg, as the refinement evaluates it"""
    t = float(np.float64(np.float32(deg))) * (math.pi / 180.0)
    st, ct = math.sin(t), math.cos(t)
    pos = np.asarray(pos, np.float64)
    phi = 2.0 * math.pi * ((pos[:, 0] * ct + pos[:, 1] * st) / lam)
    return np.cos(phi) - 1j * np.sin(phi)


def cholesky(A, pivot_ok):
    """lower L with A = L L^H (lower triangle of A read), or None at the first pivot k with not pivot_ok(k, g_k)"""
    A = np.array(A, np.complex128)
    n = A.shape[0]
    L = np.zeros_like(A)
    for k in range(n):
        g = A[k, k].real
        if not pivot_ok(k, g):
            return None
        l = math.sqrt(g)
        L[k, k] = l
        L[k + 1:, k] = A[k + 1:, k] / l
        for i in range(k + 1, n):
            for j in range(k + 1, i + 1):
                A[i, j] -= L[i, k] * np.conj(L[j, k])
    return L


def forward(L, b):
    """L^-1 b, L lower triangular with a real diagonal"""
    y = np.array(b, np.complex128)
    for k in range(len(y)):
        y[k] = (y[k] - L[k, :k] @ y[:k]) / L[k, k].real
    return y


def backward(L, y):
    """L^-H y"""
    z = np.array(y, np.complex128)
    for k in range(len(z) - 1, -1, -1):
        z[k] = (z[k] - np.conj(L[k + 1:, k]) @ z[k + 1:]) / L[k, k].real
    return z


def steering_vectors(angles, bins, table=None, pos=None, lam=None):
    """{i: a_i} over the filled slots of one window"""
    out = {}
    for i, b in enumerate(bins):
        if b < 0:
            continue
        if pos is not None:
            out[i] = steering_geo(pos, lam, angles[i])
        else:
            out[i] = np.asarray(table[int(b)], np.complex64).astype(np.complex128)
    return out


def weights(R, angles, bins, rule, loading=0.0, table=None, pos=None, lam=None):
    """complex128 [n][M] weights of one window (R [M][M] complex128, angles / bins [n]); table [K][M] for a set_table()
    table, or (pos, lam) for a geometric one"""
    n = len(bins)
    A = steering_vectors(angles, bins, table, pos, lam)
    M = (R.shape[0] if R is not None else len(next(iter(A.values())))) if A else (R.shape[0] if R is not None else 0)
    W = np.zeros((n, M), np.complex128)
    if not A:
        return W
    S = sorted(A)
    if rule == DAS:
        for i in S:
            a = A[i]
            W[i] = a / np.vdot(a, a).real
    else:
        RL = np.array(R, np.complex128)
        delta = loading * float(np.sum(np.diag(RL).real)) / M
        RL[np.diag_indices(M)] += delta
        L = cholesky(RL, lambda k, g: g > 0.0)
        if L is None:
            return np.zeros((n, M), np.complex128)
        Y = {i: forward(L, A[i]) for i in S}
        Z = {i: backward(L, Y[i]) for i in S}
        if rule == MVDR:
            for i in S:
                W[i] = Z[i] / np.vdot(Y[i], Y[i]).real
        else:
            Ym = np.array([Y[i] for i in S]).T  # [M][d]
            Zm = np.array([Z[i] for i in S]).T
            G = Ym.conj().T @ Ym
            Gd = np.diag(G).real.copy()
            C = cholesky(G, lambda k, g: g > PIVOT_REL * Gd[k])
            if C is None:
                return np.zeros((n, M), np.complex128)
            for m in range(M):  # row m of Z G^-1: u = G^-1 conj(Z[m]), w = conj(u)
                u = backward(C, forward(C, np.conj(Zm[m])))
                for r, i in enumerate(S):
                    W[i, m] = np.conj(u[r])
    if not np.all(np.isfinite(W)):
        return np.zeros((n, M), np.complex128)
    return W


def beams(x, W):
    """complex64 [n][N] beams of one window x [N * M] complex64 with its weights W [n][M]; all-zero weights give zeros"""
    n, M = W.shape
    X = np.asarray(x, np.complex64).astype(np.complex128).reshape(-1, M)  # [N][M]
    Y = X @ np.conj(W).T  # [N][n]
    Y[:, ~np.any(W != 0, axis=1)] = 0
    return np.ascontiguousarray(Y.T).astype(np.complex64)
