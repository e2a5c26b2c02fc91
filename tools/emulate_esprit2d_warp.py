#!/usr/bin/env python
"""CPU emulation (numpy fp64) of esprit2d_kernel (gr-baz_b200/csrc/music_esprit2d.cuh) and the Schur form of
esprit_eigvals (music_esprit.cuh): Psi_j by the warp Cholesky and two triangular solves, Psi_c = Psi_1 + gamma Psi_2,
the Householder reduction with Z accumulated, the single-shift complex QR over zlahqr's whole-row ranges with its
Wilkinson and exceptional shifts, the ztrevc back-substitution and the Rayleigh quotients, in the kernel's order.
`schur_ranges=False` plants the eigenvalues-only ranges (the active block only), a defect tests/test_esprit2d_oracle.py
shows the checker failing."""
import math

import numpy as np

EPS = 2.220446049250313e-16
MAX_IT = 30
EXC_EVERY = 10
EXC_SCALE = 0.75
EXC_DIR = complex(0.6, 0.8)
PIVOT = 2.0 ** -40
GAMMA = complex(0.37, 0.61)
SMIN_ABS = 2.0 ** -1022


def psi(Es, P):
    """Psi_j = G^-1 C for the doublets P [(first, second)] by the right-looking Cholesky of G, or None"""
    d = Es.shape[1]
    f = [a for a, _ in P]
    s = [b for _, b in P]
    G = Es[f].conj().T @ Es[f]
    C = Es[f].conj().T @ Es[s]
    L = np.array(G, np.complex128)
    for k in range(d):
        p = L[k, k].real
        if not p > PIVOT:
            return None
        l = math.sqrt(p)
        L[k, k] = l
        L[k + 1:, k] /= l
        for i in range(k + 1, d):
            for j in range(k + 1, i + 1):
                L[i, j] -= L[i, k] * np.conj(L[j, k])
    X = np.array(C, np.complex128)
    for k in range(d):
        X[k] = (X[k] - L[k, :k] @ X[:k]) / L[k, k].real
    for k in range(d - 1, -1, -1):
        X[k] = (X[k] - L[k + 1:, k].conj() @ X[k + 1:]) / L[k, k].real
    return X if np.all(np.isfinite(X)) else None


def schur(A, schur_ranges=True):
    """(S, Z, ok, QR steps): Psi_c = Z S Z^H by the kernel's Householder + shifted QR with Z accumulated"""
    A = np.array(A, np.complex128)
    d = A.shape[0]
    Z = np.eye(d, dtype=np.complex128)
    for k in range(d - 2):
        x0 = A[k + 1, k]
        sigma = float(np.sum(np.abs(A[k + 2:, k]) ** 2))
        if sigma == 0.0:
            continue
        ax0 = abs(x0)
        nrm = math.sqrt(ax0 * ax0 + sigma)
        ph = x0 / ax0 if ax0 > 0.0 else 1.0
        v = np.zeros(d, np.complex128)
        v[k + 1] = x0 + ph * nrm
        v[k + 2:] = A[k + 2:, k]
        tau = 2.0 / (abs(v[k + 1]) ** 2 + sigma)
        A[:, k:] -= np.outer(v, tau * (v.conj() @ A[:, k:]))
        A -= np.outer(tau * (A @ v), v.conj())
        Z -= np.outer(tau * (Z @ v), v.conj())
    hi, its, total = d - 1, 0, 0
    while hi >= 0:
        l = hi
        while l > 0:
            if abs(A[l, l - 1]) <= EPS * (abs(A[l - 1, l - 1]) + abs(A[l, l])):
                break
            l -= 1
        if l == hi:
            hi -= 1
            its = 0
            continue
        its += 1
        total += 1
        if its > MAX_IT:
            return A, Z, False, total
        if its % EXC_EVERY == 0 and its < MAX_IT:
            k = hi if its == EXC_EVERY else l
            mu = A[k, k] + EXC_SCALE * abs(A[k, k - 1] if k == hi else A[k + 1, k]) * EXC_DIR
        else:
            a, b, c, e = A[hi - 1, hi - 1], A[hi - 1, hi], A[hi, hi - 1], A[hi, hi]
            p = (a - e) * 0.5
            bc = b * c
            q = p * p + bc
            sq = math.sqrt(abs(q)) * np.exp(0.5j * math.atan2(q.imag, q.real))
            if p.real * sq.real + p.imag * sq.imag < 0.0:
                sq = -sq
            den = p + sq
            mu = e - bc / den if abs(den) ** 2 > 0.0 else e
        idx = np.arange(l, hi + 1)
        A[idx, idx] -= mu
        cend = d if schur_ranges else hi + 1
        rbeg = 0 if schur_ranges else l
        Gs = []
        for k in range(l, hi):
            x, y = A[k, k], A[k + 1, k]
            nr = math.sqrt(abs(x) ** 2 + abs(y) ** 2)
            gc, gs = (x / nr, y / nr) if nr > 0.0 else (1.0 + 0j, 0j)
            u, w = A[k, k:cend].copy(), A[k + 1, k:cend].copy()
            A[k, k:cend] = np.conj(gc) * u + np.conj(gs) * w
            A[k + 1, k:cend] = gc * w - gs * u
            Gs.append((gc, gs))
        for k, (gc, gs) in zip(range(l, hi), Gs):
            u, w = A[rbeg:hi + 1, k].copy(), A[rbeg:hi + 1, k + 1].copy()
            A[rbeg:hi + 1, k] = u * gc + w * gs
            A[rbeg:hi + 1, k + 1] = w * np.conj(gc) - u * np.conj(gs)
            u, w = Z[:, k].copy(), Z[:, k + 1].copy()
            Z[:, k] = u * gc + w * gs
            Z[:, k + 1] = w * np.conj(gc) - u * np.conj(gs)
        A[idx, idx] += mu
    return A, Z, True, total


def eigvecs(S, Z):
    """X (columns x_k = Z y_k) from the triangular S by ztrevc's back-substitution"""
    d = S.shape[0]
    Y = np.zeros((d, d), np.complex128)
    for k in range(d):
        skk = S[k, k]
        smin = max(EPS * abs(skk), SMIN_ABS)
        Y[k, k] = 1.0
        for j in range(k - 1, -1, -1):
            s = S[j, k] + S[j, j + 1:k] @ Y[j + 1:k, k]
            den = S[j, j] - skk
            if abs(den) < smin:
                den = smin
            Y[j, k] = -(s / den)
    return Z @ Y


def window(V, d, mx, my, gamma=GAMMA, schur_ranges=True):
    """(phi_1, phi_2, QR steps) of one window from its eigenvectors V (M, M, ascending, columns), or (None, None, steps)
    where the kernel reports no peaks"""
    M = V.shape[0]
    if d <= 0 or d > min((mx - 1) * my, mx * (my - 1)):
        return None, None, 0
    Es = V[:, M - d:]
    P1 = psi(Es, [(k * mx + i, k * mx + i + 1) for k in range(my) for i in range(mx - 1)])
    P2 = psi(Es, [(k * mx + i, (k + 1) * mx + i) for k in range(my - 1) for i in range(mx)]) if P1 is not None else None
    if P2 is None:
        return None, None, 0
    S, Z, ok, steps = schur(P1 + gamma * P2, schur_ranges)
    if not ok:
        return None, None, steps
    X = eigvecs(S, Z)
    xn = np.sum(np.abs(X) ** 2, axis=0)
    f1 = np.einsum("ak,ab,bk->k", X.conj(), P1, X) / xn
    f2 = np.einsum("ak,ab,bk->k", X.conj(), P2, X) / xn
    return f1, f2, steps
