#!/usr/bin/env python
"""CPU emulation (numpy fp64) of esprit_kernel and esprit_eigvals (gr-baz_b200/csrc/music_esprit.cuh): Psi by
Sherman-Morrison from the signal eigenvectors, the Householder reduction to Hessenberg form, and the single-shift complex
QR with its deflation rule, its Wilkinson and exceptional shifts and its step limit, in the kernel's update order.  The
keyword switches restore the behaviour before the fix (no exceptional shift) and plant the defects that
tests/test_gridless_oracle.py shows the checker failing."""
import math

import numpy as np

EPS = 2.220446049250313e-16
MAX_IT = 30
EXC_EVERY = 10     # an exceptional shift at the 10th and 20th step without a deflation
EXC_SCALE = 0.75   # (LAPACK zlahqr's dat1)
EXC_DIR = complex(0.6, 0.8)  # its direction: a unit vector whose angle is no rational multiple of pi


def psi(Es, den_on=True):
    """(Psi, ok) from the signal eigenvectors Es (M, d): B = E1^H E2, q = r B / (1 - |r|^2), Psi = B + r^H q"""
    M, d = Es.shape
    r = Es[M - 1]
    nr = float(np.sum(r.real ** 2 + r.imag ** 2))
    den = 1.0 - nr
    if not (d > 0 and den > 0.0):
        return None, False
    B = Es[:M - 1].conj().T @ Es[1:]
    q = (r @ B) / (den if den_on else 1.0)
    A = B + np.outer(r.conj(), q)
    return A, bool(np.all(np.isfinite(A)))


def eigvals(A, max_it=MAX_IT, exceptional=True, zero_shift=False):
    """(eigenvalues in deflation order by diagonal position, ok, total QR steps)"""
    A = np.array(A, np.complex128)
    d = A.shape[0]
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
        cols = slice(k, d)
        s = tau * (v.conj() @ A[:, cols])
        A[:, cols] -= np.outer(v, s)
        s = tau * (A @ v)
        A -= np.outer(s, v.conj())
    ev = np.zeros(d, np.complex128)
    hi, its, total = d - 1, 0, 0
    while hi >= 0:
        l = hi
        while l > 0:
            if abs(A[l, l - 1]) <= EPS * (abs(A[l - 1, l - 1]) + abs(A[l, l])):
                break
            l -= 1
        if l == hi:
            ev[hi] = A[hi, hi]
            hi -= 1
            its = 0
            continue
        its += 1
        total += 1
        if its > max_it:
            return ev, False, total
        if exceptional and its % EXC_EVERY == 0 and its < max_it:
            k = hi if its == EXC_EVERY else l
            mu = A[k, k] + EXC_SCALE * abs(A[k, k - 1] if k == hi else A[k + 1, k]) * EXC_DIR
        elif zero_shift:
            mu = 0.0
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
        G = []
        for k in range(l, hi):
            x, y = A[k, k], A[k + 1, k]
            nr = math.sqrt(abs(x) ** 2 + abs(y) ** 2)
            gc, gs = (x / nr, y / nr) if nr > 0.0 else (1.0 + 0j, 0j)
            u, w = A[k, k:hi + 1].copy(), A[k + 1, k:hi + 1].copy()
            A[k, k:hi + 1] = np.conj(gc) * u + np.conj(gs) * w
            A[k + 1, k:hi + 1] = gc * w - gs * u
            G.append((gc, gs))
        for k, (gc, gs) in zip(range(l, hi), G):
            u, w = A[l:hi + 1, k].copy(), A[l:hi + 1, k + 1].copy()
            A[l:hi + 1, k] = u * gc + w * gs
            A[l:hi + 1, k + 1] = w * np.conj(gc) - u * np.conj(gs)
        A[idx, idx] += mu
    return ev, True, total


def esprit_window(V, d, max_it=MAX_IT, exceptional=True, zero_shift=False, den_on=True):
    """One window from the eigenvectors V (M, M, ascending eigenvalues, columns) and d: (eigenvalues or None, total
    QR steps); None where the kernel reports no peaks"""
    M = V.shape[0]
    A, ok = psi(V[:, M - d:], den_on)
    if not ok:
        return None, 0
    ev, ok, total = eigvals(A, max_it, exceptional, zero_shift)
    return (ev if ok else None), total
