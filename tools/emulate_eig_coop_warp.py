#!/usr/bin/env python
"""CPU emulation (numpy fp64) of eig_coop_warp (gr-baz_b200/csrc/music_kernels.cuh): the warp-cooperative cyclic Jacobi
of the unfused M = 8 / 12 / 16 path and of the fused M = 8 fallback - round-robin parallel ordering, the column then row
updates of each step, its stopping rules and the stable ascending sort.  The keyword switches plant the defects that
tests/test_eig_oracle.py shows the eigensolver checker failing."""
import numpy as np


def pair(M, step, lane):
    if lane == 0:
        p, q = M - 1, step
    else:
        p, q = (step + lane) % (M - 1), (step - lane + (M - 1)) % (M - 1)
    return (p, q) if p < q else (q, p)


def eig(R, stop=1e-29, stagnation=True, off_by_subtraction=False, sweeps_less=0):
    """Returns (ascending eigenvalues, Vt[rank][i], sweeps).  stop: the convergence threshold on off / fro (squared
    norms); stagnation: the kernel's early exit (sweep > 2, off <= 1e-24 fro, less than a factor 4 gained);
    off_by_subtraction: off = fro - sum |a_ii|^2; sweeps_less: stop that many sweeps before the rule would."""
    A = np.array(R, np.complex128)
    M = A.shape[0]
    V = np.eye(M, dtype=np.complex128)
    prev = 1e300
    history = []
    for sweep in range(60):
        fro = float(np.sum(np.abs(A) ** 2))
        off = fro - float(np.sum(np.abs(np.diag(A)) ** 2)) if off_by_subtraction else \
            float(np.sum(np.abs(A - np.diag(np.diag(A))) ** 2))
        if off <= stop * fro or off == 0.0 or (stagnation and sweep > 2 and off <= 1e-24 * fro and off >= 0.25 * prev):
            break
        prev = off
        history.append((A.copy(), V.copy()))
        for step in range(M - 1):
            rots = []
            for lane in range(M // 2):
                p, q = pair(M, step, lane)
                g = A[p, q]
                gg = g.real * g.real + g.imag * g.imag
                rg = 1.0 / np.sqrt(gg) if gg > 0 else 0.0
                theta = min(max(0.5 * (A[q, q].real - A[p, p].real) * rg, -1e150), 1e150)
                t = np.copysign(1.0 / (abs(theta) + np.sqrt(theta * theta + 1.0)), theta) if gg > 0 else 0.0
                c = 1.0 / np.sqrt(t * t + 1.0)
                rots.append((p, q, c, t * c * g * rg))
            for p, q, c, sw in rots:
                ap, aq = A[:, p].copy(), A[:, q].copy()
                A[:, p], A[:, q] = c * ap - np.conj(sw) * aq, sw * ap + c * aq
                vp, vq = V[:, p].copy(), V[:, q].copy()
                V[:, p], V[:, q] = c * vp - np.conj(sw) * vq, sw * vp + c * vq
            for p, q, c, sw in rots:
                bp, bq = A[p, :].copy(), A[q, :].copy()
                A[p, :], A[q, :] = c * bp - sw * bq, np.conj(sw) * bp + c * bq
            for p, q, c, sw in rots:
                A[p, q] = A[q, p] = 0.0
                A[p, p], A[q, q] = A[p, p].real, A[q, q].real
    if sweeps_less and history:
        A, V = history[max(0, len(history) - sweeps_less)]
    w = np.diag(A).real.copy()
    order = np.argsort(w, kind="stable")
    Vt = V[:, order].T.copy()
    ph = np.where(np.abs(Vt[:, 0]) > 0, np.conj(Vt[:, 0]) / np.where(np.abs(Vt[:, 0]) > 0, np.abs(Vt[:, 0]), 1), 1)
    return w[order], Vt * ph[:, None], len(history)
