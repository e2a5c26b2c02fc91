"""fp64 restatement of the DML peak mode (MUSIC_B200_PEAKS_DML, include/music_b200.h): deterministic maximum likelihood
by alternating projection over the table rows, and its least-squares levels.  Test infrastructure: the definition is
written out literally, so that it can be read against the header; the product path never imports this file.

    R = the window's covariance, a_k = table row k widened to fp64, d = n or the MDL / AIC count
    S(B)    Q_B = MGS twice of the rows of B in slot order, P = I - Q_B Q_B^H, num = a^H P R P a,
            den = ||a||^2 - ||Q_B^H a||^2, candidate iff den > 2^-30 ||a||^2 and f = num / den is finite;
            the candidate of largest f, ties to the lower bin
    init    slot i = S(slots 0 .. i-1);  sweeps (<= 20, Gauss-Seidel) slot i = S(every other slot) until nothing changes
    levels  A = Q_A T, s2 = (tr R - tr(Q_A^H R Q_A)) / (M - d), p = diag(T^-1 (Q_A^H R Q_A - s2 I) T^-H)
Each search also records the winner's relative margin over the runner-up, so parity tests can tell near-ties from bugs.
"""
import numpy as np

from oracle import music_oracle as mo

import source_count_oracle as so

DEN_MIN = 2.0 ** -30
MAX_SWEEPS = 20


def rows(table_c64, m):
    """(a [K][M] complex128, ||a_k||^2 [K])"""
    a = np.asarray(table_c64).reshape(-1, m).astype(np.complex128)
    return a, np.sum(a.real * a.real + a.imag * a.imag, axis=1)


def mgs2(A):
    """modified Gram-Schmidt applied twice to the columns of A (M x r) in order: (Q, T) with A = Q T"""
    M, r = A.shape
    Q = np.zeros((M, r), np.complex128)
    T = np.zeros((r, r), np.complex128)
    for l in range(r):
        v = A[:, l].copy()
        for _ in range(2):
            for j in range(l):
                c = np.vdot(Q[:, j], v)
                v = v - c * Q[:, j]
                T[j, l] += c
        nrm = float(np.sqrt(np.sum(v.real * v.real + v.imag * v.imag)))
        Q[:, l] = v / nrm
        T[l, l] = nrm
    return Q, T


def search(R, a, na, B):
    """S(B): (winning bin or -1, relative margin over the runner-up, candidate mask, f)"""
    M = R.shape[0]
    if B:
        Q, _ = mgs2(a[list(B)].T)
        P = np.eye(M) - Q @ Q.conj().T
        Rp = P @ R @ P
        proj = a @ Q.conj()  # [K][r] = q_l^H a_k
        den = na - np.sum(proj.real * proj.real + proj.imag * proj.imag, axis=1)
    else:
        Rp = R
        den = na.copy()
    num = np.einsum("ki,ij,kj->k", a.conj(), Rp, a).real
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        f = num / den
        cand = (den > DEN_MIN * na) & np.isfinite(f)
    idx = np.nonzero(cand)[0]
    if idx.size == 0:
        return -1, np.inf, cand, f
    best = int(idx[np.argmax(f[idx])])  # argmax: the first (lowest) bin of the largest f
    rest = np.delete(f[idx], np.argmax(f[idx]))
    margin = np.inf if rest.size == 0 else (f[best] - float(rest.max())) / max(abs(f[best]), np.finfo(float).tiny)
    return best, float(margin), cand, f


def captured(R, a, slots):
    """tr(P_A R) of the rows `slots`"""
    Q, _ = mgs2(a[list(slots)].T)
    return float(np.trace(Q.conj().T @ R @ Q).real)


def levels(R, a, slots):
    """(p [d], s2): the least-squares source powers of the rows `slots` and the noise power"""
    M, d = R.shape[0], len(slots)
    Q, T = mgs2(a[list(slots)].T)
    C = Q.conj().T @ R @ Q
    s2 = (float(np.trace(R).real) - float(np.trace(C).real)) / float(M - d)
    U = np.zeros((d, d), np.complex128)  # T^-1 by back substitution, column by column
    for c in range(d):
        for i in range(c, -1, -1):
            s = (1.0 if i == c else 0.0) - sum(T[i, q] * U[q, c] for q in range(i + 1, c + 1))
            U[i, c] = s / T[i, i].real
    p = np.einsum("la,ab,lb->l", U, C - s2 * np.eye(d), U.conj()).real
    return p, s2


def empty(n):
    return {"angles": np.zeros(n, np.float32), "levels": np.zeros(n, np.float32), "bins": np.full(n, -1, np.int32),
            "margin": np.inf, "sweeps": 0, "trajectory": [], "slots": [], "p": np.zeros(0), "s2": 0.0}


def work_R(R, table_c64, n, d=None):
    """One window from its covariance R; d = n under FIXED, else the source count"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    d = n if d is None else int(d)
    a, na = rows(table_c64, M)
    K = a.shape[0]
    if d == 0 or not np.all(np.isfinite(R)) or not float(np.trace(R).real) > 0.0:
        return empty(n)
    margin = np.inf
    slots, traj = [], []
    for i in range(d):
        k, mg, _, _ = search(R, a, na, slots)
        if k < 0:
            return empty(n)
        margin = min(margin, mg)
        slots.append(k)
    traj.append(captured(R, a, slots))
    sweeps = 0
    for s in range(1, MAX_SWEEPS + 1) if d > 1 else ():
        changed = False
        sweeps = s
        for i in range(d):
            k, mg, _, _ = search(R, a, na, slots[:i] + slots[i + 1:])
            if k < 0:
                return empty(n)
            margin = min(margin, mg)
            changed = changed or k != slots[i]
            slots[i] = k
            traj.append(captured(R, a, slots))
        if not changed:
            break
    p, s2 = levels(R, a, slots)
    order = sorted(range(d), key=lambda i: (-p[i], slots[i]))
    out = empty(n)
    for r, i in enumerate(order):
        out["angles"][r] = np.float32(float(slots[i]) * 360.0 / float(K))
        out["levels"][r] = np.float32(p[i])
        out["bins"][r] = slots[i]
    out.update(margin=margin, sweeps=sweeps, trajectory=traj, slots=list(slots), p=p, s2=s2)
    return out


def work(in_c64, m, n, table_c64, rule=None):
    """One window from its samples: R, the source count (MDL / AIC, or n) and DML"""
    x = np.ascontiguousarray(in_c64, dtype=np.complex64)
    R = mo.covariance(x, m)
    d = n
    if rule is not None:
        d = so.estimate_source_count(np.linalg.eigvalsh(R), x.shape[0] // m, n, rule)[0]
    out = work_R(R, table_c64, n, d)
    out["R"] = R
    out["count"] = d
    return out
