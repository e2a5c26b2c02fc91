"""fp64 restatement of the co-array handle (music_b200_create_coarray, include/music_b200.h): the hole-free extent, the
lag table, R -> R_ss, the virtual ULA and the create checks.  Test infrastructure; the product path never imports this
file.

    U = the largest value with every lag 0 .. U - 1 some p_i - p_j;  2 <= Mv <= min(U, 16), mv = 0 -> min(U, 16)
    lag table: for l < Mv the pairs (i, j) with p_i - p_j = l in ascending i
    z_l = (1 / c_l) sum R_ij over the lag-l pairs in table order
    T_ab = z_{a-b} (a >= b), conj(z_{b-a}) (a < b);  R_ss = (1 / Mv) T T^H, entries a >= b summed over k ascending, the
    upper triangle the conjugate mirror, the diagonal real
    virtual table: the plain set_geometry() table of the Mv-element ULA at l s
"""
import math

import numpy as np

import esprit_oracle
import root_music_oracle

MAX_M = 16
EINVAL = -1


def hole_free_extent(p):
    """U: the first lag 0, 1, ... that no p_i - p_j has"""
    lags = {int(a) - int(b) for a in p for b in p if a >= b}
    U = 0
    while U in lags:
        U += 1
    return U


def resolve_mv(p, mv=0):
    """the virtual size a handle runs with, or None when mv is not valid for p"""
    cap = min(hole_free_extent(p), MAX_M)
    mv = cap if mv == 0 else mv
    return mv if 2 <= mv <= cap else None


def lag_table(p, mv):
    """[l] -> the pairs (i, j) with p_i - p_j = l, in ascending i"""
    m = len(p)
    return [[(i, j) for i in range(m) for j in range(i + 1) if int(p[i]) - int(p[j]) == l] for l in range(mv)]


def lags_z(R, table):
    """z_l = (1 / c_l) sum R_ij over the lag-l pairs in table order"""
    z = np.zeros(len(table), np.complex128)
    for l, pairs in enumerate(table):
        s = 0j
        for i, j in pairs:
            s += R[i, j]
        z[l] = s / len(pairs)
    return z


def toeplitz(z):
    mv = len(z)
    return np.array([[z[a - b] if a >= b else np.conj(z[b - a]) for b in range(mv)] for a in range(mv)])


def smoothed(R, p, mv):
    """R_ss (Mv, Mv) of one physical covariance R (m, m), literally in the definition's summation order"""
    T = toeplitz(lags_z(R, lag_table(p, mv)))
    out = np.zeros((mv, mv), np.complex128)
    for a in range(mv):
        for b in range(a + 1):
            acc = 0j
            for k in range(mv):
                acc += T[a, k] * np.conj(T[b, k])
            acc /= mv
            if a == b:
                acc = complex(acc.real, 0.0)
            out[a, b] = acc
            out[b, a] = np.conj(acc)
    return out


def smoothed_batch(R, p, mv):
    """R_ss [W][Mv][Mv] of R [W][m][m], vectorised (equal to smoothed() up to summation rounding)"""
    table = lag_table(p, mv)
    z = np.stack([sum(R[:, i, j] for i, j in pairs) / len(pairs) for pairs in table], axis=1)
    idx = np.arange(mv)
    d = idx[:, None] - idx[None, :]
    T = np.where(d >= 0, z[:, np.abs(d)], np.conj(z[:, np.abs(d)]))
    return T @ np.conj(np.transpose(T, (0, 2, 1))) / mv


def virtual_positions(step_xy, mv):
    """[Mv][x, y] of the virtual ULA l s (metres)"""
    return np.array([[l * float(step_xy[0]), l * float(step_xy[1])] for l in range(mv)], np.float64)


def steering(pos, lam, deg):
    """a(theta) [.., M], exp(-j 2 pi <p, u(theta)> / lambda)"""
    t = np.radians(np.asarray(deg, np.float64))[..., None]
    return np.exp(-2j * np.pi * (pos[:, 0] * np.cos(t) + pos[:, 1] * np.sin(t)) / lam)


def physical_positions(p, step_xy):
    return np.array([[int(q) * float(step_xy[0]), int(q) * float(step_xy[1])] for q in p], np.float64)


def exact_covariance(pos, lam, deg, powers, noise):
    """A P A^H + sigma^2 I"""
    A = steering(pos, lam, np.asarray(deg, np.float64)).T
    return (A * np.asarray(powers, np.float64)[None, :]) @ A.conj().T + noise * np.eye(pos.shape[0])


def esprit(Rss, step_xy, lam, K, n):
    """ESPRIT on R_ss: esprit_oracle on the virtual ULA"""
    return esprit_oracle.work_R(Rss, virtual_positions(step_xy, Rss.shape[0]), lam, K, n)


def roots(Rss, step_xy, lam, K, n):
    """root-MUSIC on R_ss: root_music_oracle on the virtual ULA"""
    return root_music_oracle.work_R(Rss, virtual_positions(step_xy, Rss.shape[0]), lam, K, n)


def check_create(m, n, nsamples, resolution, positions, step_xy, lam, mv):
    """EINVAL or 0: the argument checks of music_b200_create_coarray"""
    if not 2 <= m <= MAX_M or positions is None or len(positions) < m:
        return EINVAL
    p = [int(q) for q in positions[:m]]
    if p[0] != 0 or any(b <= a for a, b in zip(p, p[1:])):
        return EINVAL
    if nsamples == 0 or nsamples % m:
        return EINVAL
    if resolution == 0:
        return EINVAL
    if not (lam > 0 and math.isfinite(lam)) or not all(math.isfinite(v) for v in step_xy):
        return EINVAL
    s = math.hypot(step_xy[0], step_xy[1])
    if not (s > 0.0) or s > 0.5 * lam * (1.0 + 1e-12):
        return EINVAL
    v = resolve_mv(p, mv)
    if v is None or not 1 <= n < v:
        return EINVAL
    return 0


def circ(a, b):
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) % 360.0
    return np.minimum(d, 360.0 - d)


def worst_error(angles, truth):
    """the largest distance from a true angle to its nearest reported angle (degrees)"""
    return max(float(np.min(circ(angles, t))) for t in truth)
