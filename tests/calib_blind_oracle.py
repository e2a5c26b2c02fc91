"""fp64 numpy model of receiver self-calibration without a known source (music_b200_calib_blind_*), restating the
definition of include/music_b200.h literally.  It is Weiss-Friedlander eigenstructure calibration (1990) with the
magnitudes read from the diagonal and a multi-start phase search.

Model, as in tests/calibration_oracle.py: x_raw = G (A s + n), G = diag(g).  Input: the segment covariances R_s
[S][M][M] (each the mean raw covariance of `segment` consecutive windows; the sources may move between segments), a
table [K][M] of steering rows a_k, the source count d per segment, the kind, the start count and the seed.

  magnitudes  mag_m = sqrt(sum_s Re R_s,mm / S), scaled to sum mag_m^2 = M; t_m = 1 / mag_m; R_s <- (t_i R_s,ij) t_j.
  projectors  E_s: the M - d smallest-eigenvalue eigenvectors of the whitened R_s; Pi_s = E_s E_s^H.
  starts      phi = 1 for start 0; start p >= 1 draws element m's phase from draw(seed, p, m).
  iteration   per segment: P_s(k) = ||E_s^H (phi o a_k)||^2 / M over the table, and the d best circular local maxima of
              q = 1 / P_s under the local-maximum peak rule (q > 0, q[k] > q[k-1], q[k] >= q[k+1]; larger q first,
              lowest k on ties), in pick order; Q = sum_s sum_i D_k^H Pi_s D_k (D_k = diag(a_k)) in segment then pick
              order, and J = sum_s J_s in segment order with J_s = sum_i P_s(k_s,i) in pick order.  Then phi <- v / |v| element-wise, v the eigenvector of
              the smallest eigenvalue of Q rotated so that v_0 is real and positive.
  schedule    every start runs T1 iterations; the winner is the start with the smallest J of its last iteration (lowest
              index on ties; NaN never wins); it is polished for up to T2 iterations, stopping after the first whose
              max_m |phi_new - phi_old| <= 2^-30.
  outputs     gains mag o phi (GAIN_PHASE) or phi (PHASE); the angles of the final picks; misfit J / (S d) of the last
              iteration; the polish iterations run; the winning start.
"""
import math

import numpy as np

PHASE, GAIN_PHASE = 1, 2
T1, T2 = 24, 30
TOL = 2.0 ** -30
MAX_STARTS = 256
MASK64 = (1 << 64) - 1


def _mix64(z):
    """the splitmix64 finaliser"""
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return z ^ (z >> 31)


def draw(seed, start, element):
    """the phase in [-pi, pi) of element `element` of start `start` (>= 1): z = mix64(seed xor ((start * 256 +
    element + 1) * 0x9E3779B97F4A7C15 mod 2^64)), theta = pi (2 (z >> 11) 2^-53 - 1)"""
    key = ((start * 256 + element + 1) * 0x9E3779B97F4A7C15) & MASK64
    z = _mix64((seed & MASK64) ^ key)
    return math.pi * (2.0 * ((z >> 11) * 2.0 ** -53) - 1.0)


def start_phases(seed, starts, m):
    phi = np.ones((starts, m), np.complex128)
    for p in range(1, starts):
        for e in range(m):
            t = draw(seed, p, e)
            phi[p, e] = complex(math.cos(t), math.sin(t))
    return phi


def collinear(pos):
    """whether the element positions (M, 2) lie on one line (all coincident included)"""
    pos = np.asarray(pos, np.float64)
    d = pos - pos[0]
    f = int(np.argmax(np.sum(d * d, axis=1)))
    L2 = float(np.sum(d[f] * d[f]))
    if L2 == 0.0:
        return True
    cross = d[:, 0] * d[f, 1] - d[:, 1] * d[f, 0]
    return bool(np.max(np.abs(cross)) <= 1e-9 * L2)


def segments(R, segment):
    """the segment covariances of per-window covariances R [W][M][M]: means of `segment` consecutive windows"""
    R = np.asarray(R, np.complex128)
    return R.reshape(-1, segment, R.shape[1], R.shape[2]).sum(axis=1) / segment


def magnitudes(Rs):
    M = Rs.shape[1]
    mag = np.sqrt(np.sum(np.real(np.diagonal(Rs, axis1=1, axis2=2)), axis=0) / Rs.shape[0])
    return mag * math.sqrt(M / np.sum(mag * mag))


def noise_bases(Rs, mag, d):
    """E_s [S][M][M - d] of the whitened segment covariances"""
    t = 1.0 / mag
    Rw = (t[None, :, None] * Rs) * t[None, None, :]
    return np.linalg.eigh(Rw)[1][:, :, :Rs.shape[1] - d]


def spectra(E, phi, table):
    """P_s(k) [S][K] for the phases phi"""
    Y = np.einsum("smj,km->skj", np.conj(E), table * phi[None, :])
    return np.sum(Y.real ** 2 + Y.imag ** 2, axis=2) / table.shape[1]


def minima(P, d):
    """the bins of the d best circular local maxima of q = 1 / P, in pick order (fewer when fewer exist)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        q = 1.0 / P
    ok = (q > 0.0) & (q > np.roll(q, 1)) & (q >= np.roll(q, -1))
    k = np.nonzero(ok)[0]
    order = np.lexsort((k, -q[k]))
    return [int(x) for x in k[order[:d]]]


def iterate(E, Pi, phi, table, d):
    """one iteration's (bins [S][d] with -1 for missing picks, J, Q) at the phases phi"""
    S, M = E.shape[0], table.shape[1]
    P = spectra(E, phi, table)
    bins = -np.ones((S, d), np.int64)
    Q = np.zeros((M, M), np.complex128)
    J = 0.0
    for s in range(S):
        Js = 0.0
        for i, k in enumerate(minima(P[s], d)):
            bins[s, i] = k
            a = table[k]
            Q += (np.conj(a)[:, None] * Pi[s]) * a[None, :]
            Js += P[s, k]
        J += Js
    return bins, J, Q


def update(Q):
    v = np.linalg.eigh(Q)[1][:, 0]
    v = v * (np.conj(v[0]) / abs(v[0]))
    return v / np.abs(v)


def check(Rs, table, d, kind, starts, pos=None):
    """the definition's refusals (ValueError)"""
    S, M = Rs.shape[0], Rs.shape[1]
    if kind not in (PHASE, GAIN_PHASE):
        raise ValueError("unknown kind")
    if M < 3:
        raise ValueError("m < 3")
    if not 1 <= d <= M - 2:
        raise ValueError("d outside 1 .. m - 2")
    if S == 0:
        raise ValueError("no segments")
    if not 1 <= starts <= MAX_STARTS:
        raise ValueError("starts outside 1 .. 256")
    if pos is not None and collinear(pos):
        raise ValueError("collinear")
    if not np.all(np.isfinite(Rs)):
        raise ValueError("not finite")


def solve(Rs, table, d, kind=GAIN_PHASE, starts=32, seed=0, pos=None, trace=False):
    """(gains, angles [S][d] in degrees (NaN for missing picks), misfit, polish iterations, winner) of the segment
    covariances Rs against the table rows; with `trace` also the per-start J of the first phase and the final bins"""
    Rs = np.asarray(Rs, np.complex128)
    table = np.asarray(table, np.complex128)
    check(Rs, table, d, kind, starts, pos)
    S, M, K = Rs.shape[0], Rs.shape[1], table.shape[0]
    mag = magnitudes(Rs)
    if not np.all(np.isfinite(mag)) or not np.all(mag > 0.0):
        raise ValueError("not finite")
    E = noise_bases(Rs, mag, d)
    Pi = np.einsum("smj,snj->smn", E, np.conj(E))
    phis = start_phases(seed, starts, M)
    Js = np.zeros(starts)
    for p in range(starts):
        phi = phis[p]
        for _ in range(T1):
            _, J, Q = iterate(E, Pi, phi, table, d)
            phi = update(Q)
        phis[p], Js[p] = phi, J
    good = [p for p in range(starts) if not math.isnan(Js[p])]
    win = min(good, key=lambda p: (Js[p], p)) if good else 0
    phi = phis[win]
    used = 0
    for _ in range(T2):
        bins, J, Q = iterate(E, Pi, phi, table, d)
        new = update(Q)
        used += 1
        delta = float(np.max(np.abs(new - phi)))
        phi = new
        if delta <= TOL:
            break
    g = phi if kind == PHASE else mag * phi
    angles = np.where(bins >= 0, bins * 360.0 / K, np.nan)
    out = (g, angles, J / (S * d), used, win)
    return out + ((Js, bins) if trace else ())


def normalised(g, kind):
    """the true gains as the estimate reports them: g_0 real positive, then sum |g|^2 = M (GAIN_PHASE) or unit moduli"""
    g = np.asarray(g, np.complex128)
    g = g * (np.conj(g[0]) / abs(g[0]))
    return g / np.abs(g) if kind == PHASE else g * math.sqrt(len(g) / np.sum(np.abs(g) ** 2))


def phase_rms_deg(got, g):
    """RMS phase error in degrees of the estimate against the true gains, both with element 0 real positive"""
    e = np.angle(np.asarray(got) / normalised(g, PHASE))
    return float(math.degrees(math.sqrt(np.mean(e * e))))
