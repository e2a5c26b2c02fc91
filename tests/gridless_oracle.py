"""High-precision reference for the gridless ULA peak modes (ROOTS: the Aberth-Ehrlich root finder roots_solve, which
roots_kernel shares with manifold_kernel; ESPRIT: the Hessenberg QR of esprit_eigvals), the bounds a backward-stable
root / eigenvalue solver meets, and the windows that stress them (not a test module; the same shape as eig_oracle.py).

Reference: mpmath at eig_oracle.REF_DPS digits on the fp64 covariance R as given (the GPU's own R wherever R is not
exact, so that neither the covariance's rounding nor the eigensolver's is charged to the root stage beyond its bound).
It restates the definitions of include/music_b200.h, not the kernels' arithmetic: the noise / signal subspaces, the
coefficients c_l, every root of the reduced polynomial (mp.polyroots), the merge and selection of the slot roots, Psi
and its eigenvalues (mp.eig, with left eigenvectors for the condition numbers), the direction and the level 1 / D(t*).

Bounds (one named constant each; eps = 2^-53, beta = eig_oracle's projector bound C_PROJ M eps ||R|| / gap):
    root         |z^ - z| <= (M beta sum_k |z|^k + C_ROOT P eps sum_k |b_k| |z|^k) / |Q'(z)|
                 (a merged double root: the square root of twice that numerator over |Q''(z)|)
    ESPRIT       |phi^ - phi| <= (C_QR d eps ||Psi|| + C_SUB beta (1 + ||Psi||) / sqrt(1 - |r|^2)) / |y^H x|
    angle        compared as cos(t - alpha): |d cpsi| <= lambda / (2 pi |s|) |d arg z| + 2 float32 ulps of t* (in
                 radians) times sin psi; this stays finite at end-fire, where dt / d arg z does not
Windows whose bound exceeds CHECKED (in cpsi) or whose selection is closer than its bound to flipping are counted, not
compared.  A double root (noiseless windows) is known only to the square root of the rounding error, so its bound often
exceeds CHECKED: roots_reference compares it only where both kernel approximants must fall within ROOTS_MERGE of each
other.

One departure from the definition: the kernel deflates an outer coefficient pair only when it is exactly zero, the
reference when it is below 1e-40 |c_0|.  mp.polyroots cannot return the roots at 0 and at infinity that an exactly zero
pair means, and on an exact window mpmath leaves such a pair at about 1e-50 instead of 0.  A pair that small moves the
kept roots by about that much relative, far below every bound, and the slots are the same.
"""
import math

import mpmath as mp
import numpy as np

import eig_oracle as eo
import refine_oracle as ro
from root_music_oracle import MERGE, direction, ula_geometry

EPS = eo.EPS
C_ROOT = 16.0    # backward error of the root finder: C_ROOT P eps sum |b_k| |z|^k (the kernel stops at 8 P eps)
C_QR = 16.0      # backward error of the Hessenberg QR: C_QR d eps ||Psi||
C_SUB = 4.0      # a subspace error beta moves Psi by at most C_SUB beta (1 + ||Psi||) / sigma_min(E1)
CHECKED = 1e-4   # cpsi bounds above this are counted, not compared
F32 = 2.0 ** -23


# ---- reference ------------------------------------------------------------------------------------------------------
def _mpc(x):
    return mp.mpc(float(x.real), float(x.imag))


def subspaces(R, d):
    """mpmath eigen-decomposition of R: (ascending eigenvalues, eigenvector columns, gap at the d boundary, ||R||)"""
    R = np.asarray(R, np.complex128)
    M = R.shape[0]
    A = mp.matrix([[_mpc(R[i, j]) for j in range(M)] for i in range(M)])
    E, Q = mp.eighe(A)
    order = sorted(range(M), key=lambda i: E[i])
    w = [E[i] for i in order]
    V = mp.matrix(M, M)
    for a, k in enumerate(order):
        for i in range(M):
            V[i, a] = Q[i, k]
    gap = float(w[M - d] - w[M - d - 1]) if 0 < d < M else 0.0
    return w, V, gap, float(max(abs(x) for x in w))


def beta(M, norm, gap):
    """the eigensolver's projector bound (inf where the split is undefined)"""
    return eo.proj_bound(M, norm, gap)


def cpsi_of(z, s, lam):
    return min(1.0, max(-1.0, -math.atan2(z.imag, z.real) * lam / (2.0 * math.pi * math.hypot(s[0], s[1]))))


def slot_bound(dz, z, t, s, lam):
    """the cpsi bound of a slot at reference root / eigenvalue z and angle t (degrees) for a z-domain error dz"""
    kap = lam / (2.0 * math.pi * math.hypot(s[0], s[1]))
    darg = dz / max(abs(z) - dz, 1e-300) if dz < abs(z) else math.pi
    sinpsi = math.sqrt(max(0.0, 1.0 - cpsi_of(z, s, lam) ** 2))
    ulp = 2.0 * float(np.spacing(np.float32(max(abs(t), 1e-3)))) * math.pi / 180.0
    return kap * min(darg, math.pi) + sinpsi * ulp + 4.0 * EPS


def _level(G, pos, lam, t, dt):
    """(D at t degrees, an absolute bound on D's change over dt degrees)"""
    D, D1, D2 = ro.objective(G, pos, lam, math.radians(t))
    h = math.radians(dt)
    return D, abs(D1) * h + 0.5 * abs(D2) * h * h


def roots_reference(R, d, pos, lam):
    """ROOTS on R with d sources: dict(slots = [(t*, z, cpsi bound, D, D bound)], margin_ok, beta, t)"""
    ok, _, s = ula_geometry(pos, lam)
    assert ok
    M = R.shape[0]
    with mp.workdps(eo.REF_DPS):
        w, V, gap, norm = subspaces(R, d)
        p = M - d
        c = []
        for l in range(M):
            c.append(mp.fsum(V[i, j] * mp.conj(V[i + l, j]) for j in range(p) for i in range(M - l)))
        tiny = mp.mpf(10) ** (-(eo.REF_DPS - 10)) * abs(c[0])
        t = 0
        while t < M - 1 and abs(c[M - 1 - t]) <= tiny:
            t += 1
        H = M - 1 - t
        P = 2 * H
        b = [mp.conj(c[H - k]) if k < H else c[k - H] for k in range(P + 1)]
        z = mp.polyroots(b[::-1], maxsteps=400, extraprec=200) if P > 0 else []
        G = np.array([[complex(V[i, j]) for j in range(p)] for i in range(M)])
        bt = beta(M, norm, gap)
        ab = [float(abs(x)) for x in b]

        def deriv(zz, m):
            return abs(mp.fsum(b[k] * mp.ff(k, m) * zz ** (k - m) for k in range(m, P + 1)))

        zc = [complex(x) for x in z]
    key = [abs(x) for x in zc]
    dup = [False] * P
    merged = [False] * P
    zz = list(zc)
    for r in range(P):
        dist = [abs(zc[r] - zc[q]) if q != r else math.inf for q in range(P)]
        nn = int(np.argmin(dist))
        dist2 = [abs(zc[nn] - zc[q]) if q != nn else math.inf for q in range(P)]
        if int(np.argmin(dist2)) == r and dist[nn] <= MERGE * max(key[r], key[nn]):
            zz[r] = 0.5 * (zc[r] + zc[nn])
            dup[r] = r > nn
            merged[r] = True
    keys = [1.0 if merged[r] else key[r] for r in range(P)]
    order = sorted(range(P), key=lambda r: (keys[r], dup[r], r))
    kept = order[:H]
    td = {r: direction(zz[r], s, lam) for r in kept}
    slots_idx = sorted(kept, key=lambda r: (-keys[r], td[r], r))[:min(d, H)]
    # the bound of each root
    err = []
    with mp.workdps(eo.REF_DPS):
        for r in range(P):
            a = abs(zc[r])
            num = M * bt * sum(a ** k for k in range(P + 1)) + C_ROOT * P * EPS * sum(ab[k] * a ** k for k in range(P + 1))
            if merged[r]:
                q2 = float(deriv(z[r], 2))
                err.append(math.sqrt(2.0 * num / q2) if q2 > 0 else math.inf)
            else:
                q1 = float(deriv(z[r], 1))
                err.append(num / q1 if q1 > 0 else math.inf)
    # merged roots must merge on the GPU too; a selection margin below the bounds may flip
    margin_ok = all(not merged[r] or 2.0 * err[r] <= MERGE for r in range(P))
    if len(slots_idx) < len(kept):
        a, b2 = slots_idx[-1], sorted(kept, key=lambda r: (-keys[r], td[r], r))[len(slots_idx)]
        margin_ok = margin_ok and abs(keys[a] - keys[b2]) > err[a] + err[b2] and abs(td[a] - td[b2]) > 0
    if H < P:
        a, b2 = order[H - 1], order[H]
        recip = abs(zz[a] * np.conj(zz[b2]) - 1.0) <= err[a] + err[b2] + 1e-12
        margin_ok = margin_ok and (recip or abs(keys[a] - keys[b2]) > err[a] + err[b2])
    slots = []
    for r in slots_idx:
        tt = td[r]
        cb = slot_bound(err[r], zz[r], tt, s, lam)
        dt = math.degrees(cb / max(math.sqrt(max(0.0, 1.0 - cpsi_of(zz[r], s, lam) ** 2)), 1e-300)) if cb < 1 else 360.0
        D, dD = _level(G, pos, lam, tt, min(dt, 360.0))
        slots.append((tt, zz[r], cb, D, dD + M * M * bt + C_ROOT * M * M * EPS))
    return {"slots": slots, "margin_ok": margin_ok, "beta": bt, "t": t, "P": P}


def esprit_reference(R, d, pos, lam):
    """ESPRIT on R with d sources: dict(slots = [(t*, phi, cpsi bound, D, D bound)], margin_ok, ok, beta, psi)"""
    ok, _, s = ula_geometry(pos, lam)
    assert ok
    M = R.shape[0]
    with mp.workdps(eo.REF_DPS):
        w, V, gap, norm = subspaces(R, d)
        p = M - d
        Es = mp.matrix(M, d)
        for i in range(M):
            for a in range(d):
                Es[i, a] = V[i, p + a]
        r2 = mp.fsum(abs(Es[M - 1, a]) ** 2 for a in range(d))
        if not 1 - r2 > 0:
            return {"slots": [], "ok": False, "margin_ok": True, "beta": 0.0}
        E1 = mp.matrix(M - 1, d)
        E2 = mp.matrix(M - 1, d)
        for i in range(M - 1):
            for a in range(d):
                E1[i, a], E2[i, a] = Es[i, a], Es[i + 1, a]
        Psi = mp.inverse(E1.H * E1) * (E1.H * E2)
        ev, L, Rv = mp.eig(Psi, left=True, right=True)
        G = np.array([[complex(V[i, j]) for j in range(p)] for i in range(M)])
        bt = beta(M, norm, gap)
        pn = float(mp.mnorm(Psi, "f"))  # >= ||Psi||_2
        smin = float(mp.sqrt(1 - r2))
        conds = []
        for k in range(d):
            x = Rv.column(k)
            y = L[k, :]
            conds.append(float(mp.norm(x) * mp.norm(y) / abs((y * x)[0])))
        phis = [complex(e) for e in ev]
    slots = []
    for k in range(d):
        dz = conds[k] * (C_QR * d * EPS * pn + C_SUB * bt * (1.0 + pn) / smin)
        tt = direction(phis[k], s, lam)
        cb = slot_bound(dz, phis[k], tt, s, lam)
        sinpsi = math.sqrt(max(0.0, 1.0 - cpsi_of(phis[k], s, lam) ** 2))
        dt = math.degrees(cb / sinpsi) if cb < 1 and sinpsi > 0 else 360.0
        D, dD = _level(G, pos, lam, tt, min(dt, 360.0))
        slots.append((tt, phis[k], cb, D, dD + M * M * bt + C_ROOT * M * M * EPS))
    return {"slots": slots, "ok": True, "margin_ok": True, "beta": bt, "psi": Psi}


def cpsi_dist(c1, c2, kap):
    """|c1 - c2| measured through arg z = -c / kap, wrapped into (-pi, pi]: at |s| = lambda / 2 the end-fire directions
    cpsi = +1 and -1 are the one z = -1, and an eigenvalue or root on either side of the negative axis is either"""
    d = (c2 - c1) / kap
    d = (d + math.pi) % (2.0 * math.pi) - math.pi
    return min(abs(c1 - c2), kap * abs(d))


# ---- how much of each family must be compared ----------------------------------------------------------------------
FLOOR = 0.5
# ROOTS families built on (near-)double roots: a double root on the circle is known only to the square root of the
# rounding error, and a pair 1e-3 .. 1e-6 apart is nearly double, so most of their windows have bounds above CHECKED.
# Their finite-SNR windows (the 60 dB opposite pair, the 40 dB d = M - 1 window) keep a floor; the close pairs and the
# exact comb windows are compared only where the bound allows (the 1e-2 pair, a few combs at M = 16).
ROOTS_FLOOR = {"close pair": 0.0, "comb": 0.0, "extreme": 0.5, "opposite": 0.25}


def floor(mode, family):
    """the share of a family's windows that must be compared"""
    return ROOTS_FLOOR.get(family, FLOOR) if mode == "roots" else FLOOR


# ---- the checker ----------------------------------------------------------------------------------------------------
def check(ref, angles, levels, bins, d, n, pos, lam, K):
    """(worst cpsi error / bound over the compared slots, compared?, message or None).  Every reference slot must be
    filled by a distinct slot within its bound, no other slot filled, and every unfilled slot (0, 0, -1)."""
    _, _, s = ula_geometry(pos, lam)
    alpha = math.atan2(s[1], s[0])
    kap = lam / (2.0 * math.pi * math.hypot(s[0], s[1]))
    slots = ref["slots"]
    f = len(slots)
    if not ref["margin_ok"] or any(sl[2] > CHECKED for sl in slots):
        return 0.0, False, None
    if np.any(bins[f:] != -1) or np.any(angles[f:] != 0.0) or np.any(levels[f:] != 0.0):
        return math.inf, True, "extra or untidy slots: %s %s %s (want %d filled)" % (angles, levels, bins, f)
    if np.any(bins[:f] < 0):
        return math.inf, True, "unfilled slot: %s (want %d)" % (bins, f)
    worst = 0.0
    free = list(range(f))
    for tt, z, cb, D, dD in slots:
        cref = math.cos(math.radians(tt) - alpha)
        errs = [cpsi_dist(math.cos(math.radians(float(angles[i])) - alpha), cref, kap) / cb for i in free]
        i = free[int(np.argmin(errs))]
        e = min(errs)
        if e > 1.0:
            return e, True, "slot at %.9f deg off by %.3g of its bound (got %s)" % (tt, e, angles)
        # the mirror: t* is the lower of alpha +- psi, so the angle itself agrees where sin psi is not small
        dt = abs((float(angles[i]) - tt + 180.0) % 360.0 - 180.0)
        if dt > 1e-3 and abs(math.sin(math.radians(tt) - alpha)) > 1e-3:
            return math.inf, True, "slot at %.9f deg reported as its mirror %.9f" % (tt, float(angles[i]))
        if D > 0 and dD < 0.5 * D:
            L = 1.0 / D
            tol = L * (dD / D) / (1.0 - dD / D) + 2 * F32 * L
            if abs(float(levels[i]) - L) > tol:
                return math.inf, True, "level %.9g, want %.9g +- %.3g" % (float(levels[i]), L, tol)
        worst = max(worst, e)
        free.remove(i)
    return worst, True, None


# ---- windows --------------------------------------------------------------------------------------------------------
N = 256  # snapshots per window


def steering(M, z):
    return np.asarray(z, np.complex128) ** np.arange(M)


def z_of(theta_deg):
    """z0 of a source at theta on the half-wave x-axis ULA (helpers.ula(M, "x"))"""
    return np.exp(-1j * math.pi * math.cos(math.radians(theta_deg)))


def exact_sources(vectors, rng, S=2 ** 20):
    """x [N][M]: vector k on its own snapshots with Gaussian-integer amplitudes of total power S each (every vector has
    entries in {0, +-1, +-i}, so R is exact)"""
    M = len(vectors[0])
    snaps = []
    for v in vectors:
        a = eo.sum_of_squares(S)
        a += [0] * (len(a) % 2)
        for t in range(0, len(a), 2):
            snaps.append(complex(a[t], a[t + 1]) * [1, -1, 1j, -1j][int(rng.integers(0, 4))] * np.asarray(v))
    assert len(snaps) <= N
    x = np.zeros((N, M), np.complex128)
    x[:len(snaps)] = snaps
    x = x[rng.permutation(N)]
    assert np.array_equal(x.astype(np.complex64).astype(np.complex128), x)
    return x.astype(np.complex64)


def random_sources(M, zs, rng, snr_db=None):
    """x [N][M]: independent complex Gaussian sources at the z's, plus unit noise at snr_db (None: noiseless)"""
    X = np.zeros((N, M), np.complex128)
    amp = 1.0 if snr_db is None else 10.0 ** (snr_db / 20.0)
    for z in zs:
        X += amp * np.outer(rng.standard_normal(N) + 1j * rng.standard_normal(N), steering(M, z)) / math.sqrt(2.0)
    if snr_db is not None:
        X += (rng.standard_normal((N, M)) + 1j * rng.standard_normal((N, M))) / math.sqrt(2.0)
    return X.astype(np.complex64)


def comb(M, d, z0):
    """the comb vectors v_j (z0^m on m = j mod d, else 0): they span the steering vectors of z0 e^(2 pi i k / d)"""
    m = np.arange(M)
    return [np.where(m % d == j, z0 ** m, 0) for j in range(d)]


def families(M, seed):
    """[(family, name, x, d, exact)] for an M-element half-wave x-axis ULA"""
    rng = np.random.default_rng(seed)
    out = []
    for d in [d for d in range(2, M) if M % d == 0]:
        for z0 in (1, 1j, -1, -1j):
            out.append(("comb", "d=%d z0=%s" % (d, z0), exact_sources(comb(M, d, z0), rng), d, True))
        zs = [np.exp(2j * math.pi * k / d) * np.exp(0.3j) for k in range(d)]
        out.append(("comb control", "d=%d generic basis" % d, random_sources(M, zs, rng, 60.0), d, False))
    if M % 2 == 0 and M >= 4:
        out.append(("opposite", "+-j exact", exact_sources([steering(M, 1j), steering(M, -1j)], rng), 2, True))
        out.append(("opposite", "+-j 60 dB", random_sources(M, [1j, -1j], rng, 60.0), 2, False))
        if M >= 6:
            out.append(("opposite", "+-j, 1 exact", exact_sources([steering(M, z) for z in (1j, -1j, 1)], rng), 3, True))
    if M >= 3:
        for g in (1e-2, 1e-3, 1e-4, 1e-5, 1e-6):
            zs = [np.exp(0.7j), np.exp(1j * (0.7 + g))]
            out.append(("close pair", "gap %g noiseless" % g, random_sources(M, zs, rng), 2, False))
            out.append(("close pair", "gap %g 60 dB" % g, random_sources(M, zs, rng, 60.0), 2, False))
    for th in (0.0, 180.0, 1e-4, 180.0 - 1e-4):
        out.append(("end-fire", "%g deg" % th, random_sources(M, [z_of(th)], rng, 40.0), 1, False))
    if M >= 3:
        out.append(("end-fire", "0 and 90 exact", exact_sources([steering(M, -1), steering(M, 1)], rng), 2, True))
    for d in range(1, M):
        th = rng.uniform(5.0, 175.0, d)
        out.append(("random d", "d=%d" % d, random_sources(M, [z_of(t) for t in th], rng, 30.0), d, False))
    # d = M - 1: the sources evenly spread in spatial frequency (angles evenly spread crowd them near end-fire, where
    # the split of the last signal eigenvalue falls to ~1e-5 and no fp64 solver resolves them)
    th = np.degrees(np.arccos(np.linspace(-0.9, 0.9, M - 1)))
    out.append(("extreme", "d=M-1 noiseless", random_sources(M, [z_of(t) for t in th], rng), M - 1, False))
    out.append(("extreme", "d=M-1 40 dB", random_sources(M, [z_of(t) for t in th], rng, 40.0), M - 1, False))
    Q = eo.unitary(M, rng)
    for name, lam in eo.prescribed_spectra(M, max(1, M // 2)):
        if M >= 3:
            out.append(("prescribed", name, eo.spectrum_window(lam, Q, N), max(1, M // 2), False))
    return out
