"""fp64 restatement of (azimuth, elevation) MUSIC (music_b200_create_azel, include/music_b200.h): the grid, the table,
the flat scan, both peak rules and the 2-D refinement, with LAPACK eigenvectors.  Test infrastructure: the definition is
written out literally, step by step, so that it can be read against the header; the product path never imports it.

    az_k = k 360 / n_az,  el_i = el_lo + (i (el_hi - el_lo)) / (n_el - 1)   (degrees; el_0 = el_lo for n_el = 1)
    u = (cos el cos az, cos el sin az, sin el),  a_m = exp(-j 2 pi <p_m, u> / lambda),  b = i n_az + k
"""
import math

import numpy as np

from oracle import music_oracle as mo

import source_count_oracle as so

MAX_IT = 50
TOL = 1e-12
T_MIN = 2.0 ** -30
DEG = math.pi / 180.0


class Grid:
    def __init__(self, n_az, n_el, el_lo, el_hi):
        self.n_az, self.n_el, self.el_lo, self.el_hi = int(n_az), int(n_el), float(el_lo), float(el_hi)
        self.K = self.n_az * self.n_el

    def az_deg(self, k):
        return float(k) * 360.0 / float(self.n_az)

    def el_deg(self, i):
        if self.n_el == 1:
            return self.el_lo
        return self.el_lo + (float(i) * (self.el_hi - self.el_lo)) / float(self.n_el - 1)

    def split(self, b):
        return b // self.n_az, b % self.n_az  # (i, k)


def table(pos, lam, grid):
    """fp64 steering table [n_el][n_az][m] (the device table is this rounded to complex64, within one float32 ulp)"""
    pos = np.asarray(pos, dtype=np.float64)
    out = np.empty((grid.n_el, grid.n_az, pos.shape[0]), np.complex128)
    for i in range(grid.n_el):
        el = grid.el_deg(i) * DEG
        for k in range(grid.n_az):
            az = grid.az_deg(k) * DEG
            ux, uy, uz = math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)
            inner = pos[:, 0] * ux + pos[:, 1] * uy + pos[:, 2] * uz
            ph = 2.0 * math.pi * (inner / lam)
            out[i, k] = np.cos(ph) - 1j * np.sin(ph)
    return out


def noise_subspace(in_c64, m, n, rule=None):
    """(G = the m - d smallest-eigenvalue eigenvectors, d) of one window: d = n, or the MDL / AIC estimate"""
    R = mo.covariance(np.ascontiguousarray(in_c64, dtype=np.complex64), m)
    ev, V = np.linalg.eigh(R)
    d = n if rule is None else so.estimate_source_count(ev, in_c64.shape[0] // m, n, rule)[0]
    return V[:, : m - d], d


def spectrum(G, table_c64):
    """flat fp64 P[b] = 1 / ||G^H a_b||^2 of the (K, m) complex64 table"""
    a = np.asarray(table_c64).reshape(-1, G.shape[0]).astype(np.complex128)
    v = a @ G.conj()
    with np.errstate(divide="ignore", invalid="ignore"):
        return 1.0 / np.sum(np.abs(v) ** 2, axis=1)


def is_local_max(P, b, grid):
    p = P[b]
    if not p > 0.0:
        return False
    i, k = grid.split(b)
    for di in (-1, 0, 1):
        ii = i + di
        if ii < 0 or ii >= grid.n_el:
            continue
        for dk in (-1, 0, 1):
            j = ii * grid.n_az + (k + dk) % grid.n_az
            if j == b:
                continue
            if not (p > P[j] or (p == P[j] and b < j)):
                return False
    return True


def chebyshev(a, b, grid):
    ia, ka = grid.split(a)
    ib, kb = grid.split(b)
    dk = abs(ka - kb)
    return max(min(dk, grid.n_az - dk), abs(ia - ib))


def local_max_mask(P, grid):
    """is_local_max for every b at once (numpy): the same comparisons, neighbour by neighbour"""
    P = np.asarray(P, dtype=np.float64).reshape(grid.n_el, grid.n_az)
    B = np.arange(grid.K).reshape(grid.n_el, grid.n_az)
    with np.errstate(invalid="ignore"):
        ok = P > 0.0
        for di in (-1, 0, 1):
            for dk in (-1, 0, 1):
                if di == 0 and dk == 0:
                    continue
                Q = np.roll(P, -dk, axis=1)
                J = np.roll(B, -dk, axis=1)
                rows = np.arange(grid.n_el) + di
                valid = (rows >= 0) & (rows < grid.n_el)
                Q = Q[np.clip(rows, 0, grid.n_el - 1)]
                J = J[np.clip(rows, 0, grid.n_el - 1)]
                beats = (P > Q) | ((P == Q) & (B < J)) | (J == B)
                ok &= beats | ~valid[:, None]
    return ok.reshape(-1)


def pick_local_maxima_2d(P, n, grid, exclusion=0):
    """bins of the n strongest 2-D local maxima (descending strength, ties to the lowest b), each more than `exclusion`
    (Chebyshev) from every peak taken before it; -1 for unfilled slots"""
    P = np.asarray(P, dtype=np.float64)
    cand = [int(b) for b in np.nonzero(local_max_mask(P, grid))[0]]
    cand.sort(key=lambda b: (-P[b], b))
    taken = []
    for b in cand:
        if len(taken) == n:
            break
        if all(chebyshev(b, t, grid) > exclusion for t in taken):
            taken.append(b)
    return taken + [-1] * (n - len(taken))


def pick_top_bins(P, n):
    return [p[2] for p in mo.pick_top_n(P, n, len(P))]


def decode(bins, P, grid):
    """(azimuth, elevation, level) float32 of the slots"""
    az, el, lv = [], [], []
    for b in bins:
        if b < 0:
            az.append(0.0), el.append(0.0), lv.append(0.0)
            continue
        i, k = grid.split(b)
        az.append(grid.az_deg(k)), el.append(grid.el_deg(i)), lv.append(P[b])
    return np.array(az, np.float32), np.array(el, np.float32), np.array(lv, np.float32)


def work(in_c64, m, n, table_c64, grid, peak="top", exclusion=0, rule=None):
    """One window on the (K, m) complex64 table: dict of bins, azimuth, elevation, levels, P, count, G"""
    G, d = noise_subspace(in_c64, m, n, rule)
    P = spectrum(G, table_c64)
    bins = pick_top_bins(P, d) if peak == "top" else pick_local_maxima_2d(P, d, grid, exclusion)
    bins = list(bins) + [-1] * (n - d)
    az, el, lv = decode(bins, P, grid)
    return {"bins": np.array(bins, np.int32), "azimuth": az, "elevation": el, "levels": lv, "P": P, "count": d, "G": G}


# ---- 2-D refinement ---------------------------------------------------------------------------------------------------
def objective(G, pos, lam, ph, ep):
    """D(ph, ep), gradient (2,) and Hessian (2, 2) for the noise eigenvectors in the columns of G, angles in radians"""
    pos = np.asarray(pos, dtype=np.float64)
    x, y, z = pos[:, 0], pos[:, 1], pos[:, 2]
    sp, cp, se, ce = math.sin(ph), math.cos(ph), math.sin(ep), math.cos(ep)
    h = x * cp + y * sp
    v = y * cp - x * sp
    c = 2.0 * math.pi / lam
    th = c * (ce * h + z * se)
    tp = c * (ce * v)
    te = c * (z * ce - se * h)
    tpp = -c * (ce * h)
    tpe = -c * (se * v)
    tee = -th
    a = np.cos(th) - 1j * np.sin(th)
    da = [-1j * tp * a, -1j * te * a]
    d2 = [[(-tp * tp - 1j * tpp) * a, (-tp * te - 1j * tpe) * a], [None, (-te * te - 1j * tee) * a]]
    d2[1][0] = d2[0][1]
    Gh = G.conj().T
    s = Gh @ a
    su = [Gh @ da[0], Gh @ da[1]]
    D = float(np.sum(np.abs(s) ** 2))
    g = np.array([2.0 * np.sum((np.conj(s) * su[u]).real) for u in range(2)])
    H = np.empty((2, 2))
    for u in range(2):
        for w in range(2):
            H[u, w] = 2.0 * np.sum((np.conj(su[u]) * su[w]).real + (np.conj(s) * (Gh @ d2[u][w])).real)
    return D, g, H


def clamp(v, lo, hi):
    return lo if v < lo else (hi if v > hi else v)


def refine_slot(G, pos, lam, b, grid):
    """One filled slot with flat grid bin b.  Returns a dict: azimuth / elevation (float32 degrees), level (float32),
    kept (bool), x (radians), Db, Dx and the smallest relative gap a decision rested on (margin)"""
    i, k = grid.split(b)
    ph_b = grid.az_deg(k) * DEG
    ep_b = grid.el_deg(i) * DEG
    dph = (360.0 / float(grid.n_az)) * DEG
    dep = ((grid.el_hi - grid.el_lo) / float(grid.n_el - 1)) * DEG if grid.n_el > 1 else 0.0
    plo, phi = ph_b - dph, ph_b + dph
    elo, ehi = max(ep_b - dep, grid.el_lo * DEG), min(ep_b + dep, grid.el_hi * DEG)
    D, g, H = objective(G, pos, lam, ph_b, ep_b)
    Db = D
    x0, x1 = ph_b, ep_b
    margin = math.inf
    for _ in range(MAX_IT):
        if g[0] == 0.0 and g[1] == 0.0:
            break
        det = H[0, 0] * H[1, 1] - H[0, 1] * H[0, 1]
        if H[0, 0] > 0.0 and det > 0.0:
            s0 = -(H[1, 1] * g[0] - H[0, 1] * g[1]) / det
            s1 = -(H[0, 0] * g[1] - H[0, 1] * g[0]) / det
            margin = min(margin, abs(det) / max(abs(H[0, 0] * H[1, 1]), 1e-300))
        else:
            gn = math.sqrt(g[0] * g[0] + g[1] * g[1])
            s0 = -g[0] * dph / gn
            s1 = -g[1] * dph / gn
        s0 = clamp(x0 + s0, plo, phi) - x0
        s1 = clamp(x1 + s1, elo, ehi) - x1
        t = 1.0
        found = None
        while t > T_MIN:
            y0, y1 = x0 + t * s0, x1 + t * s1
            f = objective(G, pos, lam, y0, y1)
            if D != 0.0:
                margin = min(margin, abs(f[0] - D) / abs(D))
            if f[0] <= D:
                found = f
                break
            t *= 0.5
        if found is None:
            break
        step = max(abs(t * s0), abs(t * s1))
        x0, x1 = y0, y1
        D, g, H = found
        if step <= TOL:
            break
    out = {"Db": Db, "Dx": D, "kept": True, "x": (ph_b, ep_b), "margin": margin,
           "azimuth": np.float32(grid.az_deg(k)), "elevation": np.float32(grid.el_deg(i)),
           "level": np.float32(1.0 / Db) if Db != 0.0 else np.float32(np.inf)}
    if (x0 != ph_b or x1 != ep_b) and D <= Db:
        a = math.fmod(x0 * (180.0 / math.pi), 360.0)
        if a < 0.0:
            a += 360.0
        az = np.float32(a)
        if az >= np.float32(360.0) or az == 0.0:
            az = np.float32(0.0)
        out.update(kept=False, x=(x0, x1), azimuth=az, elevation=np.float32(x1 * (180.0 / math.pi)), level=np.float32(1.0 / D))
    return out


def box(b, grid):
    """the refinement box of flat bin b, radians: (plo, phi, elo, ehi)"""
    i, k = grid.split(b)
    ph_b, ep_b = grid.az_deg(k) * DEG, grid.el_deg(i) * DEG
    dph = (360.0 / float(grid.n_az)) * DEG
    dep = ((grid.el_hi - grid.el_lo) / float(grid.n_el - 1)) * DEG if grid.n_el > 1 else 0.0
    return ph_b - dph, ph_b + dph, max(ep_b - dep, grid.el_lo * DEG), min(ep_b + dep, grid.el_hi * DEG)


def steering(pos, lam, az_deg, el_deg):
    """unrounded fp64 steering vector at (az, el) degrees"""
    pos = np.asarray(pos, dtype=np.float64)
    az, el = az_deg * DEG, el_deg * DEG
    u = np.array([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])
    ph = 2.0 * math.pi * ((pos @ u) / lam)
    return np.cos(ph) - 1j * np.sin(ph)


def uca_xyz(m, lam, alternate_z=False):
    """m-element UCA of half-wavelength adjacent spacing in the xy-plane, or with elements alternating at z = +-lam/4"""
    r = 0.5 * lam / math.sin(math.pi / m)
    pos = [[r * math.cos(2 * math.pi * e / m), r * math.sin(2 * math.pi * e / m), 0.0] for e in range(m)]
    if alternate_z:
        for e in range(m):
            pos[e][2] = lam / 4.0 if e % 2 == 0 else -lam / 4.0
    return np.array(pos, np.float64)


def ura_xyz(rows, cols, lam):
    """rows x cols uniform rectangular array in the xy-plane, half-wavelength spacing, centred"""
    d = 0.5 * lam
    return np.array([[(c - (cols - 1) / 2.0) * d, (r - (rows - 1) / 2.0) * d, 0.0] for r in range(rows) for c in range(cols)], np.float64)


def windows(pos, lam, n_of, seed, snaps, el_range=(0.0, 90.0), noise=0.1):
    """complex64 (len(n_of), m * snaps) windows: window w holds n_of[w] unit-power sources at random off-grid (az, el)
    (el uniform in el_range) plus complex white noise of power noise^2 (20 dB at the default).  Returns (x, truth) with
    truth[w] a list of (az, el) degrees."""
    rng = np.random.default_rng(seed)
    m = pos.shape[0]
    xs, truth = [], []
    for S in n_of:
        X = noise * (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
        src = []
        for _ in range(S):
            az, el = rng.uniform(0.0, 360.0), rng.uniform(*el_range)
            X += steering(pos, lam, az, el)[:, None] * np.exp(2j * np.pi * rng.uniform(0.0, 1.0, snaps))[None, :]
            src.append((az, el))
        xs.append(X.T.reshape(-1))  # x(r, c) = in[c * m + r]
        truth.append(src)
    return np.ascontiguousarray(np.array(xs).astype(np.complex64)), truth


def direction_error(az, el, truth_az, truth_el):
    """great-circle angle in degrees between two (az, el) directions"""
    u = lambda a, e: np.array([math.cos(e * DEG) * math.cos(a * DEG), math.cos(e * DEG) * math.sin(a * DEG), math.sin(e * DEG)])
    c = float(np.clip(u(az, el) @ u(truth_az, truth_el), -1.0, 1.0))
    return math.degrees(math.acos(c))
