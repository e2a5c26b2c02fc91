"""fp64 restatement of the off-grid peak refinement (music_b200_set_refine, include/music_b200.h) and of one window's
work() under it.  Test infrastructure: the definition is written out literally, step by step, so that it can be read
against the header; the product path never imports this file.  It sits next to the tests, like source_count_oracle.py,
so that the oracle package itself is unchanged.

    a_m(t)  = exp(-j phi_m),  phi_m = 2 pi (px_m cos t + py_m sin t) / lambda,  psi_m = 2 pi (-px_m sin t + py_m cos t) / lambda
    a' = -j psi a,  a'' = (j phi - psi^2) a,  s = G^H a,  s' = G^H a',  s'' = G^H a''
    D = sum |s|^2,  D' = 2 sum Re(conj(s) s'),  D'' = 2 sum (|s'|^2 + Re(conj(s) s''))
    bracket [t_b - delta, t_b + delta], t_b = b 360 / K degrees, delta = 360 / K degrees; rtsafe on D' when
    D'(lo) < 0 < D'(hi); accept t* iff t* != t_b and D(t*) <= D(t_b).
"""
import math

import numpy as np

from oracle import music_oracle as mo

import source_count_oracle as so

MAX_IT = 50
TOL = 1e-12


def steering(pos, lam, t):
    """(a, phi, psi) of the element positions pos (M, 2) at t radians: the unrounded fp64 steering vector"""
    pos = np.asarray(pos, dtype=np.float64)
    st, ct = math.sin(t), math.cos(t)
    phi = 2.0 * math.pi * ((pos[:, 0] * ct + pos[:, 1] * st) / lam)
    psi = 2.0 * math.pi * ((pos[:, 1] * ct - pos[:, 0] * st) / lam)
    a = np.cos(phi) - 1j * np.sin(phi)
    return a, phi, psi


def objective(G, pos, lam, t):
    """D(t), D'(t), D''(t) for the noise eigenvectors in the columns of G (M, p)"""
    a, phi, psi = steering(pos, lam, t)
    a1 = -1j * psi * a
    a2 = (1j * phi - psi * psi) * a
    Gh = G.conj().T
    s, s1, s2 = Gh @ a, Gh @ a1, Gh @ a2
    D = float(np.sum(np.abs(s) ** 2))
    D1 = float(2.0 * np.sum((np.conj(s) * s1).real))
    D2 = float(2.0 * np.sum(np.abs(s1) ** 2 + (np.conj(s) * s2).real))
    return D, D1, D2


def refine_slot(G, pos, lam, b, K):
    """One filled slot with grid bin b.  Returns a dict: angle (float32 degrees), level (float32), kept (bool), theta
    (radians), and the quantities the accept decision rests on (D'(lo), D'(hi), D(t_b), D(t*))."""
    deg_b = float(b) * 360.0 / float(K)
    tb = deg_b * (math.pi / 180.0)
    delta = (360.0 / float(K)) * (math.pi / 180.0)
    Db, f, df = objective(G, pos, lam, tb)
    lo, hi = tb - delta, tb + delta
    fl = objective(G, pos, lam, lo)[1]
    fh = objective(G, pos, lam, hi)[1]
    x = tb
    if fl < 0.0 and fh > 0.0:
        dxold = hi - lo
        dx = dxold
        for _ in range(MAX_IT):
            if f == 0.0:
                break
            if ((x - hi) * df - f) * ((x - lo) * df - f) > 0.0 or abs(2.0 * f) > abs(dxold * df):
                dxold = dx
                dx = 0.5 * (hi - lo)
                x = lo + dx
            else:
                dxold = dx
                dx = f / df
                x = x - dx
            if abs(dx) <= TOL:
                break
            _, f, df = objective(G, pos, lam, x)
            if f < 0.0:
                lo = x
            else:
                hi = x
    out = {"fl": fl, "fh": fh, "Db": Db, "Dx": Db, "kept": True, "theta": tb, "angle": np.float32(deg_b),
           "level": np.float32(1.0 / Db) if Db != 0.0 else np.float32(np.inf)}
    if x != tb:
        Dx = objective(G, pos, lam, x)[0]
        out["Dx"] = Dx
        if Dx <= Db:
            a = math.fmod(x * (180.0 / math.pi), 360.0)
            if a < 0.0:
                a += 360.0
            ang = np.float32(a)
            if ang >= np.float32(360.0) or ang == 0.0:
                ang = np.float32(0.0)
            out.update(kept=False, theta=x, angle=ang, level=np.float32(1.0 / Dx))
    return out


def refine_peaks(G, bins, pos, lam, K, angles, levels):
    """The refinement of one window: every slot with bins[i] >= 0 gets the refined angle and level (copies returned,
    plus the per-slot dicts, None for unfilled slots)."""
    angles = np.array(angles, dtype=np.float32)
    levels = np.array(levels, dtype=np.float32)
    info = []
    for i, b in enumerate(bins):
        if b < 0:
            info.append(None)
            continue
        r = refine_slot(G, pos, lam, int(b), K)
        angles[i], levels[i] = r["angle"], r["level"]
        info.append(r)
    return angles, levels, info


def flip_margin(r):
    """How close (relative) the accept decision of one slot is to flipping: min over D'(lo), D'(hi) relative to the
    larger of the two, and D(t*) - D(t_b) relative to D(t_b)"""
    s = max(abs(r["fl"]), abs(r["fh"]))
    m = min(abs(r["fl"]), abs(r["fh"])) / s if s > 0 else 0.0
    if r["Dx"] != r["Db"] or not r["kept"]:
        m = min(m, abs(r["Dx"] - r["Db"]) / abs(r["Db"]))
    return m


def work(in_c64, m, n, table_c64, pos, lam, peak="top", exclusion=0, rule=None):
    """One window: oracle/music_oracle.py::work (or source_count_oracle.work under MDL / AIC) with LAPACK eigenvectors,
    then the refinement of its filled slots.  peak: "top" or "local"."""
    in_c64 = np.ascontiguousarray(in_c64, dtype=np.complex64)
    K = table_c64.shape[0]
    if rule is None:
        R = mo.covariance(in_c64, m)
        ev, V = np.linalg.eigh(R)
        r = mo.work(in_c64, m, n, table_c64)
        if peak == "local":
            picks = mo.pick_local_maxima(r["P"], n, K, exclusion)
            r["angles"] = np.array([q[0] for q in picks], np.float32)
            r["levels"] = np.array([q[1] for q in picks], np.float32)
            r["bins"] = np.array([q[2] for q in picks], np.int32)
        d = n
    else:
        r = so.work(in_c64, m, n, table_c64, rule, peak=peak, exclusion=exclusion)
        ev, V = np.linalg.eigh(mo.covariance(in_c64, m))
        d = r["count"]
    G = V[:, : m - d]
    ang, lvl, info = refine_peaks(G, r["bins"], pos, lam, K, r["angles"], r["levels"])
    return {"angles": ang, "levels": lvl, "bins": r["bins"], "grid_angles": r["angles"], "grid_levels": r["levels"],
            "P": r["P"], "count": d, "G": G, "info": info}


def angle_error(deg, truth, geometry):
    """Circular distance in degrees; on an x-axis ULA a source at t and its mirror image at -t share one steering
    vector, so the error is to the nearer of the two"""
    e = np.abs((np.asarray(deg, np.float64) - truth + 180.0) % 360.0 - 180.0)
    if geometry == "ula_x":
        e = np.minimum(e, np.abs((np.asarray(deg, np.float64) + truth + 180.0) % 360.0 - 180.0))
    if geometry == "ula_y":
        e = np.minimum(e, np.abs((np.asarray(deg, np.float64) - (180.0 - truth) + 180.0) % 360.0 - 180.0))
    return e
