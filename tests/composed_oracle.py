"""fp64 oracle of one window under ANY accepted combination of peak mode, estimator, source rule, refinement and
calibration, composed from the feature oracles next to it (nothing is restated here):

    1. covariance   calibration_oracle.covariance, then calibration_oracle.correct(R, g) when gains are set
    2. count        source_count_oracle.estimate_source_count on eigvalsh(R) (FIXED: d = n), with its margin
    3. spectrum     MUSIC: azel_oracle.spectrum over the m - d smallest eigenvectors; MVDR / Bartlett:
                    estimator_oracle.spectrum (the grid spectrum of ROOTS, ESPRIT and DML is MUSIC's)
    4. peaks        grid modes: estimator_oracle.picks; otherwise root_music_oracle / esprit_oracle / dml_oracle.work_R
                    with d = the count
    5. refinement   refine_oracle.refine_slot (MUSIC), estimator_oracle.refine_slot (MVDR, Bartlett)

work_R() runs stages 2-5 on a given covariance (the GPU's own d_R in the GPU tests, so that the conditioning of R does
not blur the later stages); covariance() is stage 1.  Test infrastructure; the product path never imports this file.
"""
import math

import numpy as np

import azel_oracle as ao
import calibration_oracle as co
import dml_oracle as dm
import esprit_oracle as es
import estimator_oracle as eo
import refine_oracle as ro
import root_music_oracle as rm
import source_count_oracle as so

PEAKS = ("top", "local", "roots", "esprit", "dml")
ESTIMATORS = ("music", "mvdr", "bartlett")
RULES = ("fixed", "mdl", "aic")


def modes(peak="top", exclusion=0, est="music", loading=0.0, rule="fixed", refine=False):
    """the settings of one handle, every one at its default unless given"""
    assert peak in PEAKS and est in ESTIMATORS and rule in RULES
    return {"peak": peak, "exclusion": int(exclusion), "est": est, "loading": float(loading), "rule": rule,
            "refine": bool(refine)}


def covariance(x, m, gains=None):
    """stage 1: the fp64 covariance of each window of x (W, N * m) complex64, corrected for the gains when given"""
    R = co.covariance(x, m)
    return R if gains is None else np.array([co.correct(r, gains) for r in R])


def count(R, N, n, rule):
    """stage 2: (d, margin of the criterion; inf under FIXED)"""
    if rule == "fixed":
        return n, math.inf
    d, crit = so.estimate_source_count(np.linalg.eigvalsh(R), N, n, rule)
    return d, so.margin(crit)


def spectrum(R, table, est, loading, d):
    """stage 3: fp64 P[k] of the estimator (MUSIC over the m - d smallest eigenvectors)"""
    if est == "music":
        _, V = np.linalg.eigh(R)
        return ao.spectrum(V[:, : R.shape[0] - d], table)
    return eo.spectrum(R, table, est, loading)


def work_R(R, md, table, geometry, n, N):
    """Stages 2-5 on one covariance R (m, m) under the settings md (modes()); table (K, m) complex64; geometry =
    (positions (m, 2), wavelength) or None for a set_table() table; N snapshots.  Returns a dict: count, margin (of the
    count), bins, angles, levels (n slots each), P (fp64 grid spectrum), and per slot `flip`, how close the oracle's
    own decision behind that slot is to going the other way (inf where nothing is close)."""
    R = np.asarray(R, np.complex128)
    K, M = np.asarray(table).reshape(-1, R.shape[0]).shape
    d, margin = count(R, N, n, md["rule"])
    grid_est = md["est"] if md["peak"] in ("top", "local") else "music"
    P = spectrum(R, table, grid_est, md["loading"], d)
    flip = np.full(n, math.inf)
    peak = md["peak"]
    if peak in ("top", "local"):
        angles, levels, bins = eo.picks(P, n, K, peak, md["exclusion"], d)
    else:
        pos, lam = geometry if geometry is not None else (None, None)
        if peak == "roots":
            r = rm.work_R(R, pos, lam, K, n, d=d)
        elif peak == "esprit":
            r = es.work_R(R, pos, lam, K, n, d=d)
        else:
            r = dm.work_R(R, table, n, d)
        angles, levels, bins = r["angles"].copy(), r["levels"].copy(), r["bins"].copy()
        flip[:] = r["margin"]
    if md["refine"]:
        pos, lam = geometry
        _, V = np.linalg.eigh(R)
        G = V[:, : M - d]
        for i, b in enumerate(bins):
            if b < 0:
                continue
            if md["est"] == "music":
                s = ro.refine_slot(G, pos, lam, int(b), K)
            else:
                s = eo.refine_slot(R, md["est"], md["loading"], pos, lam, int(b), K)
            angles[i], levels[i] = s["angle"], s["level"]
            flip[i] = ro.flip_margin(s)
    return {"count": d, "margin": margin, "bins": np.asarray(bins, np.int32), "angles": np.asarray(angles, np.float32),
            "levels": np.asarray(levels, np.float32), "P": P, "flip": flip}
