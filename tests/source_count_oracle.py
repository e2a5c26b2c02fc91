"""fp64 restatement of the per-window source count (music_b200_set_source_rule, include/music_b200.h) and of one
window's work() under it.  Test infrastructure: the definition is written out literally, loop by loop, so that it can
be read against the header; the product path never imports this file.

    for d = 0 .. n_max, p = M - d, summing i = 0 .. p-1 in ascending i:
        S = sum l_i,  G = sum log l_i
        L(d)   = N (p log(S / p) - G)
        MDL(d) = L(d) + 1/2 d (2M - d) log N
        AIC(d) = 2 L(d) + 2 d (2M - d)
    d_hat = the smallest d with the minimum criterion (NaN never wins);
    d_hat = 0 when l_0 <= 0 or any eigenvalue is not finite.
"""
import math

import numpy as np

from oracle import music_oracle as mo

RULES = {"mdl": 1, "aic": 2}


def criteria(eigvals, N, n_max, rule):
    """MDL(d) or AIC(d) for d = 0 .. n_max of ascending eigenvalues (fp64 array of n_max + 1)."""
    lam = [float(v) for v in eigvals]
    M = len(lam)
    out = np.full(n_max + 1, np.nan)
    for d in range(n_max + 1):
        p = M - d
        S = 0.0
        G = 0.0
        for i in range(p):
            S += lam[i]
            G += math.log(lam[i])
        L = N * (p * math.log(S / p) - G)
        if rule == "mdl":
            out[d] = L + 0.5 * d * (2 * M - d) * math.log(N)
        elif rule == "aic":
            out[d] = 2.0 * L + 2.0 * d * (2 * M - d)
        else:
            raise ValueError(rule)
    return out


def estimate_source_count(eigvals, N, n_max, rule):
    """(d_hat, criteria array); the criteria are all NaN where the window has no estimate (d_hat = 0 by rule)."""
    lam = np.asarray(eigvals, dtype=np.float64)
    if not (lam[0] > 0.0) or not np.all(np.isfinite(lam)):
        return 0, np.full(n_max + 1, np.nan)
    crit = criteria(lam, N, n_max, rule)
    best = None
    for d in range(n_max + 1):
        if not math.isnan(crit[d]) and (best is None or crit[d] < crit[best]):
            best = d
    return (0 if best is None else best), crit


def margin(crit):
    """relative gap between the best and the runner-up criterion (inf with fewer than two finite values)"""
    c = np.sort(crit[~np.isnan(crit)])
    if len(c) < 2:
        return math.inf
    return (c[1] - c[0]) / max(abs(c[0]), abs(c[1]))


def work(in_c64, m, n_max, table_c64, source_rule, peak="top", exclusion=0):
    """One window through oracle/music_oracle.py::work with the noise subspace of the estimated count: G is the first
    m - d_hat eigenvector columns and the peak pick is limited to d_hat slots (the rest stay (0, 0, -1)).  peak: "top"
    (the reference's n largest bins) or "local" (pick_local_maxima with `exclusion`)."""
    in_c64 = np.ascontiguousarray(in_c64, dtype=np.complex64)
    table_c64 = np.ascontiguousarray(table_c64, dtype=np.complex64)
    K = table_c64.shape[0]
    N = in_c64.shape[0] // m
    R = mo.covariance(in_c64, m)
    eigvals, eigvec = np.linalg.eigh(R)
    d, crit = estimate_source_count(eigvals, N, n_max, source_rule)
    G = eigvec[:, 0 : m - d]
    a = table_c64.astype(np.complex128)
    v = a @ G.conj()
    nrm = np.sqrt(np.sum(np.abs(v) ** 2, axis=1))
    with np.errstate(divide="ignore", invalid="ignore"):
        P = 1.0 / (nrm * nrm)
    picks = mo.pick_top_n(P, d, K) if peak == "top" else mo.pick_local_maxima(P, d, K, exclusion)
    picks = picks + [(0.0, 0.0, -1)] * (n_max - d)
    return {"count": d, "criteria": crit, "eigvals": eigvals, "P": P,
            "angles": np.array([p[0] for p in picks], dtype=np.float32),
            "levels": np.array([p[1] for p in picks], dtype=np.float32),
            "bins": np.array([p[2] for p in picks], dtype=np.int32)}


def mixed_windows(m, N, K, seed, per=3, snr_db=20.0, counts=(0, 1, 2, 3)):
    """Windows of one shape (m antennas on a uniform circular array, N snapshots, K-bin table) that mix `per` windows
    of each source count in `counts` (gr_baz_b200.synth streams, 20 dB by default).  A UCA, not a ULA: on a ULA a
    source and its mirror image share one steering vector, which makes R rank-deficient.
    Returns (table, windows (W, m * N) complex64, true counts (W,))."""
    from gr_baz_b200 import synth

    xs, truth = [], []
    table = None
    for S in counts:
        cfg = synth.config(4, m=m, n=S, snapshots=N, resolution=K, geometry="uca", snr_db=snr_db)
        if table is None:
            arr = mo.scaled_antenna_array(synth.SPACING, cfg["antenna_array"])
            table = mo.steering_table_c64(arr, K, synth.C_LIGHT / synth.FREQUENCY)
        xs.append(synth.gen_windows_numpy(cfg, seed + 7919 * S, 0, per))
        truth += [S] * per
    return table, np.concatenate(xs), np.array(truth, np.int32)
