"""GPU: every accepted combination of peak mode, estimator, source rule, refinement and calibration against one composed
fp64 oracle (tests/composed_oracle.py), the refused combinations against a Python restatement of check_modes(), the
outputs of one combination invariant under which outputs a call asks for, the kernels each call launches against a
Python restatement of the planner, every entry point, sub-batch boundaries with the settings combined, and the
calibration accumulator at multi-CTA sizes.

The oracle runs on the GPU's own covariance (d_R), which is itself checked against the fp64 covariance of the input, so
that the conditioning of R does not blur the later stages."""
import math

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import azel_oracle as ao
import beams_oracle as bo
import calibration_oracle as co
import composed_oracle as cmp
import estimator_oracle as eo
import gpu_harness as gh
import helpers
import refine_oracle as ro
import source_count_oracle as so
from helpers import LAM, check_beams, check_weights, circ, corrupt, near_half, positions, random_gains

pytestmark = pytest.mark.gpu

DEV = gh.DEV
STREAM = gh.stream
FLIP = 1e-9          # decisions the oracle sees this close to flipping may go either way (the feature tests' bound)
COUNT_MARGIN = 1e-6  # counts must be exact wherever the MDL / AIC criterion margin exceeds this
L_RTOL = 1e-5
EXCL = 3
SCAN_B = 8           # windows per scan CTA (music_kernels.cuh): the sub-batch granularity

PEAK_CODES = {"top": 0, "local": 1, "roots": 2, "esprit": 3, "dml": 4}
PEAK_NAMES = {"top": "top_bins", "local": "local_maxima", "roots": "roots", "esprit": "esprit", "dml": "dml"}
EST_CODES = {"music": 0, "mvdr": 1, "bartlett": 2}
RULE_CODES = {"fixed": 0, "mdl": 1, "aic": 2}

# ---- the settings and the Python restatement of check_modes() ---------------------------------------------------------
# peak settings: (peak, exclusion, table kind); "uca" / "ula" are geometric tables (set_geometry), "table" a set_table() one
PEAK_VALUES = [("top", 0, "uca"), ("local", 0, "uca"), ("local", EXCL, "uca"), ("roots", 0, "ula"), ("esprit", 0, "ula"),
               ("dml", 0, "uca"), ("dml", 0, "table")]
EST_VALUES = [("music", 0.0), ("mvdr", 0.01), ("mvdr", 0.0), ("bartlett", 0.0)]


def accepted(peak, excl, est, loading, refine, table, m, N):
    """check_modes() of music_b200.cu (plus the N > m conditions of set_estimator / set_source_rule), restated"""
    if est == "mvdr" and loading == 0.0 and N <= m:
        return False
    if peak in ("roots", "esprit", "dml"):
        if excl != 0 or est != "music" or refine:
            return False
        if peak != "dml" and table != "ula":
            return False
    if refine and table == "table":
        return False
    return True


def value_keys(row):
    """the setting values of a matrix row, one per setting"""
    return [("peak", (row["peak"], row["excl"], row["table"])), ("est", (row["est"], row["loading"])), ("rule", row["rule"]),
            ("refine", row["refine"]), ("calib", row["calib"])]


SHAPES = [(m, n, N) for m in (4, 7, 8, 16) for n in (1, 3 if m >= 7 else 2) for N in (256, 129)]


def base_rows():
    rows = []
    for peak, excl, table in PEAK_VALUES:
        for est, loading in EST_VALUES:
            for refine in (False, True):
                if not accepted(peak, excl, est, loading, refine, table, 4, 129):
                    continue
                for rule in ("fixed", "mdl", "aic"):
                    for calib in (False, True):
                        rows.append({"peak": peak, "excl": excl, "table": table, "est": est, "loading": loading, "rule": rule,
                                     "refine": refine, "calib": calib})
    return rows


def matrix():
    """every accepted combination once, each on a shape picked greedily so that every (setting value, shape) pair occurs;
    pairs still missing get an extra row (a copy of the first row with that value)"""
    covered = set()
    out = []
    for i, r in enumerate(base_rows()):
        keys = value_keys(r)
        best = max(range(len(SHAPES)), key=lambda s: (sum((k, SHAPES[s]) not in covered for k in keys), -((s - i) % len(SHAPES))))
        out.append(dict(r, shape=SHAPES[best]))
        covered |= {(k, SHAPES[best]) for k in keys}
    for r in list(out):
        for k in value_keys(r):
            for s in SHAPES:
                if (k, s) not in covered:
                    out.append(dict(r, shape=s))
                    covered |= {(kk, s) for kk in value_keys(r)}
    return out


MATRIX = matrix()


def row_id(r):
    m, n, N = r["shape"]
    return "%s%s-%s%s-%s%s%s-m%dn%dN%d" % (r["peak"], r["excl"] or "", r["est"], r["loading"] or "", r["rule"],
                                           "-newton" if r["refine"] else "", "-cal" if r["calib"] else "", m, n, N)


# ---- the Python restatement of the planner (plan_call + launch_cov + launch_eig_scan + enqueue_device) ---------------------
def plan(m, n, N, K, r, outs, planar=False, hop=0, beams=False, azel=False):
    """(path, scan, peaks) and the launches per sub-batch of one call; outs: the set of outputs the call asks for among
    spectrum, P64, R, eigvals, bins, counts (angles always), beams (+ weights)"""
    fixed, music = r["rule"] == "fixed", r["est"] == "music"
    local, gridless, dml = r["peak"] == "local", r["peak"] in ("roots", "esprit"), r["peak"] == "dml"
    spec, p64o = "spectrum" in outs, "P64" in outs
    planar_fusable = not planar or (hop % 2 == 0 and N % 2 == 0)
    fusable = (not azel and music and fixed and not r["refine"] and r["peak"] == "top" and n == 1 and not p64o and
               "R" not in outs and "eigvals" not in outs and not beams and not r["calib"])
    fill = 1 if fixed and "counts" in outs else 0
    if fusable and m == 4 and planar_fusable:
        return ("fused4", None, None), fill + 1, 0
    if fusable and m == 8 and not planar and not spec and N >= 128 and N % 2 == 0:
        return ("fused8", None, None), fill + 1, 0
    if planar:
        cov = 1 + ((m + 3) // 4 > 1)
    elif m == 4 or (m in (8, 16) and N >= 128 and N % (16 // m) == 0):
        cov = 1
    elif m % 4 == 0:
        cov = 1 + (m // 4 > 1)
    else:
        cov = 1
    eig = (music and (not dml or spec or p64o)) or not fixed or "eigvals" in outs
    argmax = n == 1 and not local and not gridless and not dml
    if music and (gridless or dml):
        scan = "grid" if spec or p64o else None
        p64 = scan == "grid"
    elif music and argmax and not p64o and not spec and m in (4, 8, 16):
        scan, p64 = "peak1", False
    else:
        scan, p64 = "grid", not argmax or p64o
    peaks = r["peak"] if (gridless or dml or not argmax) else None
    per = (cov + r["calib"] + eig + (not fixed) + (r["est"] == "mvdr") + (scan is not None) + (peaks is not None) + azel +
           r["refine"])
    if beams:
        per += 1 + r["calib"] + ("beams" in outs)
    ws = {"p64": p64 and not p64o, "counts": not fixed, "bins": azel or r["refine"] or (beams and "bins" not in outs),
          "wts": beams and "weights" not in outs}
    return ("unfused", scan, peaks), fill, per, ws


def launches(m, n, N, K, r, outs, W, **kw):
    """kernel launches of one device call of W windows: (kernel key, count)"""
    p = plan(m, n, N, K, r, outs, **kw)
    if p[0][0] != "unfused":
        return p[0], p[1]
    key, fill, per, ws = p
    return key, fill + per * -(-W // sub_windows(m, n, K, ws, W))


def sub_windows(m, n, K, ws, W):
    """max_sub_windows() of music_b200.cu, and the call's sub-batch size"""
    per_win = m * m * 2 * 8 * 2 + m * 8 + (K * 8 if ws["p64"] else 0) + (4 if ws["counts"] else 0) + \
        (n * 4 if ws["bins"] else 0) + (n * m * 16 if ws["wts"] else 0)
    c = (384 << 20) // per_win
    c = max(SCAN_B, min(c, 1 << 20))
    c = c // SCAN_B * SCAN_B
    return min(-(-W // SCAN_B) * SCAN_B, c)


# ---- fixtures ----------------------------------------------------------------------------------------------------------
def ula(m):
    return np.array([[0.5 * LAM * i, 0.0] for i in range(m)])


def ula_windows(pos, N, seed, counts=(0, 1, 2, 3), per=2):
    """x-axis ULA windows mixing 0 to 3 sources at 20 dB, at least 3 degrees from end-fire"""
    rng = np.random.default_rng(seed)
    m = len(pos)
    xs = []
    for S in counts:
        for _ in range(per):
            X = (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N))) / math.sqrt(2.0)
            for t in rng.uniform(3.0, 177.0, min(S, m - 1)):
                s = (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / math.sqrt(2.0)
                X += 10.0 * ro.steering(pos, LAM, math.radians(t))[0][:, None] * s[None, :]
            xs.append(X.T.reshape(-1))
    return np.ascontiguousarray(np.array(xs).astype(np.complex64))


def setup(r, seed, W_per=2):
    """(handle, raw input windows, gains or None, geometry or None) of one matrix row"""
    m, n, N = r["shape"]
    K = 360 if N == 256 else 300
    rng = np.random.default_rng(seed)
    blk = music_doa(m, n, m * N, np.ones((K, m), np.complex64), K)
    geometry = None
    if r["table"] == "ula":
        pos = ula(m)
        x = ula_windows(pos, N, seed, per=W_per)
    else:
        pos = positions("uca", m)
        _, x, _ = so.mixed_windows(m, N, K, seed, per=W_per)
    if r["table"] == "table":
        blk.set_array_response(helpers.planar_table(m, K, seed))
    else:
        blk.set_array_geometry(pos, LAM)
        geometry = (pos, LAM)
    apply(blk, r)
    g = random_gains(rng, m) if r["calib"] else None
    if g is not None:
        blk.set_calibration(g)
        x = corrupt(x, g)
    return blk, x, g, geometry, K


def apply(blk, r):
    blk.set_estimator(r["est"], r["loading"])
    blk.set_source_rule(r["rule"])
    blk.set_peak_mode(PEAK_NAMES[r["peak"]], r["excl"])
    blk.set_refine(r["refine"])


def ulps(a, b):
    return circ(a, b) / float(np.spacing(np.float32(max(abs(float(a)), abs(float(b)), 1e-3))))


# ---- the comparison with the composed oracle ------------------------------------------------------------------------------
class Tally:
    def __init__(self):
        self.slots = self.edge = 0


def check_window(got, ref, r, K, n, tie_rtol, tally, ctx, trR=None, loose=False):
    """one window's angles / levels / bins against the composed oracle; returns False when the window sits on a decision
    edge the oracle itself sees (then it is counted and skipped)"""
    ga, gl, gb = got["angles"], got.get("levels"), got.get("bins")
    d = ref["count"]
    tally.slots += d
    if gb is not None and not np.array_equal(gb, ref["bins"]):
        i = int(np.nonzero(gb != ref["bins"])[0][0])
        b, rb = int(gb[i]), int(ref["bins"][i])
        P = ref["P"]
        if r["peak"] in ("top", "local"):
            tie = b >= 0 and rb >= 0 and abs(P[b] - P[rb]) <= tie_rtol * abs(P[rb])
        elif r["peak"] in ("roots", "esprit"):
            tie = ref["flip"][i] <= FLIP or (b >= 0 and near_half(ref["angles"][i], K) and np.array_equal(np.delete(gb, i), np.delete(ref["bins"], i)))
        else:
            tie = ref["flip"][i] <= FLIP
        assert tie, (ctx, "bins", gb, ref["bins"])
        if not (r["peak"] in ("roots", "esprit") and ref["flip"][i] > FLIP):
            tally.edge += d
            return False
    for i in range(n):
        rb = int(ref["bins"][i])
        if i >= d or rb < 0:
            assert ga[i] == 0.0 and (gl is None or gl[i] == 0.0) and (gb is None or gb[i] == -1), (ctx, i, ga, gl, gb)
            continue
        ra, rl = ref["angles"][i], ref["levels"][i]
        if r["refine"] or r["peak"] in ("roots", "esprit"):
            if ref["flip"][i] <= FLIP and ulps(ga[i], ra) > 2.0:
                tally.edge += 1
                continue
            if loose:
                assert circ(ga[i], ra) <= 1e-4, (ctx, i, ga, ref["angles"])
            elif r["refine"] and r["est"] != "music":
                assert circ(ga[i], ra) <= 1e-4, (ctx, i, ga, ref["angles"])       # test_gpu_estimators.test_refine_1d
            elif r["refine"]:
                assert ulps(ga[i], ra) <= 1.0, (ctx, i, ga, ref["angles"])       # test_gpu_refine
            else:
                assert ulps(ga[i], ra) <= 2.0, (ctx, i, ga, ref["angles"])       # test_gpu_root_music / test_gpu_esprit
        else:
            assert ga[i] == ra, (ctx, i, ga, ref["angles"])
        if gl is not None:
            if r["peak"] == "dml" and not loose:
                ok = abs(float(gl[i]) - float(rl)) <= max(float(np.spacing(np.abs(np.float32(rl)))), 1e-10 * trR)
                assert ok, (ctx, i, gl, ref["levels"])                            # test_gpu_dml.level_ok
            else:
                assert abs(float(gl[i]) - float(rl)) <= L_RTOL * abs(float(rl)), (ctx, i, gl, ref["levels"])
    return True


def close_nan(a, b, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nan = np.isnan(b)
    assert np.array_equal(np.isnan(a), nan)
    return not np.any(~nan) or float(np.max(np.abs(a[~nan] - b[~nan]) / np.abs(b[~nan]))) <= rtol


OUTPUT_SETS = {"all": ("levels", "spectrum", "bins", "P64", "R", "eigvals"), "angles": (), "levels": ("levels",), "bins": ("bins",)}


def same_or_close(a, b, same_kernel, ctx):
    """byte-identical outputs where the plan ran the same peak-stage kernel; otherwise bins and angles identical and
    levels within 1e-12"""
    for k in ("angles", "bins", "counts"):
        if k in a and k in b:
            assert a[k].tobytes() == b[k].tobytes(), (ctx, k)
    if "levels" in a and "levels" in b:
        if same_kernel:
            assert a["levels"].tobytes() == b["levels"].tobytes(), (ctx, "levels")
        else:
            la, lb = a["levels"].astype(np.float64), b["levels"].astype(np.float64)
            assert np.all(np.abs(la - lb) <= 1e-12 * np.abs(lb)), (ctx, "levels", la, lb)


@pytest.mark.parametrize("r", MATRIX, ids=[row_id(r) for r in MATRIX])
def test_matrix_row(r):
    """(b) d_R, counts, bins, angles, levels, spectrum and P64 against the composed oracle; (c) the same outputs whatever
    else a call asks for; (d) every call launches the kernels the planner restatement says"""
    m, n, N = r["shape"]
    blk, x, g, geometry, K = setup(r, 1000 + MATRIX.index(r))
    W = x.shape[0]
    table = blk.array_response_c64()
    md = cmp.modes(r["peak"], r["excl"], r["est"], r["loading"], r["rule"], r["refine"])
    ctx = row_id(r)
    res = {}
    for name, outs in OUTPUT_SETS.items():
        res[name] = gh.device_call(blk, x, outs)
        key, want = launches(m, n, N, K, r, set(outs), W)
        assert res[name][1] == want, (ctx, name, res[name][1], want)
    co_outs = ("levels", "bins", "counts")
    res["counts"] = gh.device_call(blk, x, co_outs)
    key_c, want = launches(m, n, N, K, r, set(co_outs), W)
    assert res["counts"][1] == want, (ctx, "counts", res["counts"][1], want)
    full = res["all"][0]
    # d_R: the corrected fp64 covariance
    R = full["R"]
    if g is not None:
        blk.set_calibration(None)
        raw = gh.device_call(blk, x, ("R",))[0]["R"]
        blk.set_calibration(g)
        want_R = np.array([co.correct(Rw, g) for Rw in raw])
        assert np.all(np.abs(R - want_R) <= 1e-15 * np.abs(want_R)), ctx
    else:
        raw = R
    ref_raw = co.covariance(x, m)
    assert np.max(np.abs(raw - ref_raw)) <= 1e-12 * np.max(np.abs(ref_raw)), ctx
    # (c) output-set invariance
    key_all = launches(m, n, N, K, r, set(OUTPUT_SETS["all"]), W)[0]
    for name in ("angles", "levels", "bins"):
        key = launches(m, n, N, K, r, set(OUTPUT_SETS[name]), W)[0]
        same_or_close(res[name][0], full, key == key_all, (ctx, name))
    same_or_close(res["counts"][0], full, key_c == key_all, (ctx, "counts"))
    counts = res["counts"][0]["counts"]
    # (b) against the oracle on the GPU's own R
    tally = Tally()
    for w in range(W):
        ref = cmp.work_R(R[w], md, table, geometry, n, N)
        wctx = (ctx, w)
        if counts[w] != ref["count"]:
            assert ref["margin"] <= COUNT_MARGIN, (wctx, counts[w], ref["count"], ref["margin"])
            tally.edge += 1
            continue
        P = ref["P"]
        assert close_nan(full["P64"][w], P, L_RTOL), wctx
        assert close_nan(full["spectrum"][w], P, L_RTOL), wctx
        err = full["P64"][w].astype(np.float64) - P
        p_err = float(np.nanmax(np.abs(err / P))) if np.any(np.isfinite(P)) else 0.0
        got = {k: full[k][w] for k in ("angles", "levels", "bins")}
        check_window(got, ref, r, K, n, max(1e-12, 4.0 * p_err), tally, wctx, float(np.trace(R[w]).real))
    assert tally.edge <= max(1, tally.slots // 50), (ctx, tally.edge, tally.slots)
    blk.close()


# ---- (a) accepted and refused combinations -------------------------------------------------------------------------------
def test_check_modes_restatement():
    """every (peak, exclusion, estimator, refinement, table) combination: the C ABI accepts exactly the combinations the
    Python check_modes() accepts, in either setting order and with the table installed first or last (a refused table
    then fails the process call)"""
    L = _capi.load()
    m, n, N, K = 8, 2, 64, 90
    blk = music_doa(m, n, m * N, np.ones((K, m), np.complex64), K)
    h = blk._h
    x = ula_windows(ula(m), N, 3, counts=(2,), per=2)
    d_in = torch.from_numpy(x.view(np.float32)).to(DEV)
    d_ang = torch.zeros((2, n), dtype=torch.float32, device=DEV)
    tables = {"uca": lambda: blk.set_array_geometry(positions("uca", m), LAM), "ula": lambda: blk.set_array_geometry(ula(m), LAM),
              "table": lambda: blk.set_array_response(helpers.planar_table(m, K, 5))}
    n_acc = n_ref = 0
    for peak in PEAK_CODES:
        for excl in (0, EXCL):
            for est, loading in EST_VALUES:
                for refine in (False, True):
                    for tk in tables:
                        ok = accepted(peak, excl, est, loading, refine, tk, m, N)
                        n_acc += ok
                        n_ref += not ok
                        setters = {"peak": lambda: L.music_b200_set_peak_mode(h, PEAK_CODES[peak], excl),
                                   "est": lambda: L.music_b200_set_estimator(h, EST_CODES[est], loading),
                                   "refine": lambda: L.music_b200_set_refine(h, int(refine))}
                        for order, table_last in ((("peak", "est", "refine"), False), (("refine", "est", "peak"), False),
                                                  (("peak", "est", "refine"), True), (("refine", "est", "peak"), True)):
                            ctx = (peak, excl, est, loading, refine, tk, order, table_last)
                            assert L.music_b200_set_refine(h, 0) == 0 and L.music_b200_set_estimator(h, 0, 0.0) == 0
                            assert L.music_b200_set_peak_mode(h, 0, 0) == 0
                            blk.set_array_geometry(ula(m), LAM)
                            if not table_last:
                                tables[tk]()
                            rcs = [setters[s]() for s in order]
                            assert all(rc in (_capi.OK, _capi.EINVAL) for rc in rcs), ctx
                            if table_last:
                                tables[tk]()
                            rc = L.music_b200_process_device(h, d_in.data_ptr(), 2, d_ang.data_ptr(), None, None, None, STREAM())
                            torch.cuda.synchronize()
                            if ok:
                                assert rcs == [0, 0, 0] and rc == 0, (ctx, rcs, rc)
                            else:
                                assert _capi.EINVAL in rcs or rc == _capi.EINVAL, (ctx, rcs, rc)
                                if not table_last:
                                    assert _capi.EINVAL in rcs, (ctx, rcs)
    assert n_acc and n_ref
    blk.close()
    # the snapshot conditions: MDL / AIC and MVDR (and MVDR / LCMV beams) without loading need N > m
    blk = music_doa(8, 2, 8 * 8, np.ones((K, 8), np.complex64), K)
    assert L.music_b200_set_source_rule(blk._h, 1) == _capi.EINVAL and L.music_b200_set_source_rule(blk._h, 2) == _capi.EINVAL
    assert L.music_b200_set_estimator(blk._h, 1, 0.0) == _capi.EINVAL and L.music_b200_set_estimator(blk._h, 1, 0.01) == 0
    assert L.music_b200_set_beamformer(blk._h, 2, 0.0) == _capi.EINVAL and L.music_b200_set_beamformer(blk._h, 3, 0.0) == _capi.EINVAL
    assert not accepted("top", 0, "mvdr", 0.0, False, "uca", 8, 8)
    blk.close()


# ---- (e) every entry point -------------------------------------------------------------------------------------------------
def entry_rows():
    """a subset of the matrix that covers every setting value (and every m) through every entry"""
    keys = {k for r in MATRIX for k in value_keys(r)} | {("m", m) for m, _, _ in SHAPES}
    out, covered = [], set()
    while covered != keys:
        r = max(MATRIX, key=lambda q: len((set(value_keys(q)) | {("m", q["shape"][0])}) - covered))
        out.append(r)
        covered |= set(value_keys(r)) | {("m", r["shape"][0])}
    return out


ENTRY_ROWS = entry_rows()
BEAM_RULES = [("das", 0.0), ("mvdr", 0.01), ("lcmv", 0.01)]
ENTRIES = ("host", "device", "counts", "planar_host", "planar_device", "beams_host", "beams_device", "multi_host", "sharded")


def planar_streams(x, m, N, hop, W):
    """m antenna streams whose windows at hop are the windows of x at hop = N; for hop < N the overlapping windows'
    interleaved form is returned too"""
    X = x.reshape(W, N, m)
    total = (W - 1) * hop + N
    S = np.zeros((m, total), np.complex64)
    for w in range(W):
        S[:, w * hop: w * hop + N] = X[w].T
    xw = np.ascontiguousarray(np.array([S[:, w * hop: w * hop + N].T.reshape(-1) for w in range(W)]))
    return [np.ascontiguousarray(S[r]) for r in range(m)], xw


@pytest.mark.parametrize("r", ENTRY_ROWS, ids=[row_id(r) for r in ENTRY_ROWS])
def test_entries(r):
    """host, device, _counts, planar host / device (hop = N and an overlapping hop), beams host / device and, with two
    or more GPUs, the multi-device host and sharded entries: byte-identical to the device entry (planar at m > 4 against
    the oracle, which the header's R rounding allows); beam weights against beams_oracle on the corrected R"""
    m, n, N = r["shape"]
    blk, x, g, geometry, K = setup(r, 5000 + ENTRY_ROWS.index(r))
    W = x.shape[0]
    table = blk.array_response_c64()
    md = cmp.modes(r["peak"], r["excl"], r["est"], r["loading"], r["rule"], r["refine"])
    ctx = row_id(r)
    dev, _ = gh.device_call(blk, x, ("levels", "bins", "counts"))
    # host
    ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    assert blk.work(W, [x], [ang, lvl]) == W
    same_or_close({"angles": ang, "levels": lvl, "bins": blk.last_bins(), "counts": blk.last_counts()}, dev, True, (ctx, "host"))
    # planar, hop = N and an overlapping hop
    for hop in (N, N // 2 + 1):
        streams, xw = planar_streams(x, m, N, hop, W)
        devw, _ = gh.device_call(blk, xw, ("levels", "bins"))
        key_dev = launches(m, n, N, K, r, {"levels", "bins"}, W)[0]
        ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
        assert blk.work_planar(W, streams, [ang, lvl], hop=hop) == W
        ph = {"angles": ang, "levels": lvl, "bins": blk.last_bins().copy()}
        pd, nl = gh.planar_device_call(blk, streams, hop, W, ("levels", "bins"))
        key_p, want = launches(m, n, N, K, r, {"levels", "bins"}, W, planar=True, hop=hop)
        assert nl == want, (ctx, hop, nl, want)
        same_or_close(ph, pd, True, (ctx, "planar host/device", hop))
        if m <= 4:
            same_or_close(pd, devw, key_p == key_dev, (ctx, "planar", hop))
        else:
            Rq = cmp.covariance(xw, m, g)
            tally = Tally()
            for w in range(W):
                ref = cmp.work_R(Rq[w], md, table, geometry, n, N)
                if r["rule"] != "fixed" and ref["margin"] <= COUNT_MARGIN:
                    continue
                check_window({k: v[w] for k, v in pd.items()}, ref, r, K, n, 1e-9, tally, (ctx, "planar", hop, w),
                             float(np.trace(Rq[w]).real), loose=True)
            assert tally.edge <= max(1, tally.slots // 50), (ctx, tally.edge, tally.slots)
    # beams, device and host
    rule, loading = BEAM_RULES[ENTRY_ROWS.index(r) % len(BEAM_RULES)]
    blk.set_beamformer(rule, loading)
    ex, _ = gh.device_call(blk, x, ("levels", "bins", "R"))
    bd, nl = gh.device_call(blk, x, ("levels", "bins", "counts", "weights", "beams"))
    key, want = launches(m, n, N, K, r, {"levels", "bins", "counts", "weights", "beams"}, W, beams=True)
    assert nl == want, (ctx, "beams", nl, want)
    same_or_close(bd, ex, True, (ctx, "beams vs ex"))
    assert bd["counts"].tobytes() == dev["counts"].tobytes(), ctx
    wc = bd["weights"] if g is None else bd["weights"] / np.conj(co.inverse(g))[None, None, :]
    code = {"das": bo.DAS, "mvdr": bo.MVDR, "lcmv": bo.LCMV}[rule]
    check_weights(wc, ex["R"], bd, code, loading, table, geometry[0] if geometry else None, (ctx, rule))
    check_beams(x, bd["weights"], bd["beams"])
    ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    assert blk.work(W, [x], [ang, lvl]) == W
    hb = {"angles": ang, "levels": lvl, "bins": blk.last_bins(), "counts": blk.last_counts()}
    same_or_close(hb, bd, True, (ctx, "beams host"))
    assert np.array_equal(blk.last_weights(), bd["weights"]) and np.array_equal(blk.last_beams(), bd["beams"]), ctx
    blk.set_beamformer("off", 0.0)
    # multi-device host and sharded entries
    G = torch.cuda.device_count()
    if G >= 2:
        mb = music_doa(m, n, m * N, np.ones((K, m), np.complex64), K, devices=list(range(G)))
        if geometry:
            mb.set_array_geometry(*geometry)
        else:
            mb.set_array_response(table)
        apply(mb, r)
        if g is not None:
            mb.set_calibration(g)
        ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
        assert mb.work(W, [x], [ang, lvl]) == W
        same_or_close({"angles": ang, "levels": lvl, "bins": mb.last_bins(), "counts": mb.last_counts()}, dev, True, (ctx, "multi"))
        for d, sh in enumerate(gh.sharded_call(mb, x, levels=True)):
            assert sh["angles"].tobytes() == dev["angles"][d::G].tobytes(), (ctx, "sharded", d)
            assert sh["levels"].tobytes() == dev["levels"][d::G].tobytes(), (ctx, "sharded", d)
            assert sh["bins"].tobytes() == dev["bins"].tobytes(), (ctx, "sharded bins", d)
        mb.close()
    blk.close()


# ---- (f) az-el ---------------------------------------------------------------------------------------------------------
AZEL_ROWS = [{"peak": p, "excl": EXCL if p == "local" else 0, "est": e, "loading": l, "rule": ru, "refine": rf, "calib": c}
             for p in ("top", "local") for e, l in EST_VALUES for ru in ("fixed", "mdl", "aic") for rf in (False, True)
             for c in (False, True)]


def test_azel_matrix():
    """one az-el shape through peak x estimator x rule x refinement x calibration against azel_oracle and
    estimator_oracle.refine_slot_azel on the corrected fp64 covariance of the input"""
    m, n, snaps = 8, 2, 256
    grid = ao.Grid(36, 10, 0.0, 80.0)
    pos = ao.uca_xyz(m, LAM, alternate_z=True)
    x0, _ = ao.windows(pos, LAM, [0, 1, 2, 2, 1, 0], 7, snaps, (0.0, 80.0))
    g = random_gains(np.random.default_rng(8), m)
    blk = music_doa_azel(m, n, m * snaps, grid.n_az, grid.n_el, (grid.el_lo, grid.el_hi), pos, LAM)
    T = blk.array_response_c64().reshape(grid.K, m)
    edge = slots = 0
    for r in AZEL_ROWS:
        ctx = row_id(dict(r, shape=(m, n, snaps), table="azel"))
        blk.set_refine(False)
        blk.set_estimator(r["est"], r["loading"])
        blk.set_source_rule(r["rule"])
        blk.set_peak_mode(PEAK_NAMES[r["peak"]], r["excl"])
        blk.set_refine(r["refine"])
        blk.set_calibration(g if r["calib"] else None)
        x = corrupt(x0, g) if r["calib"] else x0
        W = len(x)
        o, nl = gh.device_call(blk, x, ("levels", "spectrum", "bins", "counts"))
        key, want = launches(m, n, snaps, grid.K, dict(r, peak=r["peak"]), {"levels", "spectrum", "bins", "counts"}, W, azel=True)
        assert nl == want, (ctx, nl, want)
        got = {k: o[key] for k, key in (("az", "azimuth"), ("el", "elevation"), ("lv", "levels"), ("sp", "spectrum"), ("b", "bins"),
                                         ("c", "counts"))}
        R = cmp.covariance(x, m, g if r["calib"] else None)
        for w in range(W):
            d, margin = cmp.count(R[w], snaps, n, r["rule"])
            if got["c"][w] != d:
                assert margin <= COUNT_MARGIN, (ctx, w)
                edge += 1
                continue
            P = cmp.spectrum(R[w], T, r["est"], r["loading"], d)
            assert close_nan(got["sp"][w], P, L_RTOL), (ctx, w)
            bins = ao.pick_top_bins(P, d) if r["peak"] == "top" else ao.pick_local_maxima_2d(P, d, grid, EXCL)
            bins = np.array(list(bins) + [-1] * (n - d), np.int32)
            slots += d
            gb = got["b"][w]
            if not np.array_equal(gb, bins):
                i = int(np.nonzero(gb != bins)[0][0])
                assert gb[i] >= 0 and bins[i] >= 0 and abs(P[gb[i]] - P[bins[i]]) <= 1e-9 * abs(P[bins[i]]), (ctx, w, gb, bins)
                edge += 1
                continue
            az, el, lv = ao.decode(bins, P, grid)
            _, V = np.linalg.eigh(R[w])
            for i in range(n):
                if bins[i] < 0:
                    assert got["az"][w, i] == 0 and got["el"][w, i] == 0 and got["lv"][w, i] == 0, (ctx, w, i)
                    continue
                if r["refine"]:
                    s = ao.refine_slot(V[:, : m - d], pos, LAM, int(bins[i]), grid) if r["est"] == "music" else \
                        eo.refine_slot_azel(R[w], r["est"], r["loading"], pos, LAM, int(bins[i]), grid)
                    if circ(got["az"][w, i], s["azimuth"]) > 1e-3 or abs(float(got["el"][w, i]) - float(s["elevation"])) > 1e-3:
                        assert abs(s["Dx"] - s["Db"]) <= FLIP * abs(s["Db"]), (ctx, w, i, got["az"][w, i], s)
                        edge += 1
                        continue
                    az[i], el[i], lv[i] = s["azimuth"], s["elevation"], s["level"]
                else:
                    assert got["az"][w, i] == az[i] and got["el"][w, i] == el[i], (ctx, w, i)
                assert abs(float(got["lv"][w, i]) - float(lv[i])) <= L_RTOL * abs(float(lv[i])), (ctx, w, i, got["lv"][w, i], lv[i])
    assert edge <= max(2, slots // 50), (edge, slots)
    blk.close()


# ---- (g) sub-batch boundaries with the settings combined ---------------------------------------------------------------
SUB_CASES = [
    # name, row settings, shape (m, n, N), K, W, outputs of the call, beams
    ("calib_mdl_refine_ws_bins", {"peak": "local", "excl": EXCL, "table": "uca", "est": "music", "loading": 0.0, "rule": "mdl",
                                  "refine": True, "calib": True}, (16, 2, 256), 40000, 3000, ("levels", "counts"), False),
    ("dml_spectrum", {"peak": "dml", "excl": 0, "table": "uca", "est": "music", "loading": 0.0, "rule": "fixed", "refine": False,
                      "calib": False}, (8, 2, 256), 100000, 1100, ("levels", "bins", "spectrum"), False),
    ("mvdr_local_beams_ws_wts", {"peak": "local", "excl": EXCL, "table": "uca", "est": "mvdr", "loading": 0.01, "rule": "fixed",
                                 "refine": False, "calib": False}, (8, 2, 256), 100000, 1100, ("levels", "bins", "counts", "beams"), True),
]


@pytest.mark.parametrize("name,r,shape,K,W,outs,beams", SUB_CASES, ids=[c[0] for c in SUB_CASES])
def test_sub_batches(name, r, shape, K, W, outs, beams):
    """three or more sub-batches, the last one ragged: the whole call equals per-range calls bit for bit, and the oracle
    holds on both sides of every boundary"""
    m, n, N = shape
    rng = np.random.default_rng(77)
    pos = positions("uca", m)
    blk = music_doa(m, n, m * N, np.ones((K, m), np.complex64), K)
    blk.set_array_geometry(pos, LAM)
    apply(blk, r)
    _, x, _ = so.mixed_windows(m, N, 360, 78, per=-(-W // 4))  # (the windows do not depend on the table size)
    x = x[:W]
    g = random_gains(rng, m) if r["calib"] else None
    if g is not None:
        blk.set_calibration(g)
        x = corrupt(x, g)
    if beams:
        blk.set_beamformer("mvdr", 0.01)
    d_in = torch.from_numpy(x.view(np.float32).reshape(-1)).to(DEV)
    shapes = {"levels": ((n,), torch.float32), "bins": ((n,), torch.int32), "spectrum": ((K,), torch.float32),
              "counts": ((), torch.int32), "beams": ((n, N, 2), torch.float32)}

    def run(lo, hi, into):
        ptr = lambda k: into[k][lo:hi].data_ptr() if k in into else None
        l0 = blk.launch_count()
        win = d_in[lo * m * N * 2:].data_ptr()
        if beams:
            blk.process_device_beams(win, hi - lo, ptr("angles"), ptr("levels"), ptr("spectrum"), ptr("bins"), ptr("counts"), None,
                                     ptr("beams"), stream=STREAM())
        else:
            blk.process_device(win, hi - lo, ptr("angles"), ptr("levels"), ptr("spectrum"), ptr("bins"), stream=STREAM(),
                               d_counts=ptr("counts"))
        torch.cuda.synchronize()
        return blk.launch_count() - l0

    def buffers():
        o = {"angles": torch.full((W, n), gh.SENTINEL, dtype=torch.float32, device=DEV)}
        for k in outs:
            o[k] = torch.full((W,) + shapes[k][0], gh.SENTINEL, dtype=shapes[k][1], device=DEV)
        return o

    whole = buffers()
    p = plan(m, n, N, K, r, set(outs), beams=beams)
    key, fill, per, ws = p
    sub = sub_windows(m, n, K, ws, W)
    nsub = -(-W // sub)
    assert nsub >= 3 and W % sub != 0, (sub, nsub)
    assert run(0, W, whole) == fill + per * nsub
    parts = buffers()
    for lo in range(0, W, sub):
        assert run(lo, min(W, lo + sub), parts) == fill + per
    for k in whole:
        assert torch.equal(whole[k].view(torch.int32) if whole[k].dtype != torch.int32 else whole[k],
                           parts[k].view(torch.int32) if parts[k].dtype != torch.int32 else parts[k]), (name, k)
    # the oracle on the first and last windows and on both sides of every boundary (d_R of those windows alone)
    idx = sorted({0, W - 1} | {w for b in range(sub, W, sub) for w in (b - 1, b) if w < W})
    xs = np.ascontiguousarray(x[idx])
    sel = {k: v.cpu().numpy()[idx] for k, v in whole.items()}
    blk.set_beamformer("off", 0.0)
    ex, _ = gh.device_call(blk, xs, ("levels", "bins", "R"))
    table = blk.array_response_c64()
    md = cmp.modes(r["peak"], r["excl"], r["est"], r["loading"], r["rule"], r["refine"])
    tally = Tally()
    for j, w in enumerate(idx):
        ref = cmp.work_R(ex["R"][j], md, table, (pos, LAM), n, N)
        got = {k: v[j] for k, v in sel.items() if k in ("angles", "levels", "bins")}
        if "counts" in sel and sel["counts"][j] != ref["count"]:
            assert ref["margin"] <= COUNT_MARGIN, (name, w)
            continue
        if "spectrum" in sel:
            assert close_nan(sel["spectrum"][j], ref["P"], L_RTOL), (name, w)
        check_window(got, ref, r, K, n, 1e-9, tally, (name, w), float(np.trace(ex["R"][j]).real))
    assert tally.edge <= 1, (name, tally.edge)
    if beams:
        # the beams of the boundary windows equal a call that also returns the weights, which match the oracle
        blk.set_beamformer("mvdr", 0.01)
        bd, _ = gh.device_call(blk, xs, ("levels", "bins", "counts", "weights", "beams"))
        bw = np.ascontiguousarray(sel["beams"]).view(np.float32)
        assert np.ascontiguousarray(bd["beams"]).view(np.float32).tobytes() == bw.tobytes(), name
        check_weights(bd["weights"], ex["R"], bd, bo.MVDR, 0.01, table, pos, name)
    blk.close()


# ---- 3. the calibration accumulator at multi-CTA sizes -----------------------------------------------------------------
CALIB_W = [64, 65, 128 * 64, 65536, 65537]   # 1, 2 and 128 CTAs, the 1024-CTA cap, then more than 64 windows per CTA


@pytest.mark.parametrize("m", [2, 5, 16])
def test_calibration_accumulator_sizes(m):
    """calib_solve on W windows = calibration_oracle.solve on numpy's fp64 mean (the bounds of
    test_gpu_calibration.test_estimator); a repeated call sequence gives bit-identical gains (the CTA counter re-arms);
    host and device accumulation over the same split agree bit for bit.  At m = 16 the largest W run in two sub-batches."""
    N, az = 16, 40.0
    pos = ula(2) if m == 2 else positions("uca", m)
    kind = "phase" if m == 2 else "gain_phase"
    rng = np.random.default_rng(300 + m)
    g = random_gains(rng, m)
    a0 = co.steering_1d(pos, LAM, az)
    blk = music_doa(m, 1, m * N, np.ones((360, m), np.complex64), 360)
    blk.set_array_geometry(pos, LAM)
    Wmax = max(CALIB_W)
    X = (rng.standard_normal((Wmax, N, m)) + 1j * rng.standard_normal((Wmax, N, m))) / math.sqrt(2.0)
    s = (rng.standard_normal((Wmax, N)) + 1j * rng.standard_normal((Wmax, N))) / math.sqrt(2.0)
    X += 10.0 * s[:, :, None] * a0[None, None, :]
    xr = (X * g[None, None, :]).reshape(Wmax, N * m).astype(np.complex64)
    d_all = torch.from_numpy(xr.view(np.float32).reshape(-1)).to(DEV)
    step = m * N * 2
    chunk = max(1, min(Wmax, (32 << 20) // (m * N * 8)))  # the host entry's staging chunk
    for W in CALIB_W:
        ctx = (m, W)
        x = xr[:W]
        ref, rho_ref, sw_ref = co.solve(co.covariance(x, m).mean(axis=0), a0, co.PHASE if m == 2 else co.GAIN_PHASE)
        # host accumulation (chunks of `chunk` windows)
        blk.calib_reset()
        blk.calib_accumulate(x)
        gh, rho_h, sw_h = blk.calib_solve(az, 0.0, kind)
        assert np.max(np.abs(gh - ref)) <= 1e-9 * np.max(np.abs(ref)), ctx
        assert abs(sw_h - sw_ref) <= 1 and abs(rho_h - rho_ref) <= 1e-9, ctx
        # device accumulation over the same split: the same bits, twice
        for rep in range(2):
            blk.calib_reset()
            for lo in range(0, W, chunk):
                blk.calib_accumulate_device(d_all[lo * step:].data_ptr(), min(chunk, W - lo), stream=STREAM())
            gd = blk.calib_solve(az, 0.0, kind)
            assert gd[0].tobytes() == gh.tobytes() and gd[1] == rho_h and gd[2] == sw_h, (ctx, rep)
        # one device call of all W windows (several sub-batches at m = 16): the oracle's bounds, and repeatable
        outs = []
        for rep in range(2):
            blk.calib_reset()
            blk.calib_accumulate_device(d_all.data_ptr(), W, stream=STREAM())
            outs.append(blk.calib_solve(az, 0.0, kind))
        assert outs[0][0].tobytes() == outs[1][0].tobytes(), ctx
        assert np.max(np.abs(outs[0][0] - ref)) <= 1e-9 * np.max(np.abs(ref)), ctx
    blk.close()


# ---- the matrix covers what it claims ---------------------------------------------------------------------------------
# Mutations of the CUDA shim tried on a scratch copy (one build and one run of this file each; never committed), and the
# tests of this file that failed on each.
MUTATIONS = {
    "roots_kernel gets nullptr for cnt": ["test_matrix_row"],
    "planar entries skip calib_apply_kernel": ["test_entries"],
    "p.eig false for DML with the spectrum": ["test_sub_batches"],
}


def test_matrix_self_check():
    """the matrix holds every combination the Python check_modes() accepts (with every rule and calibration), every
    setting value occurs with every m (and with every shape), every setting value and m reach every entry, and each
    listed mutation was caught by a test of this file"""
    combos = {(r["peak"], r["excl"], r["table"], r["est"], r["loading"], r["rule"], r["refine"], r["calib"]) for r in MATRIX}
    for peak, excl, table in PEAK_VALUES:
        for est, loading in EST_VALUES:
            for refine in (False, True):
                for rule in RULE_CODES:
                    for calib in (False, True):
                        ok = all(accepted(peak, excl, est, loading, refine, table, m, N) for m, _, N in SHAPES)
                        assert ok == ((peak, excl, table, est, loading, rule, refine, calib) in combos), (peak, excl, est, refine)
    pairs = {(k, r["shape"]) for r in MATRIX for k in value_keys(r)}
    values = {k for r in MATRIX for k in value_keys(r)}
    assert len(values) == len(PEAK_VALUES) + len(EST_VALUES) + 3 + 2 + 2
    for k in values:
        for s in SHAPES:
            assert (k, s) in pairs, (k, s)
    entry_values = {k for r in ENTRY_ROWS for k in value_keys(r)}
    assert entry_values == values and {r["shape"][0] for r in ENTRY_ROWS} == {m for m, _, _ in SHAPES}
    assert {("peak", p) for p in ("top", "local")} <= {("peak", r["peak"]) for r in AZEL_ROWS}
    names = {n for n in globals() if n.startswith("test_")}
    for mut, caught in MUTATIONS.items():
        assert caught and set(caught) <= names, mut
