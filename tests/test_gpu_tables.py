"""GPU: every scan path on arbitrary array-response tables installed with set_array_response - what a calibrated or
measured manifold looks like, unlike the unit-modulus steering tables of the other tests.  Several kernels screen or
guard with quantities relative to each row's own ||a_k||^2 (the fused M = 4 tensor-core screen in fp32, the complement
form's cancellation guard, the high-word screens of scan_peak1_kernel and the fused kernels' fp64 drain), so:

  A. power-of-two table scaling (2^-75 .. 2^100) is exact: P scales by 2^-2s bit for bit, bins do not move;
  B. calibrated tables (per-element gain and phase, per-row 2^j, a small perturbation) against the oracles;
  C. bit-equal duplicated rows placed across screen tiles, the decimated subsample, drain chunks, scan tiles and the
     K - 1 -> 0 wrap: the lower bin wins the tie, n = 2 reports both with equal levels;
  D. zero rows: strength 1 / 0 = +inf, the first zero row wins (Bartlett's 0 / 0 is NaN and is never picked);
  E. shape edges of the fused kernels (K from 1 to 65537) and rough spectra: a random table with ~K/3 local maxima, and
     an az-el table with more than AZEL_LM_CAP (2048) maxima per window.

The oracles: the C oracle (any table), estimator_oracle / azel_oracle on the GPU's own R, and the reference's own work()
stored in tests/golden/reference/tables.npz.  Each call's launch count shows which dispatch branch ran.

The fused M = 4 kernel starts a tensor-core (screen) pass only once one CTA holds FZ_WPT = 8 windows before the launch runs
out of them; with the few windows of groups A - D every window takes its fp64 drain, so there the fused4, fused4_jacobi
and fused4_planar rows cover the drain (as fused4_drain does on purpose) and the launch count cannot tell the two apart.
The screen itself is covered by the tests with thousands of windows and the kernel's trace (MUSIC_B200_TRACE=1), which
counts its passes: test_fused4_screen_on_scaled_and_calibrated_tables (scaling, the table limits, zero rows, ties) and
test_fused_kernels_at_table_edges (the screen's 192-row tiles and decimated subsample)."""
import numpy as np
import pytest
import torch

from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel
from oracle import c_oracle as co
from oracle import music_oracle as mo

import azel_oracle as ao
import estimator_oracle as eo
import helpers

pytestmark = pytest.mark.gpu

SENTINEL = -7
EXCL = 3        # exclusion_bins of the local-maxima paths
P_RTOL = 1e-5
K0 = 3600
W0 = 8

# path: (m, n, N, kernel launches of the call with the path's own outputs, options).  With the few windows of groups
# A - D the fused4* rows all run the fused kernel's fp64 drain, not its tensor-core screen (see the module docstring).
#   env: creation-time switches; spectrum / p64: outputs the call asks for (P64 also brings R); peak: "local";
#   est: (estimator, loading); rule: source rule; planar: the antenna streams entry
PATHS = {
    "fused4":        (4, 1, 256, 1, {}),
    "fused4_drain":  (4, 1, 256, 1, {"env": {"MUSIC_B200_MMA_FIN": "-1"}}),
    "fused4_jacobi": (4, 1, 256, 1, {"env": {"MUSIC_B200_EIG": "jacobi"}}),
    "fused4_spec":   (4, 1, 256, 1, {"spectrum": True}),
    "fused4_planar": (4, 1, 256, 1, {"planar": True}),
    "fused8":        (8, 1, 256, 1, {}),
    "peak1_4":       (4, 1, 256, 3, {"env": {"MUSIC_B200_FUSED": "0"}}),   # cov4_tma, eig, scan_peak1<4>
    "peak1_8":       (8, 1, 129, 4, {}),                                   # cov_tile x2 (odd N), eig_coop, scan_peak1<8>
    "peak1_16":      (16, 1, 256, 3, {}),                                  # covN_tma, eig_coop, scan_peak1<16>
    "scan4":         (4, 1, 256, 3, {"p64": True}),                        # scan_kernel<4>
    "scan8":         (8, 1, 256, 3, {"p64": True, "spectrum": True}),      # scan_kernel<8>
    "scan16":        (16, 1, 256, 3, {"p64": True}),                       # scan_kernel<16>
    "scan7":         (7, 1, 128, 3, {"p64": True, "spectrum": True}),      # generic cov, eig<8>, scan_kernel<0>
    "topn4":         (4, 2, 256, 4, {"spectrum": True}),                   # + topn_kernel
    "topn16":        (16, 3, 256, 4, {}),
    "local4":        (4, 2, 256, 4, {"peak": "local"}),                    # + topn_local_kernel
    "local8":        (8, 1, 256, 4, {"peak": "local"}),
    "mvdr":          (4, 1, 256, 3, {"est": ("mvdr", 0.0), "p64": True}),  # cov, mvdr_prep, scan_quad<4>
    "mvdr_loaded":   (8, 2, 256, 4, {"est": ("mvdr", 0.01), "p64": True}), # + topn_kernel
    "bartlett":      (4, 2, 256, 3, {"est": ("bartlett", 0.0), "p64": True}),  # cov, scan_quad<4>, topn_kernel
    "mdl":           (4, 2, 256, 5, {"rule": "mdl", "p64": True}),         # cov, eig, source count, scan, top-n
}


def make_handle(path, table, monkeypatch):
    m, n, N, _, o = PATHS[path]
    with monkeypatch.context() as mp:
        for k, v in o.get("env", {}).items():
            mp.setenv(k, v)
        blk = music_doa(m, n, N * m, table, table.shape[0])
    if o.get("peak") == "local":
        blk.set_peak_mode("local_maxima", EXCL)
    if "est" in o:
        blk.set_estimator(*o["est"])
    if "rule" in o:
        blk.set_source_rule(o["rule"])
    return blk


def call(blk, path, x, spectrum=None, p64=None):
    """the path's call on windows x; returns (outputs as numpy, kernel launches).  spectrum / p64 override the
    path's own choice of outputs (p64 = True: the unfused fp64 scan with P64 and R)."""
    m, n, N, _, o = PATHS[path]
    K = blk.resolution
    spectrum = o.get("spectrum", False) if spectrum is None else spectrum
    p64 = o.get("p64", False) if p64 is None else p64
    dev = torch.device("cuda:0")
    W = x.shape[0]
    out = {"angles": torch.full((W, n), SENTINEL, dtype=torch.float32, device=dev),
           "levels": torch.full((W, n), SENTINEL, dtype=torch.float32, device=dev),
           "bins": torch.full((W, n), SENTINEL, dtype=torch.int32, device=dev)}
    if spectrum:
        out["spectrum"] = torch.full((W, K), SENTINEL, dtype=torch.float32, device=dev)
    if p64:
        out["P64"] = torch.full((W, K), SENTINEL, dtype=torch.float64, device=dev)
        out["R"] = torch.zeros((W, m, m, 2), dtype=torch.float64, device=dev)
    p = lambda k: out[k].data_ptr() if k in out else None
    stream = torch.cuda.current_stream().cuda_stream
    l0 = blk.launch_count()
    if o.get("planar") and not p64:
        xs = torch.from_numpy(np.ascontiguousarray(x.reshape(W, N, m).transpose(2, 0, 1).reshape(m, W * N))).to(dev)
        blk.process_planar_device([xs[r].data_ptr() for r in range(m)], N, W, p("angles"), p("levels"), p("spectrum"),
                                  p("bins"), stream=stream)
    else:
        d_in = torch.from_numpy(x.view(np.float32)).to(dev)
        blk.process_device(d_in.data_ptr(), W, p("angles"), p("levels"), p("spectrum"), p("bins"), stream=stream,
                           d_P64=p("P64"), d_R=p("R"))
    torch.cuda.synchronize()
    launches = blk.launch_count() - l0
    res = {k: v.cpu().numpy() for k, v in out.items()}
    if "R" in res:
        res["R"] = res["R"][..., 0] + 1j * res["R"][..., 1]
    for k in ("angles", "levels", "bins") + (("spectrum",) if spectrum else ()):
        assert not np.any(res[k] == SENTINEL), (path, k, "unwritten slot")
    return res, launches


def run_path(blk, path, x):
    """the path's own call, its launch count checked"""
    got, launches = call(blk, path, x)
    assert launches == PATHS[path][3], (path, launches)
    return got


def oracle_P(path, x, table, R=None):
    """fp64 strengths the path computes, per window: the C oracle's MUSIC spectrum, the estimator's on the GPU's own
    R, or (source rule) the MUSIC spectrum of the estimated noise subspace; and the per-window count of filled slots"""
    m, n, _, _, o = PATHS[path]
    W = x.shape[0]
    with np.errstate(all="ignore"):
        if "est" in o:
            return np.stack([eo.spectrum(R[w], table, *o["est"]) for w in range(W)]), [n] * W
        if "rule" in o:
            sub = [ao.noise_subspace(x[w], m, n, o["rule"]) for w in range(W)]
            return np.stack([ao.spectrum(G, table) for G, _ in sub]), [d for _, d in sub]
        return co.work_batch(x, m, n, table)["P"], [n] * W


def oracle_bins(path, P, counts):
    m, n, _, _, o = PATHS[path]
    K = P.shape[1]
    out = np.full((P.shape[0], n), -1, np.int32)
    for w in range(P.shape[0]):
        if counts[w] == 0:
            continue
        q = mo.pick_local_maxima(P[w], counts[w], K, EXCL) if o.get("peak") == "local" else mo.pick_top_n(P[w], counts[w], K)
        for i, (_, _, b) in enumerate(q):
            out[w, i] = b
    return out


def assert_levels_at_bins(got, P, ctx, exact=False):
    """levels are float32 of P at the reported bins (+inf at a zero row), unfilled slots (0, bin -1)"""
    filled = got["bins"] >= 0
    assert np.all(got["levels"][~filled] == 0.0), ctx
    ref = np.array([[P[w, b] if b >= 0 else 0.0 for b in row] for w, row in enumerate(got["bins"])])
    if exact:
        with np.errstate(over="ignore"):  # strengths beyond the float32 range are +inf levels
            assert np.array_equal(got["levels"][filled], ref[filled].astype(np.float32)), ctx
    else:
        helpers.assert_float32_close(got["levels"][filled], ref[filled], P_RTOL, ctx)
    K = P.shape[1]
    assert np.array_equal(got["angles"][filled], (got["bins"][filled].astype(np.float64) * 360.0 / K).astype(np.float32)), ctx


def mixed_windows(table, N, seed, W=W0):
    """strong sources (n_src of them) along random rows on every other window, noise only on the rest"""
    rng = np.random.default_rng(seed)
    K, m = table.shape
    return helpers.source_windows(rng, [[table[int(rng.integers(0, K))] for _ in range(2)] if w % 2 == 0 else None
                                        for w in range(W)], m, N)


# ---- A. power-of-two table scaling is exact --------------------------------------------------------------------------
SCALES = (-75, -66, -64, -40, 0, 40, 62, 63, 64, 100)


@pytest.mark.parametrize("path", list(PATHS))
def test_power_of_two_table_scaling_is_exact(path, monkeypatch):
    """table * 2^s for s from -75 (entries near the float32 subnormals, ||a||^2 below them) to 100 (||a||^2 = 2^202, far
    beyond float32): every strength scales by exactly 2^-2s, so P64 is bit-equal to 2^-2s P64(0), the spectrum and the
    levels are float32 of that, and the bins are those of s = 0.  The fused kernels write no P64: their bins and levels
    must equal the unfused fp64 scan's on the same handle."""
    m, n, N, _, o = PATHS[path]
    table = helpers.planar_table(m, K0, 10 + m)
    x = mixed_windows(table, N, 20 + m)
    blk = make_handle(path, table, monkeypatch)
    base = run_path(blk, path, x)
    bfull, _ = call(blk, path, x, spectrum=True, p64=True)
    P0 = bfull["P64"]
    ref, counts = oracle_P(path, x, table, bfull["R"])
    helpers.assert_bins_equal_up_to_exact_ties(base["bins"], {"bins": oracle_bins(path, ref, counts), "P": ref})
    fin = np.isfinite(ref)
    assert helpers.rel_err(P0[fin], ref[fin]) <= 1e-8, path
    for s in SCALES:
        ts = (table.astype(np.complex128) * 2.0 ** s).astype(np.complex64)
        assert np.array_equal(ts.astype(np.complex128) * 2.0 ** -s, table.astype(np.complex128)), s  # exact in float32
        blk.set_array_response(ts)
        got = run_path(blk, path, x)
        full, _ = call(blk, path, x, spectrum=True, p64=True)
        Ps = P0 * 2.0 ** (-2 * s)
        ctx = (path, s)
        with np.errstate(all="ignore"):
            assert np.array_equal(full["P64"], Ps, equal_nan=True), ctx
            assert np.array_equal(full["spectrum"], Ps.astype(np.float32), equal_nan=True), ctx
            assert np.array_equal(got["bins"], base["bins"]), ctx
            assert np.array_equal(got["bins"], full["bins"]), ctx
            assert_levels_at_bins(got, Ps, ctx, exact=True)
            if "spectrum" in got:
                assert np.array_equal(got["spectrum"], Ps.astype(np.float32), equal_nan=True), ctx
    blk.close()


TRACE_WORDS, TRACE_CTAS, TRACE_LAUNCHES = 40, 1024, 32  # music_fused.cuh: FZ_TRACE, FZ_TRACE_CTAS, FZ_TRACE_LAUNCHES


def screen_passes(blk, launch):
    """tensor-core passes the fused M = 4 kernel ran in the handle's `launch`-th call (its per-CTA trace, word 13)"""
    ring = np.zeros(TRACE_LAUNCHES * TRACE_CTAS * TRACE_WORDS, np.int64)
    assert blk._lib.music_b200_debug_fused_trace(blk._h, ring.ctypes.data, TRACE_LAUNCHES * TRACE_CTAS) == 0
    rows = ring.reshape(TRACE_LAUNCHES, TRACE_CTAS, TRACE_WORDS)[launch % TRACE_LAUNCHES]
    return int(rows[rows[:, 31] != 0, 13].sum())  # (word 31: the CTA's exit time, non-zero for every CTA that ran)


SCREEN_LIMITS = (2.0 ** -100, 2.0 ** 100)  # music_b200.cu, screen_bounds_table: fl32(||a||^2) of every non-zero row
ZERO_ROWS = [(777,), (5, 1000, K0 - 1), (3, 4), (500,)]  # one, several (with the K - 1 wrap), adjacent, on the subsample


def screen_tables(geo):
    """(name, scale s or None, table, whether the screen may run, zero rows) for the screened fused M = 4 test"""
    out = []
    for s in sorted(set(SCALES) | {-52, -50, 48, 50}):  # ||a||^2 = 2^(2s + 2): 2^-102 / 2^-98 / 2^98 / 2^102 at the limits
        out.append(("2^%d" % s, s, (geo.astype(np.complex128) * 2.0 ** s).astype(np.complex64), -50 <= s <= 48, ()))
    out.append(("calibrated", None, helpers.calibrated_table(geo, 15), True, ()))
    # one row exactly at each limit, and one a float32 step beyond it (row 123 := [v, 0, 0, 0], ||a||^2 = v^2)
    for v, ok in ((2.0 ** 50, True), (2.0 ** 50 * (1 + 2.0 ** -23), False), (2.0 ** -50, True), (2.0 ** -50 * (1 - 2.0 ** -24), False)):
        t = geo.copy()
        t[123] = [v, 0, 0, 0]
        na = np.float32(np.float64(np.float32(v)) ** 2)
        assert (SCREEN_LIMITS[0] <= na <= SCREEN_LIMITS[1]) == ok
        out.append(("row ||a||^2 = %r" % float(na), None, t, ok, ()))
    for zeros in ZERO_ROWS:
        t = geo.copy()
        t[list(zeros)] = 0
        out.append(("zero rows %s" % (zeros,), None, t, True, zeros))
    return out


def test_fused4_screen_on_scaled_and_calibrated_tables(monkeypatch):
    """Enough windows per CTA that the fused M = 4 kernel runs tensor-core passes.  Its fp32 screen bounds the error
    relative to fl32(||a||^2): for a table scaled by 2^62 or more that value overflows (2^63: +inf, every d~ NaN), by
    2^-64 or less it is subnormal and the bound no longer holds.  A table with a non-zero row outside [2^-100, 2^100]
    runs on the kernel's all-fp64 drain (checked at both limits, row by row); the others - 2^-50 .. 2^48, a calibrated
    table with rows 2^-20 .. 2^20, tables with zero rows (exact in the screen: d~ = 0) - keep the screen, which the
    kernel's trace shows.  Either way bins and levels are bit-identical to the unfused fp64 scan; with zero rows the
    first zero row wins with level +inf."""
    m, n, N, W = 4, 1, 64, 8192
    geo = helpers.planar_table(m, K0, 14)
    x = mixed_windows(geo, N, 24, W=W)
    with monkeypatch.context() as mp:
        mp.setenv("MUSIC_B200_TRACE", "1")
        blk = music_doa(m, n, N * m, geo, K0)
    path = "fused4"
    tables = screen_tables(geo)
    P0 = None
    for launch, (name, s, table, screened, zeros) in enumerate(tables):
        blk.set_array_response(table)
        got = run_path(blk, path, x)
        full, _ = call(blk, path, x, spectrum=False, p64=True)
        passes = screen_passes(blk, launch)
        if s == 0:
            P0 = full["P64"]
            ref = co.work_batch(x[:64], m, n, table)
            helpers.assert_bins_equal_up_to_exact_ties(got["bins"][:64], ref)
        assert np.array_equal(got["bins"], full["bins"]), name
        assert_levels_at_bins(got, full["P64"], name, exact=True)
        assert (passes > 0) == screened, (name, passes)
        if zeros:
            assert np.all(got["bins"] == min(zeros)) and np.all(np.isposinf(got["levels"])), name
    launch = len(tables)
    for name, s, table, _, _ in tables:  # the bins of every scaled table are those of the unscaled one
        if s is not None:
            blk.set_array_response(table)
            assert np.array_equal(run_path(blk, path, x)["bins"], np.argmax(P0, axis=1)[:, None]), name
            launch += 1
    # exact ties inside the screen's candidate lists: every duplicate group of DUPLICATES, a strong source along it
    dup = geo.copy()
    for rows, _ in DUPLICATES:
        dup[list(rows[1:])] = dup[rows[0]]
    lows = [DUPLICATES[w % len(DUPLICATES)][0][0] for w in range(W)]
    xd = helpers.source_windows(np.random.default_rng(25), [[dup[k]] for k in lows], m, N, amp=100.0)
    blk.set_array_response(dup)
    got = run_path(blk, path, xd)
    assert screen_passes(blk, launch) > 0
    assert np.array_equal(got["bins"][:, 0], lows)
    blk.close()


# ---- B. calibrated tables against the oracles ------------------------------------------------------------------------
def check_against_oracle(blk, path, x, table, ctx):
    """the path's call and the fp64 call on the same handle against the oracle: bins bit-exact up to the oracle's own
    ties inside fp64 noise, levels / spectrum within 1e-5, P64 within 1e-8"""
    got = run_path(blk, path, x)
    full, _ = call(blk, path, x, spectrum=True, p64=True)
    P, counts = oracle_P(path, x, table, full["R"])
    ref = {"bins": oracle_bins(path, P, counts), "P": P}
    helpers.assert_bins_equal_up_to_exact_ties(got["bins"], ref)
    assert np.array_equal(full["bins"], got["bins"]), ctx
    assert_levels_at_bins(got, P, ctx)
    fin = np.isfinite(P)
    assert helpers.rel_err(full["P64"][fin], P[fin]) <= 1e-8, ctx
    helpers.assert_float32_close(full["spectrum"], P, P_RTOL, ctx)
    if "spectrum" in got:
        helpers.assert_float32_close(got["spectrum"], P, P_RTOL, ctx)
    return got, P


@pytest.mark.parametrize("path", list(PATHS))
def test_calibrated_table_against_oracle(path, monkeypatch):
    m, n, N, _, o = PATHS[path]
    geo = helpers.planar_table(m, K0, 30 + m)
    table = helpers.calibrated_table(geo, 31 + m)
    rng = np.random.default_rng(32 + m)
    x = helpers.source_windows(rng, [[table[int(rng.integers(0, K0))] for _ in range(n)] if w % 4 else None
                                     for w in range(W0)], m, N)
    blk = make_handle(path, table, monkeypatch)
    check_against_oracle(blk, path, x, table, path)
    blk.close()


# ---- C. duplicated rows: exact ties at bins of our choosing ----------------------------------------------------------
# K = 3600: screen tiles of 192 rows, decimated subsample = multiples of ceil(3600 / 384) = 10, drain chunk of bin k =
# (k / 32) % 16, 256-bin scan tiles
DUPLICATES = [
    ((200, 250), "same screen tile, same scan tile, other drain chunk"),
    ((100, 1000), "different screen tiles"),
    ((500, 2000), "both on the decimated subsample"),
    ((501, 2003), "both off the decimated subsample"),
    ((510, 2003), "one on, one off the decimated subsample"),
    ((64, 576), "same drain chunk"),
    ((255, 256), "adjacent scan tiles"),
    ((0, K0 - 1), "the K - 1 -> 0 wrap"),
    ((700, 1700, 3000), "triple tie"),
]


def tie_table(m, rows, src):
    """a steering table whose rows `rows` all hold row `src`'s vector"""
    t = helpers.planar_table(m, K0, 40 + m)
    for r in rows:
        t[r] = t[src]
    return t


@pytest.mark.parametrize("path", list(PATHS))
def test_duplicated_rows_tie_to_the_lowest_bin(path, monkeypatch):
    """a strong source along the duplicated vector makes the tie the peak; the result must be the oracle's with the tie
    rule applied to the bit-equal strengths: the lowest bin for n = 1, the tied bins in ascending order with equal
    levels for n = 2, both maxima (lower first) for local maxima when they are farther apart than the exclusion"""
    m, n, N, _, o = PATHS[path]
    blk = make_handle(path, helpers.planar_table(m, K0, 40 + m), monkeypatch)
    rng = np.random.default_rng(50 + m)
    for rows, what in DUPLICATES:
        for src in (rows[0], rows[-1]):  # the lower row copied upwards, and the upper one downwards
            table = tie_table(m, rows, src)
            x = helpers.source_windows(rng, [[table[src]]] * 3, m, N, amp=100.0)
            ctx = (path, rows, src, what)
            blk.set_array_response(table)
            got = run_path(blk, path, x)
            full, _ = call(blk, path, x, spectrum=True, p64=True)
            P, counts = oracle_P(path, x, table, full["R"])
            P[:, list(rows)] = P[:, [src]]  # bit-equal rows have bit-equal strengths in any exact evaluation
            ref = oracle_bins(path, P, counts)
            expect = sorted(rows)
            if o.get("peak") == "local":  # a plateau counts once, at its first bin; then the exclusion
                expect = [r for r in expect if (r - 1) % K0 not in rows]
                expect = [r for i, r in enumerate(expect) if all(min((r - q) % K0, (q - r) % K0) > EXCL for q in expect[:i])]
            for w in range(x.shape[0]):
                c = min(counts[w], len(expect))
                assert list(ref[w, :c]) == expect[:c], (ctx, ref[w], expect)
            assert np.array_equal(got["bins"], ref), (ctx, got["bins"], ref)
            assert np.array_equal(full["bins"], ref), ctx
            assert_levels_at_bins(got, P, ctx)
            tied = (ref >= 0) & np.isin(ref, rows)
            for w in range(x.shape[0]):
                lv = got["levels"][w][tied[w]]
                assert lv.size == 0 or np.all(lv == lv[0]), ctx
    blk.close()


# ---- D. zero rows ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", list(PATHS))
def test_zero_rows(path, monkeypatch):
    """a zero row has strength 1 / 0 = +inf (MUSIC, MVDR): the first zero row wins with level +inf, the spectrum is
    +inf at every zero row, with n = 2 the first two zero rows win.  Bartlett's 0 / 0 is NaN and never picked."""
    m, n, N, _, o = PATHS[path]
    geo = helpers.planar_table(m, K0, 60 + m)
    x = mixed_windows(geo, N, 61 + m, W=4)
    blk = make_handle(path, geo, monkeypatch)
    bartlett = o.get("est", ("",))[0] == "bartlett"
    for zeros in ((777,), (5, 1000, K0 - 1), (3, 4)):
        table = geo.copy()
        table[list(zeros)] = 0
        ctx = (path, zeros)
        blk.set_array_response(table)
        got, P = check_against_oracle(blk, path, x, table, ctx)
        full, _ = call(blk, path, x, spectrum=True, p64=True)
        if bartlett:
            assert np.all(np.isnan(full["spectrum"][:, list(zeros)])), ctx
            assert not np.any(np.isin(got["bins"], zeros)), ctx
            continue
        assert np.all(np.isposinf(full["spectrum"][:, list(zeros)])), ctx
        if o.get("peak") != "local":
            first = min(n, len(zeros))
            filled = got["bins"][:, :first] >= 0  # (the source rule may count no source in a noise-only window)
            assert "rule" in o or np.all(filled), ctx
            assert np.all((got["bins"][:, :first] == np.array(sorted(zeros)[:first])[None, :])[filled]), ctx
            assert np.all(np.isposinf(got["levels"][:, :first][filled])), ctx
    blk.close()


# ---- the reference's own outputs on such tables ----------------------------------------------------------------------
@pytest.mark.parametrize("path", ["fused4", "fused4_drain", "peak1_4", "scan4", "topn4", "fused4_spec"])
def test_reference_golden_tables(path, monkeypatch):
    """the CUDA paths against the reference's own work() (tests/golden/reference/tables.npz): angles bit-exact, levels
    and spectrum within 1e-5 (+inf, as the reference's, at zero rows and beyond the float32 range)"""
    m, n, N, _, o = PATHS[path]
    done = 0
    for key, gm, gn, table, x in helpers.table_golden_cases():
        if (gm, gn) != (m, n):
            continue
        ref = helpers.table_reference_outputs(key, x, table)
        with monkeypatch.context() as mp:
            for k, v in o.get("env", {}).items():
                mp.setenv(k, v)
            blk = music_doa(gm, gn, x.shape[1], table, table.shape[0])
        got, launches = call(blk, path, x, spectrum=True) if path == "fused4_spec" else call(blk, path, x)
        assert launches == PATHS[path][3], (path, key, launches)
        blk.close()
        assert np.array_equal(got["angles"], ref["angles"]), (path, key)
        helpers.assert_float32_close(got["levels"], ref["levels"], P_RTOL, (path, key))
        if "spectrum" in got:
            helpers.assert_float32_close(got["spectrum"], ref["spectrum"], P_RTOL, (path, key))
        done += 1
    assert done == 5, path


# ---- E. shape edges of the fused kernels, rough spectra --------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 191, 192, 193, 383, 384, 385, 4097, 65537])
@pytest.mark.parametrize("path", ["fused4", "fused8"])
def test_fused_kernels_at_table_edges(path, K, monkeypatch):
    """one, two, just under / at / over one and two 192-row screen tiles (the decimated subsample takes every row up to
    K = 384), and large K; a geometric and the calibrated table.  M = 4 runs 8192 windows so that the tensor-core screen
    runs (its trace counts the passes), bins and levels bit-identical to the unfused scan_peak1_kernel<4> on the same
    table, the first 64 windows against the C oracle.  M = 8 (no screen: its scan is fp64 throughout) on 16 windows."""
    m, n, N, _, _ = PATHS[path]
    geo = helpers.planar_table(m, K, 70 + K % 97)
    for name, table in (("geometric", geo), ("calibrated", helpers.calibrated_table(geo, 71))):
        ctx = (path, K, name)
        if path == "fused4":
            N = 64
            x = mixed_windows(table, N, 72 + K, W=8192)
            with monkeypatch.context() as mp:
                mp.setenv("MUSIC_B200_TRACE", "1")
                blk = music_doa(m, n, N * m, table, K)
            got = run_path(blk, path, x)
            assert screen_passes(blk, 0) > 0, ctx
            blk.close()
            with monkeypatch.context() as mp:
                mp.setenv("MUSIC_B200_FUSED", "0")
                blk = music_doa(m, n, N * m, table, K)
            unfused, launches = call(blk, path, x)
            blk.close()
            assert launches == PATHS["peak1_4"][3], ctx
            for k in ("bins", "levels", "angles"):
                assert np.array_equal(got[k], unfused[k]), (ctx, k)
            x, got = x[:64], {k: v[:64] for k, v in got.items()}
        else:
            x = mixed_windows(table, N, 72 + K, W=16)
            blk = make_handle(path, table, monkeypatch)
            got = run_path(blk, path, x)
            blk.close()
        ref = co.work_batch(x, m, n, table)
        helpers.assert_bins_equal_up_to_exact_ties(got["bins"], ref)
        assert_levels_at_bins(got, ref["P"], ctx)


@pytest.mark.parametrize("path", ["local4", "local8", "topn4", "topn16"])
def test_random_table_rough_spectrum(path, monkeypatch):
    """i.i.d. complex rows: about every third bin is a local maximum"""
    m, n, N, _, _ = PATHS[path]
    table = helpers.random_table(m, K0, 80 + m)
    x = mixed_windows(table, N, 81 + m)
    blk = make_handle(path, table, monkeypatch)
    _, P = check_against_oracle(blk, path, x, table, path)
    blk.close()
    nmax = [int(np.sum((P[w] > np.roll(P[w], 1)) & (P[w] > np.roll(P[w], -1)))) for w in range(P.shape[0])]
    assert min(nmax) > K0 // 4, nmax


@pytest.mark.parametrize("peak", ["top", "local"])
def test_azel_random_table(peak):
    """an az-el handle (360 x 91 grid) with a random table set by set_array_response: more than AZEL_LM_CAP = 2048 2-D
    local maxima per window, which sends the local-maxima kernel through its re-test branch"""
    m, n, snaps, W = 4, 2, 256, 4
    grid = ao.Grid(360, 91, 0.0, 90.0)
    table = helpers.random_table(m, grid.K, 90)
    x = mixed_windows(table, snaps, 91, W=W)
    blk = music_doa_azel(m, n, m * snaps, grid.n_az, grid.n_el, (grid.el_lo, grid.el_hi), ao.uca_xyz(m, 1.0), 1.0)
    blk.set_array_response(table.reshape(grid.n_el, grid.n_az, m))
    blk.set_peak_mode("top_bins" if peak == "top" else "local_maxima", 2)
    dev = torch.device("cuda:0")
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)
    o = {k: torch.full((W, n), SENTINEL, dtype=torch.float32, device=dev) for k in ("az", "el", "lv")}
    spec = torch.full((W, grid.K), SENTINEL, dtype=torch.float32, device=dev)
    bins = torch.full((W, n), SENTINEL, dtype=torch.int32, device=dev)
    l0 = blk.launch_count()
    blk.process_device(d_in.data_ptr(), W, o["az"].data_ptr(), o["el"].data_ptr(), o["lv"].data_ptr(), spec.data_ptr(),
                       bins.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert blk.launch_count() - l0 == 5  # cov4_tma, eig, scan, top-n / 2-D local maxima, decode
    blk.close()
    gb, gl, gs = bins.cpu().numpy(), o["lv"].cpu().numpy(), spec.cpu().numpy()
    for w in range(W):
        r = ao.work(x[w], m, n, table, grid, peak, 2)
        P = r["P"]
        if peak == "local":
            assert int(np.sum(ao.local_max_mask(P, grid))) > 2048, w
        helpers.assert_float32_close(gs[w], P, P_RTOL, w)
        for i in range(n):
            g_, o_ = int(gb[w, i]), int(r["bins"][i])
            if g_ != o_:
                assert g_ >= 0 and o_ >= 0 and abs(P[g_] - P[o_]) <= 1e-12 * P[o_], (w, i, g_, o_)
                break
            helpers.assert_float32_close(gl[w, i:i + 1], P[g_:g_ + 1], P_RTOL, (w, i))
