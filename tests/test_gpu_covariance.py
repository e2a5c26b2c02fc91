"""GPU: every covariance the estimators read, against the exact references of tests/covariance_oracle.py.

Raw kernels (process_device_ex's d_R; the launch count proves the branch): on E1 windows (and E1 scaled by 2^k, float32
subnormals included) R must be fl(S / N) bit for bit whatever the summation order; on E2 (elements 2^-60 ... 2^60 apart)
and E3 (exact zeros under large terms) every entry within its own bound; on E4 a NaN or Inf in element r must leave every
entry outside row and column r bit-identical to the window with that value 0, and make row and column r non-finite.
Every R must be exactly Hermitian with a real, non-negative diagonal.

Routes with no R port, by byte identity on E1 and E4 windows, where R is exact: the fused M = 4 kernel (Jacobi eigensolver)
against the unfused path, the fused M = 8 kernel (bins; levels within its principal solver's 1e-9), and both planar
entries against process_device on the interleaved copy.

Integration: Rbar against the recurrence at 60 digits on the device's own raw R, per entry within the bound of
covariance_oracle.integ_bounds, at forgetting factors from 2^-1074 to the largest double below 1; MDL / AIC counts
against the exact N_eff.  The worst ratio to each bound is printed with -s."""
import math

import numpy as np
import pytest

import channels_oracle as cho
import covariance_oracle as co
import gpu_harness as gh
import helpers
import source_count_oracle as sco
import test_gpu_channels as tgc
import test_gpu_focus as tgf
from helpers import LAM

pytestmark = pytest.mark.gpu

WORST = {}


def note(case, ratio):
    WORST[case] = max(WORST.get(case, 0.0), float(ratio))
    print("covariance %s: worst ratio to the bound %.3g" % (case, WORST[case]))


def raw_call(m, N, x, n=1, K=16, env=None):
    """d_R of one device call on windows x [W][N][m] (complex64), with the launches it took"""
    blk = gh.make_block(m, n, N, K=K, env=env)
    out, launches = gh.device_call(blk, np.ascontiguousarray(x.reshape(x.shape[0], -1)), ("R", "eigvals"))
    blk.close()
    return out["R"], launches


def assert_hermitian(R, ctx):
    """R_ji = conj(R_ij) off the diagonal, a real diagonal >= 0 (values: the mirrored imaginary part of an exact zero
    may carry either sign)"""
    m = R.shape[-1]
    off = ~np.eye(m, dtype=bool)
    assert np.array_equal(R[..., off], np.conj(np.swapaxes(R, -1, -2))[..., off]), ctx
    d = np.diagonal(R, axis1=-2, axis2=-1)
    assert np.all(d.imag == 0), ctx
    fin = np.isfinite(d.real)
    assert np.all(d.real[fin] >= 0), ctx


# ---- raw kernels ----
#   m  N       W: every covariance branch (launch_cov), N edges of the TMA stages and of the 32 lanes, N not a power of two
RAW = [(2, 3, 33), (2, 65536, 1), (3, 31, 3), (3, 4097, 3), (4, 5, 3), (4, 127, 33), (4, 129, 3), (4, 1000, 3),
       (4, 65536, 1), (5, 33, 3), (6, 255, 3), (7, 128, 33), (8, 9, 3), (8, 127, 3), (8, 128, 33), (8, 255, 3),
       (8, 1000, 3), (8, 65536, 1), (9, 129, 3), (10, 32, 3), (11, 4097, 1), (12, 13, 3), (12, 255, 3), (13, 33, 3),
       (14, 1000, 1), (15, 127, 3), (16, 17, 3), (16, 127, 3), (16, 129, 33), (16, 4097, 3), (16, 65536, 1)]


def expected_launches(m, N):
    return len(co.cov_kernels(m, N)) + 2  # + eigensolver + scan (n = 1, no top-n)


@pytest.mark.parametrize("m,N,W", RAW)
def test_raw_kernels_exact_windows(m, N, W):
    rng = np.random.default_rng(1000 * m + N)
    for k in (0, -140, -100, 60, 96):
        x = co.family_e1(rng, W, N, m, k)
        R, launches = raw_call(m, N, x)
        assert launches == expected_launches(m, N), (m, N, launches)
        assert_hermitian(R, (m, N, k))
        ref = co.e1_reference(x, k)
        assert np.array_equal(R, ref), (m, N, k, np.argwhere(R != ref)[:4])
    note("E1 bit-exact (%s)" % co.cov_kernels(m, N)[0], 0.0)


@pytest.mark.parametrize("m,N,W", [r for r in RAW if r[1] <= 4097])
def test_raw_kernels_dynamic_range_and_cancellation(m, N, W):
    rng = np.random.default_rng(2000 * m + N)
    kern = co.cov_kernels(m, N)[0]
    L = co.depth(kern, m, N)
    W = min(W, 3)
    fams = {"E2": co.family_e2(rng, W, N, m)}
    if N >= 4:
        fams["E3"] = co.family_e3(rng, W, N, m)[0]
        fams["E3 common"] = co.family_e3(rng, W, N, m, common=2.0 ** 20)[0]
    for name, x in fams.items():
        R, _ = raw_call(m, N, x)
        assert_hermitian(R, (m, N, name))
        worst = max(co.raw_ratios(R[w], x[w], L) for w in range(W))
        note("%s %s" % (name, kern), worst)
        assert worst <= 1.0, (m, N, name, worst)


@pytest.mark.parametrize("m,N,W", [r for r in RAW if r[1] <= 4097][::2])
@pytest.mark.parametrize("value", [math.nan, math.inf, -math.inf])
def test_raw_kernels_non_finite(m, N, W, value):
    rng = np.random.default_rng(3000 * m + N)
    bad, zero, r = co.family_e4(rng, max(W, 2), N, m, value)
    Rb, _ = raw_call(m, N, bad)
    Rz, _ = raw_call(m, N, zero)
    for w in range(len(bad)):
        keep = np.ones((m, m), bool)
        keep[r[w], :] = keep[:, r[w]] = False
        assert np.array_equal(Rb[w][keep].view(np.uint64), Rz[w][keep].view(np.uint64)), (m, N, w)
        line = np.concatenate([Rb[w][r[w], :], Rb[w][:, r[w]]])
        assert np.all(~np.isfinite(line.real) | ~np.isfinite(line.imag)), (m, N, w)


def test_raw_kernels_across_sub_batches():
    # m = 16, n = 2 under TOP_BINS keeps the fp64 spectrum of K = 65536 bins: about 750 windows per sub-batch
    m, N, W = 16, 32, 1000
    x = co.family_e1(np.random.default_rng(4), W, N, m)
    blk = gh.make_block(m, 2, N, K=65536)
    out, launches = gh.device_call(blk, x.reshape(W, -1), ("R",))
    blk.close()
    assert launches >= 2 * 5  # two sub-batches or more of 2 tile kernels, eigensolver, scan and top-n
    assert np.array_equal(out["R"], co.e1_reference(x))


# ---- routes with no R port ----
def route_windows(rng, W, N, m):
    """E1 windows with NaN windows (every fourth) and Inf windows (every eighth) among them"""
    x = co.family_e1(rng, W, N, m)
    bad, _, _ = co.family_e4(rng, W, N, m, math.nan)
    x[1::4] = bad[1::4]
    inf, _, _ = co.family_e4(rng, W, N, m, math.inf)
    x[3::8] = inf[3::8]
    return x


@pytest.mark.parametrize("N", [127, 128, 129, 255, 256, 257, 1000])
def test_fused_m4_jacobi_is_the_unfused_path(N):
    m, W = 4, 40
    pos = helpers.positions("uca", m)
    table = helpers.table_wl(pos / LAM)
    x = route_windows(np.random.default_rng(N), W, N, m).reshape(W, -1)
    env = {"MUSIC_B200_EIG": "jacobi"}
    fused_blk = gh.make_block(m, 1, N, table=table, env=env)
    fused, l_f = gh.device_call(fused_blk, x, ("levels", "bins"))
    unf, l_u = gh.device_call(fused_blk, x, ("levels", "bins", "R"))
    fused_blk.close()
    assert l_f == 1 and l_u == 3
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(fused[k].view(np.uint8), unf[k].view(np.uint8)), (N, k)


@pytest.mark.parametrize("N", [128, 256, 1000])
def test_fused_m8_covariance_is_covN(N):
    m, W = 8, 40
    pos = helpers.positions("uca", m)
    table = helpers.table_wl(pos / LAM)
    x = route_windows(np.random.default_rng(N + 8), W, N, m)
    a = np.array([1, 1j, -1, -1j] * 2, np.complex64)  # a strong source with Gaussian-integer steering: still exact
    x = (x + 64 * x[..., :1] * a).astype(np.complex64)
    blk = gh.make_block(m, 1, N, table=table)
    fused, l_f = gh.device_call(blk, x.reshape(W, -1), ("levels", "bins"))
    unf, l_u = gh.device_call(blk, x.reshape(W, -1), ("levels", "bins", "R"))
    blk.close()
    assert l_f == 1 and l_u == 3
    assert np.array_equal(fused["bins"], unf["bins"])
    none = unf["levels"] == 0  # the NaN and Inf windows: no peak, level 0, on both routes
    assert np.any(none) and np.all(fused["levels"][none] == 0)
    assert helpers.rel_err(fused["levels"][~none], unf["levels"][~none]) <= 1e-9


def planar_streams(rng, m, N, hop, W):
    """E1 antenna streams long enough for W windows of N snapshots every hop, with one NaN and one Inf sample, and the
    interleaved windows they make"""
    total = (W - 1) * hop + N
    s = co.family_e1(rng, 1, total, m)[0]  # [total][m]
    s[hop + N // 3, m - 1] = complex(math.nan, 0.0)  # inside window 1
    s[3 * hop + N // 2, 0] = complex(0.0, math.inf)  # inside window 3
    streams = [np.ascontiguousarray(s[:, i]) for i in range(m)]
    x = np.stack([s[w * hop:w * hop + N] for w in range(W)])
    return streams, x.reshape(W, -1)


def interleaved_launches(m, N, fused):
    if fused and (m == 4 or (m == 8 and N >= 128 and N % 2 == 0)):
        return 1
    return len(co.cov_kernels(m, N)) + 2


def planar_launches(m, N, hop, fused):
    """the fused M = 4 kernel reads the streams itself (even hop and N); otherwise cov_planar_kernel, eigensolver, scan"""
    if fused and m == 4 and hop % 2 == 0 and N % 2 == 0:
        return 1
    return len(co.cov_kernels(m, N, planar=True)) + 2


PLANAR = [(4, 256, 256, True), (4, 256, 64, True), (4, 256, 300, True), (4, 256, 63, True), (4, 129, 129, True),
          (4, 256, 256, False), (4, 256, 64, False), (4, 256, 300, False), (4, 256, 63, False), (4, 129, 129, False),
          (8, 128, 100, True), (12, 96, 96, True), (16, 64, 40, True), (16, 64, 65, True), (5, 40, 17, True)]


@pytest.mark.parametrize("m,N,hop,fused", PLANAR)
def test_planar_entries_are_the_interleaved_path(m, N, hop, fused):
    W = 24
    pos = helpers.positions("uca", m)
    table = helpers.table_wl(pos / LAM)
    streams, x = planar_streams(np.random.default_rng(m * 1000 + hop), m, N, hop, W)
    env = {"MUSIC_B200_EIG": "jacobi", "MUSIC_B200_FUSED": "1" if fused else "0"}
    blk = gh.make_block(m, 1, N, table=table, env=env)
    dev, l_dev = gh.device_call(blk, x, ("levels", "bins"))
    pl, l_pl = gh.planar_device_call(blk, streams, hop, W, ("levels", "bins"))
    pa, plv = np.zeros((W, 1), np.float32), np.zeros((W, 1), np.float32)
    blk.work_planar(W, streams, [pa, plv], hop=hop)
    hb = blk.last_bins().copy()
    blk.close()
    assert l_dev == interleaved_launches(m, N, fused) and l_pl == planar_launches(m, N, hop, fused), (l_dev, l_pl)
    assert not np.all(np.isfinite(x.view(np.float32)))  # the NaN and Inf samples are inside some window
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(pl[k].view(np.uint8), dev[k].view(np.uint8)), (m, N, hop, k)
    assert np.array_equal(pa.view(np.uint8), dev["angles"].view(np.uint8))
    assert np.array_equal(plv.view(np.uint8), dev["levels"].view(np.uint8)) and np.array_equal(hb, dev["bins"])


# ---- integration ----
ALPHAS = [2.0 ** -1074, 1e-300, 0.5, 0.99, 1 - 2.0 ** -20, 1 - 1e-6, 1 - 1e-8, 1 - 2.0 ** -40, math.nextafter(1.0, 0.0)]


def noise(rng, W, N, m, scale=None):
    x = (rng.standard_normal((W, N, m)) + 1j * rng.standard_normal((W, N, m))) / math.sqrt(2.0)
    if scale is not None:
        x = x * scale[:, None, None]
    return x.reshape(W, N * m).astype(np.complex64)


def integrated(m, N, x, alpha, calls, K=16):
    """(raw R from an alpha = 0 handle, Rbar from calls of the given sizes on an integrating handle)"""
    blk = gh.make_block(m, 1, N, K=K)
    R = gh.device_call(blk, x, ("R",))[0]["R"]
    blk.set_integration(alpha)
    got, w0 = [], 0
    for Wc in calls:
        out, launches = gh.device_call(blk, x[w0:w0 + Wc], ("R",))
        # one sub-batch: the covariance kernels, the three integration kernels, eigensolver and scan
        assert launches == len(co.cov_kernels(m, N)) + 5, ("every call is one sub-batch", Wc, launches)
        got.append(out["R"])
        w0 += Wc
    blk.close()
    return R, np.concatenate(got)


def check_integration(case, R, got, alpha, calls):
    hi, lo, _, _ = co.integrate_exact(R, alpha)
    bound = co.integ_bounds(R, alpha, calls)
    r = co.integ_ratios(got, hi, lo, bound)
    note("integration %s" % case, np.max(r))
    assert np.all(r <= 1.0), (case, int(np.argmax(r)), float(np.max(r)))
    assert np.array_equal(got[0], R[0])
    assert_hermitian(got, case)


@pytest.mark.parametrize("alpha", ALPHAS)
def test_integration_calls(alpha):
    m, N = 4, 16
    calls = [1, 31, 32, 33, 257, 33]
    x = noise(np.random.default_rng(7), sum(calls), N, m)
    R, got = integrated(m, N, x, alpha, calls)
    check_integration("alpha=%r calls" % alpha, R, got, alpha, calls)


@pytest.mark.parametrize("alpha", [0.99, 1 - 1e-6, 1 - 1e-8, math.nextafter(1.0, 0.0)])
def test_integration_one_long_call(alpha):
    # W > 256 INTEG_T: every thread of the carry kernel takes two tiles or more
    m, N, W = 2, 8, 256 * co.INTEG_T + 77
    x = noise(np.random.default_rng(8), W, N, m)
    R, got = integrated(m, N, x, alpha, [W])
    check_integration("alpha=%r W=%d" % (alpha, W), R, got, alpha, [W])


def test_integration_long_stream():
    m, N, W, per = 2, 8, 100000, 5000
    alpha = 1 - 1e-6
    x = noise(np.random.default_rng(9), W, N, m)
    R, got = integrated(m, N, x, alpha, [per] * (W // per))
    check_integration("1e5 windows", R, got, alpha, [per] * (W // per))


@pytest.mark.parametrize("alpha", [0.5, 0.99, 1 - 1e-8])
def test_integration_loud_then_quiet_and_alternating_signs(alpha):
    m, N, W = 4, 16, 300
    rng = np.random.default_rng(10)
    scale = np.ones(W)
    scale[5] = 2.0 ** 40  # 2^80 in R
    x = noise(rng, W, N, m, scale)
    R, got = integrated(m, N, x, alpha, [100, 200])
    check_integration("alpha=%r loud window" % alpha, R, got, alpha, [100, 200])
    # off-diagonals that change sign from window to window: element 0 negated on every other window
    y = noise(rng, W, N, m).reshape(W, N, m)
    y[1::2, :, 0] *= -1
    y[:, :, 1] = y[:, :, 0] + 0.01 * y[:, :, 1]
    R, got = integrated(m, N, y.reshape(W, -1), alpha, [W])
    check_integration("alpha=%r alternating" % alpha, R, got, alpha, [W])


@pytest.mark.parametrize("rule", ["mdl", "aic"])
@pytest.mark.parametrize("alpha", [0.99, 1 - 1e-6, 1 - 1e-8])
def test_integration_counts_use_the_exact_n_eff(rule, alpha):
    m, N, W = 8, 32, 300
    pos = helpers.positions("uca", m)
    table = helpers.table_wl(pos / LAM)
    rng = np.random.default_rng(11)
    a = helpers.steering_wl(pos / LAM, 50.0)
    s = 0.3 * (rng.standard_normal((W, N)) + 1j * rng.standard_normal((W, N)))
    x = (noise(rng, W, N, m).reshape(W, N, m) + s[..., None] * a).reshape(W, -1).astype(np.complex64)
    out = {}
    for key in ("eigvals", "counts"):  # two identical handles: one call cannot return both
        blk = gh.make_block(m, m - 1, N, table=table, rule=rule)
        blk.set_integration(alpha)
        out[key] = gh.device_call(blk, x, (key,))[0][key]
        blk.close()
    _, _, _, neff = co.integrate_exact(np.zeros((W, 1, 1)), alpha, N)
    margin = 0
    for w in range(W):
        ref = sco.estimate_source_count(out["eigvals"][w], neff[w], m - 1, rule)[0]
        lo = sco.estimate_source_count(out["eigvals"][w], neff[w] * (1 - co.C_NEFF * co.EPS), m - 1, rule)[0]
        hi = sco.estimate_source_count(out["eigvals"][w], neff[w] * (1 + co.C_NEFF * co.EPS), m - 1, rule)[0]
        if lo != ref or hi != ref:
            margin += 1
            assert out["counts"][w] in (lo, ref, hi), (w, rule)
            continue
        assert out["counts"][w] == ref, (w, rule, out["counts"][w], ref)
    print("covariance counts %s alpha=%r: %d windows inside the N_eff margin" % (rule, alpha, margin))


# ---- channels and focusing ----
#   m  F    J   first  C  taper: wrapping ranges, J = 1, 3 and 64, a batch divisor B = 1 (M = 8, F = 256, J = 3)
CHANNELS = [(2, 8, 1, 6, 3, "rect"), (4, 16, 3, 14, 4, "hann"), (4, 8, 64, 6, 4, "hann"), (8, 256, 3, 254, 3, "rect"),
            (4, 256, 2, 1, 3, "hann"), (2, 64, 5, 0, 2, "rect"), (16, 256, 1, 255, 3, "hann")]


@pytest.mark.parametrize("m,F,J,first,C,taper", CHANNELS)
def test_channel_covariances_against_the_exact_filter_bank(m, F, J, first, C, taper):
    W = 2
    x = co.channel_windows(np.random.default_rng(F * J + m), W, m, F, J, first, (first + 1) % F)
    blk = tgc.make(m, 1, F * J, 90, F, first, C, taper)
    got, _ = tgc.device_call(blk, x, ("R",))
    blk.close()
    bins = list(cho.bins_of(F, first, C))
    worst = max(max(co.channel_ratios(got["R"][:, w], x[w], m, F, bins, taper)) for w in range(W))
    note("channels F=%d J=%d %s" % (F, J, taper), worst)
    assert worst <= 1.0, worst
    assert_hermitian(got["R"], (m, F, J))


def test_all_channels_in_groups_are_the_checked_ones():
    # C = F = 256 at M = 16 takes the channels in groups; each R_c is bit for bit that of a narrow, exactly checked range
    m, F, J, taper = 16, 256, 1, "hann"
    x = co.channel_windows(np.random.default_rng(5), 2, m, F, J, 255, 0)
    full = tgc.make(m, 1, F * J, 90, F, 0, F, taper)
    R_full, _ = tgc.device_call(full, x, ("R",))
    full.close()
    narrow = tgc.make(m, 1, F * J, 90, F, 255, 3, taper)
    R_n, _ = tgc.device_call(narrow, x, ("R",))
    narrow.close()
    for c in range(3):
        assert np.array_equal(R_n["R"][c].view(np.uint64), R_full["R"][(255 + c) % F].view(np.uint64)), c


@pytest.mark.parametrize("m,F,J,first,C", [(4, 16, 4, 14, 5), (8, 64, 2, 60, 6), (4, 8, 8, 3, 1)])
def test_focused_covariance_against_the_exact_sum(m, F, J, first, C):
    K, W = 120, 3
    pos = tgf.planar_pos(m, 7 * m + F)
    x = co.channel_windows(np.random.default_rng(m + F), W, m, F, J, first, (first + 2) % F)
    x = x + tgf.noise_windows(W, m, F * J, 3) * np.float32(0.01)
    sep = tgf.make(m, 1, F * J, K, F, first, C, pos, "separate")
    R_c, _ = tgf.device_call(sep, x, ("R",))
    sep.close()
    blk = tgf.make(m, 1, F * J, K, F, first, C, pos)
    T, _ = blk.focusing()
    got, _ = tgf.device_call(blk, x, ("R",))
    blk.close()
    worst = max(co.focus_ratio(got["R"][w], T, R_c["R"][:, w]) for w in range(W))
    note("focused C=%d" % C, worst)
    assert worst <= 1.0, worst
    if C == 1:  # one channel focused onto itself is that channel, bit for bit
        assert np.array_equal(got["R"].view(np.uint64), R_c["R"][0].view(np.uint64))
