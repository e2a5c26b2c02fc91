"""GPU: the per-window source count (music_b200_set_source_rule, MDL / AIC) through every entry point.

Windows of one shape mix 0, 1, 2 and 3 sources (tests/source_count_oracle.py::mixed_windows).  For every case the
counts equal the fp64 definition on LAPACK eigenvalues and on the GPU's own; bins and angles are bit-identical to the
C oracle run at n = count, and to a FIXED handle created with n = count; levels and spectrum agree to 1e-5, and the
slots at and beyond the count are exactly (0, 0, -1)."""
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200.music_doa import music_doa
from oracle import c_oracle as co
from oracle import music_oracle as mo

import gpu_harness as gh
import helpers
import source_count_oracle as so

pytestmark = pytest.mark.gpu

P_RTOL = 1e-5
MARGIN = 1e-6
K = 720
NMAX = 3
EXCL = 3
SEED = 100
PEAKS = ("levels", "bins")
COUNTS = PEAKS + ("counts",)


def inv_norm2(table):
    a = table.astype(np.complex128)
    return 1.0 / np.sum(np.abs(a) ** 2, axis=1)


def check_against_oracles(got, x, m, N, table, rule, peak, n, counts_ref, ctx):
    """bins / angles exact and levels / spectrum to 1e-5 against the C oracle at n = count, unfilled slots exact"""
    assert np.array_equal(got["counts"], counts_ref), (ctx, got["counts"], counts_ref)
    for w in range(x.shape[0]):
        d = int(counts_ref[w])
        assert np.all(got["bins"][w, d:] == -1) and np.all(got["angles"][w, d:] == 0.0) and np.all(got["levels"][w, d:] == 0.0), (ctx, w)
    for d in sorted(set(counts_ref.tolist())):
        idx = np.nonzero(counts_ref == d)[0]
        if d == 0:
            if "spectrum" in got:
                assert helpers.rel_err(got["spectrum"][idx], np.broadcast_to(inv_norm2(table), (len(idx), K))) <= P_RTOL, ctx
            continue
        ref = co.work_batch(x[idx], m, d, table)
        if peak == "local":
            for i in range(len(idx)):
                picks = mo.pick_local_maxima(ref["P"][i], d, K, exclusion=EXCL)
                ref["angles"][i] = [q[0] for q in picks]
                ref["levels"][i] = [q[1] for q in picks]
                ref["bins"][i] = [q[2] for q in picks]
        assert np.array_equal(got["bins"][idx, :d], ref["bins"]), (ctx, d)
        assert np.array_equal(got["angles"][idx, :d], ref["angles"]), (ctx, d)
        filled = ref["bins"] >= 0
        assert np.all(got["levels"][idx, :d][~filled] == 0.0), (ctx, d)
        assert helpers.rel_err(got["levels"][idx, :d][filled], ref["levels"][filled]) <= P_RTOL, (ctx, d)
        if "spectrum" in got:
            assert helpers.rel_err(got["spectrum"][idx], ref["P"]) <= P_RTOL, (ctx, d)


CASES = [(m, N, rule, peak, spec) for m in (4, 5, 8, 12, 16) for N in (256, 4096) for rule in ("mdl", "aic")
         for peak in ("top", "local") for spec in (False, True)]


@pytest.mark.parametrize("m,N,rule,peak,spectrum", CASES, ids=lambda v: str(v))
def test_counts_and_peaks_match_oracle(m, N, rule, peak, spectrum):
    ctx = (m, N, rule, peak, spectrum)
    table, x, truth = so.mixed_windows(m, N, K, SEED + m)
    # the oracle's count, and no near-tie between the best and the runner-up criterion
    est = [so.estimate_source_count(np.linalg.eigvalsh(mo.covariance(x[w], m)), N, NMAX, rule) for w in range(len(x))]
    counts_ref = np.array([e[0] for e in est], np.int32)
    assert min(so.margin(e[1]) for e in est) > MARGIN, ctx
    assert set(counts_ref.tolist()) >= {0, 1, 2}, ctx

    blk = music_doa(m, NMAX, m * N, table.tolist(), K)
    if peak == "local":
        blk.set_peak_mode("local_maxima", EXCL)
    blk.set_source_rule(rule)
    got, _ = gh.device_call(blk, x, COUNTS + (("spectrum",) if spectrum else ()))
    check_against_oracles(got, x, m, N, table, rule, peak, NMAX, counts_ref, ctx)
    # the same definition applied to the GPU's own eigenvalues
    internals, _ = gh.device_call(blk, x, PEAKS + ("eigvals",))
    gpu_counts = [so.estimate_source_count(internals["eigvals"][w], N, NMAX, rule)[0] for w in range(len(x))]
    assert np.array_equal(gpu_counts, counts_ref), ctx
    blk.close()
    # a FIXED handle created with n = count gives the same bins on those windows
    for d in sorted(set(counts_ref.tolist()) - {0}):
        idx = np.nonzero(counts_ref == d)[0]
        fx = music_doa(m, d, m * N, table.tolist(), K)
        if peak == "local":
            fx.set_peak_mode("local_maxima", EXCL)
        ref, _ = gh.device_call(fx, x[idx], PEAKS + (("spectrum",) if spectrum else ()))
        fx.close()
        assert np.array_equal(got["bins"][idx, :d], ref["bins"]), (ctx, d)
        assert np.array_equal(got["angles"][idx, :d], ref["angles"]), (ctx, d)
        assert helpers.rel_err(got["levels"][idx, :d][ref["bins"] >= 0], ref["levels"][ref["bins"] >= 0]) <= P_RTOL, (ctx, d)


@pytest.mark.parametrize("m", [4, 8, 16])
@pytest.mark.parametrize("spectrum", [False, True])
def test_single_source_handle(m, spectrum):
    """n = 1: the count is 0 or 1; peaks-only runs scan_peak1_kernel, the spectrum the arg-max scan_kernel"""
    N = 4096
    table, x, _ = so.mixed_windows(m, N, K, SEED + 31 * m, counts=(0, 1, 2))
    est = [so.estimate_source_count(np.linalg.eigvalsh(mo.covariance(x[w], m)), N, 1, "mdl") for w in range(len(x))]
    counts_ref = np.array([e[0] for e in est], np.int32)
    assert min(so.margin(e[1]) for e in est) > MARGIN and set(counts_ref.tolist()) == {0, 1}
    blk = music_doa(m, 1, m * N, table.tolist(), K)
    blk.set_source_rule("mdl")
    got, launches = gh.device_call(blk, x, COUNTS + (("spectrum",) if spectrum else ()))
    blk.close()
    assert launches == 4, launches  # covariance + eig + count + scan
    check_against_oracles(got, x, m, N, table, "mdl", "top", 1, counts_ref, (m, spectrum))


def test_launches_m4_peak_only_and_back_to_fixed():
    m, N = 4, 1024
    table, x, _ = so.mixed_windows(m, N, K, SEED, counts=(0, 1))
    blk = music_doa(m, 1, m * N, table.tolist(), K)
    _, l_fixed = gh.device_call(blk, x, PEAKS)
    assert l_fixed == 1  # the fused kernel
    blk.set_source_rule("mdl")
    got, l_mdl = gh.device_call(blk, x, COUNTS)
    assert l_mdl == 4  # cov4_tma + eig + source count + scan_peak1, no top-n
    assert np.array_equal(got["counts"], [0] * 3 + [1] * 3)
    blk.set_source_rule("fixed")
    _, l_back = gh.device_call(blk, x, PEAKS)
    assert l_back == 1
    got, l_cnt = gh.device_call(blk, x, COUNTS)
    assert np.all(got["counts"] == 1) and l_cnt == 2  # the fused kernel plus the fill of the counts
    blk.close()


def test_sub_batches_match_per_range_calls():
    """more windows than one workspace slot holds: the whole call equals the per-sub-range calls bit for bit"""
    m, n, N, Kb, W = 4, 2, 64, 36000, 3000
    rng = np.random.default_rng(808)
    pos = 0.6 * np.stack([np.cos(2 * np.pi * np.arange(m) / m), np.sin(2 * np.pi * np.arange(m) / m)], axis=1)
    th = np.arange(Kb) * (2.0 * np.pi / Kb)
    table = np.exp(-2j * np.pi * (np.outer(np.cos(th), pos[:, 0]) + np.outer(np.sin(th), pos[:, 1]))).astype(np.complex64)
    xx = (rng.standard_normal((W, N, m)) + 1j * rng.standard_normal((W, N, m))) / np.sqrt(2.0)
    for w in range(W):
        for _ in range(w % 3):
            a = table[int(rng.integers(0, Kb))].astype(np.complex128)
            xx[w] += 5.0 * a[None, :] * (rng.standard_normal((N, 1)) + 1j * rng.standard_normal((N, 1)))
    x = xx.reshape(W, N * m).astype(np.complex64)
    blk = music_doa(m, n, N * m, table.tolist(), Kb)
    blk.set_source_rule("mdl")
    dev = torch.device("cuda:0")
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)

    def outs():
        return [torch.full((W, n), gh.SENTINEL, dtype=torch.float32, device=dev), torch.full((W, n), gh.SENTINEL, dtype=torch.float32, device=dev),
                torch.full((W, n), gh.SENTINEL, dtype=torch.int32, device=dev), torch.full((W,), gh.SENTINEL, dtype=torch.int32, device=dev)]

    def run(o, w0, nw):
        l0 = blk.launch_count()
        blk.process_device(d_in[w0].data_ptr(), nw, o[0][w0].data_ptr(), o[1][w0].data_ptr(), None, o[2][w0].data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream, d_counts=o[3][w0].data_ptr())
        torch.cuda.synchronize()
        return blk.launch_count() - l0

    per_sub = 5  # cov4_tma + eig + count + scan + top-n
    whole = outs()
    launches = run(whole, 0, W)
    assert launches % per_sub == 0 and launches // per_sub >= 2
    probe = outs()
    lo, hi = 1, W
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if run(probe, 0, mid) == per_sub:
            lo = mid
        else:
            hi = mid
    sub = lo
    assert -(-W // sub) == launches // per_sub and W % sub != 0
    parts = outs()
    for w0 in range(0, W, sub):
        assert run(parts, w0, min(sub, W - w0)) == per_sub
    for a, b in zip(whole, parts):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    counts = whole[3].cpu().numpy()
    assert set(counts.tolist()) <= {0, 1, 2} and np.all(counts >= 0)
    # the definition on both sides of every boundary, and the C oracle's bins at n = count
    idx = sorted({0, W - 1} | {w for b in range(sub, W, sub) for w in (b - 1, b) if w < W})
    bins = whole[2].cpu().numpy()
    for w in idx:
        d = so.work(x[w], m, n, table, "mdl")["count"]
        assert counts[w] == d, w
        ref = co.work_batch(x[w:w + 1], m, d, table)["bins"][0] if d else np.zeros(0, np.int32)
        assert np.array_equal(bins[w, :d], ref) and np.all(bins[w, d:] == -1), w
    blk.close()


def test_zero_and_nan_windows_have_no_sources():
    m, N = 8, 256
    table, x, _ = so.mixed_windows(m, N, K, SEED, per=2, counts=(1, 2))
    x = x.copy()
    x[0] = 0
    x[2, 17] = np.nan
    for rule in ("mdl", "aic"):
        blk = music_doa(m, NMAX, m * N, table.tolist(), K)
        blk.set_source_rule(rule)
        got, _ = gh.device_call(blk, x, COUNTS + ("spectrum",))
        blk.close()
        assert got["counts"][0] == 0 and got["counts"][2] == 0, rule
        for w in (0, 2):
            assert np.all(got["bins"][w] == -1) and np.all(got["levels"][w] == 0) and np.all(got["angles"][w] == 0)
        assert np.all(got["counts"][[1, 3]] >= 1)


def run_entries(blk, x, m, N):
    """work() (host entry) outputs and counts"""
    W = x.shape[0]
    ang, lvl = np.zeros((W, NMAX), np.float32), np.zeros((W, NMAX), np.float32)
    assert blk.work(W, [x], [ang, lvl]) == W
    return ang, lvl, blk.last_bins().copy(), blk.last_counts().copy()


def test_host_device_multi_device_and_planar_entries():
    m, N = 8, 256
    table, x, _ = so.mixed_windows(m, N, K, SEED + 5, per=5)
    W = x.shape[0]
    blk = music_doa(m, NMAX, m * N, table.tolist(), K)
    ang, lvl, bins, cnt = run_entries(blk, x, m, N)
    assert np.all(cnt == NMAX)  # FIXED: every count is n
    blk.set_source_rule("mdl")
    dref, _ = gh.device_call(blk, x, COUNTS)
    ang, lvl, bins, cnt = run_entries(blk, x, m, N)
    assert np.array_equal(cnt, dref["counts"]) and np.array_equal(bins, dref["bins"]) and np.array_equal(ang, dref["angles"])
    assert np.array_equal(lvl.view(np.int32), dref["levels"].view(np.int32))
    assert set(cnt.tolist()) >= {0, 1, 2, 3}
    # planar streams honour the rule (no counts returned)
    pa = np.zeros((W, NMAX), np.float32)
    blk.work_planar(W, helpers.antenna_streams(x, m), [pa])
    assert np.array_equal(blk.last_bins(), dref["bins"]) and np.array_equal(pa, dref["angles"])
    blk.close()
    # multi-device handles: "0" and every GPU, windows dealt round-robin, counts in stream order
    for devices in ([0], list(range(torch.cuda.device_count()))):
        mb = music_doa(m, NMAX, m * N, table.tolist(), K, devices=devices)
        mb.set_source_rule("mdl")
        a2, l2, b2, c2 = run_entries(mb, x, m, N)
        assert np.array_equal(c2, dref["counts"]) and np.array_equal(b2, dref["bins"]) and np.array_equal(a2, dref["angles"]), devices
        g, _ = gh.device_call(mb, x, COUNTS)
        assert np.array_equal(g["counts"], dref["counts"]) and np.array_equal(g["bins"], dref["bins"]), devices
        mb.close()


def test_invalid_rules_are_rejected():
    L = _capi.load()
    m, N = 4, 4
    table = np.ones((K, m), np.complex64)
    blk = music_doa(m, 1, m * N, table.tolist(), K)  # N == m: the criteria are meaningless
    for rule in (1, 2):
        assert L.music_b200_set_source_rule(blk._h, rule) == _capi.EINVAL
    assert L.music_b200_set_source_rule(blk._h, 0) == _capi.OK
    with pytest.raises(_capi.MusicB200Error):
        blk.set_source_rule("mdl")
    with pytest.raises(ValueError):
        blk.set_source_rule("bic")
    blk.close()
    blk = music_doa(m, 1, m * 5, table.tolist(), K)  # N = 5 > m
    for rule in (-1, 3, 7):
        assert L.music_b200_set_source_rule(blk._h, rule) == _capi.EINVAL
    assert L.music_b200_set_source_rule(blk._h, 1) == _capi.OK and L.music_b200_set_source_rule(blk._h, 2) == _capi.OK
    blk.close()


@pytest.mark.parametrize("rule", [1, 2])
def test_cpp_block_source_rule(rule):
    m, N = 8, 4096
    table, x, _ = so.mixed_windows(m, N, K, SEED + 8)
    W = x.shape[0]
    c = gh.run_cpp_block("test_block", struct.pack("<5I", m, NMAX, m * N, K, W), [table, table, x],
                         [("a", np.float32, W * NMAX), ("l", np.float32, W * NMAX), ("s", np.float32, W * K),
                          ("b", np.int32, W * NMAX), ("c", np.int32, W)], args=(rule,))
    ang, lvl, spec = c["a"].reshape(W, NMAX), c["l"].reshape(W, NMAX), c["s"].reshape(W, K)
    bins, counts = c["b"].reshape(W, NMAX), c["c"]
    name = {1: "mdl", 2: "aic"}[rule]
    ref = [so.estimate_source_count(np.linalg.eigvalsh(mo.covariance(x[w], m)), N, NMAX, name)[0] for w in range(W)]
    got = {"angles": ang, "levels": lvl, "spectrum": spec, "bins": bins, "counts": counts}
    check_against_oracles(got, x, m, N, table, name, "top", NMAX, np.array(ref, np.int32), ("cpp", rule))
