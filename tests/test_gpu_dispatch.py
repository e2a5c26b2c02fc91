"""GPU: every kernel instantiation the unfused and fused dispatch can choose (launch_cov, launch_eig_scan and
enqueue_device in gr-baz_b200/csrc/music_b200.cu), for every M from 2 to 16, against the fp64 C oracle.  The launch
count of each call proves which branch ran.  Also: exact invariance to power-of-two scaling at both ends of the float32
range, and the sub-batch loop of the unfused path (more windows than one workspace slot holds).

Gates: peak bins and angles bit-exact, levels / spectrum / P <= 1e-5 relative (the north-star tolerance); where the
golden fixtures hold a tighter bound (P, R, eigenvalues) the same bound is held here."""
import numpy as np
import pytest
import torch

from gr_baz_b200.music_doa import music_doa
from oracle import c_oracle as co
from oracle import music_oracle as mo

import helpers

pytestmark = pytest.mark.gpu

P_RTOL = 1e-5
SENTINEL = -7
LOCAL_EXCL = 3  # exclusion_bins of the local-maxima rows


def element_positions(geometry, m, rng):
    """random planar positions (in wavelengths) or a uniform circular array: no mirror symmetry, so no exact ties"""
    if geometry == "uca":
        a = 2.0 * np.pi * np.arange(m) / m
        return 0.6 * np.stack([np.cos(a), np.sin(a)], axis=1)
    return rng.uniform(-1.5, 1.5, (m, 2))


def steering_table(pos, K):
    """[K][m] complex64 steering vectors exp(-2 pi i <p, u(theta_k)>), theta_k = k * 360 / K degrees"""
    th = np.arange(K) * (2.0 * np.pi / K)
    phase = np.outer(np.cos(th), pos[:, 0]) + np.outer(np.sin(th), pos[:, 1])
    return np.exp(-2j * np.pi * phase).astype(np.complex64)


def make_windows(rng, table, n, N, W, signal):
    """W windows of N snapshots: unit complex noise, plus (signal == "strong") n sources of amplitude 5 on grid rows,
    or (signal == "mixed") that on every other window"""
    K, m = table.shape
    x = (rng.standard_normal((W, N, m)) + 1j * rng.standard_normal((W, N, m))) / np.sqrt(2.0)
    for w in range(W):
        if signal == "strong" or (signal == "mixed" and w % 2 == 0):
            for _ in range(n):
                a = table[int(rng.integers(0, K))].astype(np.complex128)
                x[w] += 5.0 * a[None, :] * (rng.standard_normal((N, 1)) + 1j * rng.standard_normal((N, 1)))
    return x.reshape(W, N * m).astype(np.complex64)


def rank_deficient(m, n, N):
    """R has rank min(N, m).  With N < m - n the reference itself can divide by zero; with N < n the boundary between
    noise and signal subspace falls inside the null space of R, so which vectors form G is arbitrary."""
    return N < max(n, m - n)


class Device:
    """device buffers of one call, pre-filled with a sentinel so that an unwritten slot shows"""

    def __init__(self, x, m, n, K, spectrum=False, internals=False):
        dev = torch.device("cuda:0")
        W = x.shape[0]
        self.d_in = torch.from_numpy(x.view(np.float32)).to(dev)
        self.ang = torch.full((W, n), SENTINEL, dtype=torch.float32, device=dev)
        self.lvl = torch.full((W, n), SENTINEL, dtype=torch.float32, device=dev)
        self.bins = torch.full((W, n), SENTINEL, dtype=torch.int32, device=dev)
        self.spec = torch.full((W, K), SENTINEL, dtype=torch.float32, device=dev) if spectrum else None
        self.P = torch.full((W, K), SENTINEL, dtype=torch.float64, device=dev) if internals else None
        self.R = torch.full((W, m, m, 2), SENTINEL, dtype=torch.float64, device=dev) if internals else None
        self.ev = torch.full((W, m), SENTINEL, dtype=torch.float64, device=dev) if internals else None

    def run(self, blk, w0=0, nw=None, into=None):
        """process_device on windows w0 .. w0 + nw - 1, written to the same rows of `into` (default self); returns the
        number of kernel launches the call made"""
        nw = self.d_in.shape[0] - w0 if nw is None else nw
        o = self if into is None else into
        p = lambda t: None if t is None else t[w0].data_ptr()
        l0 = blk.launch_count()
        blk.process_device(self.d_in[w0].data_ptr(), nw, p(o.ang), p(o.lvl), p(o.spec), p(o.bins),
                           stream=torch.cuda.current_stream().cuda_stream, d_P64=p(o.P), d_R=p(o.R), d_eigvals=p(o.ev))
        torch.cuda.synchronize()
        return blk.launch_count() - l0

    def host(self):
        out = {"angles": self.ang.cpu().numpy(), "levels": self.lvl.cpu().numpy(), "bins": self.bins.cpu().numpy()}
        if self.spec is not None:
            out["spectrum"] = self.spec.cpu().numpy()
        if self.P is not None:
            R = self.R.cpu().numpy()
            out.update(P=self.P.cpu().numpy(), R=R[..., 0] + 1j * R[..., 1], eigvals=self.ev.cpu().numpy())
        return out


def oracle(x, m, n, table, mode):
    """the C oracle's outputs; in local-maxima mode the peaks are oracle/music_oracle.py::pick_local_maxima of its P"""
    ref = co.work_batch(x, m, n, table)
    if mode == "local":
        K = table.shape[0]
        for w in range(x.shape[0]):
            picks = mo.pick_local_maxima(ref["P"][w], n, K, exclusion=LOCAL_EXCL)
            ref["angles"][w] = [p[0] for p in picks]
            ref["levels"][w] = [p[1] for p in picks]
            ref["bins"][w] = [p[2] for p in picks]
    return ref


def assert_matches_oracle(got, ref, ctx):
    assert np.array_equal(got["bins"], ref["bins"]), (ctx, np.argwhere(got["bins"] != ref["bins"])[:5])
    assert np.array_equal(got["angles"], ref["angles"]), ctx
    filled = ref["bins"] >= 0  # n > K, or no positive strength left: the initial (0, 0) pair
    assert np.all(got["levels"][~filled] == 0.0), ctx
    assert helpers.rel_err(got["levels"][filled], ref["levels"][filled]) <= P_RTOL, ctx
    if "spectrum" in got:
        assert helpers.rel_err(got["spectrum"], ref["P"]) <= P_RTOL, ctx


def assert_well_formed(got, K, ctx):
    """what must hold even where the values are not comparable: every slot written, bins in [-1, K), a filled slot
    carries a positive level"""
    for k in ("angles", "levels", "bins"):
        assert not np.any(got[k] == SENTINEL), (ctx, k)
    assert np.all((got["bins"] >= -1) & (got["bins"] < K)), ctx
    assert np.all(got["levels"][got["bins"] >= 0] > 0), ctx
    if "spectrum" in got:
        assert not np.any(got["spectrum"] == SENTINEL), ctx


# One row per branch.  Covariance: cov4_tma (M = 4), covN_tma (M = 8 with even N >= 128, M = 16 with N >= 128),
# cov_tile_kernel<false> (+ <true> for M > 4: 2 launches; other M % 4 == 0), cov_generic_kernel (M % 4 != 0).
# Eigensolver: eig_kernel<4, true> (M = 4), eig_coop_kernel<8/12/16>, eig_kernel<8, false> (M = 2, 3, 5, 6, 7),
# eig_kernel<MAXM, false> (M = 9, 10, 11, 13, 14, 15).  Scan: scan_kernel<4/8/16, ...>, scan_kernel<0, ...> (other M),
# scan_peak1_kernel<8/16> (n = 1, peaks only, unfused).  Top-n (n >= 2) or topn_local_kernel (local-maxima mode).
# Fused: music4_fused_kernel (M = 4, n = 1, no internals; with or without the spectrum), music8_fused_kernel (M = 8,
# n = 1, peaks only, even N >= 128).
# Expected launches per call, for the three calls of a row: (spectrum + P + R + eigenvalues, spectrum only, peaks only)
#   unfused: covariance launches + 1 eig + 1 scan (+ 1 top-n when n >= 2 or in local-maxima mode); fused: 1.
CASES = [
    # branch                                          m   n    N     K   geometry  signal    W  mode     launches
    ("generic cov E=3, eig<8>, scan<0>, N=1",          2,  1,   1,  257, "planar", "noise",  16, "top",   (3, 3, 3)),
    ("generic cov E=3, eig<8>, scan<0>",               2,  1, 256, 3600, "planar", "strong", 16, "top",   (3, 3, 3)),
    ("generic cov E=6, eig<8>, scan<0>",               3,  1, 129,  256, "uca",    "strong", 12, "top",   (3, 3, 3)),
    ("generic cov, top-n n=M-1",                       3,  2,   7, 3600, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("generic cov, top-n n=M-1",                       3,  2, 128,  255, "planar", "strong", 12, "top",   (4, 4, 4)),
    ("cov4_tma, eig<4,true>; fused M=4",               4,  1, 256, 3600, "uca",    "strong", 16, "top",   (3, 1, 1)),
    ("cov4_tma, eig<4,true>; fused M=4",               4,  1, 127,  257, "planar", "noise",  16, "top",   (3, 1, 1)),
    ("cov4_tma, scan<4>, top-n n==M-n",                4,  2,   7,  255, "planar", "strong", 12, "top",   (4, 4, 4)),
    ("cov4_tma, scan<4>, top-n n==M-n",                4,  2, 256, 3600, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("cov4_tma, scan<4>, top-n n=M-1",                 4,  3, 129,  256, "planar", "strong", 12, "top",   (4, 4, 4)),
    ("cov4_tma, rank-deficient",                       4,  3,   1,    7, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=15, eig<8>, scan<0>",              5,  1, 128, 3600, "planar", "noise",  12, "top",   (3, 3, 3)),
    ("generic cov E=15, scan<0> signal form",          5,  2, 256,  255, "uca",    "strong", 12, "top",   (4, 4, 4)),
    ("generic cov E=15, top-n n=M-1",                  5,  4,   7,  257, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("generic cov E=15, top-n n=M-1",                  5,  4, 129, 3600, "planar", "strong", 12, "top",   (4, 4, 4)),
    ("generic cov E=21, eig<8>, scan<0>",              6,  1,   7,  256, "planar", "strong", 12, "top",   (3, 3, 3)),
    ("generic cov E=21, top-n n==M-n",                 6,  3, 256, 3600, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("generic cov E=21, top-n n==M-n",                 6,  3, 127,  257, "planar", "strong", 12, "top",   (4, 4, 4)),
    ("generic cov E=21, top-n n=M-1",                  6,  5, 128,  255, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("generic cov E=28 S=9, eig<8> M=7",               7,  1, 256, 3600, "planar", "strong", 12, "top",   (3, 3, 3)),
    ("generic cov E=28 S=9, eig<8> M=7",               7,  1, 129,  255, "planar", "noise",  12, "top",   (3, 3, 3)),
    ("generic cov E=28, scan<0> signal form",          7,  3, 127, 3600, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("generic cov E=28, scan<0> signal form",          7,  3,   7,  257, "uca",    "strong", 12, "top",   (4, 4, 4)),
    ("generic cov E=28, top-n n=M-1",                  7,  6, 256,  256, "planar", "strong", 12, "top",   (4, 4, 4)),
    ("generic cov E=28, rank-deficient",               7,  6,   1, 3600, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("covN_tma<8>, eig_coop<8>; fused M=8",            8,  1, 256, 3600, "planar", "strong", 16, "top",   (3, 3, 1)),
    ("covN_tma<8>, eig_coop<8>; fused M=8",            8,  1, 128,  255, "planar", "noise",  16, "top",   (3, 3, 1)),
    ("cov_tile M=8 odd N, scan_peak1<8>",              8,  1, 129, 3600, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("cov_tile M=8 N<128, scan_peak1<8>",              8,  1, 127,  257, "uca",    "strong", 12, "top",   (4, 4, 4)),
    ("covN_tma<8>, top-n n==M-n",                      8,  4, 256, 3600, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("cov_tile M=8 N<128, top-n n==M-n",               8,  4,   7,  256, "planar", "strong", 12, "top",   (5, 5, 5)),
    ("cov_tile M=8 odd N, top-n n=M-1",                8,  7, 129, 3600, "planar", "strong", 12, "top",   (5, 5, 5)),
    ("covN_tma<8>, top-n n=M-1",                       8,  7, 128,  257, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("generic cov E=45, eig<MAXM> M=9",                9,  1, 256, 3600, "planar", "strong", 12, "top",   (3, 3, 3)),
    ("generic cov E=45, eig<MAXM> M=9",                9,  4, 129,  257, "planar", "noise",  12, "top",   (4, 4, 4)),
    ("generic cov E=45, eig<MAXM>, top-n n=M-1",       9,  8, 128,  255, "uca",    "strong", 12, "top",   (4, 4, 4)),
    ("generic cov E=45, rank-deficient",               9,  8,   7, 3600, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=55, eig<MAXM> M=10",              10,  1, 127, 3600, "planar", "noise",  12, "top",   (3, 3, 3)),
    ("generic cov E=55, eig<MAXM>, top-n n==M-n",     10,  5, 256,  256, "planar", "strong", 12, "top",   (4, 4, 4)),
    ("generic cov E=55, eig<MAXM>, top-n n=M-1",      10,  9, 128, 3600, "planar", "strong",  8, "top",   (4, 4, 4)),
    ("generic cov E=55, rank-deficient",              10,  5,   1,  255, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=66 S=3, eig<MAXM> M=11",          11,  1, 129, 3600, "planar", "strong", 12, "top",   (3, 3, 3)),
    ("generic cov E=66 S=3, eig<MAXM>, N<M",          11,  5,   7,  257, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=66 S=3, top-n n=M-1",             11, 10, 256, 3600, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=66 S=3, top-n n=M-1",             11, 10, 129,  255, "planar", "strong",  8, "top",   (4, 4, 4)),
    ("cov_tile M=12, eig_coop<12>",                   12,  1, 256, 3600, "planar", "strong",  8, "top",   (4, 4, 4)),
    ("cov_tile M=12, rank-deficient",                 12,  1,   1,  257, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("cov_tile M=12, top-n n==M-n",                   12,  6, 128, 3600, "planar", "noise",   8, "top",   (5, 5, 5)),
    ("cov_tile M=12, top-n n=M-1 > K",                12, 11, 129,    7, "planar", "strong",  8, "top",   (5, 5, 5)),
    ("generic cov E=91 S=2, eig<MAXM> M=13",          13,  1, 128, 3600, "planar", "noise",   8, "top",   (3, 3, 3)),
    ("generic cov E=91 S=2, eig<MAXM> M=13",          13,  6, 256, 3600, "planar", "strong",  8, "top",   (4, 4, 4)),
    ("generic cov E=91 S=2, top-n n=M-1",             13, 12, 127,  256, "uca",    "strong",  8, "top",   (4, 4, 4)),
    ("generic cov E=91 S=2, rank-deficient",          13, 12,   7,  257, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=105 S=2, eig<MAXM> M=14",         14,  1, 256,  255, "planar", "strong",  8, "top",   (3, 3, 3)),
    ("generic cov E=105 S=2, top-n n==M-n",           14,  7, 129, 3600, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=105 S=2, top-n n=M-1",            14, 13, 256, 3600, "planar", "strong",  8, "top",   (4, 4, 4)),
    ("generic cov E=105 S=2, top-n n=M-1",            14, 13, 128,  256, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=120 S=2, eig<MAXM> M=15",         15,  1, 127, 3600, "planar", "strong",  8, "top",   (3, 3, 3)),
    ("generic cov E=120 S=2, eig<MAXM> M=15",         15,  7, 256,  257, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=120 S=2, top-n n=M-1",            15, 14, 128, 3600, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("generic cov E=120 S=2, top-n n=M-1",            15, 14, 256,  255, "uca",    "strong",  8, "top",   (4, 4, 4)),
    ("covN_tma<16>, eig_coop<16>, scan_peak1<16>",    16,  1, 256, 3600, "planar", "strong",  8, "top",   (3, 3, 3)),
    ("covN_tma<16>, eig_coop<16>, scan_peak1<16>",    16,  1, 128,  255, "planar", "noise",   8, "top",   (3, 3, 3)),
    ("cov_tile M=16 N<128, scan_peak1<16>",           16,  1, 127, 3600, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("cov_tile M=16 N<128, rank-deficient",           16,  1,   7, 3600, "uca",    "strong",  8, "top",   (4, 4, 4)),
    ("cov_tile M=16 N<128, top-n n==M-n",             16,  8, 127, 3600, "planar", "strong",  8, "top",   (5, 5, 5)),
    ("covN_tma<16>, top-n n==M-n",                    16,  8, 256,  256, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("covN_tma<16>, top-n n=M-1",                     16, 15, 129, 3600, "planar", "strong",  8, "top",   (4, 4, 4)),
    ("covN_tma<16>, top-n n=M-1",                     16, 15, 256,  255, "planar", "noise",   8, "top",   (4, 4, 4)),
    ("cov_tile M=16, rank-deficient, n > K",          16, 15,   1,    7, "planar", "noise",   8, "top",   (5, 5, 5)),
    ("topn_local, cov4_tma (no fused kernel)",         4,  1, 128, 3600, "planar", "strong", 12, "local", (4, 4, 4)),
    ("topn_local, covN_tma<8> (no fused kernel)",      8,  1, 256, 3600, "planar", "noise",  12, "local", (4, 4, 4)),
    ("topn_local, generic cov, eig<8>",                7,  3, 256, 3600, "planar", "strong",  8, "local", (4, 4, 4)),
    ("topn_local, generic cov S=2, eig<MAXM>",        13,  6, 129, 3600, "planar", "noise",   8, "local", (4, 4, 4)),
    ("topn_local, cov_tile M=16",                     16,  8, 127,  257, "planar", "strong",  8, "local", (5, 5, 5)),
]


@pytest.mark.parametrize("row", range(len(CASES)), ids=lambda i: "%d-m%d-n%d-N%d-K%d-%s" % ((i,) + CASES[i][1:5] + (CASES[i][6],)))
def test_dispatch_branch_matches_oracle(row):
    branch, m, n, N, K, geometry, signal, W, mode, launches = CASES[row]
    ctx = (row, branch)
    rng = np.random.default_rng(1000 + row)
    table = steering_table(element_positions(geometry, m, rng), K)
    x = make_windows(rng, table, n, N, W, signal)
    blk = music_doa(m, n, N * m, table.tolist(), K)
    if mode == "local":
        blk.set_peak_mode("local_maxima", LOCAL_EXCL)
    calls = [Device(x, m, n, K, spectrum=True, internals=True), Device(x, m, n, K, spectrum=True), Device(x, m, n, K)]
    got = []
    for c, expect in zip(calls, launches):
        assert c.run(blk) == expect, (ctx, "launches")
        got.append(c.host())
    blk.close()
    for g in got:
        assert_well_formed(g, K, ctx)
    # R and its eigenvalues are defined whatever the rank: fp64 covariance of the float32 inputs, LAPACK eigenvalues
    Rref = np.stack([mo.covariance(x[w], m) for w in range(W)])
    scale = np.max(np.abs(Rref))
    assert np.max(np.abs(got[0]["R"] - Rref)) <= 1e-12 * scale, ctx
    assert np.max(np.abs(got[0]["eigvals"] - np.linalg.eigvalsh(Rref))) <= 1e-11 * scale, ctx
    if rank_deficient(m, n, N):
        return
    ref = oracle(x, m, n, table, mode)
    for g in got:
        assert_matches_oracle(g, ref, ctx)
    assert helpers.rel_err(got[0]["P"], ref["P"]) <= 1e-8, ctx  # far inside the 1e-5 gate, as on the golden fixtures


def test_dispatch_table_covers_every_branch():
    """the rows above reach each branch with a strong source and with noise only, at every M and the n / N / K edges"""
    full = [c for c in CASES if not rank_deficient(c[1], c[2], c[3])]
    assert {c[1] for c in CASES} == set(range(2, 17))
    for m in range(2, 17):
        assert {c[2] for c in CASES if c[1] == m} >= {1, m // 2, m - 1}
    assert {c[3] for c in CASES} >= {1, 7, 127, 128, 129, 256}
    assert {c[4] for c in CASES} >= {7, 255, 256, 257, 3600}
    groups = {
        "eig<MAXM,false>": lambda c: c[1] in (9, 10, 11, 13, 14, 15),
        "eig<8,false> M=7": lambda c: c[1] == 7,
        "cov_generic S=2": lambda c: c[1] in (13, 14, 15),
        "cov_tile M=12": lambda c: c[1] == 12,
        "cov_tile M=8 odd N": lambda c: c[1] == 8 and c[3] >= 128 and c[3] % 2,
        "cov_tile M=16 N<128": lambda c: c[1] == 16 and c[3] < 128,
        "covN_tma": lambda c: c[1] in (8, 16) and c[3] >= 128 and c[3] % (16 // c[1]) == 0,
        "top-n n=M-1, M=16": lambda c: c[1] == 16 and c[2] == 15,
        "top-n n==M-n": lambda c: c[2] * 2 == c[1] and c[1] >= 8,
        "fused M=4": lambda c: c[1] == 4 and c[2] == 1 and c[8] == "top",
        "fused M=8": lambda c: c[1] == 8 and c[2] == 1 and c[8] == "top" and c[3] >= 128 and c[3] % 2 == 0,
    }
    for name, hit in groups.items():
        assert {c[6] for c in full if hit(c)} == {"strong", "noise"}, name


# ---- exact power-of-two scaling at the ends of the float32 range ----------------------------------------------------
@pytest.mark.parametrize("m,n,N,spectrum,launches", [(4, 1, 256, False, 1), (8, 1, 256, False, 1), (7, 2, 129, True, 4),
                                                     (13, 6, 256, True, 4)])
def test_power_of_two_scaling_is_exact(m, n, N, spectrum, launches):
    """Windows scaled by 2^-140 (float32 subnormals), 2^-126 (the smallest normal) and 2^96: the covariance scales by an
    exact power of two, so the eigenvectors, P, the bins and the levels must be bit-identical to the unscaled run.  The
    windows are rounded to multiples of 2^-9 first, so that even the subnormal scaling is exact in float32.  M = 4 and
    M = 8 (n = 1, peaks only) run the fused kernels, M = 7 and 13 the unfused generic-M path with the spectrum."""
    K = 3600
    rng = np.random.default_rng(77 + m)
    table = steering_table(element_positions("planar", m, rng), K)
    x = make_windows(rng, table, n, N, 16, "mixed")
    x = (np.round(x.astype(np.complex128) * 512.0) / 512.0).astype(np.complex64)
    blk = music_doa(m, n, N * m, table.tolist(), K)

    def run(xs):
        c = Device(xs, m, n, K, spectrum=spectrum)
        assert c.run(blk) == launches
        return c.host()

    base = run(x)
    ref = co.work_batch(x, m, n, table)
    assert np.array_equal(base["bins"], ref["bins"]) and helpers.rel_err(base["levels"], ref["levels"]) <= P_RTOL
    for e in (-140, -126, 96):
        xs = (x.astype(np.complex128) * 2.0 ** e).astype(np.complex64)
        assert np.array_equal(xs.astype(np.complex128) * 2.0 ** -e, x.astype(np.complex128))  # the scaling is exact
        if e == -140:
            assert np.any((np.abs(xs.real) < 2.0 ** -126) & (xs.real != 0))  # subnormal inputs
        got = run(xs)
        for k in base:
            assert np.array_equal(got[k], base[k]), (e, k)
    blk.close()


# ---- the sub-batch loop of the unfused path -------------------------------------------------------------------------
SUB_CASES = [
    # m  n    N       K     W   mode     spectrum  launches per sub-batch  minimum sub-batches
    (4, 2, 64, 36000, 3000, "top", True, 4, 2),      # cov4_tma + eig + scan + top-n
    (4, 1, 64, 36000, 3000, "local", False, 4, 2),   # cov4_tma + eig + scan + topn_local
    (16, 2, 256, 160000, 1000, "top", True, 4, 3),   # covN_tma + eig + scan + top-n
]


@pytest.mark.parametrize("m,n,N,K,W,mode,spectrum,per_sub,min_subs", SUB_CASES)
def test_sub_batches_match_single_batches_and_oracle(m, n, N, K, W, mode, spectrum, per_sub, min_subs):
    """More windows than one workspace slot holds (the internal fp64 spectrum of K bins per window bounds a sub-batch):
    the call runs in several sub-batches, each of which offsets the input, the outputs and the peak descriptor by its
    first window.  The whole call must equal the same block run on each sub-range separately, bit for bit, and the
    oracle on both sides of every sub-batch boundary."""
    rng = np.random.default_rng(5150 + m + n)
    table = steering_table(element_positions("planar", m, rng), K)
    x = make_windows(rng, table, n, N, W, "mixed")
    blk = music_doa(m, n, N * m, table.tolist(), K)
    if mode == "local":
        blk.set_peak_mode("local_maxima", LOCAL_EXCL)
    whole = Device(x, m, n, K, spectrum=spectrum)
    launches = whole.run(blk)
    assert launches % per_sub == 0
    nsub = launches // per_sub
    assert nsub >= min_subs
    # the sub-batch size: the largest window count that still runs in one sub-batch
    probe = Device(x, m, n, K, spectrum=spectrum)
    lo, hi = 1, W
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if probe.run(blk, 0, mid) == per_sub:
            lo = mid
        else:
            hi = mid
    sub = lo
    assert -(-W // sub) == nsub and W % sub != 0  # several full sub-batches and a ragged last one
    # chunking independence: each sub-range on its own (one sub-batch each) gives the same bits
    parts = Device(x, m, n, K, spectrum=spectrum)
    for w0 in range(0, W, sub):
        assert whole.run(blk, w0, min(sub, W - w0), into=parts) == per_sub
    for k in ("ang", "lvl", "bins", "spec"):
        a, b = getattr(whole, k), getattr(parts, k)
        if a is not None:
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), k
    # the oracle on the first and last windows and on both sides of every boundary
    got = whole.host()
    blk.close()
    idx = sorted({0, W - 1} | {w for b in range(sub, W, sub) for w in (b - 1, b, b + 1) if w < W})
    ref = oracle(x[idx], m, n, table, mode)
    sel = {k: v[idx] for k, v in got.items()}
    assert_well_formed(got, K, "sub-batches")
    assert_matches_oracle(sel, ref, ("sub-batches", idx))
