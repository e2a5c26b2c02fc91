"""CPU half of the covariance checks (tests/covariance_oracle.py): the exact reference agrees with itself, the numpy
restatements of the kernels' summation orders pass every input family within the per-entry bound, and each planted
defect is rejected.  The integration's c and N_eff formulas of music_integrate.cuh are held to the 60-digit values."""
import math

import numpy as np
import pytest

import covariance_oracle as co

EPS = co.EPS


def windows(family, seed, N, m, W=2):
    rng = np.random.default_rng(seed)
    if family == "e1":
        return co.family_e1(rng, W, N, m)
    if family == "e1_scaled":
        return co.family_e1(rng, W, N, m, k=-100)
    if family == "e2":
        return co.family_e2(rng, W, N, m)
    if family == "e3":
        return co.family_e3(rng, W, N, m)[0]
    return co.family_e3(rng, W, N, m, common=2.0 ** 20)[0]


FAMILIES = ["e1", "e1_scaled", "e2", "e3", "e3_common"]


def checker_accepts(emulated, x, kernel, e1_k=None):
    """the GPU test's checks on one window: the per-entry bound, exact Hermitian form and, on E1 windows scaled by
    2^e1_k, bit equality with fl(S / N)"""
    N, m = x.shape
    L = co.depth("cov_generic_kernel" if kernel == "generic" else "cov_tile_kernel<false>", m, N)
    if co.raw_ratios(emulated, x, L) > 1.0:
        return False
    if e1_k is not None and not np.array_equal(emulated, co.e1_reference(x[None], e1_k)[0]):
        return False
    return np.array_equal(emulated, emulated.T.conj()) and np.all(emulated.diagonal().imag == 0)


def test_exact_sums_against_fractions():
    rng = np.random.default_rng(1)
    x = co.family_e2(rng, 1, 37, 5)[0]
    re, im = co.exact_R(x)
    X = [[(int(v.real * 2 ** 149), int(v.imag * 2 ** 149)) for v in row] for row in x.astype(np.complex128)]
    for i in range(5):
        for j in range(5):
            sre = sum(a[i][0] * a[j][0] + a[i][1] * a[j][1] for a in X)
            sim = sum(a[i][1] * a[j][0] - a[i][0] * a[j][1] for a in X)
            assert re[i, j] * 37 * 2 ** 298 == sre and im[i, j] * 37 * 2 ** 298 == sim


@pytest.mark.parametrize("k", [0, -140, 96])
def test_e1_reference_is_the_rounded_exact_quotient(k):
    x = co.family_e1(np.random.default_rng(2), 2, 129, 6, k=k)
    ref = co.e1_reference(x, k)
    for w in range(2):
        re, im = co.exact_R(x[w])
        assert np.array_equal(ref[w].real, co.rounded(re)) and np.array_equal(ref[w].imag, co.rounded(im))


@pytest.mark.parametrize("kernel,m", [("warp", 4), ("warp", 8), ("generic", 3), ("generic", 7)])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("N", [33, 255, 1000])
def test_restated_kernels_pass(kernel, m, family, N):
    x = windows(family, N + m, N, m)
    for w in range(len(x)):
        k = {"e1": 0, "e1_scaled": -100}.get(family)
        assert checker_accepts(co.emulate_R(x[w], kernel), x[w], kernel, k), (kernel, family, N)


@pytest.mark.parametrize("defect,family,N", [("f32_lane", "e2", 255), ("drop_tail", "e1", 33), ("twice_tail", "e1", 33),
                                              ("drop_tail", "e1", 1000), ("recip", "e1", 255), ("no_conj", "e1", 33)])
@pytest.mark.parametrize("kernel", ["warp", "generic"])
def test_planted_defects_fail(defect, family, N, kernel):
    m = 4 if kernel == "warp" else 5
    x = windows(family, 7, N, m, W=3)
    k = 0 if family == "e1" else None
    assert not all(checker_accepts(co.emulate_R(x[w], kernel, defect), x[w], kernel, k) for w in range(len(x))), defect


def test_e3_zeros_are_exact_and_e4_families_are_well_formed():
    x, zero = co.family_e3(np.random.default_rng(3), 1, 33, 6, common=2.0 ** 20)
    re, im = co.exact_R(x[0])
    assert all(re[i, j] == 0 and im[i, j] == 0 for i, j in zip(*np.nonzero(zero)))
    Are, _ = co.abs_sums(x[0])
    assert np.min(Are[zero]) > 2.0 ** 38
    bad, ok, r = co.family_e4(np.random.default_rng(4), 3, 40, 5, math.nan)
    assert np.all(np.isnan(bad).sum(axis=(1, 2)) == 1) and not np.any(np.isnan(ok))


# ---- integration ----
ALPHAS = [2.0 ** -1074, 1e-300, 0.5, 0.99, 1 - 2.0 ** -20, 1 - 1e-6, 1 - 1e-8, 1 - 2.0 ** -40, math.nextafter(1.0, 0.0)]


@pytest.mark.parametrize("alpha", ALPHAS)
def test_integ_c_and_neff_formulas(alpha):
    for n in (1, 31, 32, 33, 63, 1000, 10 ** 5, 10 ** 9):
        c, neff = co.exact_c_neff(alpha, n, 32)
        assert abs(co.integ_c(alpha, n) - float(c)) <= co.C_POW * EPS * float(c), (alpha, n)
        assert abs(co.integ_neff(alpha, n, 32) - float(neff)) <= co.C_NEFF * EPS * float(neff), (alpha, n)


@pytest.mark.parametrize("alpha", [1 - 1e-6, 1 - 1e-8])
def test_closed_form_c_and_naive_q_fail(alpha):
    n = 32
    c, neff = co.exact_c_neff(alpha, n, 32)
    assert abs(co.integ_c(alpha, n, closed_form=True) - float(c)) > co.C_POW * EPS * float(c)
    assert abs(co.integ_neff(alpha, n, 32, naive_q=True) - float(neff)) > co.C_NEFF * EPS * float(neff)


def _stream(W, m, seed):
    rng = np.random.default_rng(seed)
    X = (rng.standard_normal((W, 8, m)) + 1j * rng.standard_normal((W, 8, m))).astype(np.complex64).astype(np.complex128)
    return np.einsum("wti,wtj->wij", X, X.conj()) / 8


@pytest.mark.parametrize("alpha,W", [(0.99, 100), (1 - 1e-6, 70), (1 - 1e-8, 70), (0.5, 33)])
def test_restated_integration_passes_and_closed_form_fails(alpha, W):
    R = _stream(W, 2, 5)
    hi, lo, _, _ = co.integrate_exact(R, alpha)
    bound = co.integ_bounds(R, alpha, [W])
    flat = np.stack([R.real, R.imag], axis=-1).reshape(W, -1)

    def unflat(a):
        a = a.reshape(W, 2, 2, 2)
        return a[..., 0] + 1j * a[..., 1]

    good = unflat(co.emulate_integration(flat, alpha))
    assert np.max(co.integ_ratios(good, hi, lo, bound)) <= 1.0
    bad = unflat(co.emulate_integration(flat, alpha, closed_form=True))
    worst = np.max(co.integ_ratios(bad, hi, lo, bound))
    if alpha >= 1 - 1e-6:
        assert worst > 1.0, worst


def test_every_call_adds_its_carry_to_the_bound():
    # the carried error of each earlier sub-batch enters the bound with eps once, as the in-batch depth does: on
    # identity covariances (Abar = 1) at alpha near 1 the last window of 20 calls of 1000 windows gets several times the
    # in-batch allowance C_INT L(1000) eps, while the first call has no carry at all
    W, alpha = 20000, 1 - 1e-6
    R = np.broadcast_to(np.eye(2, dtype=np.complex128), (W, 2, 2))
    many = co.integ_bounds(R, alpha, [1000] * 20)
    in_batch = co.C_INT * co.integ_depth(1000) * EPS
    assert np.allclose(many[:1000, 0, 0].real, in_batch, rtol=1e-12, atol=0)
    assert many[-1, 0, 0].real > 5 * in_batch
    assert np.all(np.diff(many[999::1000, 0, 0].real) > 0)  # and it grows from call to call


# ---- channels ----
CHANNEL_CASES = [(4, 16, 3, "hann"), (2, 64, 2, "rect"), (4, 256, 1, "hann"), (3, 8, 5, "rect")]


@pytest.mark.parametrize("m,F,J,kind", CHANNEL_CASES)
def test_restated_filter_bank_passes_and_a_float32_twiddle_fails(m, F, J, kind):
    x = co.channel_windows(np.random.default_rng(F + J), 1, m, F, J, 3, 5)[0]
    bins = [3, 5, F - 1]
    tw = co.twiddles(F)
    assert max(co.channel_ratios(co.emulate_channel_R(x, m, F, bins, kind, tw), x, m, F, bins, kind)) <= 1.0
    bad = tw.copy()
    k = F // 2 - 3
    bad[k] = np.complex64(bad[k])
    assert max(co.channel_ratios(co.emulate_channel_R(x, m, F, bins, kind, bad), x, m, F, bins, kind)) > 1.0


HOST_TABLES = r"""
#include <cmath>
#include <cstdio>
struct double2 { double x, y; };
inline double2 make_double2(double x, double y) { return {x, y}; }
namespace music {
constexpr int CHAN_HANN = 1;
BODY
}
int main()
{
    static double2 tw[128];
    static double taper[256];
    for (int F = 8; F <= 256; F *= 2) {
        const double sum = music::chan_tables_host(F, music::CHAN_HANN, tw, taper);
        for (int k = 0; k < F / 2; ++k) std::printf("tw %d %d %a %a\n", F, k, tw[k].x, tw[k].y);
        for (int t = 0; t < F; ++t) std::printf("taper %d %d %a\n", F, t, taper[t]);
        std::printf("sum %d %a\n", F, sum);
    }
}
"""


def test_host_tables_are_correctly_rounded(tmp_path):
    """chan_tables_host, compiled by the host compiler with a two-line double2: every twiddle is the correctly rounded
    exp(-2 pi i k / F) for F = 8 ... 256, and every Hann value is 1/2 - 1/2 c in one rounding of that correctly rounded
    cosine (so within eps h + eps / 2 of the exact taper)"""
    import os
    import subprocess
    import mpmath as mp
    src = open(os.path.join(os.path.dirname(__file__), "..", "gr-baz_b200", "csrc", "music_channels.cuh")).read()
    body = src[src.index("inline void chan_cos_sin"):src.rindex("}  // namespace music")]
    (tmp_path / "t.cc").write_text(HOST_TABLES.replace("BODY", body))
    subprocess.check_call(["c++", "-O2", "-std=c++17", "-o", str(tmp_path / "t"), str(tmp_path / "t.cc")])
    out = subprocess.run([str(tmp_path / "t")], capture_output=True, text=True, check=True).stdout.split("\n")
    tw, taper = {}, {}
    for line in filter(None, out):
        f = line.split()
        if f[0] == "tw":
            tw[int(f[1]), int(f[2])] = complex(float.fromhex(f[3]), float.fromhex(f[4]))
        elif f[0] == "taper":
            taper[int(f[1]), int(f[2])] = float.fromhex(f[3])
    for F in (8, 16, 32, 64, 128, 256):
        ref = co.twiddles(F)
        assert all(tw[F, k] == ref[k] for k in range(F // 2)), F
        with mp.workdps(50):
            for t in range(F):
                c = float(mp.cospi(mp.mpf(2 * t) / F))
                h = mp.mpf(1) / 2 - mp.cospi(mp.mpf(2 * t) / F) / 2
                assert taper[F, t] == 0.5 - 0.5 * c, (F, t)
                assert abs(taper[F, t] - h) <= EPS * h + EPS / 2, (F, t)
