"""GPU: the ROOTS and ESPRIT peak modes against the mpmath reference and bounds of tests/gridless_oracle.py on the
adversarial window families (comb / cyclic Psi, vanishing outer coefficients, close pairs, end-fire, d = M - 1,
prescribed spectra) for M in {2, 4, 5, 6, 8, 12, 16}, on the GPU's own covariance (d_R).

Under FIXED every slot the reference fills must be filled within its bound, no other slot filled, and every unfilled
slot (0, 0, -1).  Under MDL, every window whose count equals the planted d must give the FIXED outputs bit for bit.
Windows whose bound or selection margin is too wide to compare are counted and printed per family."""
import numpy as np
import pytest

import gpu_harness as gh
import gridless_oracle as go
from helpers import LAM, ula

pytestmark = pytest.mark.gpu

K = 3600


def by_d(fams):
    groups = {}
    for f in fams:
        groups.setdefault(f[3], []).append(f)
    return groups


@pytest.mark.parametrize("mode", ["roots", "esprit"])
@pytest.mark.parametrize("M", [2, 4, 5, 6, 8, 12, 16])
def test_gridless_within_bounds(mode, M):
    pos = ula(M, "x")
    fams = go.families(M, 9000 + M)
    ref_of = go.roots_reference if mode == "roots" else go.esprit_reference
    stats = {}
    for d, group in sorted(by_d(fams).items()):
        x = np.stack([g[2].reshape(-1) for g in group])
        fixed = gh.make_block(M, d, go.N, K, pos=pos, rule="fixed", mode=mode)
        got, lf = gh.device_call(fixed, x, ("levels", "bins", "R"))
        fixed.close()
        mdl = gh.make_block(M, d, go.N, K, pos=pos, rule="mdl", mode=mode)
        gm, lm = gh.device_call(mdl, x, ("levels", "bins", "counts"))
        mdl.close()
        # covariance + eigensolver + root / ESPRIT kernel (+ the source count), as test_gpu_root_music counts them;
        # M = 12 runs one more eigensolver launch (test_gpu_eigensolvers: eig_coop_kernel<12>)
        want = 3 + (M == 12)
        assert (lf, lm) == (want, want + 1), (lf, lm, want)
        for w, (fam, name, xw, _, exact) in enumerate(group):
            ctx = (mode, M, d, fam, name)
            R = got["R"][w]
            if fam == "comb":
                m = np.arange(M)
                off = (m[:, None] - m[None, :]) % d != 0
                assert np.all(R[off] == 0) and np.all(R[~off] != 0), ctx  # the eigensolver sees the block structure
            ref = ref_of(R, d, pos, LAM)
            e, compared, msg = go.check(ref, got["angles"][w], got["levels"][w], got["bins"][w], d, d, pos, LAM, K)
            assert msg is None, (ctx, msg)
            wst, c, sk = stats.get(fam, (0.0, 0, 0))
            stats[fam] = (max(wst, e), c + compared, sk + (not compared))
            if gm["counts"][w] == d:
                for k in ("angles", "levels", "bins"):
                    assert np.array_equal(gm[k][w], got[k][w]), (ctx, "mdl", k)
    for fam, (wst, c, sk) in sorted(stats.items()):
        print("%s M=%d %s: worst error %.3g of its bound, %d checked, %d skipped" % (mode, M, fam, wst, c, sk))
    for fam, (wst, c, sk) in sorted(stats.items()):
        assert c >= go.floor(mode, fam) * (c + sk), (mode, M, fam, c, sk)  # the reasons for lower floors: go.ROOTS_FLOOR


@pytest.mark.parametrize("mode", ["roots", "esprit"])
def test_scaled_exact_windows_are_bit_identical(mode):
    for M in (4, 8, 12):
        pos = ula(M, "x")
        fams = [f for f in go.families(M, 77 + M) if f[4]]
        for d, group in sorted(by_d(fams).items()):
            x = np.stack([g[2].reshape(-1) for g in group])
            blk = gh.make_block(M, d, go.N, K, pos=pos, mode=mode)
            base, _ = gh.device_call(blk, x, ("levels", "bins"))
            assert np.all(base["bins"] >= 0), (M, d, base["bins"])  # every slot of an exact window is filled
            for e in (-140, 96):
                y = (x.astype(np.complex128) * 2.0 ** e).astype(np.complex64)
                assert np.array_equal(y.astype(np.complex128) * 2.0 ** -e, x.astype(np.complex128))
                got, _ = gh.device_call(blk, y, ("levels", "bins"))
                assert np.array_equal(got["angles"], base["angles"]) and np.array_equal(got["bins"], base["bins"]), (M, d, e)
                assert np.array_equal(got["levels"], base["levels"]), (M, d, e)  # Pi, hence D, does not scale
            blk.close()


@pytest.mark.parametrize("mode", ["roots", "esprit"])
def test_coherent_channel_handle(mode):
    """the same checker on a coherent music_doa_channels handle: the reference runs on the focused covariance R_foc
    the device reports, with the reference channel's wavelength"""
    import focus_oracle as fo
    import channels_oracle as ch
    from test_gpu_focus import FC, FS, device_call, make, path_windows

    m, n, K, F, J, first, C, W = 6, 2, 360, 16, 8, 12, 8, 8
    lam_ref = ch.wavelengths(F, first, C, FC, FS)[fo.ref_channel(C)]
    pos = np.stack([np.arange(m) * lam_ref / 2.0, np.zeros(m)], axis=1)
    blk = make(m, n, F * J, K, F, first, C, pos)
    blk.set_peak_mode(mode, 0)
    x = path_windows(W, pos, F * J, 900 + len(mode), degs=(35.0, 120.0))
    got, _ = device_call(blk, x, ("levels", "bins", "R"))
    blk.close()
    ref_of = go.roots_reference if mode == "roots" else go.esprit_reference
    checked, worst = 0, 0.0
    for w in range(W):
        ref = ref_of(got["R"][w], n, pos, lam_ref)
        e, compared, msg = go.check(ref, got["angles"][0, w], got["levels"][0, w], got["bins"][0, w], n, n, pos, lam_ref, K)
        assert msg is None, (mode, w, msg)
        checked += compared
        worst = max(worst, e)
    print("%s coherent channels: worst error %.3g of its bound, %d of %d checked" % (mode, worst, checked, W))
    assert checked >= W // 2, checked
