"""The IAA estimator on the GPU: the spectrum against tests/iaa_oracle.py on the GPU's own R, every entry point against
process_device_ex, failure windows, the mode rules, channel and az-el handles, and the seeded cases IAA is for."""
import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200.music_doa_azel import music_doa_azel

from oracle import music_oracle as mo

import azel_oracle as ao
import gpu_harness as gh
import helpers
import iaa_oracle as io
from helpers import LAM, array_wl, table_wl

pytestmark = pytest.mark.gpu

OUT = ("levels", "bins", "spectrum", "P64", "R")
WORST = {"ratio": 0.0}  # the largest max_k |P_device - P| / bound seen by check_against_oracle (printed by the parity tests)


def einval(f):
    with pytest.raises(_capi.MusicB200Error):
        f()


def iaa_block(tab, n, snaps, iters=15, loading=0.0, mode=None, rule=None, devices=None, pos=None):
    blk = gh.make_block(tab.shape[1], n, snaps, table=tab, pos=pos, est=("iaa", loading), rule=rule, mode=mode,
                        devices=devices)
    blk.set_iaa_iterations(iters)
    return blk


def two_source_windows(pos, W, seed, snaps, coherent=False):
    rng = np.random.default_rng(seed)
    th = [rng.uniform(0.0, 360.0, 2) for _ in range(W)]
    return helpers.angle_windows(pos, th, coherent, W, seed, snaps=snaps)


def check_against_oracle(out, tab, n, iters, loading, rng, ctx, peak="top"):
    """per window: P64 within the oracle's own rounding-order bound, the spectrum its float cast, bins exact except at
    near-ties under that bound, levels the float P at the bin.  Returns the number of near-ties."""
    ties = 0
    K = tab.shape[0]
    for w in range(len(out["P64"])):
        R, got = out["R"][w], out["P64"][w]
        ref = io.spectrum(R, tab, iters, loading)
        if np.all(np.isnan(ref)):
            assert np.all(np.isnan(got)) and np.all(out["bins"][w] == -1), (ctx, w)
            continue
        tol = io.bound(R, tab, iters, loading, rng, ref)
        assert np.max(np.abs(got - ref)) <= tol, (ctx, w, np.max(np.abs(got - ref)), tol)
        WORST["ratio"] = max(WORST["ratio"], float(np.max(np.abs(got - ref))) / tol)
        assert np.array_equal(out["spectrum"][w], got.astype(np.float32)), (ctx, w)
        rb = io.window(R, tab, n, iters, loading, peak)["bins"]
        if not np.array_equal(out["bins"][w], rb):
            gb, rb_ = out["bins"][w], rb
            assert all(abs(ref[g] - ref[r]) <= 2 * tol for g, r in zip(gb, rb_) if g >= 0 and r >= 0), (ctx, w, gb, rb_)
            ties += 1
        for s, b in enumerate(out["bins"][w]):
            if b >= 0:
                assert out["levels"][w][s] == np.float32(got[b]), (ctx, w, s)
    return ties


# ---- against the oracle ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2, 4, 7, 8, 16])
def test_parity_geometric(m):
    pos = array_wl("uca", m)
    tab = table_wl(pos, 360)
    rng = np.random.default_rng(m)
    ties = total = 0
    for snaps in (64, max(2, m // 2)):
        x = two_source_windows(pos, 6, 10 * m + snaps, snaps, coherent=snaps == 64)
        for iters in (1, 15):
            for loading in (0.0, 0.05):
                for n, peak in ((1, "top"), (min(2, m - 1), "local")):
                    blk = iaa_block(tab, n, snaps, iters, loading, mode="local_maxima" if peak == "local" else None)
                    out, _ = gh.device_call(blk, x, OUT)
                    blk.close()
                    ties += check_against_oracle(out, tab, n, iters, loading, rng, (m, snaps, iters, loading, n), peak)
                    total += len(x)
    assert ties <= 0.05 * total, (ties, total)
    print("IAA parity M = %d: worst error / bound so far %.3g" % (m, WORST["ratio"]))


def test_parity_set_table_rows():
    """calibrated rows with power-of-two factors, zero rows and duplicate rows (M = 8 and M = 16)"""
    for m in (8, 16):
        tab = helpers.calibrated_table(table_wl(array_wl("uca", m), 360), m)
        tab[[3, 90, 200]] = 0
        tab[250] = tab[40]
        pos = array_wl("uca", m)
        x = two_source_windows(pos, 6, m, 64)
        rng = np.random.default_rng(m)
        for loading in (0.0, 0.01):
            blk = iaa_block(tab, 2, 64, 15, loading, mode="local_maxima")
            out, _ = gh.device_call(blk, x, OUT)
            blk.close()
            assert np.all(out["P64"][:, [3, 90, 200]] == 0.0)
            assert np.array_equal(out["P64"][:, 250], out["P64"][:, 40])
            check_against_oracle(out, tab, 2, 15, loading, rng, ("table", m, loading), "local")


# ---- entry points and determinism --------------------------------------------------------------------------------------
def test_entries_agree():
    m, n, snaps = 8, 2, 64
    pos = array_wl("uca", m)
    tab = table_wl(pos, 360)
    x = two_source_windows(pos, 21, 5, snaps, coherent=True)
    make = lambda devices=None: iaa_block(tab, n, snaps, 5, 0.0, mode="local_maxima", devices=devices)
    blk = make()
    ref, _ = gh.device_call(blk, x, ("levels", "bins", "spectrum", "P64", "R"))
    cn, _ = gh.device_call(blk, x, ("levels", "bins", "counts"))
    blk.set_beamformer("das", 0.0)  # read by the beams entry points only
    bm, _ = gh.device_call(blk, x, ("levels", "bins", "spectrum", "weights", "beams"))
    # a window's outputs do not depend on its place in the batch
    order = np.random.default_rng(1).permutation(len(x))
    sh, _ = gh.device_call(blk, x[order], ("levels", "bins", "P64"))
    one, _ = gh.device_call(blk, x[7:8], ("levels", "bins", "P64"))
    blk.close()
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(cn[k], ref[k]), k
        assert np.array_equal(sh[k], ref[k][order]), k
        assert np.array_equal(one[k][0], ref[k][7]), k
    assert np.array_equal(sh["P64"], ref["P64"][order]) and np.array_equal(one["P64"][0], ref["P64"][7])
    for k in ("angles", "levels", "bins", "spectrum"):
        assert np.array_equal(bm[k], ref[k]), k
    ent = gh.entry_outputs(make, x, spectrum=True, planar_outputs=("levels", "bins", "spectrum"))
    for name, o in ent.items():
        if name == "planar_launches":
            continue
        for d in (o if isinstance(o, list) else [o]):
            if name == "sharded":
                g = ent["sharded"].index(d)
                G = len(ent["sharded"])
                assert np.array_equal(d["angles"], ref["angles"][g::G]), name
                assert np.array_equal(d["bins"], ref["bins"]), name
                continue
            for k in ("angles", "levels", "bins", "spectrum"):
                if k in d and d[k] is not None:
                    assert np.array_equal(d[k], ref[k]), (name, k)


def test_sub_batch_split():
    """a sub-batch split (host chunks of different sizes) changes no byte"""
    m, n, snaps = 4, 1, 32
    pos = array_wl("uca", m)
    tab = table_wl(pos, 720)
    x = two_source_windows(pos, 37, 6, snaps)
    blk = iaa_block(tab, n, snaps, 15, 0.0)
    ref, _ = gh.device_call(blk, x, ("levels", "bins", "P64"))
    parts = [gh.device_call(blk, x[a:b], ("levels", "bins", "P64"))[0] for a, b in ((0, 9), (9, 10), (10, 37))]
    blk.close()
    for k in ("angles", "levels", "bins", "P64"):
        assert np.array_equal(np.concatenate([p[k] for p in parts]), ref[k]), k


# ---- composition ---------------------------------------------------------------------------------------------------------
def test_counts_match_mvdr_and_integration_feeds_iaa():
    m, n, snaps = 8, 3, 64
    pos = array_wl("uca", m)
    tab = table_wl(pos, 360)
    x = two_source_windows(pos, 12, 8, snaps)
    a = iaa_block(tab, n, snaps, 15, 0.01, rule="mdl")
    b = gh.make_block(m, n, snaps, table=tab, est=("mvdr", 0.01), rule="mdl")
    ca, _ = gh.device_call(a, x, ("counts", "bins"))
    cb, _ = gh.device_call(b, x, ("counts",))
    assert np.array_equal(ca["counts"], cb["counts"])
    for w in range(len(x)):
        assert np.all(ca["bins"][w][ca["counts"][w]:] == -1)
    b.close()
    a.set_integration(0.8)
    a.set_source_rule("fixed")
    out, _ = gh.device_call(a, x, OUT)
    a.close()
    check_against_oracle(out, tab, n, 15, 0.01, np.random.default_rng(2), "integration")
    assert not np.allclose(out["R"][-1], mo.covariance(x[-1], m))  # R is the integrated R


# ---- failure windows -----------------------------------------------------------------------------------------------------
def test_failure_windows():
    m, n, snaps = 4, 2, 16
    pos = array_wl("uca", m)
    tab = table_wl(pos, 360)
    x = two_source_windows(pos, 6, 3, snaps)
    x[1] = 0
    x[3, 5] = np.nan
    a0 = helpers.steering_wl(pos, 33.0)
    x[4] = (a0[None, :] * np.exp(1j * np.arange(snaps))[:, None]).reshape(-1).astype(np.complex64)  # noiseless, rank one
    blk = iaa_block(tab, n, snaps, 15, 0.0)
    out, _ = gh.device_call(blk, x, OUT)
    blk.close()
    for w in (1, 3):
        assert np.all(np.isnan(out["P64"][w])) and np.all(np.isnan(out["spectrum"][w]))
        assert np.all(out["bins"][w] == -1) and not np.any(out["angles"][w]) and not np.any(out["levels"][w])
    check_against_oracle(out, tab, n, 15, 0.0, np.random.default_rng(3), "failure")


# ---- mode rules ----------------------------------------------------------------------------------------------------------
def test_mode_rules_and_default_restored():
    m, n, snaps = 8, 2, 8
    pos = array_wl("x", m)
    tab = table_wl(pos, 360)
    blk = gh.make_block(m, n, snaps, table=tab, pos=pos * LAM)
    blk.set_estimator("iaa", 0.0)  # loading 0 with N <= m
    for mode in ("roots", "esprit", "manifold", "dml", "wsf"):
        einval(lambda: blk.set_peak_mode(mode, 0))
    einval(lambda: blk.set_refine(True))
    einval(lambda: blk.set_refine("joint"))
    einval(lambda: blk.set_estimator("iaa", -1.0))
    einval(lambda: blk.set_estimator("iaa", float("nan")))
    einval(lambda: blk.set_estimator("iaa", float("inf")))
    for bad in (0, 65, -3):
        einval(lambda: blk.set_iaa_iterations(bad))
    blk.set_iaa_iterations(1)
    blk.set_iaa_iterations(64)
    blk.set_estimator("music", 0.0)
    for mode in ("roots", "dml"):
        blk.set_peak_mode(mode, 0)
        einval(lambda: blk.set_estimator("iaa", 0.0))
    blk.set_peak_mode("top_bins", 0)
    blk.set_refine(True)
    einval(lambda: blk.set_estimator("iaa", 0.0))
    blk.set_refine(False)
    blk.close()
    # MUSIC again restores the default path: outputs and launch count of a fresh handle
    x = two_source_windows(pos, 8, 4, 64)
    for nn in (1, 2):
        fresh = gh.make_block(m, nn, 64, table=tab)
        used = gh.make_block(m, nn, 64, table=tab)
        used.set_estimator("iaa", 0.1)
        used.set_iaa_iterations(3)
        gh.device_call(used, x, ("levels",))
        used.set_estimator("music", 0.0)
        for outs in ((), ("levels", "bins"), ("levels", "bins", "spectrum")):
            a, la = gh.device_call(fresh, x, outs)
            b, lb = gh.device_call(used, x, outs)
            assert la == lb, (nn, outs)
            for k in a:
                assert np.array_equal(a[k], b[k]), (nn, outs, k)
        fresh.close()
        used.close()


def test_multi_device_iterations_apply_to_every_device():
    m, n, snaps = 4, 1, 32
    pos = array_wl("uca", m)
    tab = table_wl(pos, 360)
    x = two_source_windows(pos, 10, 9, snaps)
    G = torch.cuda.device_count()
    one = iaa_block(tab, n, snaps, 4)
    multi = iaa_block(tab, n, snaps, 4, devices=list(range(G)))
    a = gh.host_call(one, x, spectrum=True)
    b = gh.host_call(multi, x, spectrum=True)
    one.close()
    multi.close()
    for k in ("angles", "levels", "spectrum", "bins"):
        assert np.array_equal(a[k], b[k]), k


# ---- az-el and channel handles -------------------------------------------------------------------------------------------
def azel_block(grid, pos, n, snaps, mode="local_maxima", lam=1.0):
    blk = music_doa_azel(pos.shape[0], n, pos.shape[0] * snaps, grid.n_az, grid.n_el, (grid.el_lo, grid.el_hi), pos * lam, lam)
    blk.set_estimator("iaa", 0.0)
    blk.set_peak_mode(mode, 0)
    return blk


@pytest.mark.parametrize("N", [256, 8])
def test_coherent_azel_ura(N):
    """the seeded coherent az-el case: the device finds both paths in at least as many windows as the oracle on the
    same windows, and its spectrum is the oracle's on the covariance of the same windows"""
    pos, grid, tab, x = io.azel_case(N)
    blk = azel_block(grid, pos, 2, N)
    out, _ = gh.device_call(blk, x, ("levels", "spectrum", "bins"))
    blk.close()
    dev = ora = 0
    for w in range(len(x)):
        R = mo.covariance(x[w], 16)
        P = io.spectrum(R, tab, 15)
        assert np.max(np.abs(out["spectrum"][w] - P)) <= 1e-5 * np.max(P), w
        ora += io.azel_found(ao.pick_local_maxima_2d(P, 2, grid), grid)
        dev += io.azel_found(out["bins"][w], grid)
    assert dev >= ora - 1 and dev >= (12 if N == 256 else 10), (dev, ora)


def test_coherent_ula_and_fewer_snapshots():
    tab, x, truth = io.ula_case("coherent")
    blk = iaa_block(tab, 2, 64, 15, 0.0, mode="local_maxima")
    out, _ = gh.device_call(blk, x, ("bins",))
    blk.close()
    dev = sum(io.ula_resolved(out["bins"][w], truth) for w in range(len(x)))
    assert dev == 60, dev
    tab, x, truth = io.ula_case("coherent", W=20, N=4)
    blk = iaa_block(tab, 2, 4, 15, 0.0, mode="local_maxima")
    out, _ = gh.device_call(blk, x, ("bins", "R"))
    blk.close()
    dev = sum(io.ula_resolved(out["bins"][w], truth) for w in range(len(x)))
    ora = sum(io.ula_resolved(io.window(out["R"][w], tab, 2, peak="local")["bins"], truth) for w in range(len(x)))
    assert dev >= ora - 1, (dev, ora)


@pytest.mark.parametrize("combine", ["separate", "coherent"])
def test_channel_handles(combine):
    import channels_oracle as ch
    import focus_oracle as fo
    from gr_baz_b200.music_doa_channels import music_doa_channels

    m, n, K, F, J, first, C, W = 6, 2, 360, 16, 8, 12, 8, 6
    fc, fs = 400e6, 56e6
    lam_ref = ch.wavelengths(F, first, C, fc, fs)[fo.ref_channel(C)]
    pos = fo.uca(m, lam_ref)
    blk = music_doa_channels(m, n, m * F * J, K, F, (first, C), "hann", combine, pos, 1.0, fc, fs)
    blk.set_estimator("iaa", 0.01)
    blk.set_peak_mode("local_maxima", 0)
    rng = np.random.default_rng(41)
    x = np.stack([fo.two_paths(rng, pos, F * J, degs=(40.0, 110.0), noise=0.3, fc=fc, fs=fs) for _ in range(W)])
    Cr = C if combine == "separate" else 1
    o = {k: torch.full(s, gh.SENTINEL, dtype=t, device=gh.DEV) for k, (s, t) in
         {"angles": ((Cr, W, n), torch.float32), "levels": ((Cr, W, n), torch.float32), "bins": ((Cr, W, n), torch.int32),
          "spectrum": ((Cr, W, K), torch.float32), "R": ((Cr, W, m, m, 2), torch.float64)}.items()}
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    blk.process_device(d_in.data_ptr(), W, o["angles"].data_ptr(), o["levels"].data_ptr(), o["spectrum"].data_ptr(),
                       o["bins"].data_ptr(), None, o["R"].data_ptr(), stream=gh.stream())
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in o.items()}
    R = got["R"][..., 0] + 1j * got["R"][..., 1]
    rr = np.random.default_rng(5)
    for c in range(Cr):
        tab = blk.array_response_c64(c if combine == "separate" else fo.ref_channel(C))
        for w in range(W):
            ref = io.spectrum(R[c, w], tab, 15, 0.01)
            tol = io.bound(R[c, w], tab, 15, 0.01, rr, ref)
            assert np.max(np.abs(got["spectrum"][c, w] - ref)) <= tol + float(np.spacing(np.float32(np.max(ref)))), (c, w)
    blk.close()


# ---- the CRB and tracks entries, and the az-el host entry ------------------------------------------------------------------
def dev_out(spec, fill=gh.SENTINEL):
    return {k: torch.full(s, fill, dtype=t, device=gh.DEV) for k, (s, t) in spec.items()}


def numpy_of(o):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def test_crb_and_tracks_entries_1d():
    """under IAA the CRB and tracks entries give the angles, levels and bins of process_device_ex, the CRB entry the bound
    of those angles, and the tracks entry with a CRB output the CRB entry's bound"""
    import crb_oracle as co
    m, n, snaps = 8, 2, 64
    pos = array_wl("uca", m)
    x = two_source_windows(pos, 11, 14, snaps)
    W = len(x)
    blk = gh.make_block(m, n, snaps, K=360, pos=pos * LAM, est=("iaa", 0.0), mode="local_maxima")
    ref, _ = gh.device_call(blk, x, ("levels", "bins", "spectrum", "R"))
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    f32, i32 = torch.float32, torch.int32
    c = dev_out({"angles": ((W, n), f32), "levels": ((W, n), f32), "spectrum": ((W, 360), f32), "bins": ((W, n), i32),
                 "std": ((W, n), f32)})
    blk.process_device_crb(d_in.data_ptr(), W, c["angles"].data_ptr(), c["std"].data_ptr(), c["levels"].data_ptr(),
                           c["spectrum"].data_ptr(), c["bins"].data_ptr(), stream=gh.stream())
    c = numpy_of(c)
    for k in ("angles", "levels", "bins", "spectrum"):
        assert np.array_equal(c[k], ref[k]), k
    crb, _ = co.crb_outputs(ref["R"], ref["angles"], ref["bins"], snaps, pos * LAM, LAM)
    assert np.allclose(c["std"], crb, rtol=1e-3, atol=0, equal_nan=True)
    blk.set_tracking("fixed")
    t = dev_out({"angles": ((W, n), f32), "levels": ((W, n), f32), "spectrum": ((W, 360), f32), "bins": ((W, n), i32),
                 "slot_track": ((W, n), i32), "std": ((W, n), f32)})
    blk.process_device_tracks(d_in.data_ptr(), W, t["angles"].data_ptr(), t["slot_track"].data_ptr(), t["levels"].data_ptr(),
                              t["spectrum"].data_ptr(), t["bins"].data_ptr(), None, None, None, t["std"].data_ptr(),
                              stream=gh.stream())
    t = numpy_of(t)
    blk.close()
    for k in ("angles", "levels", "bins", "spectrum"):
        assert np.array_equal(t[k], ref[k]), k
    assert np.array_equal(t["std"], c["std"], equal_nan=True)
    assert np.all(t["slot_track"][ref["bins"] < 0] == -1) and np.all(t["slot_track"] >= -1)


def test_azel_entries():
    """on an az-el handle under IAA the host, CRB and tracks entries give the azimuths, elevations, levels, bins and
    spectrum of process_azel_device, and the tracks entry the CRB entry's bound"""
    grid = ao.Grid(72, 10, 0.0, 90.0)
    pos = ao.ura_xyz(3, 3, LAM)
    rng = np.random.default_rng(2)
    A = np.array([ao.steering(pos, LAM, 40.0, 20.0), ao.steering(pos, LAM, 200.0, 50.0)])
    x = io._windows(rng, A, (1.0, 0.7), 32, 20.0, False, 13)
    W, n, K = len(x), 2, grid.K
    blk = azel_block(grid, pos / LAM, n, 32, lam=LAM)
    ref, _ = gh.device_call(blk, x, ("levels", "spectrum", "bins"))
    host = gh.host_call(blk, x, spectrum=True)
    for k in ("azimuth", "elevation", "levels", "spectrum", "bins"):
        assert np.array_equal(host[k], ref[k]), k
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    f32, i32 = torch.float32, torch.int32
    shape = {"azimuth": ((W, n), f32), "elevation": ((W, n), f32), "levels": ((W, n), f32), "spectrum": ((W, K), f32),
             "bins": ((W, n), i32), "crb": ((W, n, 3), f32)}
    c = dev_out(shape)
    blk.process_device_crb(d_in.data_ptr(), W, c["azimuth"].data_ptr(), c["elevation"].data_ptr(), c["crb"].data_ptr(),
                           c["levels"].data_ptr(), c["spectrum"].data_ptr(), c["bins"].data_ptr(), stream=gh.stream())
    c = numpy_of(c)
    blk.set_tracking("fixed")
    t = dev_out(dict(shape, slot_track=((W, n), i32)))
    blk.process_device_tracks(d_in.data_ptr(), W, t["azimuth"].data_ptr(), t["elevation"].data_ptr(), t["slot_track"].data_ptr(),
                              t["levels"].data_ptr(), t["spectrum"].data_ptr(), t["bins"].data_ptr(), None, t["crb"].data_ptr(),
                              stream=gh.stream())
    t = numpy_of(t)
    blk.close()
    for k in ("azimuth", "elevation", "levels", "spectrum", "bins"):
        assert np.array_equal(c[k], ref[k]), k
        assert np.array_equal(t[k], ref[k]), k
    assert np.array_equal(t["crb"], c["crb"], equal_nan=True)
    filled = ref["bins"] >= 0
    assert np.all(np.isfinite(c["crb"][filled][:, :2]) | np.isnan(c["crb"][filled][:, :2]))
    assert np.all(t["slot_track"][~filled] == -1)


# ---- mode rules on the az-el and channel handles, in both setter orders -------------------------------------------------
def test_mode_rules_azel_and_channels():
    from gr_baz_b200.music_doa_channels import music_doa_channels
    import channels_oracle as ch
    import focus_oracle as fo

    grid = ao.Grid(36, 5, 0.0, 90.0)
    az = azel_block(grid, ao.ura_xyz(3, 3, 1.0), 2, 8, mode="top_bins")
    az.set_iaa_iterations(2)
    einval(lambda: az.set_iaa_iterations(0))
    for setter in (lambda: az.set_peak_mode("esprit", 0), lambda: az.set_refine(True)):
        einval(setter)
    az.set_estimator("music", 0.0)
    az.set_peak_mode("esprit", 0)
    einval(lambda: az.set_estimator("iaa", 0.0))
    az.set_peak_mode("local_maxima", 0)
    az.set_refine(True)
    einval(lambda: az.set_estimator("iaa", 0.0))
    az.set_refine(False)
    az.set_estimator("iaa", 0.0)  # loading 0 with N = 8 < m = 9
    az.close()

    m, n, K, F, J, first, C = 6, 2, 360, 16, 8, 12, 8
    fc, fs = 400e6, 56e6
    lam_ref = ch.wavelengths(F, first, C, fc, fs)[fo.ref_channel(C)]
    pos = fo.uca(m, lam_ref)
    for combine in ("separate", "coherent", "incoherent"):
        blk = music_doa_channels(m, n, m * F * J, K, F, (first, C), "hann", combine, pos, 1.0, fc, fs)
        if combine == "incoherent":
            einval(lambda: blk.set_estimator("iaa", 0.0))
            blk.close()
            continue
        blk.set_estimator("iaa", 0.0)
        blk.set_iaa_iterations(7)
        einval(lambda: blk.set_iaa_iterations(65))
        modes = ("dml", "wsf") if combine == "coherent" else ()
        for mode in modes:
            einval(lambda: blk.set_peak_mode(mode, 0))
        if combine == "coherent":
            einval(lambda: blk.set_refine(True))
        blk.set_estimator("music", 0.0)
        for mode in modes:
            blk.set_peak_mode(mode, 0)
            einval(lambda: blk.set_estimator("iaa", 0.0))
        blk.set_peak_mode("local_maxima", 0)
        if combine == "coherent":
            blk.set_refine(True)
            einval(lambda: blk.set_estimator("iaa", 0.0))
            blk.set_refine(False)
        blk.set_estimator("iaa", 0.01)
        blk.close()


# ---- the C++ blocks ----------------------------------------------------------------------------------------------------------
def test_cpp_blocks():
    """set_estimator(4) and set_iaa_iterations on baz_music_doa, baz_music_doa_azel and baz_music_doa_channels give the
    outputs of the Python blocks"""
    import struct

    from gr_baz_b200.music_doa_channels import music_doa_channels
    import channels_oracle as ch
    import focus_oracle as fo

    # 1-D
    m, n, K, snaps, W = 8, 2, 360, 32, 9
    pos = array_wl("uca", m) * LAM
    x = two_source_windows(pos / LAM, W, 3, snaps, coherent=True)
    got = gh.run_cpp_block("test_block_iaa", struct.pack("<7Id", 0, m, n, m * snaps, W, 6, 1, 0.02) + struct.pack("<Id", K, LAM),
                           [np.ascontiguousarray(pos), x],
                           [("angles", np.float32, W * n), ("levels", np.float32, W * n), ("spectrum", np.float32, W * K),
                            ("bins", np.int32, W * n)])
    blk = gh.make_block(m, n, snaps, K=K, pos=pos, est=("iaa", 0.02), mode="local_maxima")
    blk.set_iaa_iterations(6)
    ang, lvl, spec = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32), np.zeros((W, K), np.float32)
    blk.work(W, [x], [ang, lvl, spec])
    for k, v in (("angles", ang), ("levels", lvl), ("spectrum", spec), ("bins", blk.last_bins())):
        assert np.array_equal(got[k], v.ravel()), k
    blk.close()

    # az-el
    grid = ao.Grid(36, 10, 0.0, 90.0)
    p3 = ao.ura_xyz(3, 3, LAM)
    m, n, snaps = 9, 2, 8
    xa = io._windows(np.random.default_rng(4), np.array([ao.steering(p3, LAM, 40.0, 20.0)]), (1.0,), snaps, 20.0, False, W)
    got = gh.run_cpp_block("test_block_iaa", struct.pack("<7Id", 1, m, n, m * snaps, W, 4, 1, 0.0) +
                           struct.pack("<2I3d", grid.n_az, grid.n_el, grid.el_lo, grid.el_hi, LAM),
                           [np.ascontiguousarray(p3), xa],
                           [("azimuth", np.float32, W * n), ("elevation", np.float32, W * n), ("levels", np.float32, W * n),
                            ("spectrum", np.float32, W * grid.K), ("bins", np.int32, W * n)])
    az = azel_block(grid, p3 / LAM, n, snaps, lam=LAM)
    az.set_iaa_iterations(4)
    ports = [np.zeros((W, n), np.float32) for _ in range(3)] + [np.zeros((W, grid.K), np.float32)]
    az.work(W, [xa], ports)
    for k, v in zip(("azimuth", "elevation", "levels", "spectrum"), ports):
        assert np.array_equal(got[k], v.ravel()), k
    assert np.array_equal(got["bins"], az.last_bins().ravel())
    az.close()

    # channels (separate and coherent)
    m, n, K, F, J, first, C = 6, 2, 360, 16, 8, 12, 8
    fc, fs = 400e6, 56e6
    lam_ref = ch.wavelengths(F, first, C, fc, fs)[fo.ref_channel(C)]
    pc = fo.uca(m, lam_ref)
    rng = np.random.default_rng(41)
    xc = np.stack([fo.two_paths(rng, pc, F * J, degs=(40.0, 110.0), noise=0.3, fc=fc, fs=fs) for _ in range(4)])
    for combine, code in (("separate", 0), ("coherent", 2)):
        rows = C if combine == "separate" else 1
        Wc = len(xc)
        got = gh.run_cpp_block("test_block_iaa", struct.pack("<7Id", 2, m, n, m * F * J, Wc, 5, 1, 0.01) +
                               struct.pack("<5I2d", K, F, first, C, code, fc, fs), [np.ascontiguousarray(pc), xc],
                               [("angles", np.float32, Wc * rows * n), ("levels", np.float32, Wc * rows * n),
                                ("spectrum", np.float32, Wc * rows * K), ("bins", np.int32, Wc * rows * n)])
        blk = music_doa_channels(m, n, m * F * J, K, F, (first, C), "hann", combine, pc, 1.0, fc, fs)
        blk.set_estimator("iaa", 0.01)
        blk.set_iaa_iterations(5)
        blk.set_peak_mode("local_maxima", 0)
        ang, lvl, spec = (np.zeros((Wc, rows * n), np.float32), np.zeros((Wc, rows * n), np.float32),
                          np.zeros((Wc, rows * K), np.float32))
        blk.work(Wc, [xc], [ang, lvl, spec])
        for k, v in (("angles", ang), ("levels", lvl), ("spectrum", spec), ("bins", blk.last_bins())):
            assert np.array_equal(got[k], np.asarray(v).ravel()), (combine, k)
        blk.close()
