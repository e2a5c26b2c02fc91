"""The WSF peak mode and the JOINT refinement on the GPU: bins and refined angles against tests/wsf_oracle.py on the
GPU's own R, every entry point against process_device_ex, the mode rules, and what the modes are for (the RMSE against
the CRB, and coherent paths)."""
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi

import crb_oracle as co
import gpu_harness as gh
import helpers
import wsf_oracle as wo
from helpers import LAM, array_wl, table_wl

pytestmark = pytest.mark.gpu

FLIP = 1e-9
PEAKS = ("levels", "bins")


def handle(pos, tab, n, snaps, mode="wsf", joint=True, rule=None, devices=None):
    blk = gh.make_block(tab.shape[1], n, snaps, table=tab, pos=None if pos is None else pos * LAM, rule=rule, mode=mode,
                        devices=devices)
    if joint:
        blk.set_refine("joint")
    return blk


def windows(pos, seed, W, snaps=256):
    """per group of four (20 dB): a coherent pair, an uncorrelated pair, three uncorrelated sources and one source"""
    rng = np.random.default_rng(seed)
    out = []
    for w in range(W):
        S = (2, 2, 3, 1)[w % 4]
        th = rng.uniform(0.0, 360.0, S)
        out.append(helpers.angle_windows(pos, [th], w % 4 == 0, 1, seed + w, snaps=snaps))
    return np.concatenate(out)


def oracle(R, tab, n, d, mode, pos, joint):
    return wo.window_R(R, tab, n, d, mode, pos, 1.0, joint)


def permuted(R, tab, pos, n, d, mode, joint, perm):
    """the oracle on the same problem with the elements in another order: its spread is the summation-order spread"""
    return oracle(R[np.ix_(perm, perm)], np.ascontiguousarray(tab[:, perm]), n, d, mode, pos[perm], joint)


def check_window(g, R, tab, pos, n, d, mode, joint, rng, ctx):
    """bins exact (or a near-tie: returns 1), refined angles and levels within the oracle's own summation-order spread
    (at least two float32 ulps)"""
    ref = oracle(R, tab, n, d, mode, pos, joint)
    if not np.array_equal(g["bins"], ref["bins"]):
        assert ref["margin"] <= FLIP, (ctx, g["bins"], ref["bins"], ref["margin"])
        return 1
    alt = permuted(R, tab, pos, n, d, mode, joint, rng.permutation(R.shape[0]))
    # Two slots on one source (n above the number of sources in the window) refine to within a few bins of each other,
    # where V is nearly flat along their difference and the path depends on rounding: the oracle on these windows,
    # with and without the elements permuted, ends up to 0.03 degrees apart.  Those windows are held to their box only.
    th = ref.get("theta")
    bin_deg = 360.0 / len(tab)
    loose = joint and th is not None and any(helpers.circ(np.degrees(th[i]), np.degrees(th[j])) < 4.0 * bin_deg
                                             for i in range(len(th)) for j in range(i))
    for i in range(n):
        if ref["bins"][i] < 0:
            assert g["angles"][i] == 0.0 and g["levels"][i] == 0.0, ctx
            continue
        if loose:
            assert helpers.circ(g["angles"][i], ref["bins"][i] * bin_deg) <= bin_deg * (1 + 1e-6), ctx
            continue
        spread = helpers.circ(ref["angles"][i], alt["angles"][i])
        tol = max(4.0 * spread, 2.0 * float(np.spacing(np.float32(max(ref["angles"][i], 1.0)))))
        assert helpers.circ(g["angles"][i], ref["angles"][i]) <= tol, (ctx, i, g["angles"], ref["angles"], alt["angles"])
        lsp = abs(float(ref["levels"][i]) - float(alt["levels"][i]))
        ltol = max(4.0 * lsp, 2.0 * float(np.spacing(np.abs(np.float32(ref["levels"][i])))), 1e-10 * float(np.trace(R).real))
        if helpers.circ(g["angles"][i], ref["angles"][i]) == 0.0:
            assert abs(float(g["levels"][i]) - float(ref["levels"][i])) <= ltol, (ctx, i, g["levels"], ref["levels"])
    return 0


# ---- parity with the oracle ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,m", [("uca", 4), ("uca", 8), ("random", 8), ("x", 8), ("uca", 16)])
def test_parity_with_oracle(kind, m):
    pos = array_wl(kind, m, seed=m)
    tab = table_wl(pos, 360)
    x = windows(pos, 10 * m, 24)
    rng = np.random.default_rng(m)
    edge = total = 0
    for mode, joint in (("wsf", False), ("wsf", True), ("dml", True)):
        for n in (1, 2, 3):
            for rule in ("fixed", "mdl"):
                blk = handle(pos, tab, n, 256, mode, joint, rule)
                out, _ = gh.device_call(blk, x, PEAKS + ("R",))
                cnt, _ = gh.device_call(blk, x, PEAKS + ("counts",))
                blk.close()
                for k in ("angles", "levels", "bins"):
                    assert np.array_equal(cnt[k], out[k]), k
                for w in range(len(x)):
                    g = {k: out[k][w] for k in ("angles", "levels", "bins")}
                    edge += check_window(g, out["R"][w], tab, pos, n, int(cnt["counts"][w]), mode, joint, rng,
                                         (kind, m, mode, joint, n, rule, w))
                    total += 1
    assert edge <= 0.02 * total, (edge, total)


# ---- entry points ------------------------------------------------------------------------------------------------------
def test_entries_agree():
    """host, device, _counts, planar, multi-device, sharded, and the beams and CRB entries under WSF + JOINT: the same
    angles, levels and bins as process_device_ex"""
    m, n, snaps = 8, 2, 256
    pos = array_wl("uca", m)
    tab = table_wl(pos, 720)
    x = windows(pos, 3, 16, snaps)
    make = lambda devices=None: handle(pos, tab, n, snaps, devices=devices)
    blk = make()
    ref, _ = gh.device_call(blk, x, PEAKS + ("spectrum", "P64", "R"))
    cn, _ = gh.device_call(blk, x, PEAKS + ("counts",))
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(cn[k], ref[k]), k
    W = len(x)
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    o = {k: torch.full(s, gh.SENTINEL, dtype=t, device=gh.DEV) for k, (s, t) in
         {"angles": ((W, n), torch.float32), "levels": ((W, n), torch.float32), "bins": ((W, n), torch.int32),
          "std": ((W, n), torch.float32)}.items()}
    blk.process_device_crb(d_in.data_ptr(), W, o["angles"].data_ptr(), o["std"].data_ptr(), o["levels"].data_ptr(), None,
                           o["bins"].data_ptr(), stream=gh.stream())
    torch.cuda.synchronize()
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(o[k].cpu().numpy(), ref[k]), k
    crb, _ = co.crb_outputs(ref["R"], ref["angles"], ref["bins"], snaps, pos, 1.0)
    assert np.allclose(o["std"].cpu().numpy(), crb, rtol=1e-3, atol=0, equal_nan=True)
    blk.set_beamformer("das")
    bw, _ = gh.device_call(blk, x, PEAKS + ("weights",))
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(bw[k], ref[k]), k
    blk.set_beamformer("off")
    blk.set_tracking("fixed")
    t = {k: torch.full(s, gh.SENTINEL, dtype=d, device=gh.DEV) for k, (s, d) in
         {"angles": ((W, n), torch.float32), "levels": ((W, n), torch.float32), "bins": ((W, n), torch.int32),
          "slot_track": ((W, n), torch.int32)}.items()}
    blk.process_device_tracks(d_in.data_ptr(), W, t["angles"].data_ptr(), t["slot_track"].data_ptr(), t["levels"].data_ptr(),
                              None, t["bins"].data_ptr(), stream=gh.stream())
    torch.cuda.synchronize()
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(t[k].cpu().numpy(), ref[k]), k
    st = t["slot_track"].cpu().numpy()
    assert np.all(st[ref["bins"] < 0] == -1) and np.all(st >= -1)
    blk.close()
    e = gh.entry_outputs(make, x, multi_device=False)
    for name in ("host", "planar_host", "planar_device") + tuple(k for k in e if k.startswith("multi_")):
        for k in ("angles", "levels", "bins"):
            if k in e[name]:
                assert np.array_equal(e[name][k], ref[k]), (name, k)
    G = torch.cuda.device_count()
    for g, sh in enumerate(e.get("sharded", [])):
        assert np.array_equal(sh["angles"], ref["angles"][g::G]) and np.array_equal(sh["bins"], ref["bins"]), g


def test_default_and_dml_paths_are_untouched():
    """JOINT off: DML's outputs do not depend on whether a WSF handle ran before; WSF with JOINT off reports grid angles"""
    m, n, snaps = 8, 2, 256
    pos = array_wl("uca", m)
    tab = table_wl(pos, 360)
    x = windows(pos, 5, 16, snaps)
    blk = handle(pos, tab, n, snaps, "dml", False)
    a, _ = gh.device_call(blk, x, PEAKS)
    blk.set_peak_mode("wsf", 0)
    blk.set_refine("joint")
    gh.device_call(blk, x, PEAKS)
    blk.set_refine("off")
    ws, _ = gh.device_call(blk, x, PEAKS)
    filled = ws["bins"] >= 0
    assert np.array_equal(ws["angles"][filled], (ws["bins"][filled] * 1.0).astype(np.float32))
    blk.set_peak_mode("dml", 0)
    b, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(a[k], b[k]), k


# ---- mode rules -------------------------------------------------------------------------------------------------------
def einval(f):
    with pytest.raises(_capi.MusicB200Error):
        f()


def test_invalid_combinations():
    m, n, snaps = 8, 2, 256
    pos = array_wl("uca", m)
    tab = table_wl(pos, 360)
    blk = handle(pos, tab, n, snaps, "wsf", False)
    assert blk.refine == 0
    einval(lambda: blk.set_peak_mode("wsf", 1))            # exclusion
    einval(lambda: blk.set_refine("newton"))               # NEWTON under WSF
    einval(lambda: blk.set_estimator("mvdr", 0.1))         # estimator under WSF
    blk.set_peak_mode("top_bins", 0)
    einval(lambda: blk.set_refine("joint"))                # JOINT under a grid mode
    blk.set_refine("newton")
    einval(lambda: blk.set_peak_mode("wsf", 0))            # WSF under NEWTON
    blk.set_refine("off")
    for mode in ("local_maxima", "manifold"):
        blk.set_peak_mode(mode, 0)
        einval(lambda: blk.set_refine("joint"))
    blk.set_peak_mode("top_bins", 0)
    blk.set_estimator("mvdr", 0.1)
    einval(lambda: blk.set_peak_mode("wsf", 0))            # WSF under MVDR
    blk.set_estimator("music", 0.0)
    blk.set_peak_mode("dml", 0)
    blk.set_refine("joint")
    assert blk.refine == 2
    einval(lambda: blk.set_peak_mode("local_maxima", 0))   # a grid mode under JOINT
    blk.set_peak_mode("wsf", 0)
    # a set_table() table under JOINT: the call refuses, with no fall-back
    blk.set_array_response(tab)
    x = windows(pos, 1, 4)
    einval(lambda: gh.device_call(blk, x, PEAKS))
    blk.close()
    with pytest.raises(ValueError):
        handle(pos, tab, n, snaps, "wsf", False).set_refine("sideways")


# ---- what the modes are for -------------------------------------------------------------------------------------------
def correlated_windows(pos, th, rho, W, seed, snr_db=20.0, snaps=256):
    rng = np.random.default_rng(seed)
    m = pos.shape[0]
    amp = 10.0 ** (snr_db / 20.0)
    A = helpers.steering_wl(pos, th).T
    xs = []
    for _ in range(W):
        X = (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
        s1 = (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps)) / np.sqrt(2.0)
        s2 = (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps)) / np.sqrt(2.0)
        s2 = rho * s1 + np.sqrt(1.0 - rho * rho) * s2
        X += amp * (A[:, :1] * s1[None, :] + A[:, 1:2] * s2[None, :])
        xs.append(X.T.reshape(-1))
    return np.ascontiguousarray(np.array(xs).astype(np.complex64))


def rmse_over_crb(blk, x, th, n):
    W = len(x)
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    ang = torch.zeros((W, n), dtype=torch.float32, device=gh.DEV)
    std = torch.zeros((W, n), dtype=torch.float32, device=gh.DEV)
    bins = torch.zeros((W, n), dtype=torch.int32, device=gh.DEV)
    blk.process_device_crb(d_in.data_ptr(), W, ang.data_ptr(), std.data_ptr(), None, None, bins.data_ptr(), stream=gh.stream())
    torch.cuda.synchronize()
    a, s = ang.cpu().numpy().astype(np.float64), std.cpu().numpy().astype(np.float64)
    err = np.stack([np.min(helpers.circ(a, t), axis=1) for t in th], 1)
    return float(np.sqrt(np.mean(err ** 2)) / np.mean(s))


# UCA 8, sources at 40.3 and 75.6 degrees, 20 dB each, 256 snapshots, 500 windows.  tests/wsf_oracle.py on these
# seeds: WSF + JOINT RMSE / mean CRB std = 1.000 (rho = 0) and 1.008 (rho = 0.7); fine-grid MUSIC local maxima (what
# NEWTON converges to) 1.003 and 1.139.  Thresholds: WSF at most 1.05; MUSIC + NEWTON at least 1.08 x WSF at rho = 0.7.
STAT_TH = np.array([40.3, 75.6])


@pytest.mark.parametrize("rho", [0.0, 0.7])
def test_rmse_against_the_crb(rho):
    pos = array_wl("uca", 8)
    tab = table_wl(pos, 360)
    x = correlated_windows(pos, STAT_TH, rho, 500, 7)
    blk = handle(pos, tab, 2, 256)
    wsf = rmse_over_crb(blk, x, STAT_TH, 2)
    blk.close()
    assert wsf <= 1.05, (rho, wsf)
    if rho > 0:
        mus = gh.make_block(8, 2, 256, table=tab, pos=pos * LAM, mode="local_maxima", refine=True)
        music = rmse_over_crb(mus, x, STAT_TH, 2)
        mus.close()
        assert music >= 1.08 * wsf, (wsf, music)


def test_coherent_paths_resolved_by_wsf():
    """the seeded coherent UCA 8 row of the DML resolution table (two paths 40 degrees apart): WSF under FIXED n = 2
    resolves what its oracle resolves on the GPU's R, MUSIC's local maxima far fewer"""
    pos, tab, x, th = helpers.resolution_case("uca", 8, True, 40)
    blk = handle(pos, tab, 2, helpers.SNAPS, joint=False)
    out, _ = gh.device_call(blk, x, PEAKS + ("R",))
    blk.close()
    got = sum(helpers.resolved(out["angles"][w], th[w]) for w in range(len(x)))
    want = sum(helpers.resolved(wo.wsf_R(out["R"][w], tab, 2)["angles"], th[w]) for w in range(len(x)))
    assert abs(got - want) <= 1, (got, want)
    loc = gh.make_block(8, 2, helpers.SNAPS, table=tab, mode="local_maxima")
    lo, _ = gh.device_call(loc, x, PEAKS)
    loc.close()
    music = sum(helpers.resolved([a for a, b in zip(lo["angles"][w], lo["bins"][w]) if b >= 0], th[w]) for w in range(len(x)))
    assert music * 3 < got, (music, got)


def test_cpp_block():
    """the C++ block through set_array_geometry(), set_peak_mode(6, 0) and set_refine_mode(2) equals the Python block"""
    m, n, K, snaps, Wn = 8, 2, 360, 256, 16
    pos = array_wl("uca", m)
    x = windows(pos, 78, Wn, snaps)
    geo = np.concatenate([[LAM], (pos * LAM).ravel()]).astype(np.float64)
    c = gh.run_cpp_block("test_block_wsf", struct.pack("<5I", m, n, m * snaps, K, Wn), [geo, x],
                         [("a", np.float32, Wn * n), ("l", np.float32, Wn * n), ("s", np.float32, Wn * K),
                          ("b", np.int32, Wn * n)])
    blk = gh.make_block(m, n, snaps, K=K, pos=pos * LAM, mode="wsf")
    blk.set_refine("joint")
    ang, lvl, spec = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32), np.zeros((Wn, K), np.float32)
    blk.work(Wn, [x], [ang, lvl, spec])
    assert np.array_equal(c["a"], ang.ravel()) and np.array_equal(c["l"], lvl.ravel()) and np.array_equal(c["s"], spec.ravel())
    assert np.array_equal(c["b"], blk.last_bins().ravel()) and np.all(c["b"] >= 0)
    blk.close()


def test_coherent_channel_handle():
    """a COHERENT channel handle takes WSF as it takes DML (one problem per window on the focused R and the reference
    channel's table) and refuses JOINT"""
    import channels_oracle as ch
    import focus_oracle as fo
    from gr_baz_b200.music_doa_channels import music_doa_channels

    m, n, K, F, J, first, C, W = 6, 2, 360, 16, 8, 12, 8, 6
    fc, fs = 400e6, 56e6
    lam_ref = ch.wavelengths(F, first, C, fc, fs)[fo.ref_channel(C)]
    pos = fo.uca(m, lam_ref)
    blk = music_doa_channels(m, n, m * F * J, K, F, (first, C), "hann", "coherent", pos, 1.0, fc, fs)
    blk.set_peak_mode("wsf", 0)
    einval(lambda: blk.set_refine("joint"))
    rng = np.random.default_rng(41)
    x = np.stack([fo.two_paths(rng, pos, F * J, degs=(40.0, 110.0), noise=0.3, fc=fc, fs=fs) for _ in range(W)])
    o = {k: torch.full(s, gh.SENTINEL, dtype=t, device=gh.DEV) for k, (s, t) in
         {"angles": ((1, W, n), torch.float32), "levels": ((1, W, n), torch.float32), "bins": ((1, W, n), torch.int32),
          "R": ((W, m, m, 2), torch.float64)}.items()}
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    blk.process_device(d_in.data_ptr(), W, o["angles"].data_ptr(), o["levels"].data_ptr(), None, o["bins"].data_ptr(), None,
                       o["R"].data_ptr(), stream=gh.stream())
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in o.items()}
    R = got["R"][..., 0] + 1j * got["R"][..., 1]
    tab = blk.array_response_c64(fo.ref_channel(C))
    blk.close()
    edge = 0
    for w in range(W):
        ref = wo.wsf_R(R[w], tab, n)
        if not np.array_equal(got["bins"][0, w], ref["bins"]):
            assert ref["margin"] <= FLIP, (w, got["bins"][0, w], ref["bins"])
            edge += 1
            continue
        assert np.array_equal(got["angles"][0, w], ref["angles"]), w
        tol = [max(float(np.spacing(np.abs(np.float32(r)))), 1e-10 * float(np.trace(R[w]).real)) for r in ref["levels"]]
        assert all(abs(float(g) - float(r)) <= t for g, r, t in zip(got["levels"][0, w], ref["levels"], tol)), w
    assert edge <= 1
