"""GPU: the root-MUSIC peak mode (MUSIC_B200_PEAKS_ROOTS) against its fp64 definition (tests/root_music_oracle.py,
numpy.roots on LAPACK eigenvectors), through every entry point, and the other peak modes unchanged.

The oracle runs on the GPU's own covariance (d_R), so what is compared is the root stage itself."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, synth
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import refine_oracle as ro
import root_music_oracle as rm

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = synth.C_LIGHT / synth.FREQUENCY
SENTINEL = -7
FLIP = 1e-9     # selections the oracle sees this close to flipping may go either way
L_RTOL = 1e-5


def ula(m, kind):
    """x-axis, y-axis, an oblique offset ULA and the x-axis ULA in reversed order, lambda / 2 apart"""
    axis, p0, rev = {"x": (0.0, (0.0, 0.0), False), "y": (90.0, (0.0, 0.0), False),
                     "oblique": (30.0, (0.7, -1.3), False), "reversed": (0.0, (0.0, 0.0), True)}[kind]
    a = math.radians(axis)
    pos = np.array([[p0[0] + 0.5 * i * math.cos(a), p0[1] + 0.5 * i * math.sin(a)] for i in range(m)])
    return pos[::-1].copy() if rev else pos


def axis_deg(pos):
    s = rm.ula_geometry(pos, LAM)[2]
    return math.degrees(math.atan2(s[1], s[0]))


def source_angles(rng, S, alpha, min_cos=0.05):
    """S angles over [0, 360), at least 2 degrees from end-fire, with distinct cos(t - alpha)"""
    while True:
        t = rng.uniform(0.0, 360.0, S)
        off = (t - alpha) % 180.0
        if np.any(np.minimum(off, 180.0 - off) < 2.0):
            continue
        cs = np.cos(np.radians(t - alpha))
        if S < 2 or np.min(np.abs(np.subtract.outer(cs, cs))[np.triu_indices(S, 1)]) >= min_cos:
            return t


def windows(pos, plan, seed, snaps):
    """complex64 windows; plan[w] = (sources, snr_db or None for noiseless); returns (x, truth per window)"""
    rng = np.random.default_rng(seed)
    m = pos.shape[0]
    alpha = axis_deg(pos)
    xs, truth = [], []
    for S, snr in plan:
        X = np.zeros((m, snaps), np.complex128)
        if snr is not None:
            X += (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
        angs = source_angles(rng, S, alpha) if S else np.zeros(0)
        amp = 1.0 if snr is None else 10.0 ** (snr / 20.0)
        for t in angs:
            a = ro.steering(pos, LAM, math.radians(t))[0]
            X += amp * a[:, None] * (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps))[None, :] / np.sqrt(2.0)
        xs.append(X.T.reshape(-1))
        truth.append(angs)
    return np.ascontiguousarray(np.array(xs).astype(np.complex64)), truth


def handle(m, n, K, pos, snaps, mode="roots", rule="fixed", devices=None):
    blk = music_doa(m, n, m * snaps, np.ones((K, m), np.complex64), K, devices=devices)
    blk.set_array_geometry(pos, LAM)
    blk.set_source_rule(rule)
    blk.set_peak_mode(mode, 0)
    return blk


def dev_call(blk, x, n, K, spectrum=False, p64=False, R=False, counts=False):
    """one process_device_ex call (or process_device_counts with counts); returns (outputs, kernel launches)"""
    dev = torch.device("cuda:0")
    Wn, m = x.shape[0], blk.m
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)
    o = {"angles": torch.full((Wn, n), SENTINEL, dtype=torch.float32, device=dev),
         "levels": torch.full((Wn, n), SENTINEL, dtype=torch.float32, device=dev),
         "bins": torch.full((Wn, n), SENTINEL, dtype=torch.int32, device=dev)}
    if spectrum:
        o["spectrum"] = torch.full((Wn, K), SENTINEL, dtype=torch.float32, device=dev)
    if p64:
        o["P64"] = torch.full((Wn, K), SENTINEL, dtype=torch.float64, device=dev)
    if R:
        o["R"] = torch.zeros((Wn, m, m, 2), dtype=torch.float64, device=dev)
    if counts:
        o["counts"] = torch.full((Wn,), SENTINEL, dtype=torch.int32, device=dev)
    p = lambda k: o[k].data_ptr() if k in o else None
    l0 = blk.launch_count()
    blk.process_device(d_in.data_ptr(), Wn, p("angles"), p("levels"), p("spectrum"), p("bins"),
                       stream=torch.cuda.current_stream().cuda_stream, d_P64=p("P64"), d_R=p("R"), d_counts=p("counts"))
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    if "R" in out:
        out["R"] = out["R"][..., 0] + 1j * out["R"][..., 1]
    return out, blk.launch_count() - l0


def circ(a, b):
    d = abs(float(a) - float(b)) % 360.0
    return min(d, 360.0 - d)


def near_half(tdeg, K):
    f = tdeg * K / 360.0
    return abs(f - math.floor(f) - 0.5) <= 1e-6


# ---- parity with the oracle ------------------------------------------------------------------------------------------
PLAN = [(0, 0.0), (1, 40.0), (2, 40.0), (1, 20.0), (2, 20.0), (3, 20.0), (1, 0.0), (2, 0.0), (3, 0.0), (1, None),
        (2, None), (3, 10.0)]


@pytest.mark.parametrize("m", [2, 3, 4, 5, 8, 12, 16])
def test_parity_with_oracle(m):
    """angles within 2 float32 ulps, levels within 1e-5, bins equal (except at half-bin ties), counts equal to a
    TOP_BINS handle's under MDL; noiseless (double-root) windows within 5e-4 degrees of the truth"""
    snaps = 512
    edge = total = 0
    for n in (1, 2, 3):
        if n >= m:
            continue
        for gi, kind in enumerate(("x", "y", "oblique", "reversed")):
            pos = ula(m, kind)
            plan = [(min(S, m - 1), snr) for S, snr in PLAN]
            x, truth = windows(pos, plan, 1000 * m + 10 * n + gi, snaps)
            for rule in ("fixed", "mdl"):
                K = 3600 if (gi + n) % 2 else 360
                blk = handle(m, n, K, pos, snaps, rule=rule)
                out, _ = dev_call(blk, x, n, K, R=True)
                counts = None
                if rule == "mdl":
                    cnt, _ = dev_call(blk, x, n, K, counts=True)
                    top = handle(m, n, K, pos, snaps, mode="top_bins", rule=rule)
                    tc, _ = dev_call(top, x, n, K, counts=True)
                    top.close()
                    assert np.array_equal(cnt["counts"], tc["counts"]), (m, n, kind)
                    assert np.array_equal(cnt["angles"], out["angles"]) and np.array_equal(cnt["bins"], out["bins"])
                    counts = tc["counts"]
                blk.close()
                for w in range(len(x)):
                    ctx = (m, n, kind, rule, K, w, plan[w])
                    d = n if counts is None else int(counts[w])
                    ref = rm.work_R(out["R"][w], pos, LAM, K, n, d=d)
                    ga, gl, gb = out["angles"][w], out["levels"][w], out["bins"][w]
                    assert np.all(gb[d:] == -1) and np.all(ga[d:] == 0.0) and np.all(gl[d:] == 0.0), ctx
                    if plan[w][1] is None:
                        if d != len(truth[w]):
                            continue  # a noise subspace inside the null space of R is not unique
                        want = sorted(min(t % 360.0, (2.0 * axis_deg(pos) - t) % 360.0) for t in truth[w])
                        got = sorted(float(a) for a in ga[:d])
                        assert max(circ(g, t) for g, t in zip(got, want)) <= 5e-4, (ctx, got, want)
                        continue
                    total += d
                    if ref["margin"] <= FLIP and not np.array_equal(gb, ref["bins"]):
                        edge += d
                        continue
                    for i in range(d):
                        ra = ref["angles"][i]
                        tol = 2.0 * float(np.spacing(np.float32(max(abs(float(ra)), abs(float(ga[i])), 1e-3))))
                        assert circ(ga[i], ra) <= tol, (ctx, i, ga, ref["angles"])
                        assert abs(float(gl[i]) - float(ref["levels"][i])) <= L_RTOL * abs(float(ref["levels"][i])), (ctx, i, gl, ref["levels"])
                        if gb[i] != ref["bins"][i]:
                            assert near_half(float(ra), K), (ctx, i, gb, ref["bins"])
    assert edge <= 0.01 * max(total, 1), (edge, total)


def test_degenerate_windows():
    """NaN and all-zero windows report (0, 0, -1); MDL with d = 0 reports no peak"""
    m, n, K, snaps = 4, 2, 360, 256
    pos = ula(m, "x")
    x, _ = windows(pos, [(2, 20.0), (2, 20.0), (0, 0.0), (2, 20.0)], 5, snaps)
    x[0] = 0
    x[1, 17] = np.nan
    for rule in ("fixed", "mdl"):
        blk = handle(m, n, K, pos, snaps, rule=rule)
        out, _ = dev_call(blk, x, n, K)
        empty = [0, 1] if rule == "fixed" else [0, 1, 2]
        for w in empty:
            assert np.all(out["bins"][w] == -1) and np.all(out["angles"][w] == 0.0) and np.all(out["levels"][w] == 0.0), (rule, w, out)
        assert np.all(out["bins"][3] >= 0) and np.all(out["levels"][3] > 0.0)
        blk.close()


# ---- entry points ------------------------------------------------------------------------------------------------------
def test_entries_agree():
    """host, device, _ex, _counts and planar (at the fused-eligible M = 4 / n = 1 shape) agree byte for byte; with the
    spectrum port the spectrum and P64 are a LOCAL_MAXIMA handle's, byte for byte"""
    m, n, K, snaps, Wn = 4, 1, 3600, 1024, 24
    pos = ula(m, "x")
    x, _ = windows(pos, [(1, 20.0)] * Wn, 31, snaps)
    blk = handle(m, n, K, pos, snaps)
    ref, _ = dev_call(blk, x, n, K)
    assert np.all(ref["bins"] >= 0)
    ex, _ = dev_call(blk, x, n, K, spectrum=True, p64=True, R=True)
    cn, _ = dev_call(blk, x, n, K, counts=True)
    for o in (ex, cn):
        assert all(np.array_equal(o[k], ref[k]) for k in ("angles", "levels", "bins"))
    assert np.all(cn["counts"] == n)
    loc = handle(m, n, K, pos, snaps, mode="local_maxima")
    lo, _ = dev_call(loc, x, n, K, spectrum=True, p64=True)
    loc.close()
    assert np.array_equal(lo["spectrum"], ex["spectrum"]) and np.array_equal(lo["P64"], ex["P64"])
    ang, lvl, spec = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32), np.zeros((Wn, K), np.float32)
    blk.work(Wn, [x], [ang, lvl, spec])
    assert np.array_equal(ang, ref["angles"]) and np.array_equal(lvl, ref["levels"]) and np.array_equal(blk.last_bins(), ref["bins"])
    assert np.array_equal(spec, ex["spectrum"])
    streams = [np.ascontiguousarray(x.reshape(Wn, snaps, m)[:, :, r].reshape(-1)) for r in range(m)]
    pa, pl = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32)
    blk.work_planar(Wn, streams, [pa, pl])
    assert np.array_equal(pa, ref["angles"]) and np.array_equal(pl, ref["levels"]) and np.array_equal(blk.last_bins(), ref["bins"])
    dev = torch.device("cuda:0")
    d_streams = [torch.from_numpy(s.view(np.float32)).to(dev) for s in streams]
    da = torch.zeros((Wn, n), dtype=torch.float32, device=dev)
    l0 = blk.launch_count()
    blk.process_planar_device([t.data_ptr() for t in d_streams], snaps, Wn, da.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert blk.launch_count() - l0 == 3  # the planar covariance, eig, roots: never the fused kernel
    assert np.array_equal(da.cpu().numpy(), ref["angles"])
    blk.close()
    G = torch.cuda.device_count()
    for devices in ([0], list(range(G))):
        mb = handle(m, n, K, pos, snaps, devices=devices)
        a2, l2 = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32)
        mb.work(Wn, [x], [a2, l2])
        assert np.array_equal(a2, ref["angles"]) and np.array_equal(l2, ref["levels"]), devices
        g, _ = dev_call(mb, x, n, K)
        assert np.array_equal(g["angles"], ref["angles"]) and np.array_equal(g["bins"], ref["bins"]), devices
        mb.close()
    if G < 2:
        return
    mb = handle(m, n, K, pos, snaps, devices=list(range(G)))
    ins, angs, bins_all = [], [], []
    for g in range(G):
        d = torch.device("cuda", g)
        ins.append(torch.from_numpy(np.ascontiguousarray(x[g::G]).view(np.float32)).to(d))
        angs.append(torch.zeros((len(x[g::G]), n), dtype=torch.float32, device=d))
        bins_all.append(torch.full((Wn, n), SENTINEL, dtype=torch.int32, device=d))
    mb.process_device_sharded([t.data_ptr() for t in ins], Wn, [t.data_ptr() for t in angs], None, [t.data_ptr() for t in bins_all])
    for g in range(G):
        torch.cuda.synchronize(g)
    for g in range(G):
        assert np.array_equal(angs[g].cpu().numpy(), ref["angles"][g::G]), g
        assert np.array_equal(bins_all[g].cpu().numpy(), ref["bins"]), g
    mb.close()


def test_launch_counts_and_sub_batches():
    """per sub-batch: covariance + eig + roots, +1 source count under MDL, +1 scan with the spectrum"""
    m, n, K, snaps = 4, 1, 3600, 256
    pos = ula(m, "x")
    x, _ = windows(pos, [(1, 20.0)], 3, snaps)
    for rule, spectrum, want in (("fixed", False, 3), ("mdl", False, 4), ("fixed", True, 4), ("mdl", True, 5)):
        blk = handle(m, n, K, pos, snaps, rule=rule)
        _, launches = dev_call(blk, x, n, K, spectrum=spectrum)
        assert launches == want, (rule, spectrum, launches)
        blk.close()
    # several sub-batches (the internal fp64 spectrum of K bins per window bounds one); the whole call equals its halves
    Kb, Wb, Nb = 36000, 3000, 64
    xb, _ = windows(pos, [(1, 20.0)] * Wb, 808, Nb)
    blk = handle(m, n, Kb, pos, Nb)
    whole, launches = dev_call(blk, xb, n, Kb, spectrum=True)
    assert launches % 4 == 0 and launches // 4 >= 2, launches
    first, _ = dev_call(blk, xb[: Wb // 2], n, Kb, spectrum=True)
    second, _ = dev_call(blk, xb[Wb // 2:], n, Kb, spectrum=True)
    for k in ("angles", "levels", "bins", "spectrum"):
        assert np.array_equal(whole[k], np.concatenate([first[k], second[k]])), k
    blk.close()


def test_switching_back_to_top_bins():
    """TOP_BINS after ROOTS is byte-identical to a fresh handle and runs the fused kernel once per call at the C2 shape"""
    cfg = synth.config(2, snapshots=4096)
    x = synth.gen_windows_numpy(cfg, 11, 0, 64)
    pos = ula(4, "x")
    fresh = handle(4, 1, cfg["resolution"], pos, cfg["snapshots"], mode="top_bins")
    ref, l_ref = dev_call(fresh, x, 1, cfg["resolution"])
    fresh.close()
    blk = handle(4, 1, cfg["resolution"], pos, cfg["snapshots"])
    _, l_roots = dev_call(blk, x, 1, cfg["resolution"])
    assert l_roots == 3
    blk.set_peak_mode("top_bins", 0)
    got, l_top = dev_call(blk, x, 1, cfg["resolution"])
    assert l_ref == l_top == 1
    assert all(np.array_equal(got[k], ref[k]) for k in ("angles", "levels", "bins"))
    blk.close()


# ---- what the mode is for ----------------------------------------------------------------------------------------------
def test_mirror_case():
    """M = 4 x-axis ULA, sources at 40 and 110 degrees at 20 dB: the root mode reports both in every window (the local
    maximum rule spends its second slot on the mirror of the first)"""
    m, n, K, snaps, Wn = 4, 2, 3600, 4096, 100
    pos = ula(m, "x")
    rng = np.random.default_rng(40)
    xs = []
    for _ in range(Wn):
        X = (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
        for t in (40.0, 110.0):
            a = ro.steering(pos, LAM, math.radians(t))[0]
            X += 10.0 * a[:, None] * (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps))[None, :] / np.sqrt(2.0)
        xs.append(X.T.reshape(-1))
    x = np.array(xs).astype(np.complex64)
    blk = handle(m, n, K, pos, snaps)
    out, _ = dev_call(blk, x, n, K)
    blk.close()
    got = np.sort(out["angles"], axis=1)
    assert np.all(np.abs(got[:, 0] - 40.0) < 1.0) and np.all(np.abs(got[:, 1] - 110.0) < 1.0), got


@pytest.mark.parametrize("m,th", [(4, (70.0, 78.0)), (8, (30.0, 36.0))])
def test_resolution(m, th):
    """0 dB, 1024 snapshots: both sources within half their separation in at least 90 % of windows"""
    n, K, snaps, Wn = 2, 3600, 1024, 200
    pos = ula(m, "x")
    rng = np.random.default_rng(7 * m)
    xs = []
    for _ in range(Wn):
        X = (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / np.sqrt(2.0)
        for t in th:
            a = ro.steering(pos, LAM, math.radians(t))[0]
            X += a[:, None] * (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps))[None, :] / np.sqrt(2.0)
        xs.append(X.T.reshape(-1))
    x = np.array(xs).astype(np.complex64)
    blk = handle(m, n, K, pos, snaps)
    out, _ = dev_call(blk, x, n, K)
    blk.close()
    got = np.sort(out["angles"], axis=1)
    ok = np.all(np.abs(got - np.array(th)[None, :]) < (th[1] - th[0]) / 2.0, axis=1)
    assert ok.mean() >= 0.9, ok.mean()


# ---- invalid combinations ----------------------------------------------------------------------------------------------
def test_invalid_combinations():
    m, n, K, snaps = 4, 1, 360, 64
    pos = ula(m, "x")
    L = _capi.load()
    blk = music_doa(m, n, m * snaps, np.ones((K, m), np.complex64), K)
    EINVAL = _capi.EINVAL
    # a set_table() table has no geometry
    assert L.music_b200_set_peak_mode(blk._h, 2, 0) == EINVAL
    blk.set_array_geometry(pos, LAM)
    assert L.music_b200_set_peak_mode(blk._h, 2, 1) == EINVAL  # exclusion_bins must be 0
    # MVDR / Bartlett / NEWTON, in either order
    for kind, loading in (("mvdr", 0.01), ("bartlett", 0.0)):
        blk.set_estimator(kind, loading)
        assert L.music_b200_set_peak_mode(blk._h, 2, 0) == EINVAL
        blk.set_estimator("music", 0.0)
    blk.set_refine(True)
    assert L.music_b200_set_peak_mode(blk._h, 2, 0) == EINVAL
    blk.set_refine(False)
    assert L.music_b200_set_peak_mode(blk._h, 2, 0) == _capi.OK
    assert L.music_b200_set_estimator(blk._h, 1, 0.01) == EINVAL
    assert L.music_b200_set_estimator(blk._h, 2, 0.0) == EINVAL
    assert L.music_b200_set_refine(blk._h, 1) == EINVAL
    assert L.music_b200_set_estimator(blk._h, 0, 0.0) == _capi.OK
    # non-ULA geometries: a UCA, one element off the line, 0.6 lambda spacing
    uca = np.asarray([[0.5 * math.cos(2 * math.pi * i / m), 0.5 * math.sin(2 * math.pi * i / m)] for i in range(m)])
    bent = ula(m, "x")
    bent[2, 1] += 1e-5 * 0.5
    x, _ = windows(pos, [(1, 20.0)], 2, snaps)
    for bad in (uca, bent, ula(m, "x") * 1.2):
        blk.set_array_geometry(bad, LAM)  # set_geometry() itself keeps its behaviour
        with pytest.raises(_capi.MusicB200Error):
            dev_call(blk, x, n, K)
        assert L.music_b200_set_peak_mode(blk._h, 2, 0) == EINVAL
        blk.set_array_geometry(pos, LAM)
        assert L.music_b200_set_peak_mode(blk._h, 2, 0) == _capi.OK
    # set_table() after set_peak_mode(ROOTS): the call fails, no fall-back to grid peaks
    blk.set_array_response(np.ones((K, m), np.complex64))
    with pytest.raises(_capi.MusicB200Error):
        dev_call(blk, x, n, K)
    ang = np.zeros((1, n), np.float32)
    with pytest.raises(_capi.MusicB200Error):
        blk.work(1, [x], [ang])
    with pytest.raises(ValueError):
        blk.set_peak_mode("root")
    blk.close()
    # az-el handles
    az = music_doa_azel(m, n, m * snaps, 36, 3, (0.0, 30.0), np.c_[pos, np.zeros(m)], LAM)
    assert L.music_b200_set_peak_mode(az._h, 2, 0) == EINVAL
    with pytest.raises(_capi.MusicB200Error):
        az.set_peak_mode("roots")
    az.close()


def test_cpp_block():
    """the C++ block through set_peak_mode(2, 0) equals the Python block"""
    exe = os.path.join(ROOT, "lib", "_build", "test_block_roots")
    m, n, K, snaps, Wn = 8, 2, 720, 256, 16
    pos = ula(m, "oblique")
    x, _ = windows(pos, [(2, 20.0)] * Wn, 77, snaps)
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        fin, fout = os.path.join(td, "in.bin"), os.path.join(td, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("<6I", m, n, m * snaps, K, Wn, 1))
            f.write(struct.pack("<d", LAM))
            f.write(np.ascontiguousarray(pos, np.float64).tobytes())
            f.write(x.view(np.float32).tobytes())
        r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        raw = open(fout, "rb").read()
    o = 0
    take = lambda cnt, dt: np.frombuffer(raw[o:o + 4 * cnt], dt)
    ca = take(Wn * n, np.float32); o += 4 * Wn * n
    cl = take(Wn * n, np.float32); o += 4 * Wn * n
    cs = take(Wn * K, np.float32); o += 4 * Wn * K
    cb = take(Wn * n, np.int32); o += 4 * Wn * n
    cc = take(Wn, np.int32)
    blk = handle(m, n, K, pos, snaps, rule="mdl")
    ang, lvl, spec = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32), np.zeros((Wn, K), np.float32)
    blk.work(Wn, [x], [ang, lvl, spec])
    assert np.array_equal(ca, ang.ravel()) and np.array_equal(cl, lvl.ravel()) and np.array_equal(cs, spec.ravel())
    assert np.array_equal(cb, blk.last_bins().ravel()) and np.array_equal(cc, blk.last_counts())
    assert np.all(cc == 2) and np.all(cb >= 0)
    blk.close()
