#!/usr/bin/env python
"""Small invocations of the kernels compute-sanitizer should look at (SURVEY.md section 5): run as
  compute-sanitizer --tool racecheck|memcheck|synccheck python tools/sanitize_targets.py <target>
targets: fused (C1-size windows, 2000 of them + a ragged 1187 + a drain-only 9), fused_jacobi, fused8, covn8, covn16, eig16, esprit2d,
gridless_roots, crb, tracks, wsf, iaa, multi,
lifecycle (every handle kind created, retuned, grown and destroyed through the host entry points; run it under
  compute-sanitizer --tool memcheck --leak-check full, which reports what a handle leaves allocated)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from gr_baz_b200 import synth
from gr_baz_b200.music_doa import music_doa

target = sys.argv[1] if len(sys.argv) > 1 else "fused"
dev = torch.device("cuda:0")


def synth_table(m, K):
    """a UCA table of m elements, lambda / 2 between neighbours"""
    k = np.arange(m)
    r = 0.25 / np.sin(np.pi / m) if m > 2 else 0.25
    pos = np.stack([r * np.cos(2 * np.pi * k / m), r * np.sin(2 * np.pi * k / m)], 1)
    th = np.arange(K) * 2 * np.pi / K
    return np.exp(-2j * np.pi * (np.outer(np.cos(th), pos[:, 0]) + np.outer(np.sin(th), pos[:, 1]))).astype(np.complex64)


def run(cfg, counts, devices=None):
    resp, _ = bench.table_for(cfg)
    Wmax = max(counts)
    d_in = synth.gen_windows_torch(cfg, 1234, 0, Wmax, dev)
    blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], resp, cfg["resolution"], devices=devices)
    a = torch.empty((Wmax, cfg["n"]), dtype=torch.float32, device=dev)
    l = torch.empty_like(a)
    b = torch.empty((Wmax, cfg["n"]), dtype=torch.int32, device=dev)
    for W in counts:
        blk.process_device(d_in.data_ptr(), W, a.data_ptr(), l.data_ptr(), None, b.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    print(target, "ok: bins[:8] =", b[:8, 0].cpu().numpy().tolist(), "launches", blk.launch_count())
    blk.close()


if target in ("fused", "fused_jacobi"):
    if target == "fused_jacobi":
        os.environ["MUSIC_B200_EIG"] = "jacobi"
    run(synth.config(1), (2000, 1187, 9))
elif target in ("covn8", "fused8"):  # M = 8, n = 1 takes the fused M = 8 kernel by default; covn8 = the three-kernel path
    if target == "covn8":
        os.environ["MUSIC_B200_FUSED"] = "0"
    run(synth.config(4, snapshots=1024, resolution=360), (600, 37))
elif target == "covn16":
    run(synth.config(5, snapshots=512, resolution=360), (300, 19))
elif target == "eig16":
    run(synth.config(5, snapshots=128, resolution=180), (64,))
elif target == "esprit2d":
    # 2-D ESPRIT on az-el handles (music_esprit2d.cuh): 4 x 4 and 2 x 4 lattices, a ragged window count (the last CTA's
    # idle warps), d = n on noise windows
    from gr_baz_b200.music_doa_azel import music_doa_azel
    lam = 0.5
    for rows, cols, n in ((4, 4, 3), (2, 4, 2)):
        m = rows * cols
        pos = np.array([[c * 0.25, r * 0.25, 0.0] for r in range(rows) for c in range(cols)])
        rng = np.random.default_rng(m)
        W = 301
        x = ((rng.standard_normal((W, 64 * m)) + 1j * rng.standard_normal((W, 64 * m))) * 0.1).astype(np.complex64)
        az = music_doa_azel(m, n, 64 * m, 72, 19, (0.0, 90.0), pos, lam)
        az.set_peak_mode("esprit", 0)
        outs = [np.zeros((W, s), np.float32) for s in (n, n, n, az.resolution)]
        az.work(W, [x], outs)
        print("esprit2d ok", m, outs[0][:2])
        az.close()
elif target == "gridless_roots":
    # the shared root finder of ROOTS and MANIFOLD (music_roots.cuh): ROOTS on x-axis ULAs (one warp per window), MANIFOLD
    # on UCA 8 (L = 32, one warp), UCA 16 (L = 46, three warps) and a UCA 16 at 0.85 lambda (L = 63, four warps); a
    # ragged window count with a zero window and a NaN window
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import manifold_oracle as mf
    from helpers import LAM, plan_windows, ula

    for mode, m, n, pos in (("roots", 4, 1, ula(4, "x")), ("roots", 16, 3, ula(16, "x")), ("manifold", 8, 2, mf.uca(8, 0.5, LAM)),
                            ("manifold", 16, 3, mf.uca(16, 0.5, LAM)), ("manifold", 16, 3, mf.uca(16, 0.85, LAM))):
        W = 37
        x, _ = plan_windows(pos, [(1 + w % n, 20.0) for w in range(W)], m, 256)
        x[3] = 0
        x[5, 11] = np.nan
        blk = music_doa(m, n, m * 256, np.ones((360, m), np.complex64), 360)
        blk.set_array_geometry(pos, LAM)
        blk.set_peak_mode(mode, 0)
        ang = np.zeros((W, n), np.float32)
        blk.work(W, [x], [ang])
        print(target, "ok", mode, m, ang[:2].tolist())
        blk.close()
elif target == "crb":
    # the CRB kernel (music_crb.cuh): 1-D at M = 3, 8 and 16 with n up to M - 1 (every slot filled by DML, so d = 15 at
    # M = 16), and az-el at M = 16 with n = 15 (30 parameters, the largest shared-memory footprint); a zero window and a
    # NaN window among them
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from gr_baz_b200.music_doa_azel import music_doa_azel
    from helpers import LAM

    W = 37
    for m, n, mode in ((3, 2, "dml"), (8, 3, "local_maxima"), (16, 15, "dml")):
        rng = np.random.default_rng(m)
        x = ((rng.standard_normal((W, 64 * m)) + 1j * rng.standard_normal((W, 64 * m)))).astype(np.complex64)
        x[3] = 0
        x[5, 11] = np.nan
        k = np.arange(m)
        pos = np.stack([0.5 * LAM * np.cos(2 * np.pi * k / m) * m / 6, 0.5 * LAM * np.sin(2 * np.pi * k / m) * m / 6], 1)
        blk = music_doa(m, n, 64 * m, np.ones((360, m), np.complex64), 360)
        blk.set_array_geometry(pos, LAM)
        blk.set_peak_mode(mode, 0)
        blk.set_crb(True)
        blk.work(W, [x], [np.zeros((W, n), np.float32)])
        print(target, "ok", m, n, mode, blk.last_crb()[:2].tolist())
        blk.close()
    m, n = 16, 15
    rng = np.random.default_rng(16)
    x = ((rng.standard_normal((W, 64 * m)) + 1j * rng.standard_normal((W, 64 * m)))).astype(np.complex64)
    x[3] = 0
    pos = rng.uniform(-0.6, 0.6, (m, 3)) * LAM
    az = music_doa_azel(m, n, 64 * m, 36, 9, (0.0, 80.0), pos, LAM)
    az.set_peak_mode("local_maxima", 0)
    az.set_crb(True)
    az.work(W, [x], [np.zeros((W, n), np.float32) for _ in range(3)])
    print(target, "ok az-el", az.last_crb()[:1, :2].tolist())
    az.close()
elif target == "wsf":
    # the WSF matrix and the JOINT refinement (music_wsf.cuh): M = 3, 8 and 16 with n up to M - 1 (d = 15 at M = 16, the
    # largest shared-memory footprint), under WSF and DML; a zero window and a NaN window among them
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from helpers import LAM

    W = 37
    for m, n, mode in ((3, 2, "wsf"), (8, 3, "dml"), (16, 15, "wsf")):
        rng = np.random.default_rng(m)
        x = ((rng.standard_normal((W, 64 * m)) + 1j * rng.standard_normal((W, 64 * m)))).astype(np.complex64)
        x[3] = 0
        x[5, 11] = np.nan
        k = np.arange(m)
        pos = np.stack([0.5 * LAM * np.cos(2 * np.pi * k / m) * m / 6, 0.5 * LAM * np.sin(2 * np.pi * k / m) * m / 6], 1)
        blk = music_doa(m, n, 64 * m, np.ones((360, m), np.complex64), 360)
        blk.set_array_geometry(pos, LAM)
        blk.set_peak_mode(mode, 0)
        blk.set_refine("joint")
        ang = np.zeros((W, n), np.float32)
        blk.work(W, [x], [ang])
        print(target, "ok", m, n, mode, ang[:2].tolist())
        blk.close()
elif target == "iaa":
    # the IAA kernel (music_iaa.cuh): M = 2, 4 and 16 (T = 8, 8 and 4 windows per CTA; the partial sums alias the tile
    # region, M = 16 has the largest shared-memory footprint), a ragged window count (37: the last CTA is partly
    # empty), a zero window and a NaN window (both fail before the first pass), and at M = 4 a noiseless rank-one window
    # with loading 0, then a run with the spectrum port and a split into host chunks
    W = 37
    for m, n, loading in ((2, 1, 0.0), (4, 2, 0.0), (16, 3, 0.01)):
        rng = np.random.default_rng(m)
        N = 32
        x = ((rng.standard_normal((W, N * m)) + 1j * rng.standard_normal((W, N * m)))).astype(np.complex64)
        x[3] = 0
        x[5, 11] = np.nan
        if m == 4:
            x[7] = np.tile(np.exp(1j * np.arange(m) * 0.7), N).astype(np.complex64)
        blk = music_doa(m, n, N * m, synth_table(m, 360), 360)
        blk.set_estimator("iaa", loading)
        blk.set_iaa_iterations(3)
        ang = np.zeros((W, n), np.float32)
        spec = np.zeros((W, 360), np.float32)
        blk.work(W, [x], [ang, np.zeros((W, n), np.float32), spec])
        blk.work(9, [x[28:]], [ang[:9]])
        print(target, "ok", m, n, ang[:2].tolist(), bool(np.isnan(spec[3]).all()), bool(np.isnan(spec[5]).all()))
        blk.close()
elif target == "tracks":
    # the tracker (music_track.cuh): 32 rows and 15 slots in 1-D (CRB variance, every slot filled by DML) and az-el, a wide
    # gate so that ambiguous clusters reach the assignment solve, a zero window and a NaN window (a failed CRB) among
    # them, and a ragged window count over several input chunks
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from gr_baz_b200.music_doa_azel import music_doa_azel
    from helpers import LAM

    W, m, n = 101, 16, 15
    rng = np.random.default_rng(32)
    x = ((rng.standard_normal((W, 64 * m)) + 1j * rng.standard_normal((W, 64 * m)))).astype(np.complex64)
    x[3] = 0
    x[5, 11] = np.nan
    k = np.arange(m)
    pos = np.stack([0.5 * LAM * np.cos(2 * np.pi * k / m) * m / 6, 0.5 * LAM * np.sin(2 * np.pi * k / m) * m / 6], 1)
    blk = music_doa(m, n, 64 * m, np.ones((360, m), np.complex64), 360)
    blk.set_array_geometry(pos, LAM)
    blk.set_peak_mode("dml", 0)
    blk.set_tracking("crb", q=1.0, floor_deg=2.0, gate=1e4, confirm_hits=2, confirm_window=3, max_misses=2, max_tracks=32)
    blk.work(W, [x], [np.zeros((W, n), np.float32)])
    print(target, "ok 1-D", blk.last_tracks()[0][:2].tolist())
    blk.close()
    az = music_doa_azel(m, n, 64 * m, 36, 9, (0.0, 80.0), rng.uniform(-0.6, 0.6, (m, 3)) * LAM, LAM)
    az.set_peak_mode("local_maxima", 0)
    az.set_tracking("crb", q=1.0, floor_deg=2.0, gate=1e4, confirm_hits=1, confirm_window=1, max_misses=2, max_tracks=32)
    az.work(W, [x], [np.zeros((W, n), np.float32) for _ in range(3)])
    print(target, "ok az-el", az.last_tracks()[1][:1].tolist())
    az.close()
elif target == "multi":
    cfg = synth.config(1)
    resp, table = bench.table_for(cfg)
    W = 300
    x = synth.gen_windows_numpy(cfg, 7, 0, W)
    blk = music_doa(4, 1, cfg["nsamples"], resp, cfg["resolution"], devices=list(range(torch.cuda.device_count())))
    ang = np.zeros((W, 1), np.float32)
    blk.work(W, [x], [ang])
    print("multi ok", ang[:4, 0])
    blk.close()
elif target == "lifecycle":
    # Host entry points only: device memory torch allocated would be reported as a leak.  The primary context is reset
    # at the end, because compute-sanitizer reports the allocations still live when a context is destroyed.  The handles
    # take turns on the same input arrays, so none registers caller memory (a range stays registered to the handle that
    # registered it).
    import ctypes

    os.environ["MUSIC_B200_HOSTREG"] = "0"

    from gr_baz_b200.music_doa_azel import music_doa_azel
    from gr_baz_b200.music_doa_channels import music_doa_channels

    cfg = synth.config(1)
    resp, table = bench.table_for(cfg)
    rng = np.random.default_rng(5)
    m, n, ns, K = cfg["m"], cfg["n"], cfg["nsamples"], cfg["resolution"]
    x = synth.gen_windows_numpy(cfg, 9, 0, 600)
    pos = np.array([[0.5 * i, 0.0] for i in range(m)]) * synth.C_LIGHT / synth.FREQUENCY
    lam = synth.C_LIGHT / synth.FREQUENCY

    def work(blk, W, ports):
        outs = [np.zeros((W, s), np.float32) for s in ports]
        blk.work(W, [x[:W]], outs)

    for devices in (None, [0]):
        blk = music_doa(m, n, ns, resp, K, devices=devices)
        work(blk, 16, [n, n])                      # fused path
        blk.set_array_geometry(pos, lam)           # retunes: every slot refilled after it has been current
        blk.set_array_response(resp)
        blk.set_array_geometry(pos[::-1].copy(), lam)
        blk.set_source_rule("mdl")                 # unfused: workspace and staging grow
        work(blk, 40, [n, n])
        work(blk, 600, [n, n, K])
        blk.set_beamformer("das")
        work(blk, 300, [n, n])
        blk.set_source_rule("fixed")
        blk.set_beamformer("off")
        if devices is None:
            blk.calibrate(x[:64], 0.0, kind="phase")
            blk.reduce_angles(np.zeros((8, n), np.float32), np.ones((8, n), np.float32), weighted=True)
            blk.reduce_spectrum(np.ones((8, K), np.float32))
            blk.gather_attach(1, 0, [blk.gather_create(64)])
        blk.close()
    az = music_doa_azel(m, n, ns, 36, 4, (0.0, 45.0), np.c_[pos, np.zeros(m)], lam)
    for i in range(3):
        az.set_array_geometry(np.c_[pos * (1.0 + 0.1 * i), np.zeros(m)], lam)
    outs = [np.zeros((100, s), np.float32) for s in (n, n, n, az.resolution)]
    az.work(100, [x[:100]], outs)
    az.close()
    for combine in ("separate", "incoherent", "coherent"):
        ch = music_doa_channels(m, n, ns, 90, 16, (14, 5), "hann", combine, np.asarray(synth.antenna_array("uca", m)), 0.3, 400e6, 56e6)
        ch.set_array_geometry(np.asarray(synth.antenna_array("uca", m)) * 0.35, 420e6, 56e6)
        if combine == "coherent":
            ch.set_focusing(10, 60)
        else:
            ch.set_array_response(rng.standard_normal((90, m)) + 1j * rng.standard_normal((90, m)))
        ch.set_array_geometry(np.asarray(synth.antenna_array("uca", m)) * 0.3, 380e6, 56e6)
        for W in (8, 200):
            ch.process_host(x, W, spectrum=True, counts=combine != "incoherent", R=True)
        ch.close()
    libcuda = ctypes.CDLL("libcuda.so.1")
    dev0 = ctypes.c_int()
    assert libcuda.cuDeviceGet(ctypes.byref(dev0), 0) == 0
    assert libcuda.cuDevicePrimaryCtxReset(dev0) == 0
    print("lifecycle ok")
