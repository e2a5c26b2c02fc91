#!/usr/bin/env python
"""Cost of receiver calibration (music_b200_set_calibration, music_b200_calib_*) on bench.py's workloads.

  python tools/bench_calibration.py [--steps 20] [--rounds 3]

On bench.py's resident C2 (M = 4, 4096 snapshots, K = 3600, n = 1, 10 000 windows) and C5 (M = 16, n = 2, 4096
windows) windows and tables, two handles are timed alternately (`steps` back-to-back process_device calls per handle
per round, CUDA events on the launch stream):
  plain        no calibration (the fused kernel at C2);
  calibrated   seeded complex gains set (the unfused plan plus calib_apply_kernel).
Also reported:
  stage_ms     per-stage times of both handles (cov, eig, scan, top-n); the calibrated cov slot includes the apply kernel;
  apply_ms     calib_apply_kernel's own time per step (torch.profiler) and its share of the calibrated cov slot;
  accumulate   music_b200_calib_accumulate_device over the resident windows: windows/s and input GB/s;
  gain_error   after one solve on windows of one 20 dB source at a known direction (the resident window shape and
               count, corrupted by the seeded gains): the largest phase error (degrees) and magnitude error (relative);
  card         the card's name, power limit and maximum SM clock, read in the same run.
Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (the workload and table of bench.py, unchanged)
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa import music_doa  # noqa: E402

SOURCE_DEG = 57.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def seeded_gains(m, seed):
    rng = np.random.default_rng(seed)
    return 10.0 ** (rng.uniform(-3.0, 3.0, m) / 20.0) * np.exp(1j * rng.uniform(-math.pi, math.pi, m))


def calibration_windows(pos, lam, g, W, N, dev, seed):
    """W windows [N][M] of one 20 dB source at SOURCE_DEG plus unit noise, corrupted by g, as interleaved float32"""
    gen = torch.Generator(device=dev).manual_seed(seed)
    m = len(pos)
    t = math.radians(SOURCE_DEG)
    phi = 2.0 * math.pi * (pos[:, 1] * math.sin(t) + pos[:, 0] * math.cos(t)) / lam
    a = torch.tensor(np.exp(-1j * phi) * g, dtype=torch.complex128, device=dev)
    gt = torch.tensor(g, dtype=torch.complex128, device=dev)
    out = torch.empty((W, N, m), dtype=torch.complex64, device=dev)
    for w0 in range(0, W, 512):
        w1 = min(W, w0 + 512)
        s = torch.randn((w1 - w0, N, 1), dtype=torch.complex128, device=dev, generator=gen) * 10.0
        nz = torch.randn((w1 - w0, N, m), dtype=torch.complex128, device=dev, generator=gen)
        out[w0:w1] = (s * a + nz * gt).to(torch.complex64)
    return torch.view_as_real(out).reshape(W, -1).contiguous()


def run(cfg, W, args, dev, stream):
    n, K, m = cfg["n"], cfg["resolution"], cfg["m"]
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg["id"], 0, W, dev, out=d_in)
    pos = np.array([[synth.SPACING * x, synth.SPACING * y] for x, y in cfg["antenna_array"]])
    lam = synth.C_LIGHT / synth.FREQUENCY
    g = seeded_gains(m, 1000 + cfg["id"])
    table = bench.table_for(cfg)[1]
    blks = {}
    for k in ("plain", "calibrated"):
        b = music_doa(m, n, cfg["nsamples"], table, K)
        b.set_array_geometry(pos, lam)
        if n > 1:
            b.set_peak_mode("local_maxima", 0)
        blks[k] = b
    blks["calibrated"].set_calibration(g)
    ang = torch.empty((W, n), dtype=torch.float32, device=dev)
    lvl = torch.empty((W, n), dtype=torch.float32, device=dev)
    bins = torch.empty((W, n), dtype=torch.int32, device=dev)

    def call(k):
        blks[k].process_device(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), None, bins.data_ptr(), stream=stream.cuda_stream)

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            f()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for k in blks:
        for _ in range(3):
            call(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in blks}
    for _ in range(args.rounds):
        for k in blks:
            ms[k].append(timed(lambda: call(k)))
    stage = {}
    for k, b in blks.items():
        b.set_stage_timing(True)
        for _ in range(3):
            call(k)
        torch.cuda.synchronize()
        s, _ = b.stage_times_ms()
        b.set_stage_timing(False)
        stage[k] = dict(zip(("cov", "eig", "scan", "topn"), [v / 3 for v in s]))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call("calibrated")
        torch.cuda.synchronize()
    apply_ms = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in prof.key_averages()
                   if "calib_apply_kernel" in e.key) / 1e3 / 5
    # accumulation over the resident windows
    b = blks["plain"]
    b.calib_reset()
    b.calib_accumulate_device(d_in.data_ptr(), W, stream=stream.cuda_stream)
    torch.cuda.synchronize()
    acc_ms = []
    for _ in range(args.rounds):
        b.calib_reset()
        acc_ms.append(timed(lambda: b.calib_accumulate_device(d_in.data_ptr(), W, stream=stream.cuda_stream)))
    best = min(acc_ms)
    # gain error after one solve on one-source windows of the same shape and count
    del d_in
    torch.cuda.empty_cache()
    x = calibration_windows(pos, lam, g, W, cfg["snapshots"], dev, 2000 + cfg["id"])
    b.calib_reset()
    b.calib_accumulate_device(x.data_ptr(), W, stream=stream.cuda_stream)
    torch.cuda.synchronize()
    est, rho, sweeps = b.calib_solve(SOURCE_DEG)
    want = g * np.conj(g[0]) / abs(g[0])
    want = want * math.sqrt(m / np.sum(np.abs(want) ** 2))
    for bb in blks.values():
        bb.close()
    return {"windows_per_step": W, "ms_per_step": ms, "stage_ms": stage,
            "apply_ms": apply_ms, "apply_share_of_cov_slot": apply_ms / stage["calibrated"]["cov"] if stage["calibrated"]["cov"] else None,
            "accumulate": {"ms": acc_ms, "windows_per_s": W / (best * 1e-3), "input_GBps": W * cfg["nsamples"] * 8 / (best * 1e-3) / 1e9},
            "gain_error": {"phase_deg": float(np.max(np.abs(np.degrees(np.angle(est / want))))),
                           "magnitude_rel": float(np.max(np.abs(np.abs(est) / np.abs(want) - 1.0))),
                           "residual": rho, "sweeps": sweeps}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    res = {"steps_per_round": args.steps, "rounds": args.rounds, "card": card()}
    for c in (2, 5):
        cfg, W = bench.workload(c)
        res["c%d" % c] = run(cfg, W, args, dev, stream)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
