#!/usr/bin/env python
"""Cost of the IAA estimator (music_iaa.cuh) on bench.py's workloads and on one az-el grid.

  python tools/bench_iaa.py [--steps 5] [--rounds 3]

On bench.py's resident C2 (M = 4, K = 3600), C3 (M = 8, K = 7200) and C5 (M = 16, K = 3600) windows and tables, with
I = 5 and I = 15, and on a 4 x 4 URA over a 360 x 91 az-el grid (1024 windows of 64 snapshots, I = 15):
  ms_per_step    process_device calls timed by CUDA events on the launch stream (best of `rounds`);
  iaa_ms         the scan slot of the stage timing, where iaa_kernel runs;
  fma            the fp64 FMA the algorithm needs, 3 K M^2 per window per pass, I + 1 passes;
  fp64_bound_ms  fma over the FP64 FFMA rate, 64 DFMA / clock / SM at the card's maximum SM clock;
  share          fp64_bound_ms / iaa_ms;
  card           the card's name, power limit and maximum SM clock, read in the same run.
Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (the workload and table of bench.py, unchanged)
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa import music_doa  # noqa: E402
from gr_baz_b200.music_doa_azel import music_doa_azel  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def sm_clock_hz(c):
    try:
        return float(c.split(",")[-1].strip().split()[0]) * 1e6
    except Exception:
        return None


def measure(blk, d_in, W, n, iters, args, stream, clock):
    dev = d_in.device
    blk.set_estimator("iaa", 0.0)
    blk.set_iaa_iterations(iters)
    ang = torch.empty((W, n), dtype=torch.float32, device=dev)
    ang2 = torch.empty_like(ang)
    lvl = torch.empty_like(ang)
    azel = isinstance(blk, music_doa_azel)
    if azel:
        f = lambda: blk.process_device(d_in.data_ptr(), W, ang.data_ptr(), ang2.data_ptr(), lvl.data_ptr(), stream=stream.cuda_stream)
    else:
        f = lambda: blk.process_device(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), None, None, stream=stream.cuda_stream)
    f()
    torch.cuda.synchronize()
    best = None
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            f()
        e1.record(stream)
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1) / args.steps
        best = t if best is None else min(best, t)
    blk.set_stage_timing(True)
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    s, _ = blk.stage_times_ms()
    blk.set_stage_timing(False)
    iaa_ms = s[2] / 3
    M, K = blk.m, blk.resolution
    fma = 3.0 * K * M * M * (iters + 1) * W
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bound = fma / (64.0 * sms * clock) * 1e3 if clock else None
    return {"windows": W, "m": M, "K": K, "iterations": iters, "ms_per_step": best, "iaa_ms": iaa_ms, "fma": fma,
            "fp64_bound_ms": bound, "share": bound / iaa_ms if bound and iaa_ms else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    c = card()
    clock = sm_clock_hz(c)
    res = {"steps": args.steps, "rounds": args.rounds, "card": c}
    for cid in (2, 3, 5):
        cfg, W = bench.workload(cid)
        d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
        synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg["id"], 0, W, dev, out=d_in)
        blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], bench.table_for(cfg)[1], cfg["resolution"])
        for iters in (5, 15):
            res["c%d_i%d" % (cid, iters)] = measure(blk, d_in, W, cfg["n"], iters, args, stream, clock)
        blk.close()
        del d_in
        torch.cuda.empty_cache()
    import azel_oracle as ao
    import iaa_oracle as io
    pos = ao.ura_xyz(4, 4, 1.0)
    W, N = 1024, 64
    x = io._windows(np.random.default_rng(1), np.array([ao.steering(pos, 1.0, 40.0, 20.0), ao.steering(pos, 1.0, 70.0, 36.0)]),
                    (1.0, 0.8), N, 20.0, True, W)
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)
    blk = music_doa_azel(16, 2, 16 * N, 360, 91, (0.0, 90.0), pos, 1.0)
    res["azel_360x91_i15"] = measure(blk, d_in, W, 2, 15, args, stream, clock)
    blk.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
