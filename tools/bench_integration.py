#!/usr/bin/env python
"""Cost of covariance integration across windows (music_b200_set_integration) on bench.py's workloads.

  python tools/bench_integration.py [--steps 20] [--rounds 3] [--alpha 0.95]

On bench.py's resident C2 (M = 4, 4096 snapshots, K = 3600), C3 (M = 8, 8192 snapshots, K = 7200) and C5 (M = 16, n = 2,
4096 snapshots) windows and tables, two handles are timed alternately (`steps` back-to-back process_device calls per
handle per round, CUDA events on the launch stream):
  plain        integration off (the fused kernel at C2 and C3);
  integrated   alpha set (the unfused plan plus integ_tiles_kernel, integ_carry_kernel and integ_apply_kernel).
Also reported:
  stage_ms     per-stage times of both handles (cov, eig, scan, top-n); the integrated cov slot includes the integration;
  integ_ms     the three integration kernels' own time per step (torch.profiler), their share of the integrated step
               and of its cov slot;
  bytes        what the integration moves per step: the tile pass reads R, the apply pass reads and writes it
               (16 M^2 bytes per window each way), the carry pass reads and writes the tile aggregates; and the
               8 N M bytes per window the covariance kernel reads, for comparison;
  integ_GBps   those bytes over integ_ms, and their share of the 3.35 TB/s HBM3 data-sheet peak of an H100 SXM;
  card         the card's name, power limit and maximum SM clock, read in the same run.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (the workload and table of bench.py, unchanged)
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa import music_doa  # noqa: E402

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
INTEG_T = 32        # windows per tile (music_integrate.cuh)
KERNELS = ("integ_tiles_kernel", "integ_carry_kernel", "integ_apply_kernel")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def integration_bytes(W, m, sub):
    """bytes the three kernels move for W windows run in sub-batches of at most `sub` windows"""
    E8 = 2 * m * m * 8
    total = 0
    for w0 in range(0, W, sub):
        Ws = min(sub, W - w0)
        tiles = (Ws + INTEG_T - 1) // INTEG_T
        total += Ws * E8 * 3 + tiles * E8 * 3
    return total


def run(cfg, W, args, dev, stream):
    n, K, m = cfg["n"], cfg["resolution"], cfg["m"]
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg["id"], 0, W, dev, out=d_in)
    pos = np.array([[synth.SPACING * x, synth.SPACING * y] for x, y in cfg["antenna_array"]])
    lam = synth.C_LIGHT / synth.FREQUENCY
    table = bench.table_for(cfg)[1]
    blks = {}
    for k in ("plain", "integrated"):
        b = music_doa(m, n, cfg["nsamples"], table, K)
        b.set_array_geometry(pos, lam)
        if n > 1:
            b.set_peak_mode("local_maxima", 0)
        blks[k] = b
    blks["integrated"].set_integration(args.alpha)
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
        s, chunks = b.stage_times_ms()
        b.set_stage_timing(False)
        stage[k] = dict(zip(("cov", "eig", "scan", "topn"), [v / 3 for v in s]))
        stage[k]["sub_batches"] = chunks / 3
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call("integrated")
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for kn in KERNELS:
            if kn in e.key:
                per[kn] = per.get(kn, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / 5
    integ_ms = sum(per.values())
    sub = int(round(W / stage["integrated"]["sub_batches"])) if stage["integrated"]["sub_batches"] else W
    nbytes = integration_bytes(W, m, max(sub, 1))
    step = min(ms["integrated"])
    for b in blks.values():
        b.close()
    return {"windows_per_step": W, "m": m, "snapshots": cfg["snapshots"], "ms_per_step": ms, "stage_ms": stage,
            "integ_ms": integ_ms, "integ_kernel_ms": per,
            "integ_share_of_step": integ_ms / step if step else None,
            "integ_share_of_cov_slot": integ_ms / stage["integrated"]["cov"] if stage["integrated"]["cov"] else None,
            "bytes": {"integration_per_step": nbytes, "integration_per_window": nbytes / W,
                      "covariance_input_per_window": 8 * cfg["snapshots"] * m},
            "integ_GBps": nbytes / (integ_ms * 1e-3) / 1e9 if integ_ms else None,
            "integ_share_of_hbm_peak": nbytes / (integ_ms * 1e-3) / HBM_PEAK if integ_ms else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--alpha", type=float, default=0.95)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    res = {"steps_per_round": args.steps, "rounds": args.rounds, "alpha": args.alpha, "card": card()}
    for c in (2, 3, 5):
        cfg, W = bench.workload(c)
        res["c%d" % c] = run(cfg, W, args, dev, stream)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
