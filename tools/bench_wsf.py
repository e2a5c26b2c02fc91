#!/usr/bin/env python
"""Cost of the WSF peak mode and the JOINT refinement (music_wsf.cuh) on bench.py's workloads.

  python tools/bench_wsf.py [--steps 20] [--rounds 3]

On bench.py's resident C2 (M = 4, n = 1, 4096 snapshots, K = 3600), C3 (M = 8, n = 1, 8192 snapshots, K = 7200) and C5
(M = 16, n = 2, 4096 snapshots, K = 3600) windows and tables, with a geometric table installed, three calls on one handle
are timed alternately (`steps` back-to-back process_device calls per kind per round, CUDA events on the launch stream):
  dml        the DML peak mode, refinement off;
  wsf        the WSF peak mode, refinement off;
  wsf_joint  the WSF peak mode with JOINT.
Also reported:
  stage_ms            per-stage times of each call (cov, eig, scan, top-n): wsf_x_kernel is timed in the eigensolver
                      slot, joint_kernel in the top-n slot;
  x_ms, joint_ms      the two kernels' own times per step (torch.profiler, in a run of their own) and their shares of
                      the wsf_joint step;
  card                the card's name, power limit and maximum SM clock, read in the same run.
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

KINDS = {"dml": ("dml", "off"), "wsf": ("wsf", "off"), "wsf_joint": ("wsf", "joint")}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def run(cfg, W, args, dev, stream):
    n, K, m = cfg["n"], cfg["resolution"], cfg["m"]
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg["id"], 0, W, dev, out=d_in)
    pos = np.array([[synth.SPACING * x, synth.SPACING * y] for x, y in cfg["antenna_array"]])
    lam = synth.C_LIGHT / synth.FREQUENCY
    blk = music_doa(m, n, cfg["nsamples"], bench.table_for(cfg)[1], K)
    blk.set_array_geometry(pos, lam)
    ang = torch.empty((W, n), dtype=torch.float32, device=dev)
    lvl = torch.empty_like(ang)
    bins = torch.empty((W, n), dtype=torch.int32, device=dev)

    def call(kind):
        mode, refine = KINDS[kind]
        blk.set_refine("off")
        blk.set_peak_mode(mode, 0)
        blk.set_refine(refine)
        return lambda: blk.process_device(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), None, bins.data_ptr(),
                                          stream=stream.cuda_stream)

    def timed(kind):
        f = call(kind)
        f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            f()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for k in KINDS:
        f = call(k)
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in KINDS}
    for _ in range(args.rounds):
        for k in KINDS:
            ms[k].append(timed(k))
    stage = {}
    for k in KINDS:
        f = call(k)
        blk.set_stage_timing(True)
        for _ in range(3):
            f()
        torch.cuda.synchronize()
        s, _ = blk.stage_times_ms()
        blk.set_stage_timing(False)
        stage[k] = dict(zip(("cov", "eig", "scan", "topn"), [v / 3 for v in s]))
    f = call("wsf_joint")
    f()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            f()
        torch.cuda.synchronize()
    kern = {"wsf_x_kernel": 0.0, "joint_kernel": 0.0}
    for e in prof.key_averages():
        for name in kern:
            if name in e.key:
                kern[name] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / 5
    filled = float((bins >= 0).float().mean())
    blk.close()
    step = min(ms["wsf_joint"])
    return {"windows_per_step": W, "m": m, "n": n, "snapshots": cfg["snapshots"], "ms_per_step": ms, "stage_ms": stage,
            "x_ms": kern["wsf_x_kernel"], "joint_ms": kern["joint_kernel"],
            "x_share_of_step": kern["wsf_x_kernel"] / step if step else None,
            "joint_share_of_step": kern["joint_kernel"] / step if step else None, "filled_share": filled}


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
    for c in (2, 3, 5):
        cfg, W = bench.workload(c)
        res["c%d" % c] = run(cfg, W, args, dev, stream)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
