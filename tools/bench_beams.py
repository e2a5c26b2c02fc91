#!/usr/bin/env python
"""Cost of the beamformed source signals (music_b200_process_device_beams) against the peak-only paths.

  python tools/bench_beams.py [--steps 20] [--rounds 3]

On bench.py's resident C2 (M = 4, 4096 snapshots, K = 3600, n = 1, 10 000 windows) and C5 (M = 16, n = 2, 4096
windows) windows and tables, each handle is timed alternately (`steps` back-to-back calls per handle per round, CUDA
events on the launch stream):
  plain        process_device (the fused kernel at C2);
  ex_R         process_device_ex with d_R (the unfused plan a beams call runs);
  das / mvdr / lcmv   process_device_beams with weights and beams.
Also reported:
  stage_ms     per-stage times (cov, eig, scan, top-n slot = peak rule + beam weights + beam apply under beams);
  apply        the beam_apply_kernel's own time per step (torch.profiler), its byte floor (input read + beams written)
               and the achieved bytes/s;
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

import torch  # noqa: E402

import bench  # noqa: E402  (the workload and table of bench.py, unchanged)
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa import music_doa  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def run(cfg, W, args, dev, stream):
    n, K, m, N = cfg["n"], cfg["resolution"], cfg["m"], cfg["snapshots"]
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg["id"], 0, W, dev, out=d_in)
    table = bench.table_for(cfg)[1]
    variants = {"plain": "off", "ex_R": "off", "das": "das", "mvdr": "mvdr", "lcmv": "lcmv"}
    blks = {}
    for k, rule in variants.items():
        b = music_doa(m, n, cfg["nsamples"], table, K)
        if n > 1:
            b.set_peak_mode("local_maxima", 0)
        b.set_beamformer(rule, 0.0)
        blks[k] = b
    ang = torch.empty((W, n), dtype=torch.float32, device=dev)
    lvl = torch.empty((W, n), dtype=torch.float32, device=dev)
    bins = torch.empty((W, n), dtype=torch.int32, device=dev)
    R = torch.empty((W, m, m, 2), dtype=torch.float64, device=dev)
    wts = torch.empty((W, n, m, 2), dtype=torch.float64, device=dev)
    beams = torch.empty((W, n, N, 2), dtype=torch.float32, device=dev)

    def call(k):
        b, s = blks[k], stream.cuda_stream
        if k == "plain":
            b.process_device(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), None, bins.data_ptr(), stream=s)
        elif k == "ex_R":
            b.process_device(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), None, bins.data_ptr(), stream=s, d_R=R.data_ptr())
        else:
            b.process_device_beams(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), None, bins.data_ptr(), None, wts.data_ptr(),
                                   beams.data_ptr(), stream=s)

    def timed(k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            call(k)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for k in variants:
        for _ in range(3):
            call(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k in variants:
            ms[k].append(timed(k))
    stage = {}
    for k in variants:
        b = blks[k]
        b.set_stage_timing(True)
        for _ in range(3):
            call(k)
        torch.cuda.synchronize()
        s, _ = b.stage_times_ms()
        b.set_stage_timing(False)
        stage[k] = dict(zip(("cov", "eig", "scan", "topn_slot"), [v / 3 for v in s]))
    # the apply kernel on its own: kernel time from the profiler over a few beams calls
    apply_ms = {}
    for k in ("das", "mvdr", "lcmv"):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                call(k)
            torch.cuda.synchronize()
        tot = {}
        for e in prof.key_averages():
            for name in ("beam_weights_kernel", "beam_apply_kernel"):
                if name in e.key:
                    tot[name] = tot.get(name, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / 5
        apply_ms[k] = tot
    for b in blks.values():
        b.close()
    bytes_floor = W * N * m * 8 + W * n * N * 8
    ap = [v.get("beam_apply_kernel", 0.0) for v in apply_ms.values()]
    best = min(ap) if ap and min(ap) > 0 else None
    return {"windows_per_step": W, "ms_per_step": ms, "stage_ms": stage, "beam_kernels_ms": apply_ms,
            "apply_byte_floor_GB": bytes_floor / 1e9,
            "apply_achieved_TBps": None if best is None else bytes_floor / (best * 1e-3) / 1e12}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    res = {"steps_per_round": args.steps, "rounds": args.rounds}
    for c in (2, 5):
        cfg, W = bench.workload(c)
        res["c%d" % c] = run(cfg, W, args, dev, stream)
        torch.cuda.empty_cache()
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
