#!/usr/bin/env python
"""Cost and accuracy of the MVDR and Bartlett spectra (music_b200_set_estimator) against MUSIC on the bench.py workloads.

  python tools/bench_estimators.py [--steps 50] [--rounds 3]

For configs 2 (M = 4, n = 1) and 5 (M = 16, n = 2), on bench.py's resident windows and table, a MUSIC handle (the
default path), an MVDR handle (loading 0) and a Bartlett handle are timed alternately: `steps` back-to-back
process_device calls per handle per round, CUDA events on the launch stream.  Also reported:
  *_stage_ms   per-stage times (cov, eig slot = eigensolver or MVDR preparation, scan, top-n slot);
  *_scan_floor the quadratic-form scan's FP64 floor from its DFMA count per (window, bin) at 64 DFMA/clk/SM x SMs x the
               maximum SM clock, and the fraction of it the measured scan stage achieves;
  *_err_deg    RMS / max angle error against the synthetic truth, over the slots where every estimator is within 1 degree
               (x-axis ULA: to the nearer of a source and its mirror image), and how many slots were excluded;
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

KINDS = ("music", "mvdr", "bartlett")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def max_sm_clock_hz():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out) * 1e6
    except Exception:
        return 1.98e9


def angle_error(deg, truth, geometry):
    d = np.asarray(deg, np.float64)[:, :, None]
    t = np.asarray(truth, np.float64)[:, None, :]
    e = np.abs((d - t + 180.0) % 360.0 - 180.0)
    if geometry == "ula_x":
        e = np.minimum(e, np.abs((d + t + 180.0) % 360.0 - 180.0))
    return e.min(axis=2)


def err_stats(errs):
    ok = np.all(np.stack([e < 1.0 for e in errs.values()]), axis=0)
    out = {k: [float(np.sqrt(np.mean(e[ok] ** 2))), float(e[ok].max())] for k, e in errs.items()}
    out["slots_excluded"] = int((~ok).sum())
    return out


def quad_dfma(kind, M):
    """DFMA per (window, bin) of the quadratic-form scan (music_estimators.cuh)"""
    if kind == "mvdr":
        return 2 * M * (M + 1) + 2 * M
    return 2 * M * (M - 1) + 5 * M


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clk = max_sm_clock_hz()
    res = {"steps_per_round": args.steps, "rounds": args.rounds}
    for base in (2, 5):
        cfg, W = bench.workload(base)
        n, K = cfg["n"], cfg["resolution"]
        seed = synth.BASE_SEED + base
        d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
        synth.gen_windows_torch(cfg, seed, 0, W, dev, out=d_in)
        truth, _ = synth.window_params(cfg, seed, 0, W)
        table = bench.table_for(cfg)[1]
        blks = {}
        for k in KINDS:
            blks[k] = music_doa(cfg["m"], n, cfg["nsamples"], table, K)
            blks[k].set_estimator(k)
        outs = {k: (torch.empty((W, n), dtype=torch.float32, device=dev), torch.empty((W, n), dtype=torch.float32, device=dev),
                    torch.empty((W, n), dtype=torch.int32, device=dev)) for k in KINDS}

        def call(k):
            a, l, b = outs[k]
            blks[k].process_device(d_in.data_ptr(), W, a.data_ptr(), l.data_ptr(), None, b.data_ptr(), stream=stream.cuda_stream)

        def timed(k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                call(k)
            e1.record(stream)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.steps

        for k in KINDS:
            for _ in range(5):
                call(k)
        torch.cuda.synchronize()
        ms = {k: [] for k in KINDS}
        for _ in range(args.rounds):
            for k in KINDS:
                ms[k].append(timed(k))
        o = {k: [t.cpu().numpy() for t in v] for k, v in outs.items()}
        stage = {}
        for k in KINDS:
            b = blks[k]
            b.set_stage_timing(True)
            for _ in range(5):
                call(k)
            torch.cuda.synchronize()
            s, _ = b.stage_times_ms()
            b.set_stage_timing(False)
            stage[k] = dict(zip(("cov", "eig_slot", "scan", "topn_slot"), [v / 5 for v in s]))
        floor = {}
        for k in ("mvdr", "bartlett"):
            f_ms = quad_dfma(k, cfg["m"]) * W * K / (64.0 * sms * clk) * 1e3
            floor[k] = {"dfma_per_window_bin": quad_dfma(k, cfg["m"]), "floor_ms": f_ms,
                        "achieved_fraction": f_ms / stage[k]["scan"] if stage[k]["scan"] > 0 else None}
        res["c%d" % base] = {"windows_per_step": W, "ms_per_step": ms,
                             "err_deg": err_stats({k: angle_error(o[k][0], truth, cfg["geometry"]) for k in KINDS})}
        res["c%d_stage_ms" % base] = stage
        res["c%d_scan_floor" % base] = floor
        for b in blks.values():
            b.close()
        del d_in
        torch.cuda.empty_cache()
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
