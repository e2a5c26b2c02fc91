#!/usr/bin/env python
"""Cost of the per-window source count (music_b200_set_source_rule) on the bench.py workload of one BASELINE config.

  python tools/bench_source_count.py [--config 2] [--rule mdl] [--steps 50] [--rounds 3]

Two handles on the same resident windows: the default rule (FIXED) and the chosen rule through
music_b200_process_device_counts.  Each round times `steps` back-to-back calls of one handle and then of the other
(CUDA events on the launch stream), alternating, so that both see the same clocks.  Prints one JSON line: both step
times per round, the fraction of windows whose count equals the synthetic source count, whether the bins equal the
default rule's where the count is n, the stage times of the unfused path with and without the count kernel (the count
kernel runs inside the eig slot), and the card's name and power limit read in the same run.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--rule", default="mdl", choices=["mdl", "aic"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    cfg, W = bench.workload(args.config)
    resp, _ = bench.table_for(cfg)
    n, K, M = cfg["n"], cfg["resolution"], cfg["m"]
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, synth.BASE_SEED + args.config, 0, W, dev, out=d_in)
    stream = torch.cuda.current_stream()
    out = {k: (torch.empty((W, n), dtype=torch.float32, device=dev), torch.empty((W, n), dtype=torch.float32, device=dev),
               torch.empty((W, n), dtype=torch.int32, device=dev)) for k in ("fixed", "rule")}
    d_cnt = torch.empty((W,), dtype=torch.int32, device=dev)
    blk = {"fixed": music_doa(M, n, cfg["nsamples"], resp, K), "rule": music_doa(M, n, cfg["nsamples"], resp, K)}
    blk["rule"].set_source_rule(args.rule)

    def call(k):
        a, l, b = out[k]
        blk[k].process_device(d_in.data_ptr(), W, a.data_ptr(), l.data_ptr(), None, b.data_ptr(), stream=stream.cuda_stream,
                              d_counts=d_cnt.data_ptr() if k == "rule" else None)

    def timed(k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            call(k)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for k in ("fixed", "rule"):
        for _ in range(5):
            call(k)
    torch.cuda.synchronize()
    ms = {"fixed": [], "rule": []}
    for _ in range(args.rounds):
        for k in ("fixed", "rule"):
            ms[k].append(timed(k))

    counts = d_cnt.cpu().numpy()
    true_count = len(cfg["fixed_sources"]) if cfg.get("fixed_sources") else n
    full = torch.from_numpy(counts == n).to(dev)
    bins_equal = bool(torch.equal(out["rule"][2][full], out["fixed"][2][full]))

    def stages(b, reps=5):
        b.set_stage_timing(True)
        for _ in range(reps):
            b.process_device(d_in.data_ptr(), W, out["rule"][0].data_ptr(), None, None, out["rule"][2].data_ptr(), stream=stream.cuda_stream)
        torch.cuda.synchronize()
        s, _ = b.stage_times_ms()
        b.set_stage_timing(False)
        return [v / reps for v in s]

    # the unfused path of the default rule (what the rule runs, minus the count kernel)
    old = os.environ.get("MUSIC_B200_FUSED")
    os.environ["MUSIC_B200_FUSED"] = "0"
    unfused = music_doa(M, n, cfg["nsamples"], resp, K)
    if old is None:
        del os.environ["MUSIC_B200_FUSED"]
    else:
        os.environ["MUSIC_B200_FUSED"] = old
    s_fixed = stages(unfused)
    s_rule = stages(blk["rule"])
    unfused.close()
    for b in blk.values():
        b.close()
    print(json.dumps({
        "config": args.config, "rule": args.rule, "windows_per_step": W, "steps_per_round": args.steps,
        "default_rule_ms_per_step": ms["fixed"], "rule_ms_per_step": ms["rule"],
        "rule_windows_per_s": W / (min(ms["rule"]) * 1e-3),
        "fraction_count_equals_true_sources": float(np.mean(counts == true_count)), "true_sources": true_count,
        "windows_with_count_n": int(full.sum().item()), "bins_equal_default_rule_where_count_is_n": bins_equal,
        "stage_ms_unfused_fixed": dict(zip(("cov", "eig", "scan", "topn"), s_fixed)),
        "stage_ms_rule": dict(zip(("cov", "eig_and_count", "scan", "topn"), s_rule)),
        "card": card()}))


if __name__ == "__main__":
    main()
