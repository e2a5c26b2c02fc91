#!/usr/bin/env python
"""Cost and accuracy of the root-MUSIC peak mode (MUSIC_B200_PEAKS_ROOTS) against the grid peak paths.

  python tools/bench_roots.py [--steps 50] [--rounds 3]

C2 (M = 4 x-axis ULA, 4096 snapshots, K = 3600, n = 1) on bench.py's resident windows and table: TOP_BINS (the fused
kernel), ROOTS, ROOTS with the spectrum port, and LOCAL_MAXIMA + Newton refinement, timed alternately (`steps`
back-to-back process_device calls per handle per round, CUDA events on the launch stream).  A second row runs config 5's
shape (M = 16, n = 2) on an x-axis ULA with sources near 40 and 110 degrees, where ROOTS skips a 16-element scan:
LOCAL_MAXIMA against ROOTS.  Also reported:
  *_stage_ms       per-stage times (cov, eig, scan, top-n slot = the root kernel under ROOTS);
  *_roots_ms_per_10k  the root kernel's time per 10 000 windows;
  *_err_deg        RMS / max angle error against the synthetic truth (to the nearer of a source and its mirror image), over
                   the slots where every variant is within 1 degree, and how many slots were excluded;
  card             the card's name, power limit and maximum SM clock, read in the same run.
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

LAM = synth.C_LIGHT / synth.FREQUENCY


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def angle_error(deg, truth):
    """x-axis ULA: each slot against the nearest source or mirror image"""
    d = np.asarray(deg, np.float64)[:, :, None]
    t = np.asarray(truth, np.float64)[:, None, :]
    e = np.minimum(np.abs((d - t + 180.0) % 360.0 - 180.0), np.abs((d + t + 180.0) % 360.0 - 180.0))
    return e.min(axis=2)


def err_stats(errs):
    """RMS / max over the slots where every variant is within 1 degree (the rest: end-fire windows, counted)"""
    ok = np.all(np.stack([e < 1.0 for e in errs.values()]), axis=0)
    out = {k: [float(np.sqrt(np.mean(e[ok] ** 2))), float(e[ok].max())] for k, e in errs.items()}
    out["slots_excluded"] = int((~ok).sum())
    return out


def run(cfg, W, variants, args, dev, stream):
    """variants: name -> (peak mode, refine, spectrum).  Returns the result dict of one workload."""
    n, K, m = cfg["n"], cfg["resolution"], cfg["m"]
    seed = synth.BASE_SEED + cfg["id"]
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, seed, 0, W, dev, out=d_in)
    truth, _ = synth.window_params(cfg, seed, 0, W)
    table = bench.table_for(cfg)[1]
    pos = np.asarray([[synth.SPACING * x, synth.SPACING * y] for x, y in cfg["antenna_array"]], np.float64)
    blks, outs = {}, {}
    for k, (mode, refine, spectrum) in variants.items():
        b = music_doa(m, n, cfg["nsamples"], table, K)
        if mode != "top_bins" or refine:
            b.set_array_geometry(pos, LAM)
        b.set_peak_mode(mode, 0)
        b.set_refine(refine)
        blks[k] = b
        outs[k] = [torch.empty((W, n), dtype=torch.float32, device=dev), torch.empty((W, n), dtype=torch.float32, device=dev),
                   torch.empty((W, n), dtype=torch.int32, device=dev),
                   torch.empty((W, K), dtype=torch.float32, device=dev) if spectrum else None]

    def call(k):
        a, l, b, s = outs[k]
        blks[k].process_device(d_in.data_ptr(), W, a.data_ptr(), l.data_ptr(), None if s is None else s.data_ptr(), b.data_ptr(),
                               stream=stream.cuda_stream)

    def timed(k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            call(k)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for k in variants:
        for _ in range(5):
            call(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k in variants:
            ms[k].append(timed(k))
    err = err_stats({k: angle_error(outs[k][0].cpu().numpy(), truth) for k in variants})
    stage, per10k = {}, {}
    for k in variants:
        b = blks[k]
        b.set_stage_timing(True)
        for _ in range(5):
            call(k)
        torch.cuda.synchronize()
        s, _ = b.stage_times_ms()
        b.set_stage_timing(False)
        stage[k] = dict(zip(("cov", "eig", "scan", "topn_slot"), [v / 5 for v in s]))
        if variants[k][0] == "roots":
            per10k[k] = stage[k]["topn_slot"] * 1e4 / W
    for b in blks.values():
        b.close()
    return {"windows_per_step": W, "ms_per_step": ms, "stage_ms": stage, "roots_ms_per_10k": per10k, "err_deg": err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    res = {"steps_per_round": args.steps, "rounds": args.rounds}
    cfg, W = bench.workload(2)
    res["c2"] = run(cfg, W, {"top_bins": ("top_bins", False, False), "roots": ("roots", False, False),
                             "roots_spectrum": ("roots", False, True), "local_refine": ("local_maxima", True, False)},
                    args, dev, stream)
    torch.cuda.empty_cache()
    cfg16 = synth.config(5, geometry="ula_x", fixed_sources=(40.0, 110.0))
    W16 = bench.workload(5)[1]
    res["m16_ula_n2"] = run(cfg16, W16, {"local_maxima": ("local_maxima", False, False), "roots": ("roots", False, False)},
                            args, dev, stream)
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
