#!/usr/bin/env python
"""Cost and accuracy of the manifold-separation root-MUSIC peak mode (MUSIC_B200_PEAKS_MANIFOLD) against the grid peak
paths, on the uniform circular arrays of BASELINE configs 3 and 4 (UCA 8) and 5 (UCA 16).

  python tools/bench_manifold.py [--steps 20] [--rounds 3]

Per config shape, on bench.py's resident windows and table (K = 7200 / 3600 / 3600):
  ms_per_step      TOP_BINS (the path bench.py measures), LOCAL_MAXIMA (the unfused scan and peak kernel), MANIFOLD and
                   LOCAL_MAXIMA + NEWTON, timed alternately (`steps` back-to-back process_device calls per handle per
                   round, CUDA events on the launch stream);
  stage_ms         per-stage times (cov, eig, scan, top-n slot = the manifold kernel under MANIFOLD);
  us_per_10k       scan + peak pick (LOCAL_MAXIMA: scan and top-n slot) against the manifold kernel, per 10 000 windows;
  err_deg          at 0, 10 and 20 dB: RMS and max angle error of every slot against the nearest true source, and the
                   share of slots more than 1 degree off, for TOP_BINS, LOCAL_MAXIMA + NEWTON and MANIFOLD;
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
VARIANTS = {"top_bins": ("top_bins", False), "local_maxima": ("local_maxima", False), "manifold": ("manifold", False),
            "local_newton": ("local_maxima", True)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def slot_error(deg, truth):
    """each slot against the nearest true source (a UCA has no mirror image), degrees"""
    d = np.asarray(deg, np.float64)[:, :, None]
    t = np.asarray(truth, np.float64)[:, None, :]
    return np.abs((d - t + 180.0) % 360.0 - 180.0).min(axis=2)


class Handles:
    def __init__(self, cfg, dev):
        n, K, m = cfg["n"], cfg["resolution"], cfg["m"]
        table = bench.table_for(cfg)[1]
        pos = np.asarray([[synth.SPACING * x, synth.SPACING * y] for x, y in cfg["antenna_array"]], np.float64)
        self.cfg, self.dev, self.blks = cfg, dev, {}
        for k, (mode, refine) in VARIANTS.items():
            b = music_doa(m, n, cfg["nsamples"], table, K)
            if mode != "top_bins":
                b.set_array_geometry(pos, LAM)
            b.set_peak_mode(mode, 0)
            b.set_refine(refine)
            self.blks[k] = b

    def outputs(self, W):
        n = self.cfg["n"]
        return [torch.empty((W, n), dtype=torch.float32, device=self.dev), torch.empty((W, n), dtype=torch.float32, device=self.dev),
                torch.empty((W, n), dtype=torch.int32, device=self.dev)]

    def call(self, k, d_in, W, out, stream):
        a, l, b = out
        self.blks[k].process_device(d_in.data_ptr(), W, a.data_ptr(), l.data_ptr(), None, b.data_ptr(), stream=stream.cuda_stream)

    def close(self):
        for b in self.blks.values():
            b.close()


def timing(cfg_id, args, dev, stream):
    cfg, W = bench.workload(cfg_id)
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg_id, 0, W, dev, out=d_in)
    hs = Handles(cfg, dev)
    outs = {k: hs.outputs(W) for k in VARIANTS}

    def timed(k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            hs.call(k, d_in, W, outs[k], stream)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for k in VARIANTS:
        for _ in range(3):
            hs.call(k, d_in, W, outs[k], stream)
    torch.cuda.synchronize()
    ms = {k: [] for k in VARIANTS}
    for _ in range(args.rounds):
        for k in VARIANTS:
            ms[k].append(timed(k))
    stage = {}
    for k in ("local_maxima", "manifold"):
        b = hs.blks[k]
        b.set_stage_timing(True)
        for _ in range(5):
            hs.call(k, d_in, W, outs[k], stream)
        torch.cuda.synchronize()
        s, _ = b.stage_times_ms()
        b.set_stage_timing(False)
        stage[k] = dict(zip(("cov", "eig", "scan", "topn_slot"), [v / 5 for v in s]))
    hs.close()
    per10k = {"scan_plus_peaks": (stage["local_maxima"]["scan"] + stage["local_maxima"]["topn_slot"]) * 1e7 / W,
              "manifold_kernel": stage["manifold"]["topn_slot"] * 1e7 / W}
    return {"windows_per_step": W, "ms_per_step": ms, "stage_ms": stage, "us_per_10k": per10k}


def accuracy(cfg_id, W, dev, stream):
    res = {}
    for snr in (0.0, 10.0, 20.0):
        cfg = synth.config(cfg_id, snr_db=snr)
        seed = synth.BASE_SEED + 100 * cfg_id + int(snr)
        d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
        synth.gen_windows_torch(cfg, seed, 0, W, dev, out=d_in)
        truth, _ = synth.window_params(cfg, seed, 0, W)
        hs = Handles(cfg, dev)
        row = {}
        for k in ("top_bins", "local_newton", "manifold"):
            out = hs.outputs(W)
            hs.call(k, d_in, W, out, stream)
            torch.cuda.synchronize()
            e = slot_error(out[0].cpu().numpy(), truth)
            row[k] = {"rms": float(np.sqrt(np.mean(e ** 2))), "max": float(e.max()), "over_1deg": float(np.mean(e > 1.0))}
        hs.close()
        res["%d_dB" % int(snr)] = row
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--accuracy-windows", type=int, default=2048)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    res = {"steps_per_round": args.steps, "rounds": args.rounds}
    for cid in (3, 4, 5):
        res["c%d" % cid] = timing(cid, args, dev, stream)
        res["c%d" % cid]["err_deg"] = accuracy(cid, args.accuracy_windows, dev, stream)
        torch.cuda.empty_cache()
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
