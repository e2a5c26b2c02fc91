#!/usr/bin/env python
"""Cost and coherent-source resolution of the DML peak mode (MUSIC_B200_PEAKS_DML) against the grid peak paths.

  python tools/bench_dml.py [--steps 20] [--rounds 3]

C2 (M = 4 x-axis ULA, 4096 snapshots, K = 3600, n = 1) on bench.py's resident windows and table: TOP_BINS (the fused
kernel), Bartlett TOP_BINS and DML, timed alternately (`steps` back-to-back process_device calls per handle per round,
CUDA events on the launch stream).  A second row runs config 5's shape (M = 16 UCA, n = 2, its two fixed sources):
LOCAL_MAXIMA, Bartlett and DML.  Also reported:
  *_stage_ms       per-stage times (cov, eig, scan, top-n slot = the DML kernel under DML);
  dml_sweeps       the AP sweep-count distribution of the oracle (tests/dml_oracle.py) on the first 200 windows' R;
  coherent_uca16   resolved windows (both sources within 2 degrees) of 500 windows of two coherent sources 20 degrees
                   apart at 20 dB on a UCA 16 (K = 360), DML against MUSIC LOCAL_MAXIMA;
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (the workload and table of bench.py, unchanged)
import dml_oracle as dm  # noqa: E402
import helpers  # noqa: E402
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa import music_doa  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def run(cfg, W, variants, args, dev, stream):
    """variants: name -> (peak mode, estimator).  Returns the result dict of one workload."""
    n, K, m = cfg["n"], cfg["resolution"], cfg["m"]
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg["id"], 0, W, dev, out=d_in)
    table = bench.table_for(cfg)[1]
    blks, outs = {}, {}
    for k, (mode, est) in variants.items():
        b = music_doa(m, n, cfg["nsamples"], table, K)
        b.set_estimator(est, 0.0)
        b.set_peak_mode(mode, 0)
        blks[k] = b
        outs[k] = [torch.empty((W, n), dtype=torch.float32, device=dev) for _ in range(2)] + [torch.empty((W, n), dtype=torch.int32, device=dev)]

    def call(k, R=None):
        a, l, b = outs[k]
        blks[k].process_device(d_in.data_ptr(), W, a.data_ptr(), l.data_ptr(), None, b.data_ptr(), stream=stream.cuda_stream,
                               d_R=None if R is None else R.data_ptr())

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
    Wr = 200
    R = torch.zeros((W, m, m, 2), dtype=torch.float64, device=dev)
    call("dml", R)
    torch.cuda.synchronize()
    Rn = R[:Wr].cpu().numpy()
    Rn = Rn[..., 0] + 1j * Rn[..., 1]
    tab = np.asarray(table, np.complex64).reshape(K, m)
    sweeps = [dm.work_R(Rn[w], tab, n)["sweeps"] for w in range(Wr)]
    for b in blks.values():
        b.close()
    return {"windows_per_step": W, "ms_per_step": ms, "stage_ms": stage,
            "dml_sweeps": {str(s): sweeps.count(s) for s in sorted(set(sweeps))}}


def coherent_uca16(dev):
    """resolved windows of a seeded coherent UCA 16 stream (two sources 20 degrees apart, 20 dB, 1024 snapshots)"""
    W, m, n, snaps = 500, 16, 2, helpers.SNAPS
    rng = np.random.default_rng(16)
    th = rng.uniform(0.0, 360.0, W)
    th = np.stack([th, (th + 20.0) % 360.0], axis=1)
    pos = helpers.array_wl("uca", m)
    tab = helpers.table_wl(pos)
    x = helpers.angle_windows(pos, th, True, W, 17)
    res = {}
    for mode in ("dml", "local_maxima"):
        b = music_doa(m, n, m * snaps, tab, tab.shape[0])
        b.set_peak_mode(mode, 0)
        ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
        b.work(W, [x], [ang, lvl])
        bins = b.last_bins()
        b.close()
        res[mode] = int(sum(helpers.resolved([a for a, k in zip(ang[w], bins[w]) if k >= 0], th[w]) for w in range(W)))
    res["windows"] = W
    return res


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
    cfg, W = bench.workload(2)
    res["c2"] = run(cfg, W, {"top_bins": ("top_bins", "music"), "bartlett": ("top_bins", "bartlett"), "dml": ("dml", "music")},
                    args, dev, stream)
    torch.cuda.empty_cache()
    cfg5, W5 = bench.workload(5)
    res["c5_shape"] = run(cfg5, W5, {"local_maxima": ("local_maxima", "music"), "bartlett": ("local_maxima", "bartlett"),
                                     "dml": ("dml", "music")}, args, dev, stream)
    torch.cuda.empty_cache()
    res["coherent_uca16"] = coherent_uca16(dev)
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
