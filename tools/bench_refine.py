#!/usr/bin/env python
"""Cost and accuracy of the off-grid peak refinement (music_b200_set_refine) on the bench.py workloads.

  python tools/bench_refine.py [--steps 50] [--rounds 3]

Every comparison times two handles on the same resident windows (bench.py's windows and seeds for configs 2 and 5),
`steps` back-to-back process_device calls of one and then of the other per round (CUDA events on the launch stream),
alternating, so that both see the same clocks:
  c2_off_vs_on        config 2 (M = 4, K = 3600): refinement off (the fused kernel) against on;
  c2_k360_vs_k3600    config 2's windows at K = 360 with refinement against K = 3600 without it, with the RMS / max
                      angle error of each against the synthetic truth (synth.window_params; on the x-axis ULA a source
                      and its mirror image are one direction, so the error is to the nearer of the two; slots where
                      a handle peaks on the wrong end-fire lobe are counted rather than averaged, see err_stats);
  c5_off_vs_on        config 5 (M = 16, n = 2), both with the local-maxima peak rule, off against on;
plus the per-stage times (stage_times_ms: cov, eig, scan, top-n slot, the refine kernel runs in the last) of the
refining handles and of their unfused counterparts, and the card's name and power limit read in the same run.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def angle_error(deg, truth, geometry):
    """(W, n) reported angles against (W, S) true angles: per slot, the distance to the nearest true source"""
    d = np.asarray(deg, np.float64)[:, :, None]
    t = np.asarray(truth, np.float64)[:, None, :]
    e = np.abs((d - t + 180.0) % 360.0 - 180.0)
    if geometry == "ula_x":
        e = np.minimum(e, np.abs((d + t + 180.0) % 360.0 - 180.0))
    return e.min(axis=2)


def err_stats(errs):
    """name -> per-slot errors: RMS and max of each over the slots where every handle is within 1 degree of the truth.
    At half-wavelength spacing a ULA's two end-fire directions (0 and 180 degrees) have nearly one steering vector, so a
    few windows near end-fire peak on the wrong side whatever the grid; those are counted, not averaged in."""
    ok = np.all(np.stack([e < 1.0 for e in errs.values()]), axis=0)
    out = {k: [float(np.sqrt(np.mean(e[ok] ** 2))), float(e[ok].max())] for k, e in errs.items()}
    out["slots_off_lobe_excluded"] = int((~ok).sum())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    lam = synth.C_LIGHT / synth.FREQUENCY

    def make(cfg, K, refine, local=False, fused=True):
        old = os.environ.get("MUSIC_B200_FUSED")
        if not fused:
            os.environ["MUSIC_B200_FUSED"] = "0"
        try:
            b = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], np.ones((K, cfg["m"]), np.complex64), K)
        finally:
            if not fused:
                if old is None:
                    del os.environ["MUSIC_B200_FUSED"]
                else:
                    os.environ["MUSIC_B200_FUSED"] = old
        b.set_array_geometry([[synth.SPACING * x, synth.SPACING * y] for x, y in cfg["antenna_array"]], lam)
        if local:
            b.set_peak_mode("local_maxima", 3)
        if refine:
            b.set_refine(True)
        return b

    def compare(d_in, W, n, blks):
        outs = {k: (torch.empty((W, n), dtype=torch.float32, device=dev), torch.empty((W, n), dtype=torch.float32, device=dev),
                    torch.empty((W, n), dtype=torch.int32, device=dev)) for k in blks}

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

        for k in blks:
            for _ in range(5):
                call(k)
        torch.cuda.synchronize()
        ms = {k: [] for k in blks}
        for _ in range(args.rounds):
            for k in blks:
                ms[k].append(timed(k))
        return ms, {k: [t.cpu().numpy() for t in v] for k, v in outs.items()}

    def stages(b, d_in, W, n, reps=5):
        a = torch.empty((W, n), dtype=torch.float32, device=dev)
        bb = torch.empty((W, n), dtype=torch.int32, device=dev)
        b.set_stage_timing(True)
        for _ in range(reps):
            b.process_device(d_in.data_ptr(), W, a.data_ptr(), None, None, bb.data_ptr(), stream=stream.cuda_stream)
        torch.cuda.synchronize()
        s, _ = b.stage_times_ms()
        b.set_stage_timing(False)
        return dict(zip(("cov", "eig", "scan", "topn_slot"), [v / reps for v in s]))

    res = {"steps_per_round": args.steps}
    # ---- config 2 ------------------------------------------------------------------------------------------------
    cfg, W = bench.workload(2)
    seed = synth.BASE_SEED + 2
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, seed, 0, W, dev, out=d_in)
    truth, _ = synth.window_params(cfg, seed, 0, W)
    blks = {"off": make(cfg, 3600, False), "on": make(cfg, 3600, True)}
    ms, o = compare(d_in, W, 1, blks)
    res["c2_off_vs_on"] = {"windows_per_step": W, "off_fused_ms_per_step": ms["off"], "on_ms_per_step": ms["on"],
                           "bins_equal": bool(np.array_equal(o["off"][2], o["on"][2])),
                           "err_deg_rms_max": err_stats({k: angle_error(o[k][0], truth, cfg["geometry"]) for k in blks})}
    unfused = make(cfg, 3600, False, fused=False)
    res["c2_stage_ms"] = {"unfused_off": stages(unfused, d_in, W, 1), "on": stages(blks["on"], d_in, W, 1)}
    unfused.close()
    for b in blks.values():
        b.close()
    blks = {"k3600_off": make(cfg, 3600, False), "k360_on": make(cfg, 360, True)}
    ms, o = compare(d_in, W, 1, blks)
    res["c2_k360_vs_k3600"] = {"k3600_off_ms_per_step": ms["k3600_off"], "k360_on_ms_per_step": ms["k360_on"],
                               "err_deg_rms_max": err_stats({k: angle_error(o[k][0], truth, cfg["geometry"]) for k in blks})}
    res["c2_stage_ms"]["k360_on"] = stages(blks["k360_on"], d_in, W, 1)
    for b in blks.values():
        b.close()
    del d_in
    torch.cuda.empty_cache()
    # ---- config 5 ------------------------------------------------------------------------------------------------
    cfg, W = bench.workload(5)
    seed = synth.BASE_SEED + 5
    d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
    synth.gen_windows_torch(cfg, seed, 0, W, dev, out=d_in)
    truth, _ = synth.window_params(cfg, seed, 0, W)
    blks = {"off": make(cfg, 3600, False, local=True), "on": make(cfg, 3600, True, local=True)}
    ms, o = compare(d_in, W, 2, blks)
    res["c5_local_maxima_off_vs_on"] = {
        "windows_per_step": W, "off_ms_per_step": ms["off"], "on_ms_per_step": ms["on"],
        "bins_equal": bool(np.array_equal(o["off"][2], o["on"][2])),
        "err_deg_rms_max": err_stats({k: angle_error(o[k][0], truth, cfg["geometry"]) for k in blks})}
    res["c5_stage_ms"] = {"off": stages(blks["off"], d_in, W, 2), "on": stages(blks["on"], d_in, W, 2)}
    for b in blks.values():
        b.close()
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
