#!/usr/bin/env python
"""Cost of the angle tracker (music_b200_process_device_tracks, music_track.cuh) at bench.py's array shapes.

  python tools/bench_tracks.py [--windows 10000] [--steps 5] [--rounds 3]

At bench.py's C2, C3 and C5 shapes (M, snapshots and grid), on the device's geometric table, windows of 0, 1 and 4
sources (3 on the M = 4 array) moving slowly over 20 dB noise are run through one handle (local-maximum peaks with n = max(1, sources) slots, FIXED variance, 8 rows),
alternately timed (CUDA events, `steps` back-to-back calls per kind per round):
  unfused   process_device_ex with d_R: the unfused plan a tracks call also runs;
  tracks    process_device_tracks: the same plan plus track_kernel.
Plus the stress case: M = 16, noise only, n = 15 slots, 32 rows and a wide gate (ambiguous clusters in every window).
Reported per case: track_kernel's own time per call (torch.profiler), per 10 000 windows and per window, and its share
of the tracks call; the card's name, power limit and maximum SM clock, read in the same run.  Prints one JSON line.
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

import bench  # noqa: E402  (the shapes and tables of bench.py, unchanged)
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa import music_doa  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def windows(table, S, W, N, dev, seed):
    """complex64 [W][N * m] (interleaved snapshots) on the device: unit noise plus S sources of 20 dB, each moving by one
    table bin every 50 windows from its own start"""
    g = torch.Generator(device=dev).manual_seed(seed)
    K, m = table.shape
    X = torch.randn((W, N, m), generator=g, device=dev, dtype=torch.complex64)
    tab = torch.from_numpy(table).to(dev)
    w = torch.arange(W, device=dev)
    for s in range(S):
        bins = ((s * K) // max(S, 1) + K // 16 + w // 50) % K
        sig = 10.0 * torch.randn((W, N), generator=g, device=dev, dtype=torch.complex64)
        X += sig[:, :, None] * tab[bins][:, None, :]
    return torch.view_as_real(X.reshape(W, N * m)).reshape(W, N * m * 2).contiguous()


def run(cfg, S, W, args, dev, stream, n=None, rows=8, gate=16.0):
    m, N, K = cfg["m"], cfg["snapshots"], cfg["resolution"]
    n = n or max(1, S)
    table = bench.table_for(cfg)[1]
    pos = np.array([[synth.SPACING * x, synth.SPACING * y] for x, y in cfg["antenna_array"]])
    blk = music_doa(m, n, cfg["nsamples"], table, K)
    blk.set_array_geometry(pos, synth.C_LIGHT / synth.FREQUENCY)
    blk.set_peak_mode("local_maxima", 0)
    blk.set_tracking("fixed", q=1e-3, floor_deg=0.5, gate=gate, confirm_hits=2, confirm_window=3, max_misses=3, max_tracks=rows)
    d_in = windows(table, S, W, N, dev, 7 + S)
    t = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)
    ang, lvl, bins = t((W, n), torch.float32), t((W, n), torch.float32), t((W, n), torch.int32)
    R = t((W, m, m, 2), torch.float64)
    slot, ids, state = t((W, n), torch.int32), t((W, rows), torch.int32), t((W, rows, 3), torch.float32)
    calls = {
        "unfused": lambda: blk.process_device(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), None, bins.data_ptr(),
                                              stream=stream.cuda_stream, d_R=R.data_ptr()),
        "tracks": lambda: blk.process_device_tracks(d_in.data_ptr(), W, ang.data_ptr(), slot.data_ptr(), lvl.data_ptr(), None,
                                                    bins.data_ptr(), d_track_ids=ids.data_ptr(), d_track_state=state.data_ptr(),
                                                    stream=stream.cuda_stream),
    }

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            f()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for f in calls.values():
        for _ in range(2):
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in calls}
    for _ in range(args.rounds):
        for k, f in calls.items():
            ms[k].append(timed(f))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            calls["tracks"]()
        torch.cuda.synchronize()
    trk_ms = 0.0
    for e in prof.key_averages():
        if "track_kernel" in e.key:
            trk_ms += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / 3
    filled = float((slot >= 0).float().mean())
    confirmed = float((ids >= 0).sum(1).float().mean())
    blk.close()
    del d_in, R
    torch.cuda.empty_cache()
    step = min(ms["tracks"])
    return {"windows": W, "m": m, "n": n, "sources": S, "rows": rows, "ms_per_call": ms, "track_kernel_ms": trk_ms,
            "track_ms_per_10k_windows": trk_ms * 1e4 / W, "track_us_per_window": trk_ms * 1e3 / W,
            "track_share_of_call": trk_ms / step if step else None, "slots_with_a_track": filled,
            "confirmed_tracks_per_window": confirmed}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    res = {"steps_per_round": args.steps, "rounds": args.rounds, "card": card()}
    for c in (2, 3, 5):
        cfg, _ = bench.workload(c)
        for S in (0, 1, 4):
            res["c%d_s%d" % (c, S)] = run(cfg, min(S, cfg["m"] - 1), args.windows, args, dev, stream)
    cfg, _ = bench.workload(5)
    res["stress_c5_n15_t32"] = run(cfg, 0, args.windows, args, dev, stream, n=15, rows=32, gate=1e4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
