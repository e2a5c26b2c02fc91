"""Time the self-calibration solve (music_b200_calib_blind_solve) and the share of each of its kernels, at M = 4 / 8 / 16,
32 starts, 64 segments of one window (256 snapshots, one source each) and a 3600-row table.

The solve time is a host clock around the call, which ends in a device synchronise (median of --reps calls after one
warm-up).  The kernel shares come from torch.profiler in a separate run of one solve.  Prints one JSON line per M with
the GPU's name and power limit.  Usage: python tools/bench_calib_blind.py [--reps 5] [--out DIR]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gr_baz_b200.music_doa import music_doa  # noqa: E402

import helpers  # noqa: E402
from test_gpu_calibration import windows  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name(0) + ", unknown"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing measured")
    info = gpu_info()
    K, S, snaps, starts = 3600, 64, 256, 32
    for m in (4, 8, 16):
        pos = helpers.array_wl("uca", m)
        rng = np.random.default_rng(m)
        g = helpers.random_gains(rng, m)
        degs = [[360.0 * s / S + rng.uniform(0.0, 360.0 / S)] for s in range(S)]
        x = helpers.corrupt(windows(pos, degs, m + 1, snaps), g)
        blk = music_doa(m, 1, m * snaps, np.ones((K, m), np.complex64), K)
        blk.set_array_geometry(pos, helpers.LAM)
        blk.calib_blind_reset()
        blk.calib_blind_accumulate(x, 1)
        blk.calib_blind_solve(1, starts=starts)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            gains, _, st = blk.calib_blind_solve(1, starts=starts)
            ts.append(time.perf_counter() - t0)
        ref = g * (np.conj(g[0]) / abs(g[0]))
        phase_rms = float(math.degrees(math.sqrt(np.mean(np.angle(gains / ref) ** 2))))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            blk.calib_blind_solve(1, starts=starts)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                t = getattr(e, "device_time_total", None) or e.cuda_time_total
                kern[e.key.split("(")[0].split("<")[0].replace("void ", "").replace("music::", "")] = t
        tot = sum(kern.values()) or 1.0
        shares = {k: round(v / tot, 4) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
        forms = starts * S * K * 12 + S * K * 30  # scan rows of the 12 iterations and at most 30 polish iterations
        rec = {"m": m, "starts": starts, "segments": S, "rows": K, "solve_ms": round(1e3 * float(np.median(ts)), 3),
               "kernel_ms": round(tot / 1e3, 3), "kernel_share": shares, "quadratic_forms_upper_bound": forms,
               "misfit": st["misfit"], "polish": st["polish"], "phase_rms_deg": phase_rms, "gpu": info}
        print(json.dumps(rec))
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "bench_calib_blind_m%d.json" % m), "w") as f:
                json.dump(rec, f)
        blk.close()


if __name__ == "__main__":
    main()
