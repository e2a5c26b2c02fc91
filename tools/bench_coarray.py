#!/usr/bin/env python
"""Cost of the co-array handle (music_b200_create_coarray, music_coarray.cuh) against plain handles.

  python tools/bench_coarray.py [--windows 100000] [--steps 3] [--rounds 2]

Shapes (N = 1024 snapshots per window, K = 3600, resident windows of complex Gaussian samples):
  mra4     {0, 1, 4, 6}, Mv = 7, n = 5
  nested6  {0, 1, 2, 3, 7, 11}, Mv = 12, n = 9
  nested8  {0, 1, 2, 3, 4, 9, 14, 19} truncated to Mv = 16, n = 12
For each shape, under the LOCAL_MAXIMA grid mode and under ESPRIT:
  coarray_wps        windows/s of process_device on the co-array handle (CUDA events on the launch stream, best of
                     `rounds` runs of `steps` calls, after a warm-up call);
  coarray_kernel_ms  coarray_kernel's time per call (torch.profiler, CUDA activities, a run of its own) and its share of
                     the call;
  bytes, fma         what coarray_kernel needs per call: m^2 + Mv^2 complex fp64 (16 bytes) per window; 4 Mv real FMA per
                     entry of the lower triangle of R_ss, Mv (Mv + 1) / 2 entries;
  hbm_bound_ms, fp64_bound_ms  bytes over 3.35 TB/s and fma over 64 DFMA / clock / SM at the card's maximum SM clock;
  plain_m_wps        the same call on a plain handle of the same m physical elements (n = m - 1; the grid mode only, the
                     sparse array is not a ULA);
  plain_ula_wps      a plain Mv-element ULA handle with n sources: what the full array would cost.
card: the card's name, power limit and maximum SM clock, read in the same run.  Prints one JSON line.
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

from gr_baz_b200.music_doa import music_doa  # noqa: E402
from gr_baz_b200.music_doa_coarray import music_doa_coarray  # noqa: E402

SHAPES = [("mra4", [0, 1, 4, 6], 7, 5), ("nested6", [0, 1, 2, 3, 7, 11], 12, 9),
          ("nested8", [0, 1, 2, 3, 4, 9, 14, 19], 16, 12)]
N, K, LAM = 1024, 3600, 1.0
STEP = (0.5, 0.0)
HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def sm_clock_hz(c):
    try:
        return float(c.split(",")[-1].strip().split()[0]) * 1e6
    except Exception:
        return None


def timed(f, args, stream):
    f()
    torch.cuda.synchronize()
    best = None
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            f()
        e1.record(stream)
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1) / args.steps
        best = t if best is None else min(best, t)
    return best


def call(blk, d_in, W, stream):
    ang = torch.empty((W, blk.n), dtype=torch.float32, device=d_in.device)
    lvl = torch.empty_like(ang)
    return lambda: blk.process_device(d_in.data_ptr(), W, ang.data_ptr(), lvl.data_ptr(), stream=stream.cuda_stream)


def kernel_ms(f, name, calls=3):
    """the summed device time of the kernels whose name holds `name`, per call (a profiled run of its own)"""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            f()
        torch.cuda.synchronize()
    total = 0.0
    for ev in prof.key_averages():
        if name in ev.key:
            total += getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
    return total / 1e3 / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    c = card()
    clock = sm_clock_hz(c)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    W = args.windows
    res = {"windows": W, "N": N, "K": K, "steps": args.steps, "rounds": args.rounds, "card": c}
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    for name, p, mv, n in SHAPES:
        m = len(p)
        d_in = torch.randn((W, m * N * 2), dtype=torch.float32, device=dev, generator=g)
        r = {"m": m, "mv": mv, "n": n}
        blk = music_doa_coarray(m, n, m * N, K, p, STEP, LAM, mv)
        plain = music_doa(m, m - 1, m * N, np.ones((K, m), np.complex64), K)
        plain.set_array_geometry([[q * STEP[0], q * STEP[1]] for q in p], LAM)
        plain.set_peak_mode("local_maxima")
        r["plain_m_wps"] = W / timed(call(plain, d_in, W, stream), args, stream) * 1e3
        plain.close()
        for mode in ("local_maxima", "esprit"):
            blk.set_peak_mode(mode)
            f = call(blk, d_in, W, stream)
            ms = timed(f, args, stream)
            kms = kernel_ms(f, "coarray_kernel")
            nbytes = 16.0 * (m * m + mv * mv) * W
            fma = 4.0 * mv * (mv * (mv + 1) / 2) * W
            hbm_ms = nbytes / HBM * 1e3
            fp64_ms = fma / (64.0 * sms * clock) * 1e3 if clock else None
            r[mode] = {"coarray_wps": W / ms * 1e3, "call_ms": ms, "coarray_kernel_ms": kms, "share_of_call": kms / ms,
                       "bytes": nbytes, "fma": fma, "hbm_bound_ms": hbm_ms, "fp64_bound_ms": fp64_ms,
                       "bound_share": max(hbm_ms, fp64_ms or 0.0) / kms if kms else None}
        blk.close()
        del d_in
        torch.cuda.empty_cache()
        # the full array: a plain Mv-element ULA with the same snapshots per window
        d_ula = torch.randn((W, mv * N * 2), dtype=torch.float32, device=dev, generator=g)
        ula = music_doa(mv, n, mv * N, np.ones((K, mv), np.complex64), K)
        ula.set_array_geometry([[l * STEP[0], l * STEP[1]] for l in range(mv)], LAM)
        for mode in ("local_maxima", "esprit"):
            ula.set_peak_mode(mode)
            r["plain_ula_%s_wps" % mode] = W / timed(call(ula, d_ula, W, stream), args, stream) * 1e3
        ula.close()
        del d_ula
        torch.cuda.empty_cache()
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
