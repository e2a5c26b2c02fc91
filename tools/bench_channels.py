#!/usr/bin/env python
"""Cost of the frequency-channelised modes (music_b200_create_channels) on the bench.py workloads.

  python tools/bench_channels.py [--steps 20] [--rounds 3] [--nfft 64]

For configs 2 (M = 4) and 5 (M = 16), on bench.py's resident windows (larger than L2), channel handles with C = 1, 8 and
64 channels of an nfft-point filter bank (Hann, SEPARATE) and a plain handle on the unfused path (it is asked for R) are
timed alternately in one session: back-to-back process_device calls per handle per round, CUDA events on the launch
stream.  Reported per handle:
  ms_per_step      every round's mean step time;
  stage_ms         per-stage times (cov slot = the filter bank, or the plain covariance kernel; eig slot; scan; top-n slot);
  cov_hbm_fraction the covariance slot against the HBM floor of reading the windows once and writing R (data-sheet
                   3.35 TB/s; a floor, not a rate that was reached);
  cov_fp64_fraction the same slot against the FP64 floor of its instruction count (FFT butterflies, taper, rank-one updates;
                   2 M^2 DFMA per snapshot for the plain kernel) at 64 FP64 instructions/clk/SM x SMs x the maximum SM clock;
  card             the card's name, power limit and maximum SM clock, read in the same run.
Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (the workload and table of bench.py, unchanged)
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa import music_doa  # noqa: E402
from gr_baz_b200.music_doa_channels import music_doa_channels  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
SAMPLE_RATE = 56e6
CHANNELS = (1, 8, 64)
SMEM_MAX = 232448


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


def batch_segments(M, F, J):
    """segments per batch of chan_cov_kernel (music_channels.cuh, chan_batch)"""
    return max(b for b in range(1, J + 1) if J % b == 0 and (b == 1 or b * F * M <= 2048))


def channel_groups(M, N, F, C):
    """passes over a window: the channel groups of chan_cov_kernel (music_channels.cuh, chan_group_size)"""
    B = batch_segments(M, F, N // F)
    fixed = 128 + 3 * B * F * M * 8 + B * M * (F + 1) * 16 + (F // 2) * 16 + F * 8 + 512
    cg = min(C, (SMEM_MAX - fixed) // (M * (M + 1) // 2 * 16))
    return (C + cg - 1) // cg


def filter_bank_fp64(M, N, F, C):
    """FP64 instructions per window of chan_cov_kernel: per pass 8 per radix-2 butterfly and 2 per sample for the taper,
    plus 4 DFMA per (segment, channel, Hermitian-half entry)"""
    J = N // F
    fft = J * M * ((F // 2) * int(math.log2(F)) * 8 + 2 * F)
    return channel_groups(M, N, F, C) * fft + J * C * (M * (M + 1) // 2) * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--nfft", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clk = max_sm_clock_hz()
    F = args.nfft
    res = {"rounds": args.rounds, "nfft": F, "taper": "hann", "combine": "separate"}
    for base in (2, 5):
        cfg, W = bench.workload(base)
        M, N, n, K = cfg["m"], cfg["snapshots"], cfg["n"], cfg["resolution"]
        d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
        synth.gen_windows_torch(cfg, synth.BASE_SEED + base, 0, W, dev, out=d_in)
        blks = {"plain": music_doa(M, n, cfg["nsamples"], bench.table_for(cfg)[1], K)}
        for C in CHANNELS:
            blks["C%d" % C] = music_doa_channels(M, n, cfg["nsamples"], K, F, ((F - C // 2) % F, C), "hann", "separate",
                                                 cfg["antenna_array"], synth.SPACING, synth.FREQUENCY, SAMPLE_RATE)
        rows = {k: (1 if k == "plain" else b.chan_count) for k, b in blks.items()}
        outs = {k: (torch.empty((r * W, n), dtype=torch.float32, device=dev), torch.empty((r * W, n), dtype=torch.int32, device=dev))
                for k, r in rows.items()}
        d_R = torch.empty((W, M, M, 2), dtype=torch.float64, device=dev)  # the plain handle: asks for R, so the unfused kernels

        def call(k):
            a, b = outs[k]
            if k == "plain":
                blks[k].process_device(d_in.data_ptr(), W, a.data_ptr(), None, None, b.data_ptr(), stream=stream.cuda_stream,
                                       d_R=d_R.data_ptr())
            else:
                blks[k].process_device(d_in.data_ptr(), W, a.data_ptr(), None, None, b.data_ptr(), stream=stream.cuda_stream)

        def timed(k, steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(steps):
                call(k)
            e1.record(stream)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / steps

        steps = {}
        for k in blks:
            call(k)
            call(k)
            torch.cuda.synchronize()
            steps[k] = max(2, min(args.steps, int(1500.0 / max(timed(k, 1), 1e-3))))  # about 1.5 s per round at most
        ms = {k: [] for k in blks}
        for _ in range(args.rounds):
            for k in blks:
                ms[k].append(timed(k, steps[k]))
        out = {"windows_per_step": W, "steps_per_round": steps, "ms_per_step": ms}
        for k, b in blks.items():
            b.set_stage_timing(True)
            for _ in range(3):
                call(k)
            torch.cuda.synchronize()
            s, _ = b.stage_times_ms()
            b.set_stage_timing(False)
            stage = dict(zip(("cov", "eig_slot", "scan", "topn_slot"), [v / 3 for v in s]))
            C = rows[k]
            hbm_ms = W * (N * M * 8 + C * M * M * 16) / HBM_BYTES_PER_S * 1e3
            ops = 2 * M * M * N if k == "plain" else filter_bank_fp64(M, N, F, C)
            fp64_ms = W * ops / (64.0 * sms * clk) * 1e3
            out[k] = {"stage_ms": stage, "cov_hbm_floor_ms": hbm_ms, "cov_fp64_floor_ms": fp64_ms, "fp64_instructions_per_window": ops,
                      "cov_hbm_fraction": hbm_ms / stage["cov"], "cov_fp64_fraction": fp64_ms / stage["cov"],
                      "channel_groups": 1 if k == "plain" else channel_groups(M, N, F, C)}
        res["c%d" % base] = out
        for b in blks.values():
            b.close()
        del d_in, d_R, outs
        torch.cuda.empty_cache()
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
