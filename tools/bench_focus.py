#!/usr/bin/env python
"""Cost of the COHERENT combine of a channel handle (focusing, music_focus.cuh) against the INCOHERENT one on the bench.py
workloads.

  python tools/bench_focus.py [--steps 20] [--rounds 3] [--nfft 64]

For configs 2 (M = 4) and 5 (M = 16), on bench.py's resident windows (larger than L2), channel handles with C = 1, 8 and
64 channels of an nfft-point filter bank (Hann), INCOHERENT and COHERENT, are timed alternately in one session:
back-to-back process_device calls per handle per round, CUDA events on the launch stream.  Reported per handle:
  ms_per_step       every round's mean step time;
  stage_ms          per-stage times (cov slot = the filter bank, and under COHERENT the focus kernel; eig slot; scan;
                    top-n slot);
  coherent only:
  focus_ms          chan_focus_kernel's own time per call and chan_cov_kernel's, from torch.profiler's CUDA activity
                    (CUPTI kernel records) in a separate pass; the profiler is off while the steps are timed.  The kernel is
                    enqueued inside the library call, so no CUDA event can sit right around it from here, and the
                    difference of two handles' cov slots does not isolate it: a COHERENT handle runs larger sub-batches,
                    so its chan_cov_kernel launches differ from an INCOHERENT handle's;
  focus_fp64_floor_ms  its DFMA count (4 M^3 for Y = R T^H plus 4 M m(m+1)/2 for the upper half of T Y, per window and
                    channel other than the reference) at 64 FP64 instructions/clk/SM x SMs x the maximum SM clock;
  focus_hbm_floor_ms   reading the C R_c and writing R_foc once at the data-sheet 3.35 TB/s (floors, not rates that were
                    reached);
  setup_ms          a retune, set_array_geometry() on the host clock: C table builds, the B_c accumulation, the polar factors and
                    the errors (the whole grid);
  card              the card's name, power limit and maximum SM clock, read in the same run.
Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (the workload of bench.py, unchanged)
from bench_channels import HBM_BYTES_PER_S, SAMPLE_RATE, card, max_sm_clock_hz  # noqa: E402
from gr_baz_b200 import synth  # noqa: E402
from gr_baz_b200.music_doa_channels import music_doa_channels  # noqa: E402

CHANNELS = (1, 8, 64)


def focus_dfma(M, C):
    """DFMA per window of chan_focus_kernel"""
    return (C - 1) * (4 * M ** 3 + 4 * M * (M * (M + 1) // 2))


def kernel_ms(call, names, calls=3):
    """device time per call of the kernels whose names contain each of `names`, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            call()
        torch.cuda.synchronize()
    out = {}
    for name in names:
        us = 0.0
        for e in prof.key_averages():
            if name in e.key:
                us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        out[name] = us / 1e3 / calls
    return out


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
    res = {"rounds": args.rounds, "nfft": F, "taper": "hann"}
    for base in (2, 5):
        cfg, W = bench.workload(base)
        M, n, K = cfg["m"], cfg["n"], cfg["resolution"]
        d_in = torch.empty((W, cfg["nsamples"] * 2), dtype=torch.float32, device=dev)
        synth.gen_windows_torch(cfg, synth.BASE_SEED + base, 0, W, dev, out=d_in)
        blks, setup = {}, {}
        for C in CHANNELS:
            for combine in ("incoherent", "coherent"):
                blks["%s_C%d" % (combine, C)] = music_doa_channels(M, n, cfg["nsamples"], K, F, ((F - C // 2) % F, C), "hann", combine,
                                                                   cfg["antenna_array"], synth.SPACING, synth.FREQUENCY, SAMPLE_RATE)
                if combine == "coherent":
                    b = blks["coherent_C%d" % C]
                    t0 = time.perf_counter()
                    b.set_array_geometry(np.asarray(cfg["antenna_array"], dtype=np.float64) * synth.SPACING, synth.FREQUENCY, SAMPLE_RATE)
                    setup["coherent_C%d" % C] = (time.perf_counter() - t0) * 1e3
        outs = {k: (torch.empty((W, n), dtype=torch.float32, device=dev), torch.empty((W, n), dtype=torch.int32, device=dev)) for k in blks}

        def call(k):
            a, b = outs[k]
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
            for C in CHANNELS:  # INCOHERENT and COHERENT of one C back to back
                for combine in ("incoherent", "coherent"):
                    k = "%s_C%d" % (combine, C)
                    ms[k].append(timed(k, steps[k]))
        out = {"windows_per_step": W, "steps_per_round": steps, "ms_per_step": ms}
        for k, b in blks.items():
            b.set_stage_timing(True)
            for _ in range(3):
                call(k)
            torch.cuda.synchronize()
            s, _ = b.stage_times_ms()
            b.set_stage_timing(False)
            out[k] = {"stage_ms": dict(zip(("cov", "eig_slot", "scan", "topn_slot"), [v / 3 for v in s]))}
            if k.startswith("coherent"):
                C = b.chan_count
                kt = kernel_ms(lambda: call(k), ("chan_focus_kernel", "chan_cov_kernel"))
                fp64_ms = W * focus_dfma(M, C) / (64.0 * sms * clk) * 1e3
                hbm_ms = W * (C + 1) * M * M * 16 / HBM_BYTES_PER_S * 1e3
                out[k].update({"focus_ms": kt["chan_focus_kernel"], "chan_cov_ms": kt["chan_cov_kernel"],
                               "focus_share_of_chan_cov": kt["chan_focus_kernel"] / kt["chan_cov_kernel"] if kt["chan_cov_kernel"] else None,
                               "focus_fp64_floor_ms": fp64_ms, "focus_hbm_floor_ms": hbm_ms, "setup_ms": setup[k]})
        res["c%d" % base] = out
        for b in blks.values():
            b.close()
        del d_in, outs
        torch.cuda.empty_cache()
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
