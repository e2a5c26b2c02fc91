#!/usr/bin/env python
"""Cost and accuracy of 2-D ESPRIT on az-el handles (MUSIC_B200_PEAKS_ESPRIT on a planar lattice) against the grid
peak paths of the same handle kind.

  python tools/bench_esprit2d.py [--windows 2000] [--steps 10] [--rounds 3]

Shapes: a 4 x 4 URA with n = 2 and a 2 x 4 URA with n = 1, half-wavelength steps, N = 4096 snapshots, a 360 x 91 grid
over el [0, 90], sources of unit power at random (az, el in [5, 85]) with white noise at 20 dB per element, generated
on the device.  Per shape:
  ms_per_step    ESPRIT, TOP_BINS, LOCAL_MAXIMA and LOCAL_MAXIMA + NEWTON on the same resident windows, timed alternately
                 (`steps` back-to-back process_device calls per handle per round, CUDA events on the launch stream);
  ms_per_10k     the same per 10 000 windows (median round);
  stage_ms       per-stage times per step (cov, eig, scan, top-n slot = the ESPRIT kernel under ESPRIT, the peak pick
                 + decode (+ refinement) otherwise);
  esprit_kernel_ms_per_10k   the ESPRIT kernel's own time (its top-n slot);
  rms_deg        RMS great-circle error of every true source against its nearest unused report;
  card           the card's name, power limit and maximum SM clock, read in the same run.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import azel_oracle as ao  # noqa: E402
import esprit2d_oracle as eo  # noqa: E402
from gr_baz_b200.music_doa_azel import music_doa_azel  # noqa: E402

LAM = 0.5
N = 4096
GRID = ao.Grid(360, 91, 0.0, 90.0)
VARIANTS = {"esprit": ("esprit", False), "top_bins": ("top_bins", False), "local_maxima": ("local_maxima", False),
            "local_newton": ("local_maxima", True)}
SHAPES = {"ura4x4_n2": (4, 4, 2), "ura2x4_n1": (2, 4, 1)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing does not depend on it
        out = "nvidia-smi unavailable (%s)" % e
    return out or torch.cuda.get_device_name(0)


def windows(pos, n, W, seed, dev, noise=0.1):
    """complex64 windows [W][N * M] (x(r, c) = in[c M + r]) on the device and the true (az, el) per window"""
    g = torch.Generator(device=dev).manual_seed(seed)
    rng = np.random.default_rng(seed)
    M = pos.shape[0]
    truth = [[(rng.uniform(0.0, 360.0), rng.uniform(5.0, 85.0)) for _ in range(n)] for _ in range(W)]
    A = torch.tensor(np.array([[ao.steering(pos, LAM, az, el) for az, el in t] for t in truth]), dtype=torch.complex64, device=dev)
    out = torch.empty((W, N, M), dtype=torch.complex64, device=dev)
    for w0 in range(0, W, 256):
        w1 = min(W, w0 + 256)
        ph = torch.rand((w1 - w0, n, N), generator=g, device=dev) * (2.0 * math.pi)
        s = torch.polar(torch.ones_like(ph), ph)
        x = torch.einsum("wkm,wkt->wtm", A[w0:w1], s)
        nz = torch.complex(torch.randn((w1 - w0, N, M), generator=g, device=dev), torch.randn((w1 - w0, N, M), generator=g, device=dev))
        out[w0:w1] = x + nz * (noise / math.sqrt(2.0))
    return out.reshape(W, N * M), truth


def shape_run(name, args, dev, stream):
    mx, my, n = SHAPES[name]
    pos = eo.lattice_xyz(mx, my, (0.5 * LAM, 0.0), (0.0, 0.5 * LAM))
    M, W = pos.shape[0], args.windows
    x, truth = windows(pos, n, W, 4242 + M, dev)
    d_in = torch.view_as_real(x).reshape(W, -1).contiguous()
    blks, outs = {}, {}
    for k, (mode, refine) in VARIANTS.items():
        b = music_doa_azel(M, n, M * N, GRID.n_az, GRID.n_el, (GRID.el_lo, GRID.el_hi), pos, LAM)
        b.set_peak_mode(mode, 0)
        b.set_refine(refine)
        blks[k] = b
        outs[k] = [torch.empty((W, n), dtype=torch.float32, device=dev) for _ in range(3)] + [torch.empty((W, n), dtype=torch.int32, device=dev)]

    def call(k):
        a, e, l, bn = outs[k]
        blks[k].process_device(d_in.data_ptr(), W, a.data_ptr(), e.data_ptr(), l.data_ptr(), None, bn.data_ptr(), None,
                               stream=stream.cuda_stream)

    def timed(k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            call(k)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for k in VARIANTS:
        for _ in range(2):
            call(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in VARIANTS}
    for _ in range(args.rounds):
        for k in VARIANTS:
            ms[k].append(timed(k))
    stage = {}
    for k in VARIANTS:
        blks[k].set_stage_timing(True)
        for _ in range(3):
            call(k)
        torch.cuda.synchronize()
        s, _ = blks[k].stage_times_ms()
        blks[k].set_stage_timing(False)
        stage[k] = dict(zip(("cov", "eig", "scan", "topn_slot"), [v / 3 for v in s]))
    rms = {}
    for k in VARIANTS:
        call(k)
        torch.cuda.synchronize()
        az, el = outs[k][0].cpu().numpy(), outs[k][1].cpu().numpy()
        errs = []
        for w in range(W):
            errs += eo.matched_errors(list(zip(az[w].astype(float), el[w].astype(float))), truth[w])
        rms[k] = math.sqrt(float(np.mean(np.square(errs))))
    for b in blks.values():
        b.close()
    per10k = {k: float(np.median(v)) * 1e4 / W for k, v in ms.items()}
    return {"windows_per_step": W, "ms_per_step": ms, "ms_per_10k": per10k, "stage_ms": stage,
            "esprit_kernel_ms_per_10k": stage["esprit"]["topn_slot"] * 1e4 / W,
            "grid_scan_plus_pick_ms_per_10k": (stage["local_maxima"]["scan"] + stage["local_maxima"]["topn_slot"]) * 1e4 / W,
            "rms_deg": rms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU path only")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    res = {"steps_per_round": args.steps, "rounds": args.rounds, "grid": [GRID.n_az, GRID.n_el, GRID.el_lo, GRID.el_hi], "N": N}
    res["card"] = card()
    for name in SHAPES:
        res[name] = shape_run(name, args, dev, stream)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
