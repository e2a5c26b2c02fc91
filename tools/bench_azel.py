"""Cost and accuracy of (azimuth, elevation) MUSIC (music_b200_create_azel) on synthetic windows.

Shapes: an 8-element UCA with N = 4096 snapshots on 360 x 46 and 360 x 91 grids over el in [0, 90] (n = 1, the
n largest bins), and a 16-element UCA with n = 2 and the 2-D local-maximum rule.  For each: the device call time (CUDA
events), the per-stage times from stage_times_ms, the local-maximum kernel's rate on the fp64 spectrum bytes it reads,
the cost of the refinement and the RMS (az, el) error against the synthetic truth with and without it.  Windows hold
unit-power sources at random off-grid directions (el in [10, 80]) plus white noise at 20 dB, generated on the device.

    python tools/bench_azel.py [--windows W] [--reps R] [--out results/bench_azel.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gr_baz_b200.music_doa_azel import music_doa_azel  # noqa: E402

LAM = 1.0


def uca(m):
    r = 0.5 * LAM / math.sin(math.pi / m)
    return np.array([[r * math.cos(2 * math.pi * e / m), r * math.sin(2 * math.pi * e / m), 0.0] for e in range(m)])


def windows(pos, n, W, N, seed, dev):
    """complex64 (W, m * N) on the device and the true (az, el) degrees (W, n)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    m = pos.shape[0]
    az = torch.rand((W, n), generator=g, device=dev, dtype=torch.float64) * 360.0
    el = 10.0 + torch.rand((W, n), generator=g, device=dev, dtype=torch.float64) * 70.0
    P = torch.tensor(pos, device=dev)
    X = torch.complex(torch.randn((W, m, N), generator=g, device=dev), torch.randn((W, m, N), generator=g, device=dev)) * (0.1 / math.sqrt(2))
    for s in range(n):
        a, e = torch.deg2rad(az[:, s]), torch.deg2rad(el[:, s])
        u = torch.stack([torch.cos(e) * torch.cos(a), torch.cos(e) * torch.sin(a), torch.sin(e)], 1)
        ph = 2 * math.pi * (u @ P.T) / LAM  # (W, m)
        st = torch.exp(-1j * ph).to(torch.complex64)
        sig = torch.exp(2j * math.pi * torch.rand((W, 1, N), generator=g, device=dev)).to(torch.complex64)
        X += st[:, :, None] * sig
    x = X.transpose(1, 2).reshape(W, m * N).contiguous()  # x(r, c) = in[c * m + r]
    return x, az.cpu().numpy(), el.cpu().numpy()


def run(blk, x, n, K, reps):
    dev = x.device
    W = x.shape[0]
    az = torch.zeros((W, n), dtype=torch.float32, device=dev)
    el, lv = torch.zeros_like(az), torch.zeros_like(az)
    st = torch.cuda.current_stream().cuda_stream
    call = lambda: blk.process_device(x.data_ptr(), W, az.data_ptr(), el.data_ptr(), lv.data_ptr(), stream=st)
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    blk.set_stage_timing(True)
    call()
    stages, _ = blk.stage_times_ms()
    blk.set_stage_timing(False)
    return ms, stages, az.cpu().numpy(), el.cpu().numpy()


def rms_error(az, el, taz, tel):
    """RMS azimuth and elevation error in degrees, each output slot matched to the nearest true source"""
    ea, ee = [], []
    for w in range(az.shape[0]):
        for i in range(az.shape[1]):
            d = [abs((az[w, i] - taz[w, s] + 180.0) % 360.0 - 180.0) + abs(el[w, i] - tel[w, s]) for s in range(taz.shape[1])]
            s = int(np.argmin(d))
            ea.append((az[w, i] - taz[w, s] + 180.0) % 360.0 - 180.0)
            ee.append(el[w, i] - tel[w, s])
    return float(np.sqrt(np.mean(np.square(ea)))), float(np.sqrt(np.mean(np.square(ee))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_azel needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    N = 4096
    shapes = [dict(m=8, n=1, n_az=360, n_el=46, peak="top_bins"), dict(m=8, n=1, n_az=360, n_el=91, peak="top_bins"),
              dict(m=16, n=2, n_az=360, n_el=91, peak="local_maxima")]
    results = []
    for sh in shapes:
        m, n, K = sh["m"], sh["n"], sh["n_az"] * sh["n_el"]
        pos = uca(m)
        blk = music_doa_azel(m, n, m * N, sh["n_az"], sh["n_el"], (0.0, 90.0), pos, LAM)
        blk.set_peak_mode(sh["peak"], 2)
        x, taz, tel = windows(pos, n, a.windows, N, 1234 + m, dev)
        r = dict(sh, windows=a.windows, snapshots=N)
        for refine in (False, True):
            blk.set_refine(refine)
            ms, stages, az, el = run(blk, x, n, K, a.reps)
            key = "refined" if refine else "grid"
            r[key] = dict(ms_per_call=ms, ms_per_10k_windows=ms * 1e4 / a.windows,
                          stage_ms=dict(zip(("cov", "eig", "scan", "topn"), stages)), rms_deg=rms_error(az, el, taz, tel))
        r["refine_cost_ms_per_10k_windows"] = r["refined"]["ms_per_10k_windows"] - r["grid"]["ms_per_10k_windows"]
        if sh["peak"] == "local_maxima":
            # the top-n slot holds the 2-D local-maximum kernel and the decode (refinement off); the P64 bytes it reads
            r["local_max_p64_GBps"] = a.windows * K * 8 / (r["grid"]["stage_ms"]["topn"] * 1e-3) / 1e9
        blk.close()
        results.append(r)
        print(json.dumps(r))
    out = dict(card=card, results=results)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(dict(card=card)))


if __name__ == "__main__":
    main()
