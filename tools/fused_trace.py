#!/usr/bin/env python
"""Per-CTA trace of the fused M = 4 kernel (MUSIC_B200_TRACE=1) over back-to-back calls on the bench.py config-2 windows:
when each role finished, how busy the eigensolver / scan warps were, and how the CTAs of consecutive calls share the SMs -
how long each SM's input stream stands still between one call's last covariance and the next call's first bulk copy.
Run on the GPU box: python tools/fused_trace.py [calls]"""
import os
import sys

os.environ["MUSIC_B200_TRACE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from gr_baz_b200 import synth
from gr_baz_b200.music_doa import music_doa

WORDS, CTAS, RING = 40, 1024, 32  # FZ_TRACE, FZ_TRACE_CTAS, FZ_TRACE_LAUNCHES (music_fused.cuh)
WARM = 3
CALLS = int(sys.argv[1]) if len(sys.argv) > 1 else 20
assert WARM + CALLS <= RING

cfg, W = bench.workload(2)
resp, _ = bench.table_for(cfg)
dev = torch.device("cuda:0")
d_in = synth.gen_windows_torch(cfg, synth.BASE_SEED + 2, 0, W, dev)
blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], resp, cfg["resolution"])
a = torch.empty((W, 1), dtype=torch.float32, device=dev)
l = torch.empty_like(a)
b = torch.empty((W, 1), dtype=torch.int32, device=dev)
st = torch.cuda.current_stream()


def call():
    blk.process_device(d_in.data_ptr(), W, a.data_ptr(), l.data_ptr(), None, b.data_ptr(), stream=st.cuda_stream)


for _ in range(WARM):
    call()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(st)
for _ in range(CALLS):
    call()
e1.record(st)
torch.cuda.synchronize()
step_us = e0.elapsed_time(e1) * 1e3 / CALLS
ring = np.zeros((RING * CTAS, WORDS), np.int64)
blk._lib.music_b200_debug_fused_trace(blk._h, ring.ctypes.data, RING * CTAS)
ring = ring.reshape(RING, CTAS, WORDS)
grid = int((ring[WARM, :, 31] != 0).sum())
L = ring[WARM:WARM + CALLS, :grid]  # [call][CTA][word]
print("device %s, %d back-to-back calls of W = %d, grid %d CTAs: %.1f us per call (TRACE build)" % (torch.cuda.get_device_name(0), CALLS, W, grid, step_us))

tr = L[-1]  # per-role cycle counts of the last call
cov_end = tr[:, 0]
print("cycles (mean over the CTAs of the last call):")
print("  last cov warp done   %9.0f   (first cov warp done %9.0f)" % (cov_end.mean(), tr[:, 1].mean()))
print("  eig warp exit        %9.0f   busy %9.0f in %5.1f rounds -> %7.0f cyc/round" % (tr[:, 8].mean(), tr[:, 9].mean(), tr[:, 10].mean(), (tr[:, 9] / np.maximum(tr[:, 10], 1)).mean()))
print("  scan warps exit      %9.0f   busy %9.0f in %5.1f passes -> %7.0f cyc/pass" % (tr[:, 11].mean(), tr[:, 12].mean(), tr[:, 13].mean(), (tr[:, 12] / np.maximum(tr[:, 13], 1)).mean()))
print("  scan: exact-evaluation phase %9.0f cycles, candidates/CTA %7.1f, full-fp64 fallbacks/CTA %5.2f" % (tr[:, 14].mean(), tr[:, 7].mean(), tr[:, 15].mean()))
print("  scan thread 0 inside the sweeps: issue+slot-wait %9.0f, tile-arrival wait %9.0f, loads+MMA+post %9.0f" % (tr[:, 4].mean(), tr[:, 5].mean(), tr[:, 6].mean()))
print("  tensor-core passes ended %9.0f, windows taken by the fp64 drain workers %5.1f / CTA, Jacobi rounds %5.2f / CTA" % (tr[:, 16].mean(), tr[:, 17].mean(), tr[:, 19].mean()))
print("  CTA done (all outputs written) %9.0f mean, %9.0f max; after the last covariance warp: %9.0f mean" % (tr[:, 18].mean(), tr[:, 18].max(), (tr[:, 18] - cov_end).mean()))
print("  drain: %5.2f groups / CTA, last group finished %9.0f (%9.0f after the last covariance warp)" % (tr[:, 20].mean(), tr[:, 23].mean(), (tr[:, 23] - cov_end).mean()))

# %globaltimer (ns): word 2 CTA start, 32 first input bytes arrived, 33 last covariance warp done, 31 CTA exit; word 30 %smid
start, first, cend, end, sm = L[..., 2], L[..., 32], L[..., 33], L[..., 31], L[..., 30]
print("globaltimer, mean over %d x %d CTAs (us):" % (CALLS, grid))
print("  CTA lifetime %.1f; head (start -> first input bytes) %.2f; tail (last covariance -> exit) %.2f"
      % ((end - start).mean() / 1e3, (first - start).mean() / 1e3, (end - cend).mean() / 1e3))
gaps, streams, resident = [], [], []
for s in np.unique(sm):
    rows = [(c, i) for c in range(CALLS) for i in range(grid) if sm[c, i] == s]
    resident.append(max(sum(1 for c2, i2 in rows if start[c2, i2] <= start[c, i] < end[c2, i2]) for c, i in rows))
    for c in range(CALLS - 1):  # the CTA of call c on this SM -> the CTA of call c + 1 on this SM
        prev = [i for cc, i in rows if cc == c]
        nxt = [i for cc, i in rows if cc == c + 1]
        if prev and nxt:
            gaps.append((first[c + 1, nxt].min() - end[c, prev].max()) / 1e3)
    iv = sorted((first[c, i], cend[c, i]) for c, i in rows)
    lo, hi = iv[0][0], max(e for _, e in iv)
    cov, cur0, cur1 = 0, iv[0][0], iv[0][1]
    for a0, a1 in iv[1:]:  # union of the streaming intervals of every CTA on this SM
        if a0 > cur1:
            cov += cur1 - cur0
            cur0, cur1 = a0, a1
        else:
            cur1 = max(cur1, a1)
    cov += cur1 - cur0
    streams.append(1.0 - cov / max(hi - lo, 1))
gaps = np.array(gaps)
print("  SMs %d; CTAs resident together on one SM: max %d; exit -> next call's first input bytes on the same SM: mean %.2f, min %.2f, max %.2f"
      % (len(resident), max(resident), gaps.mean(), gaps.min(), gaps.max()))
print("  share of the run in which an SM streams no input (no CTA between its first bytes and its last covariance): mean %.2f %%, max %.2f %%"
      % (100 * np.mean(streams), 100 * np.max(streams)))
print("  (head + tail) / call: %.2f %%" % (100 * ((first - start).mean() + (end - cend).mean()) / 1e3 / step_us))
