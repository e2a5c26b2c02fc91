import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
from gr_baz_b200 import synth
from gr_baz_b200.music_doa import music_doa
from oracle import c_oracle as co
import helpers
from helpers import streams_for, form_windows
cfg = synth.config(2, snapshots=1024)
N, hop, W = 1024, 512, 1500
table = helpers.table_for(cfg)
streams = streams_for(cfg, 77, (W - 1) * hop + N)
x = form_windows(streams, hop, W, N)
ref = co.work_batch(x, cfg["m"], cfg["n"], table)
blk = music_doa(cfg["m"], cfg["n"], cfg["nsamples"], table.tolist(), cfg["resolution"])
ang = np.zeros((W, 1), np.float32); lvl = np.zeros((W, 1), np.float32)
blk.work_planar(W, streams, [ang, lvl], hop=hop)
b_pl = blk.last_bins().copy()
blk.work(W, [x], [ang, lvl])
b_il = blk.last_bins().copy()
spec = np.zeros((W, cfg["resolution"]), np.float32)
blk.work(W, [x], [ang, lvl, spec])
b_il3 = blk.last_bins().copy()
for name, b in (("planar", b_pl), ("interleaved-fused", b_il), ("interleaved-3k", b_il3)):
    bad = np.nonzero(b[:, 0] != ref["bins"][:, 0])[0]
    print(name, "mismatches", len(bad), bad[:10])
    for w in bad[:6]:
        P = ref["P"][w]
        print("  w", w, "got", b[w, 0], "ref", ref["bins"][w, 0], "P[got]=%.17g P[ref]=%.17g rel=%.3e" % (P[b[w, 0]], P[ref["bins"][w, 0]], abs(P[b[w,0]]-P[ref["bins"][w,0]])/P[ref["bins"][w,0]]))
