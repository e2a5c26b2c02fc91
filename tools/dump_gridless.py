#!/usr/bin/env python
"""Outputs of the polynomial-rooting peak modes (ROOTS and MANIFOLD) on a fixed set of seeded windows, for comparing
two builds of the library byte for byte.

  python tools/dump_gridless.py dump LIB OUT.npz      run every case against the library at LIB
  python tools/dump_gridless.py compare A.npz B.npz   list the arrays that differ; exit status 1 if any does
  python tools/dump_gridless.py run LIB TOOL [ARGS]   run the tool script TOOL with the library at LIB

The cases: ROOTS on x-axis ULAs (M = 2, 3, 4, 5, 8, 12, 16) and MANIFOLD on UCAs (m = 3, 4, 5, 8, 12, 16) and on
random planar arrays, n = 1 .. 3 under the FIXED and MDL rules, on the seeded windows of the GPU tests (noiseless ones
included) and their degenerate windows (zero, NaN, d = 0, every element at one point); ROOTS on the adversarial
families of tests/gridless_oracle.py; and the windows of the C2, M = 16 x-ULA and C3 - C5 timing shapes.  Each case
stores the angles, levels, bins and counts of one device call.
"""
import os
import runpy
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

from gr_baz_b200 import _capi  # noqa: E402


def use_library(path):
    path = os.path.abspath(path)
    _capi.lib_path = lambda: path


def cases():
    """yields (name, make_block() arguments, windows)"""
    import bench
    import torch
    import gridless_oracle as go
    import manifold_oracle as mf
    from gr_baz_b200 import synth
    from helpers import LAM, PLAN, plan_windows, ula
    from test_gpu_manifold import planar

    for mode, geos in (("roots", [("ula", m, ula(m, "x")) for m in (2, 3, 4, 5, 8, 12, 16)]),
                       ("manifold", [("uca", m, mf.uca(m, 0.5, LAM)) for m in (3, 4, 5, 8, 12, 16)]
                        + [("planar", m, planar(m, 40 + m)) for m in (5, 8, 12)])):
        for kind, m, pos in geos:
            for n in (1, 2, 3):
                if n >= m:
                    continue
                x, _ = plan_windows(pos, [(min(S, m - 1), snr) for S, snr in PLAN], 3000 * m + 10 * n + len(kind), 512)
                deg, _ = plan_windows(pos, [(n, 20.0), (n, 20.0), (0, 0.0), (n, 20.0)], 5 + m, 512)
                deg[0] = 0
                deg[1, 17] = np.nan
                for rule in ("fixed", "mdl"):
                    K = 3600 if (m + n) % 2 else 360
                    yield "%s_%s%d_n%d_%s" % (mode, kind, m, n, rule), dict(m=m, n=n, snaps=512, K=K, pos=pos, rule=rule, mode=mode), x
                    yield "%s_%s%d_n%d_%s_degenerate" % (mode, kind, m, n, rule), dict(m=m, n=n, snaps=512, K=K, pos=pos, rule=rule, mode=mode), deg
        # seeded noisy windows, 1 to 3 sources at 0 to 40 dB
        m = 16
        pos = geos[-1][2] if mode == "roots" else mf.uca(m, 0.5, LAM)
        rng = np.random.default_rng(9)
        plan = [(int(rng.integers(1, 4)), float(rng.choice([0.0, 10.0, 20.0, 40.0]))) for _ in range(2000)]
        x, _ = plan_windows(pos, plan, 99, 256)
        yield "%s_m16_seeded" % mode, dict(m=m, n=3, snaps=256, K=3600, pos=pos, mode=mode), x
    x, _ = plan_windows(mf.uca(5, 0.5, LAM), [(2, 20.0)] * 4, 5, 256)
    yield "manifold_one_point", dict(m=5, n=2, snaps=256, K=360, pos=np.zeros((5, 2)), mode="manifold"), x
    for M in (2, 4, 5, 6, 8, 12, 16):
        groups = {}
        for f in go.families(M, 9000 + M):
            groups.setdefault(f[3], []).append(f[2].reshape(-1))
        for d, xs in sorted(groups.items()):
            for rule in ("fixed", "mdl"):
                yield "roots_family_M%d_d%d_%s" % (M, d, rule), dict(m=M, n=d, snaps=go.N, K=3600, pos=ula(M, "x"), rule=rule, mode="roots"), np.stack(xs)
    # the timing shapes of tools/bench_roots.py and tools/bench_manifold.py, on their synthetic windows
    for name, cid, cfg, mode in (("c2", 2, synth.config(2), "roots"),
                                 ("m16_ula", 5, synth.config(5, geometry="ula_x", fixed_sources=(40.0, 110.0)), "roots"),
                                 ("c3", 3, synth.config(3), "manifold"), ("c4", 4, synth.config(4), "manifold"),
                                 ("c5", 5, synth.config(5), "manifold")):
        W = bench.workload(cid)[1]
        x = synth.gen_windows_torch(cfg, synth.BASE_SEED + cfg["id"], 0, W, torch.device("cuda:0")).cpu().numpy().view(np.complex64)
        pos = np.asarray([[synth.SPACING * a, synth.SPACING * b] for a, b in cfg["antenna_array"]], np.float64)
        yield "%s_%s" % (mode, name), dict(m=cfg["m"], n=cfg["n"], snaps=cfg["snapshots"], K=cfg["resolution"], pos=pos,
                                           lam=synth.C_LIGHT / synth.FREQUENCY, mode=mode), x


def dump(out_path):
    import gpu_harness as gh

    res = {}
    for name, kw, x in cases():
        kw = dict(kw)
        blk = gh.make_block(kw.pop("m"), kw.pop("n"), kw.pop("snaps"), kw.pop("K"), **kw)
        out, _ = gh.device_call(blk, np.ascontiguousarray(x, np.complex64), ("levels", "bins", "counts"))
        blk.close()
        for k in ("angles", "levels", "bins", "counts"):
            res["%s/%s" % (name, k)] = out[k]
    np.savez(out_path, **res)
    print("%d cases, %d arrays -> %s" % (len(res) // 4, len(res), out_path))


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    diff = sorted(set(a.files) ^ set(b.files))
    diff += [k for k in sorted(set(a.files) & set(b.files)) if a[k].tobytes() != b[k].tobytes() or a[k].dtype != b[k].dtype]
    filled = sum(int((a[k] >= 0).sum()) for k in a.files if k.endswith("/bins"))
    print("%d arrays (%d filled slots) compared, %d differ%s" % (len(a.files), filled, len(diff), (": " + ", ".join(diff)) if diff else ""))
    return 1 if diff else 0


if __name__ == "__main__":
    cmd = sys.argv[1] if len(sys.argv) > 1 else ""
    if cmd == "dump" and len(sys.argv) == 4:
        use_library(sys.argv[2])
        dump(sys.argv[3])
    elif cmd == "compare" and len(sys.argv) == 4:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    elif cmd == "run" and len(sys.argv) >= 4:
        use_library(sys.argv[2])
        sys.argv = sys.argv[3:]
        runpy.run_path(sys.argv[0], run_name="__main__")
    else:
        sys.exit(__doc__)
