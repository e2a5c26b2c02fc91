#!/usr/bin/env python
"""Generates tests/golden/reference/work.npz: what the reference's own work() returns on the inputs of
tests/test_ref_shim.py and tests/test_gpu_zz_reference_source.py (case lists and random sweeps in tests/helpers.py;
the wide-array sweep's keys come last, after every earlier key); and
tests/golden/reference/interface.json: the signature of the reference's GRC descriptor and the C++ declarations of its
block header that tests/test_boundary_files.py holds ours to.

The reference is gr-baz's lib/baz_music_doa.cc, compiled unmodified against stand-in GNU Radio / Armadillo headers into
oracle/_ref/ (`make -C oracle ref`, which needs a gr-baz checkout; see oracle/Makefile).  The tests compare against the
stored outputs, so they need neither that checkout nor the compiled library.

Run from the repo root:   python tests/golden/reference/make_reference_golden.py
"""
import json
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gr_baz_b200 import synth  # noqa: E402
from oracle import ref_build  # noqa: E402

import helpers  # noqa: E402

SAMPLED_BINS = 32  # spectrum columns stored per case besides the top bins and their neighbours
NEIGHBOURS = 2


def spectrum_bins(K, angles, seed):
    """Columns of the spectrum to store: all for small grids, else a seeded sample plus every window's top bins +-2."""
    if K <= SAMPLED_BINS + 16:
        return np.arange(K, dtype=np.int32)
    rng = np.random.default_rng(seed)
    pick = set(rng.choice(K, SAMPLED_BINS, replace=False).tolist())
    tops = np.rint(np.asarray(angles, np.float64) * K / 360.0).astype(np.int64) % K
    for b in np.unique(tops):
        pick.update(((b + d) % K) for d in range(-NEIGHBOURS, NEIGHBOURS + 1))
    return np.array(sorted(pick), dtype=np.int32)


def store(out, key, x, ref, K, seed, finite=True):
    bins = spectrum_bins(K, ref["angles"], seed)
    out.append((key, helpers.sha256(x), finite, ref["angles"], ref["levels"], ref["spectrum"][:, bins], bins))


def pack(cases):
    """One flat array per field, rows located by the (W, n, columns) table: a few arrays instead of hundreds."""
    return {"keys": np.array([c[0] for c in cases]), "in_sha256": np.array([c[1] for c in cases]),
            "finite": np.array([c[2] for c in cases]),
            "shape": np.array([(c[3].shape[0], c[3].shape[1], len(c[6])) for c in cases], np.int64),
            "angles": np.concatenate([c[3].ravel() for c in cases]), "levels": np.concatenate([c[4].ravel() for c in cases]),
            "spectrum": np.concatenate([c[5].ravel() for c in cases]), "bins": np.concatenate([c[6] for c in cases])}


def write_interface():
    src = os.path.dirname(os.path.dirname(ref_build.REFERENCE))  # the gr-baz checkout the `ref` target compiles from
    grc = helpers.grc_signature(ET.parse(os.path.join(src, "grc", "baz_music_doa.xml")).getroot())
    with open(os.path.join(src, "lib", "baz_music_doa.h")) as f:
        header = helpers.normalized_declarations(f.read())
    declared = [d for d in helpers.CPP_SURFACE if helpers.normalized_declarations(d) in header]
    with open(helpers.REFERENCE_INTERFACE, "w") as f:
        json.dump({"grc_signature": grc, "header_declarations": declared}, f, indent=1)
        f.write("\n")


def main():
    write_interface()
    if not ref_build.build():
        raise SystemExit("oracle/_ref/libbaz_music_ref.so could not be built (needs the gr-baz sources, oracle/Makefile)")
    out = []
    seed = 0
    for path in helpers.golden_files():
        cfg, _, table, wins, _ = helpers.load_golden(path)
        x = np.stack([w["in"] for w in wins])
        key = "fixture_" + os.path.basename(path)[:-4]
        store(out, key, x, ref_build.work_batch(x, cfg["m"], cfg["n"], table), cfg["resolution"], seed)
        seed += 1
    for kind, cases, s0 in (("oracle", helpers.ORACLE_CASES, helpers.ORACLE_SEED), ("gpu", helpers.GPU_CASES, helpers.GPU_SEED)):
        for i, (base, over, W) in enumerate(cases):
            cfg, table, x = helpers.case_windows(base, over, W, s0)
            store(out, helpers.case_key(kind, i), x, ref_build.work_batch(x, cfg["m"], cfg["n"], table), cfg["resolution"], seed)
            seed += 1
    base, over, W, s = helpers.MIRROR_CASE
    cfg = synth.config(base, **over)
    x = synth.gen_windows_numpy(cfg, s, 0, W)
    store(out, "mirror", x, ref_build.work_batch(x, cfg["m"], cfg["n"], helpers.table_for(cfg)), cfg["resolution"], seed)
    seed += 1
    for kind, shapes in (("random", helpers.random_small_shapes), ("wide", helpers.random_wide_shapes)):
        for trial, m, n, snaps, K, table, x in shapes():
            ref = ref_build.work_batch(x, m, n, table)
            finite = bool(np.all(np.isfinite(ref["levels"])) and np.all(np.isfinite(ref["spectrum"])))
            store(out, helpers.case_key(kind, trial), x, ref, K, seed, finite)
            seed += 1
    path = helpers.REFERENCE_GOLDEN
    np.savez_compressed(path, **pack(out))
    print("%s: %d cases, %d bytes" % (path, len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
