#!/usr/bin/env python
"""Generates tests/golden/reference/tables.npz: what the reference's own work() returns on arbitrary array-response
tables (helpers.table_golden_cases: tables scaled by 2^63 and 2^-70, a calibrated table, duplicated rows, zero rows).
The full angles, levels and spectrum of every case are stored, with the sha256 of the inputs and of the table.

The reference is gr-baz's lib/baz_music_doa.cc, compiled unmodified against stand-in GNU Radio / Armadillo headers into
oracle/_ref/ (`make -C oracle ref`, which needs a gr-baz checkout; see oracle/Makefile).

Run from the repo root:   python tests/golden/reference/make_reference_tables_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_build  # noqa: E402

import helpers  # noqa: E402


def main():
    if not ref_build.build():
        raise SystemExit("oracle/_ref/libbaz_music_ref.so could not be built (needs the gr-baz sources, oracle/Makefile)")
    out = {}
    for key, m, n, table, x in helpers.table_golden_cases():
        with np.errstate(all="ignore"):
            ref = ref_build.work_batch(x, m, n, table)
        out[key + "/in_sha256"] = np.array(helpers.sha256(x))
        out[key + "/table_sha256"] = np.array(helpers.sha256(table))
        for f in ("angles", "levels", "spectrum"):
            out[key + "/" + f] = ref[f]
    np.savez_compressed(helpers.REFERENCE_TABLES, **out)
    print("%s: %d cases, %d bytes" % (helpers.REFERENCE_TABLES, len(out) // 5, os.path.getsize(helpers.REFERENCE_TABLES)))


if __name__ == "__main__":
    main()
