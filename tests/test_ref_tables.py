"""CPU: the oracle restatements against the reference's own work() on arbitrary array-response tables - scaled by 2^63
and 2^-70, calibrated, with duplicated rows and with zero rows (helpers.table_golden_cases; the reference's outputs are
stored in tests/golden/reference/tables.npz by make_reference_tables_golden.py).  This pins what the GPU tests of
tests/test_gpu_tables.py take from the oracles on such tables: a zero row has strength 1 / 0 = +inf and the first one
wins, bit-equal rows tie and the lower bin comes first, strengths beyond the float32 range become +inf / tiny levels."""
import numpy as np
import pytest

from oracle import c_oracle as co
from oracle import music_oracle as mo

import helpers

CASES = list(helpers.table_golden_cases())


@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracles_follow_the_reference_on_arbitrary_tables(case):
    key, m, n, table, x = CASES[case]
    ref = helpers.table_reference_outputs(key, x, table)
    with np.errstate(all="ignore"):
        c = co.work_batch(x, m, n, table, want_spectrum=True)
        py = [mo.work(x[w], m, n, table) for w in range(x.shape[0])]
    assert np.array_equal(c["angles"], ref["angles"]), key
    helpers.assert_float32_close(c["levels"], ref["levels"], 1.2e-7, key)
    helpers.assert_float32_close(c["spectrum"], ref["spectrum"], 1.2e-7, key)
    for w, p in enumerate(py):
        assert np.array_equal(p["angles"], ref["angles"][w]), (key, w)
        helpers.assert_float32_close(p["levels"], ref["levels"][w], 1.2e-7, (key, w))


def test_reference_semantics_of_zero_and_duplicated_rows():
    """what the reference itself decides, independently of any restatement"""
    K = 400
    for key, m, n, table, x in CASES:
        ref = helpers.table_reference_outputs(key, x, table)
        bins = np.rint(ref["angles"].astype(np.float64) * K / 360.0).astype(np.int64)
        if key.startswith("zero"):
            z = helpers.TABLE_ZERO_ROWS
            assert np.all(bins == np.array(z[:n])[None, :]), key        # the first zero rows, in bin order
            assert np.all(np.isposinf(ref["levels"])), key
            assert np.all(np.isposinf(ref["spectrum"][:, list(z)])), key
        elif key.startswith("duplicate"):
            for w, (src, dst) in ((0, helpers.TABLE_DUPLICATES[0]), (2, helpers.TABLE_DUPLICATES[1])):
                assert list(bins[w]) == [src, dst][:n], (key, w)        # the tie is the peak; lower bin first
                if n == 2:
                    assert ref["levels"][w, 0] == ref["levels"][w, 1], (key, w)
        elif key.startswith("scaled-70"):
            assert np.all(np.isposinf(ref["levels"])), key               # 2^140 P overflows float32
