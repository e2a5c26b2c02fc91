"""CPU: the oracle of the COHERENT combine (tests/focus_oracle.py) has the properties the definition promises, and on the
two-path wideband case the focused covariance resolves what the incoherent combine cannot."""
import numpy as np

import channels_oracle as ch
import composed_oracle as cmp
import focus_oracle as fo


def small_case(m=6, C=9, band=1.0):
    """a planar m-element array and C channel wavelengths spanning +-band * 7.5 % of 1 GHz"""
    pos = np.random.default_rng(m).uniform(-0.2, 0.2, (m, 2))
    f = fo.FC * (1.0 + band * np.linspace(-0.075, 0.075, C))
    return pos, ch.C0 / f


def test_focusing_matrices_are_unitary_and_the_reference_is_the_identity():
    pos, lams = small_case()
    for first, count in ((0, None), (350, 40), (100, 3)):
        T, err = fo.focusing(pos, lams, fo.K, first, count)
        ref = fo.ref_channel(len(lams))
        assert np.array_equal(T[ref], np.eye(len(pos))) and err[ref] == 0.0
        for c in range(len(lams)):
            assert np.max(np.abs(T[c] @ T[c].conj().T - np.eye(len(pos)))) <= 1e-12, (first, count, c)


def test_white_noise_stays_white():
    pos, lams = small_case()
    T, _ = fo.focusing(pos, lams, fo.K)
    s2 = 0.37
    R = np.stack([s2 * np.eye(len(pos), dtype=np.complex128)] * len(lams))
    assert np.max(np.abs(fo.focus(R, T) - s2 * np.eye(len(pos)))) <= 1e-15


def test_zero_bandwidth_focuses_with_the_identity():
    pos, lams = small_case()
    T, err = fo.focusing(pos, np.full(len(lams), lams[0]), fo.K)
    assert np.max(np.abs(T - np.eye(len(pos))[None])) <= 1e-12
    assert np.max(err) <= 1e-12


def test_the_error_falls_as_the_sector_and_the_band_narrow():
    pos, lams = fo.geometry()
    full = fo.focusing(pos, lams, fo.K)[1].max()
    assert abs(full - 0.215) <= 5e-4  # UCA 8, +-7.5 %, the whole grid
    sectors = [fo.focusing(pos, lams, fo.K, 300, n)[1].max() for n in (360, 180, 60)]
    assert sectors[0] > sectors[1] > sectors[2] and abs(fo.focusing(pos, lams, fo.K, 40, 60)[1].max() - 0.054) <= 5e-4
    half = ch.C0 / (fo.FC + 0.5 * (ch.C0 / lams - fo.FC))
    assert fo.focusing(pos, half, fo.K)[1].max() < 0.6 * full
    pos4 = fo.uca(4, ch.C0 / fo.FC)
    assert abs(fo.focusing(pos4, lams, fo.K)[1].max() - 0.118) <= 5e-4


def test_a_singular_sector_is_refused():
    pos, lams = small_case()
    try:
        fo.focusing(pos, lams, fo.K, 0, 1)  # beta keeps one bin's B_c regular
    except ValueError:
        raise AssertionError("a one-bin sector with beta > 0 must stay regular")
    fo_beta, fo.BETA = fo.BETA, 0.0
    try:
        raised = False
        try:
            fo.focusing(pos, lams, fo.K, 0, 1)  # rank one without beta
        except ValueError:
            raised = True
        assert raised
    finally:
        fo.BETA = fo_beta


def test_two_paths_are_resolved_only_after_focusing():
    W = 20
    pos, lams, x = fo.scenario(W, 7)
    T, _ = fo.focusing(pos, lams, fo.K)
    tab_ref = ch.table(pos, lams[fo.ref_channel(fo.C)], fo.K)
    tabs = np.stack([ch.table(pos, lam, fo.K) for lam in lams])
    md = cmp.modes(peak="local")
    focused = incoherent = 0
    for w in range(W):
        R = ch.covariances(x[w], len(pos), fo.F, fo.FIRST, fo.C, "rect")
        r = cmp.work_R(fo.focus(R, T), md, tab_ref, None, 2, fo.J * fo.C)
        focused += fo.resolved(r["angles"])
        incoherent += fo.resolved(ch.incoherent(R, tabs, 2, "local", 0)[1][0])
    assert focused >= 18 and incoherent <= 2, (focused, incoherent)


def test_mdl_counts_both_paths_from_all_looks():
    W = 20
    pos, lams, x = fo.scenario(W, 11, noise=1.0)
    T, _ = fo.focusing(pos, lams, fo.K)
    R = [ch.covariances(x[w], len(pos), fo.F, fo.FIRST, fo.C, "hann") for w in range(W)]
    counts = [cmp.count(fo.focus(r, T), fo.J * fo.C, len(pos) - 1, "mdl")[0] for r in R]
    assert counts.count(2) >= 18, counts
    per_channel = [cmp.count(r[fo.ref_channel(fo.C)], fo.J, len(pos) - 1, "mdl")[0] for r in R]
    assert per_channel.count(1) >= 18, per_channel  # each channel alone sees one (rank-one) source


def test_mdl_over_counts_at_high_snr():
    """the documented caveat: the focusing error leaks signal power into the noise eigenvalues"""
    pos, lams, x = fo.scenario(4, 7)
    T, _ = fo.focusing(pos, lams, fo.K)
    counts = [cmp.count(fo.focus(ch.covariances(w, len(pos), fo.F, fo.FIRST, fo.C, "rect"), T), fo.J * fo.C, len(pos) - 1, "mdl")[0]
              for w in x]
    assert min(counts) > 2, counts
