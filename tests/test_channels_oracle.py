"""CPU: the definition of the frequency-channelised modes (tests/channels_oracle.py) and the two cases they exist for -
emitters at different frequencies from different directions, and one wideband source seen through tables built for the
wrong wavelength."""
import math

import numpy as np
import pytest

import calibration_oracle as co
import channels_oracle as ch
import composed_oracle as cmp
import source_count_oracle as so

FC, FS = 400e6, 56e6  # a 56 MHz band at 400 MHz: 14 % fractional bandwidth


def noise_window(rng, m, N, sigma=1.0):
    return ch.interleave(sigma * (rng.standard_normal((N, m)) + 1j * rng.standard_normal((N, m))) / math.sqrt(2.0))


@pytest.mark.parametrize("m,F,J", [(4, 8, 1), (4, 64, 8), (7, 16, 5), (16, 256, 2)])
def test_rect_parseval_gives_the_plain_covariance(m, F, J):
    rng = np.random.default_rng(m * F)
    x = noise_window(rng, m, F * J)
    R = ch.covariances(x, m, F, 0, F, "rect")
    plain = co.covariance(x[None, :], m)[0]
    assert np.max(np.abs(R.sum(axis=0) / F - plain)) <= 1e-13 * np.max(np.abs(plain))


def test_definition_against_a_direct_dft():
    """np.fft.fft is the sum in the header, bin by bin"""
    rng = np.random.default_rng(3)
    m, F, J = 3, 8, 2
    x = noise_window(rng, m, F * J)
    X = x.reshape(-1, m).astype(np.complex128)
    h = ch.taper(F, "hann")
    for first, C in ((0, 8), (6, 4)):
        R = ch.covariances(x, m, F, first, C, "hann")
        for c in range(C):
            b = (first + c) % F
            acc = np.zeros((m, m), complex)
            for j in range(J):
                v = sum(h[t] * X[j * F + t] * np.exp(-2j * math.pi * b * t / F) for t in range(F))
                acc += np.outer(v, v.conj())
            assert np.allclose(R[c], acc / (J * np.sum(h * h)), rtol=0, atol=1e-13 * np.max(np.abs(acc)))


def test_channel_and_offset_mapping():
    F, fs = 8, 8000.0
    assert list(ch.bins_of(F, 0, 8)) == [0, 1, 2, 3, 4, 5, 6, 7]
    assert list(ch.offsets(F, 0, 8, fs)) == [0.0, 1000.0, 2000.0, 3000.0, -4000.0, -3000.0, -2000.0, -1000.0]  # b = F / 2 is -fs / 2
    assert list(ch.bins_of(F, 6, 4)) == [6, 7, 0, 1]  # a range that wraps through the negative frequencies
    assert list(ch.offsets(F, 6, 4, fs)) == [-2000.0, -1000.0, 0.0, 1000.0]
    lam = ch.wavelengths(F, 6, 4, 100000.0, fs)
    assert np.array_equal(lam, ch.C0 / (100000.0 + np.array([-2000.0, -1000.0, 0.0, 1000.0])))


@pytest.mark.parametrize("kind", ch.TAPERS)
def test_white_noise_has_its_power_in_every_channel(kind):
    """the normalisation J sum h^2: tr R_c / m ~ sigma^2 whatever the taper"""
    rng = np.random.default_rng(11)
    m, F, J, sigma = 4, 32, 512, 1.7
    R = ch.covariances(noise_window(rng, m, F * J, sigma), m, F, 0, F, kind)
    p = np.real(np.trace(R, axis1=1, axis2=2)) / m
    assert np.max(np.abs(p / sigma ** 2 - 1.0)) < 0.15


def test_two_emitters_in_two_channels_are_separated():
    """The motivating case: two transmitters at different frequencies from different directions.  Each channel's n = 1
    MUSIC peak is its own emitter; the plain covariance of the same window holds both and its n = 1 peak is neither
    reliably."""
    m, F, J, K = 4, 64, 64, 360
    lam0 = ch.C0 / FC
    pos = ch.ula_pos(m, lam0)
    chans, degs = (6, 58), (50.0, 120.0)
    tables = np.stack([ch.table(pos, l, K) for l in ch.wavelengths(F, 0, F, FC, FS)])
    md = cmp.modes()
    hits = {0: 0, 1: 0}
    plain_hits = 0
    trials = 20
    for seed in range(trials):
        rng = np.random.default_rng(100 + seed)
        x = ch.two_emitters(rng, pos, FC, FS, F, F * J, chans, degs, amps=(1.0, 1.0))
        R = ch.covariances(x, m, F, 0, F, "hann")
        for i, (c, deg) in enumerate(zip(chans, degs)):
            r = cmp.work_R(R[c], md, tables[c], None, 1, J)
            hits[i] += abs(float(r["angles"][0]) - deg) <= 1.0
        plain = cmp.work_R(co.covariance(x[None, :], m)[0], md, ch.table(pos, lam0, K), None, 1, F * J)
        a = float(plain["angles"][0])
        plain_hits += min(abs(a - degs[0]), abs(a - degs[1])) <= 1.0
    assert hits[0] == trials and hits[1] == trials
    assert plain_hits <= trials // 2  # two equal sources in one R with n = 1: a blend


def test_wideband_source_needs_per_channel_tables():
    """One source white across a 14 % band near end-fire of a line array (lambda / 2 at the top of the band, so that no
    channel has a grating lobe): with each channel's own table the channel estimates are unbiased; with the
    centre-frequency table their error grows with |f_c|; the incoherent combine is at least as good as the median
    single channel."""
    m, F, J, K = 4, 16, 256, 1440
    lam0 = ch.C0 / FC
    pos = ch.ula_pos(m, ch.C0 / (FC + FS / 2))
    deg = 20.0
    # the bin at -fs / 2 and its neighbours hold both band edges (the spectrum wraps there): a range that leaves them out
    first, C = F // 2 + 2, F - 3
    off = ch.offsets(F, first, C, FS)
    tables = np.stack([ch.table(pos, l, K) for l in ch.wavelengths(F, first, C, FC, FS)])
    centre = ch.table(pos, lam0, K)
    md = cmp.modes()
    trials = 12
    err_own = np.zeros((trials, C))
    err_centre = np.zeros((trials, C))
    err_inc = np.zeros(trials)
    for s in range(trials):
        rng = np.random.default_rng(500 + s)
        x = ch.white_source(rng, pos, FC, FS, F * J, deg)
        R = ch.covariances(x, m, F, first, C, "hann")
        for c in range(C):
            err_own[s, c] = float(cmp.work_R(R[c], md, tables[c], None, 1, J)["angles"][0]) - deg
            err_centre[s, c] = float(cmp.work_R(R[c], md, centre, None, 1, J)["angles"][0]) - deg
        _, (ang, _, _) = ch.incoherent(R, tables, 1)
        err_inc[s] = float(ang[0]) - deg
    bias_own, bias_centre = err_own.mean(axis=0), err_centre.mean(axis=0)
    assert np.max(np.abs(bias_own)) <= 0.5
    steps = np.unique(np.abs(off))
    grown = np.array([np.mean(np.abs(bias_centre[np.abs(off) == f])) for f in steps])
    assert grown[0] <= 0.25 and np.all(np.diff(grown) > 0) and grown[-1] >= 5.0
    assert np.all(np.sign(bias_centre[off > 0.3 * FS]) != np.sign(bias_centre[off < -0.3 * FS]))
    rms = lambda e: math.sqrt(float(np.mean(np.square(e))))
    assert rms(err_inc) <= np.median([rms(err_own[:, c]) for c in range(C)])


def test_mdl_counts_occupied_and_empty_channels_from_the_segments():
    """MDL with J looks per channel: 1 in the two occupied channels, 0 in channels holding noise only"""
    m, F, J = 4, 32, 128
    pos = ch.ula_pos(m, ch.C0 / FC)
    rng = np.random.default_rng(77)
    chans = (3, 27)
    x = ch.two_emitters(rng, pos, FC, FS, F, F * J, chans, (40.0, 130.0), noise=0.1, walk=0.002)
    R = ch.covariances(x, m, F, 0, F, "hann")
    counts = [so.estimate_source_count(np.linalg.eigvalsh(R[c]), J, 2, "mdl")[0] for c in range(F)]
    # the Hann main lobe puts a tone at a bin centre into its two neighbours as well
    near = {(c + d) % F for c in chans for d in (-1, 0, 1)}
    assert all(counts[c] == 1 for c in chans)
    assert all(counts[c] == 0 for c in range(F) if c not in near)
