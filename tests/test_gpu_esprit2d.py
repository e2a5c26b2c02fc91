"""GPU: 2-D ESPRIT on az-el handles (MUSIC_B200_PEAKS_ESPRIT on a planar lattice) against its fp64 definition
(tests/esprit2d_oracle.py, LAPACK eigh / solve / eig), against the truth, against the grid peak modes, through both
entry points and the C++ block, and every refusal.

Az-el handles have no R port, so the parity windows are quantised: samples on a 2^-9 grid below 4 in magnitude and
N = 512 snapshots make every product and sum of the covariance exact in fp64, so the host's R is the device's bit for
bit (calibration gains are signed powers of two, or j times one, so the correction is exact too)."""
import math
import struct

import numpy as np
import pytest

from gr_baz_b200 import _capi
from gr_baz_b200.music_doa_azel import music_doa_azel

import azel_oracle as ao
import esprit2d_oracle as eo
import gpu_harness as gh
from helpers import LAM

pytestmark = pytest.mark.gpu

ESPRIT = 3
H = 0.5 * LAM
N = 512
DIR_TOL = 2e-5    # degrees on the sphere, plus one float32 ulp per angle where the fp64 value sits on a rounding boundary
L_RTOL = 1e-5
GAP = 1e-9        # eigengap guard: (lambda_{M-d} - lambda_{M-d-1}) / lambda_max below this leaves E_s ill-determined
PEAKS = ("levels", "bins")


def lattices():
    c, s = math.cos(math.radians(33.0)), math.sin(math.radians(33.0))
    r = lambda v: (c * v[0] - s * v[1], s * v[0] + c * v[1])
    return {"2x2": eo.lattice_xyz(2, 2, (H, 0.0), (0.0, H)),
            "2x4": ao.ura_xyz(4, 2, LAM),
            "3x3": eo.lattice_xyz(3, 3, (H, 0.0), (0.0, H), p0=(0.4, -0.3, 0.1)),
            "4x4": ao.ura_xyz(4, 4, LAM),
            "rotated_skew3x4": eo.lattice_xyz(3, 4, r((0.9 * H, 0.0)), r((0.35 * H, 0.85 * H)))}


def handle(pos, n, grid, mode="esprit", rule="fixed", gains=None):
    blk = music_doa_azel(pos.shape[0], n, pos.shape[0] * N, grid.n_az, grid.n_el, (grid.el_lo, grid.el_hi), pos, LAM)
    if rule != "fixed":
        blk.set_source_rule(rule)
    if gains is not None:
        blk.set_calibration(gains)
    if mode is not None:
        blk.set_peak_mode(mode, 0)
    return blk


def quantised_windows(pos, n_of, seed, noise=0.1, el_range=(0.0, 88.0)):
    x, truth = ao.windows(pos, LAM, n_of, seed, N, el_range=el_range, noise=noise)
    q = 2.0 ** -9
    x = (np.round(x.real.astype(np.float64) / q) * q + 1j * np.round(x.imag.astype(np.float64) / q) * q).astype(np.complex64)
    assert np.max(np.abs(x.real)) < 4 and np.max(np.abs(x.imag)) < 4
    return x, truth


def host_R(x, m, gains=None):
    X = x.reshape(-1, m).astype(np.complex128)
    R = X.T @ X.conj() / X.shape[0]
    if gains is not None:
        c = 1.0 / np.asarray(gains, np.complex128)
        R = (c[:, None] * R) * np.conj(c)[None, :]
    return R


def chord_deg(a, b):
    u = lambda t: np.array([math.cos(math.radians(t[1])) * math.cos(math.radians(t[0])),
                            math.cos(math.radians(t[1])) * math.sin(math.radians(t[0])), math.sin(math.radians(t[1]))])
    return math.degrees(float(np.linalg.norm(u(a) - u(b))))


def near_half_bin(az, el, grid):
    fa = az * grid.n_az / 360.0 + 0.5
    fe = (el - grid.el_lo) * (grid.n_el - 1) / (grid.el_hi - grid.el_lo) + 0.5 if grid.n_el > 1 else 0.25
    return abs(fa - round(fa)) < 1e-6 or abs(fe - round(fe)) < 1e-6


@pytest.mark.parametrize("name", sorted(lattices()))
def test_parity_with_oracle(name):
    """directions within DIR_TOL of the oracle's on the sphere, levels within 1e-5, bins equal except at half-bin ties,
    unfilled slots (0, 0, 0, -1); under FIXED and MDL, with and without calibration"""
    pos = lattices()[name]
    m = pos.shape[0]
    mx, my, _, _ = eo.lattice(pos, LAM)
    dmax = eo.d_max(mx, my)
    grid = ao.Grid(360, 91, 0.0, 90.0)
    n = min(2, dmax)
    plan = [min(S, n) for S in (1, 2, 2, 1, 2, 2, 2, 1)] * 4
    x, _ = quantised_windows(pos, plan, 100 + m)
    gains = np.array([[1, 2, -1, 0.5, 1j, -2, 1, -0.5j][i % 8] for i in range(m)], np.complex128)
    compared = skipped = 0
    for rule in ("fixed", "mdl"):
        for g in (None, gains):
            blk = handle(pos, n, grid, rule=rule, gains=g)
            out, _ = gh.device_call(blk, x, PEAKS + ("counts",))
            blk.close()
            for w in range(len(x)):
                d = n if rule == "fixed" else int(out["counts"][w])
                ctx = (name, rule, g is not None, w, d)
                R = host_R(x[w], m, g)
                ev = np.linalg.eigvalsh(R)
                if 0 < d < m and (ev[m - d] - ev[m - d - 1]) / ev[-1] < GAP:
                    skipped += 1
                    continue
                ref = eo.work_R(R, d, pos, LAM, grid, n)
                az, el, lv, bn = out["azimuth"][w], out["elevation"][w], out["levels"][w], out["bins"][w]
                f = int(np.sum(ref["bins"] >= 0))
                assert np.array_equal(bn >= 0, ref["bins"] >= 0), (ctx, bn, ref["bins"])
                assert np.all(az[f:] == 0) and np.all(el[f:] == 0) and np.all(lv[f:] == 0), ctx
                src = ref["sources"]
                for i in range(f):
                    # a slot pair whose fp64 levels are this close may be ordered either way: compare as a set
                    j = i
                    if any(abs(src[i][0] - src[k][0]) <= 1e-9 * src[i][0] for k in range(f) if k != i):
                        j = min(range(f), key=lambda k: chord_deg((az[i], el[i]), (src[k][1], src[k][2])))
                    ra, re_ = float(ref["az"][j]), float(ref["el"][j])
                    tol = DIR_TOL + float(np.spacing(np.float32(max(ra, 1.0)))) + float(np.spacing(np.float32(max(abs(re_), 1.0))))
                    assert chord_deg((float(az[i]), float(el[i])), (ra, re_)) <= tol, (ctx, i, az, el, ref["az"], ref["el"])
                    assert abs(float(lv[i]) - float(ref["levels"][j])) <= L_RTOL * float(ref["levels"][j]), (ctx, i, lv, ref["levels"])
                    if bn[i] != ref["bins"][j]:
                        assert near_half_bin(src[j][1], src[j][2], grid), (ctx, i, bn, ref["bins"])
                    compared += 1
    print("%s: %d slots compared, %d windows skipped at the eigengap guard" % (name, compared, skipped))
    assert skipped <= 0.02 * 4 * len(x), skipped


@pytest.mark.parametrize("name", sorted(lattices()))
def test_noiseless_truth(name):
    """noiseless windows, d = 1 .. min(d_max, 3): every source within 1e-3 degrees of the truth"""
    pos = lattices()[name]
    m = pos.shape[0]
    mx, my, _, _ = eo.lattice(pos, LAM)
    n = min(eo.d_max(mx, my), 3, m - 1)
    grid = ao.Grid(360, 91, 0.0, 90.0)
    x, truth = ao.windows(pos, LAM, [1 + w % n for w in range(24)], 7 + m, N, el_range=(0.0, 85.0), noise=0.0)
    for S in range(1, n + 1):
        idx = [w for w in range(len(x)) if len(truth[w]) == S]
        blk = handle(pos, S, grid)
        out, _ = gh.device_call(blk, x[idx])
        blk.close()
        for r, w in enumerate(idx):
            got = list(zip(out["azimuth"][r].astype(float), out["elevation"][r].astype(float)))
            errs = eo.matched_errors(got, truth[w])
            assert max(errs) <= 1e-3, (name, w, got, truth[w])


def test_accuracy_against_grid_modes():
    """4 x 4 URA, two sources at 20 dB per element, 360 x 46 grid: ESPRIT's RMS direction error below TOP_BINS's and
    within eo.RMS_FACTOR of LOCAL_MAXIMA + NEWTON's (the bounds test_esprit2d_oracle.test_accuracy_model sets)"""
    pos = ao.ura_xyz(4, 4, LAM)
    grid = ao.Grid(360, 46, 0.0, 90.0)
    x, truth = ao.windows(pos, LAM, [2] * 200, 11, N, el_range=(5.0, 80.0))
    rms = {}
    for key, mode, refine in (("esprit", "esprit", False), ("top_bins", "top_bins", False), ("newton", "local_maxima", True)):
        blk = handle(pos, 2, grid, mode=mode)
        if refine:
            blk.set_refine(True)
        out, _ = gh.device_call(blk, x)
        blk.close()
        errs = []
        for w in range(len(x)):
            errs += eo.matched_errors(list(zip(out["azimuth"][w].astype(float), out["elevation"][w].astype(float))), truth[w])
        rms[key] = math.sqrt(float(np.mean(np.square(errs))))
    print("RMS direction error (degrees):", rms)
    assert rms["esprit"] < rms["top_bins"], rms
    assert rms["esprit"] <= eo.RMS_FACTOR * rms["newton"], rms


def test_entries_launches_and_spectrum():
    """host and device entries byte-identical; covariance + eigensolver + ESPRIT per call (+1 source count, +1 scan
    with the spectrum), no decode; the spectrum bit-identical to a TOP_BINS handle's"""
    pos = ao.ura_xyz(4, 2, LAM)
    grid = ao.Grid(72, 19, 0.0, 90.0)
    x, _ = ao.windows(pos, LAM, [1, 2, 2, 0, 2] * 4, 21, N)
    for rule, spectrum, want in (("fixed", False, 3), ("mdl", False, 4), ("fixed", True, 4), ("mdl", True, 5)):
        blk = handle(pos, 2, grid, rule=rule)
        dev, launches = gh.device_call(blk, x, PEAKS + (("spectrum",) if spectrum else ()))
        assert launches == want, (rule, spectrum, launches)
        cnt, _ = gh.device_call(blk, x, PEAKS + ("counts",))
        host = gh.host_call(blk, x, spectrum=spectrum)
        for k in ("azimuth", "elevation", "levels", "bins") + (("spectrum",) if spectrum else ()):
            assert np.array_equal(host[k], dev[k]) and (k == "spectrum" or np.array_equal(cnt[k], dev[k])), (rule, k)
        assert np.array_equal(host["counts"], cnt["counts"]), rule
        blk.close()
        if spectrum:
            top = handle(pos, 2, grid, mode="top_bins", rule=rule)
            ref, _ = gh.device_call(top, x, ("spectrum",))
            top.close()
            assert np.array_equal(ref["spectrum"], dev["spectrum"]), rule


def test_retunes_and_set_table():
    """lattice -> UCA fails the call (no fall-back), -> lattice again equals a fresh handle; set_table() fails the call
    until a lattice geometry is installed again"""
    pos = ao.ura_xyz(4, 4, LAM)
    grid = ao.Grid(72, 19, 0.0, 90.0)
    x, _ = ao.windows(pos, LAM, [2] * 6, 31, N)
    fresh = handle(pos, 2, grid)
    ref, _ = gh.device_call(fresh, x, PEAKS)
    fresh.close()
    blk = handle(pos, 2, grid)
    blk.set_array_geometry(ao.uca_xyz(16, LAM), LAM)
    with pytest.raises(_capi.MusicB200Error):
        gh.device_call(blk, x, PEAKS)
    with pytest.raises(_capi.MusicB200Error):
        blk.work(len(x), [x], [np.zeros((len(x), 2), np.float32), np.zeros((len(x), 2), np.float32)])
    blk.set_array_geometry(pos, LAM)
    got, _ = gh.device_call(blk, x, PEAKS)
    for k in ("azimuth", "elevation", "levels", "bins"):
        assert np.array_equal(got[k], ref[k]), k
    blk.set_array_response(blk.array_response_c64())
    with pytest.raises(_capi.MusicB200Error):
        gh.device_call(blk, x, PEAKS)
    blk.set_array_geometry(pos, LAM)
    got, _ = gh.device_call(blk, x, PEAKS)
    assert np.array_equal(got["azimuth"], ref["azimuth"])
    blk.set_peak_mode("top_bins", 0)  # the grid modes still run on the same handle
    gh.device_call(blk, x, PEAKS)
    blk.close()


def test_refusals():
    L = _capi.load()
    EINVAL = _capi.EINVAL
    grid = ao.Grid(36, 10, 0.0, 90.0)
    pos = ao.ura_xyz(4, 4, LAM)
    blk = handle(pos, 2, grid, mode=None)
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 1) == EINVAL  # exclusion_bins must be 0
    for kind, loading in (("mvdr", 0.01), ("bartlett", 0.0)):
        blk.set_estimator(kind, loading)
        assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
        blk.set_estimator("music", 0.0)
    blk.set_refine(True)
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
    blk.set_refine(False)
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == _capi.OK
    assert L.music_b200_set_estimator(blk._h, 1, 0.01) == EINVAL
    assert L.music_b200_set_estimator(blk._h, 2, 0.0) == EINVAL
    assert L.music_b200_set_refine(blk._h, 1) == EINVAL
    for mode in (2, 4, 5):  # ROOTS, DML, MANIFOLD stay refused on az-el handles, lattice or not
        assert L.music_b200_set_peak_mode(blk._h, mode, 0) == EINVAL, mode
    blk.close()
    # n > d_max: a 2 x 2 lattice resolves at most 2 sources
    sq = eo.lattice_xyz(2, 2, (H, 0.0), (0.0, H))
    blk = handle(sq, 3, grid, mode=None)
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
    assert "at most 2" in L.music_b200_last_error(blk._h).decode()
    blk.close()
    # geometries that fail the lattice condition, and a set_table() table
    for bad in (ao.uca_xyz(8, LAM), ao.uca_xyz(8, LAM, alternate_z=True), np.c_[np.arange(8) * H, np.zeros(8), np.zeros(8)]):
        blk = handle(bad, 1, grid, mode=None)
        assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
        assert "lattice" in L.music_b200_last_error(blk._h).decode()
        blk.close()
    blk = handle(pos, 1, grid, mode=None)
    blk.set_array_response(blk.array_response_c64())
    assert L.music_b200_set_peak_mode(blk._h, ESPRIT, 0) == EINVAL
    blk.close()


def test_cpp_block():
    """the C++ az-el block with peak mode 3 and MDL equals the Python block"""
    pos = ao.ura_xyz(4, 4, LAM)
    m, n, Wn = 16, 2, 12
    grid = ao.Grid(72, 19, 0.0, 90.0)
    x, _ = ao.windows(pos, LAM, [n] * Wn, 55, N)
    c = gh.run_cpp_block("test_block_azel", struct.pack("<10I", m, n, m * N, grid.n_az, grid.n_el, Wn, ESPRIT, 0, 1, 0) +
                         struct.pack("<3d", grid.el_lo, grid.el_hi, LAM), [np.ascontiguousarray(pos), x],
                         [(k, np.float32, Wn * size) for k, size in (("azimuth", n), ("elevation", n), ("levels", n),
                                                                     ("spectrum", grid.K), ("bins", n), ("counts", 1))])
    got = {k: v.reshape(Wn, -1) for k, v in c.items()}
    py = handle(pos, n, grid, rule="mdl")
    outs = [np.zeros((Wn, n), np.float32) for _ in range(3)] + [np.zeros((Wn, grid.K), np.float32)]
    py.work(Wn, [x], outs)
    for k, v in zip(("azimuth", "elevation", "levels", "spectrum"), outs):
        assert np.array_equal(got[k], v), k
    assert np.array_equal(got["bins"].view(np.int32), py.last_bins()), "bins"
    assert np.all(py.last_bins() >= 0)
    py.close()
