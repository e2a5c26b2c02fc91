"""GPU tests of the co-array handle (music_b200_create_coarray, include/music_b200.h) against tests/coarray_oracle.py:
R_ss and the peaks on seeded and exact-covariance windows, every accepted entry, the unfused dispatch at Mv = 4 and 8,
the calibration workflow, every refusal, the retune, and the C++ block."""
import struct

import numpy as np
import pytest
import torch

import coarray_oracle as co
import gpu_harness as gh
import helpers
import integration_oracle as io
from calibration_oracle import correct
from gr_baz_b200 import _capi
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_coarray import music_doa_coarray
from oracle import music_oracle as mo

pytestmark = pytest.mark.gpu

MRA4 = [0, 1, 4, 6]
NESTED6 = [0, 1, 2, 3, 7, 11]
NESTED8 = [0, 1, 2, 3, 4, 9, 14, 19]
LAM = 1.0
STEP = (0.5, 0.0)
DEV = gh.DEV


def make(p, n, snaps, K=360, mv=0, mode=None, refine=False):
    blk = music_doa_coarray(len(p), n, len(p) * snaps, K, p, STEP, LAM, mv)
    if mode is not None:
        blk.set_peak_mode(mode)
    if refine:
        blk.set_refine(True)
    return blk


def windows(p, deg, W, seed, snr_db=20.0, snaps=1024):
    """W windows of uncorrelated complex Gaussian sources at the angles deg (same in every window), snr_db each over
    unit noise, on the physical elements of p"""
    rng = np.random.default_rng(seed)
    m, d = len(p), len(deg)
    A = co.steering(co.physical_positions(p, STEP), LAM, np.asarray(deg, np.float64)).T  # (m, d)
    amp = 10.0 ** (snr_db / 20.0)
    S = amp * (rng.standard_normal((W, d, snaps)) + 1j * rng.standard_normal((W, d, snaps))) / np.sqrt(2.0)
    X = np.einsum("md,wdn->wmn", A, S) + (rng.standard_normal((W, m, snaps)) + 1j * rng.standard_normal((W, m, snaps))) / np.sqrt(2.0)
    return np.ascontiguousarray(X.transpose(0, 2, 1).reshape(W, -1).astype(np.complex64))


def physical_R(x, m):
    return np.stack([mo.covariance(w, m) for w in x])


def dev_call(blk, x, spectrum=False, R=True, counts=False):
    """process_device (process_device_counts with counts) on the windows x: numpy outputs, R as complex [W][Mv][Mv]"""
    W, n, K, mv = x.shape[0], blk.n, blk.resolution, blk.virtual_size
    f32, f64, i32 = torch.float32, torch.float64, torch.int32
    o = {"angles": torch.full((W, n), -7, dtype=f32, device=DEV), "levels": torch.full((W, n), -7, dtype=f32, device=DEV),
         "bins": torch.full((W, n), -7, dtype=i32, device=DEV)}
    if spectrum:
        o["spectrum"] = torch.full((W, K), -7, dtype=f32, device=DEV)
    if R:
        o["R"] = torch.full((W, mv, mv, 2), np.nan, dtype=f64, device=DEV)
        o["eigvals"] = torch.full((W, mv), np.nan, dtype=f64, device=DEV)
    if counts:
        o["counts"] = torch.full((W,), -7, dtype=i32, device=DEV)
    p = lambda k: o[k].data_ptr() if k in o else None
    d_in = torch.from_numpy(x.view(np.float32)).to(DEV)
    l0 = blk.launch_count()
    blk.process_device(d_in.data_ptr(), W, p("angles"), p("levels"), p("spectrum"), p("bins"), stream=gh.stream(), d_R=p("R"),
                       d_eigvals=p("eigvals"), d_counts=p("counts"))
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    if R:
        out["R"] = out["R"][..., 0] + 1j * out["R"][..., 1]
    return out, blk.launch_count() - l0


def rel(got, ref):
    return float(np.max(np.abs(got - ref)) / np.max(np.abs(ref)))


def sorted_close(got, ref, tol):
    return float(np.max(np.abs(np.sort(np.asarray(got, np.float64)) - np.sort(np.asarray(ref, np.float64))))) <= tol


# ---- R_ss against the oracle ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [MRA4, NESTED8])
@pytest.mark.parametrize("calibrated", [False, True])
@pytest.mark.parametrize("alpha", [0.0, 0.8])
def test_R_output(p, calibrated, alpha):
    m, W = len(p), 96
    n = co.resolve_mv(p) - 1
    x = windows(p, np.linspace(25.0, 155.0, n), W, 1 + m, snr_db=5.0, snaps=256)
    blk = make(p, n, 256, mode="esprit")
    R = physical_R(x, m)
    if calibrated:
        g = helpers.random_gains(np.random.default_rng(5), m)
        blk.set_calibration(g)
        R = correct(R, g)
    if alpha:
        blk.set_integration(alpha)
        R = io.integrate(R, alpha)[0]
    out, _ = dev_call(blk, x)
    mv = blk.virtual_size
    ref = co.smoothed_batch(R, p, mv)
    assert rel(out["R"], ref) <= 1e-12
    assert np.all(np.diagonal(out["R"], axis1=1, axis2=2).imag == 0.0)
    assert np.array_equal(out["R"], np.conj(np.transpose(out["R"], (0, 2, 1))))
    assert np.max(np.abs(out["eigvals"] - np.linalg.eigvalsh(ref))) <= 1e-10 * np.max(np.abs(ref))
    blk.close()


# ---- peaks on the GPU's own R_ss ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("p, n", [(MRA4, 6), (NESTED6, 9)])
@pytest.mark.parametrize("mode", ["esprit", "roots"])
def test_gridless_against_oracle(p, n, mode):
    W, K = 64, 3600
    x = windows(p, np.linspace(20.0, 160.0, n) + 1.3, W, 10 + n, snr_db=10.0, snaps=2048)
    blk = make(p, n, 2048, K=K, mode=mode)
    out, _ = dev_call(blk, x)
    solve = co.esprit if mode == "esprit" else co.roots
    for w in range(W):
        ref = solve(out["R"][w], STEP, LAM, K, n)
        assert sorted_close(out["angles"][w], ref["angles"], 1e-3), (w, out["angles"][w], ref["angles"])
        assert np.all(out["bins"][w] >= 0)
        for a, b in zip(np.sort(out["angles"][w]), np.sort(ref["angles"])):
            if not helpers.near_half(b, K):
                assert int(np.floor(a * K / 360.0 + 0.5)) % K == int(np.floor(b * K / 360.0 + 0.5)) % K
    blk.close()


@pytest.mark.parametrize("p, n", [(MRA4, 6), (NESTED8, 12)])
def test_grid_against_oracle(p, n):
    W, K = 32, 720
    x = windows(p, np.linspace(20.0, 160.0, n), W, 20 + n, snr_db=10.0, snaps=1024)
    blk = make(p, n, 1024, K=K)
    out, _ = dev_call(blk, x, spectrum=True)
    table = blk.array_response_c64().astype(np.complex128)
    mv = blk.virtual_size
    for w in range(W):
        V = np.linalg.eigh(out["R"][w])[1]
        G = V[:, : mv - n]
        P = 1.0 / np.sum(np.abs(table.conj() @ G) ** 2, axis=1)
        assert np.max(np.abs(out["spectrum"][w] - P) / P) <= 1e-5
        top = np.sort(P)[::-1][:n]
        assert np.max(np.abs(np.sort(P[out["bins"][w]])[::-1] - top) / top) <= 1e-9  # the top-n bins, up to near-ties
        assert np.max(np.abs(out["levels"][w] - P[out["bins"][w]]) / P[out["bins"][w]]) <= 1e-5
    blk.close()
    # NEWTON on the virtual ULA's analytic steering: every refined angle stays within a bin of its local maximum
    blk = make(p, n, 1024, K=K, mode="local_maxima", refine=True)
    out, _ = dev_call(blk, x)
    filled = out["bins"] >= 0
    assert np.all(np.isfinite(out["angles"])) and filled.any()
    d = co.circ(out["angles"][filled], out["bins"][filled] * 360.0 / K)
    assert np.max(d) <= 360.0 / K
    blk.close()


# ---- exact covariances: orthogonal tones ------------------------------------------------------------------------------
def tone_windows(p, deg, powers, sigma, snaps=1024):
    """one window whose sample covariance is exactly A P A^H + sigma^2 I before the float32 rounding of its samples:
    every source and every element's noise a tone of its own integer frequency over the window"""
    m, d = len(p), len(deg)
    t = np.arange(snaps)
    A = co.steering(co.physical_positions(p, STEP), LAM, np.asarray(deg)).T
    S = np.sqrt(np.asarray(powers))[:, None] * np.exp(2j * np.pi * np.outer(np.arange(1, d + 1) * 7, t) / snaps)
    Nz = sigma * np.exp(2j * np.pi * np.outer(np.arange(1, m + 1) * 7 + 3, t) / snaps)
    X = A @ S + Nz
    return np.ascontiguousarray(X.T.reshape(1, -1).astype(np.complex64))


@pytest.mark.parametrize("mode", ["esprit", "roots"])
def test_exact_covariance_six_sources_on_four_antennas(mode):
    K, n = 3600, 6
    rng = np.random.default_rng(3)
    xs, truths = [], []
    for _ in range(8):
        deg = np.sort(rng.uniform(20.0, 160.0, n))
        while np.min(np.diff(deg)) < 12.0:
            deg = np.sort(rng.uniform(20.0, 160.0, n))
        xs.append(tone_windows(MRA4, deg, rng.uniform(0.5, 2.0, n), 0.3))
        truths.append(deg)
    x = np.concatenate(xs)
    blk = make(MRA4, n, 1024, K=K, mode=mode)
    out, _ = dev_call(blk, x)
    solve = co.esprit if mode == "esprit" else co.roots
    for w, deg in enumerate(truths):
        Rss = co.smoothed(mo.covariance(x[w], 4), MRA4, 7)  # the same float32 windows, fp64
        ref = solve(Rss, STEP, LAM, K, n)
        e_ref = co.worst_error(ref["angles"], deg)
        ulp = 2.0 * float(np.spacing(np.float32(180.0)))
        # the float32 samples move the angles by e_ref; the GPU's R_ss differs from the oracle's by summation order only
        assert sorted_close(out["angles"][w], ref["angles"], ulp + 1e-6), (out["angles"][w], ref["angles"])
        assert co.worst_error(out["angles"][w], deg) <= e_ref + ulp + 1e-6
        assert e_ref <= 1e-3
    blk.close()


# ---- seeded statistical cases -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p, n, snaps, W", [(MRA4, 6, 4096, 40), (NESTED6, 9, 2048, 30)])
def test_statistical(p, n, snaps, W):
    rng = np.random.default_rng(50 + n)
    deg = np.linspace(25.0, 155.0, n) + rng.uniform(-3.0, 3.0, n)
    x = windows(p, deg, W, 60 + n, snr_db=10.0, snaps=snaps)
    blk = make(p, n, snaps, K=3600, mode="esprit")
    out, _ = dev_call(blk, x, R=False)
    mv = blk.virtual_size
    got = np.array([co.worst_error(out["angles"][w], deg) for w in range(W)])
    ref = np.array([co.worst_error(co.esprit(co.smoothed(mo.covariance(x[w], len(p)), p, mv), STEP, LAM, 3600, n)["angles"], deg)
                    for w in range(W)])
    assert np.median(got) <= np.median(ref) + 1e-3 and np.max(got) <= np.max(ref) + 1e-3, (np.median(got), np.max(got), ref)
    blk.close()


def test_more_sources_than_antennas():
    t = np.ones((360, 4), np.complex64)
    with pytest.raises(ValueError):
        music_doa(4, 6, 4 * 1024, t, 360)
    blk = make(MRA4, 6, 1024, mode="esprit")
    assert blk.virtual_size == 7
    out, _ = dev_call(blk, windows(MRA4, np.linspace(30, 150, 6), 4, 9), R=False)
    assert np.all(out["bins"] >= 0)
    blk.close()


# ---- entries ------------------------------------------------------------------------------------------------------------
def test_entries_give_the_device_bits():
    p, n, W, snaps = NESTED6, 7, 50, 512
    x = windows(p, np.linspace(30.0, 150.0, n), W, 77, snaps=snaps)
    blk = make(p, n, snaps, K=720, mode="esprit")
    ref, _ = dev_call(blk, x, R=False)
    cnt, _ = dev_call(blk, x, R=False, counts=True)
    assert np.all(cnt["counts"] == n)
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(cnt[k], ref[k])
    host = gh.host_call(blk, x)
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(host[k], ref[k]), k
    # host chunk splits
    a, l = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    for s, e in ((0, 17), (17, 50)):
        blk.work(e - s, [np.ascontiguousarray(x[s:e])], [a[s:e], l[s:e]])
    assert np.array_equal(a, ref["angles"]) and np.array_equal(l, ref["levels"])
    # planar host and device entries: the planar covariance sums in another order
    streams = helpers.antenna_streams(x, len(p))
    pa, pl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    blk.work_planar(W, streams, [pa, pl])
    assert np.max(np.abs(pa - ref["angles"])) <= 1e-3
    pd, _ = gh.planar_device_call(blk, streams, snaps, W, ("levels", "bins"))
    assert np.max(np.abs(pd["angles"] - ref["angles"])) <= 1e-3
    # tracks under FIXED variance: the same peaks
    blk.set_tracking("fixed", max_tracks=16)
    st = torch.full((W, n), -7, dtype=torch.int32, device=DEV)
    ang = torch.full((W, n), -7, dtype=torch.float32, device=DEV)
    d_in = torch.from_numpy(x.view(np.float32)).to(DEV)
    blk.process_device_tracks(d_in.data_ptr(), W, ang.data_ptr(), st.data_ptr(), stream=gh.stream())
    torch.cuda.synchronize()
    assert np.array_equal(ang.cpu().numpy(), ref["angles"])
    assert (st.cpu().numpy() >= 0).any()
    # reducers and the table
    mean, _, _ = blk.reduce_angles(ref["angles"])
    assert mean.shape == (n,)
    assert blk.array_response_c64().shape == (720, 12)
    blk.close()


def test_integration_carries_across_calls():
    p, n, W = MRA4, 5, 80
    x = windows(p, np.linspace(30.0, 150.0, n), W, 31, snr_db=0.0, snaps=128)
    one = make(p, n, 128, mode="esprit")
    one.set_integration(0.9)
    a, _ = dev_call(one, x)
    two = make(p, n, 128, mode="esprit")
    two.set_integration(0.9)
    b1, _ = dev_call(two, x[:33])
    b2, _ = dev_call(two, x[33:])
    assert rel(np.concatenate([b1["R"], b2["R"]]), a["R"]) <= 1e-13
    assert rel(a["R"], co.smoothed_batch(io.integrate(physical_R(x, 4), 0.9)[0], p, 7)) <= 1e-12
    one.close()
    two.close()


@pytest.mark.parametrize("p, mv", [([0, 1, 3], 0), ([0, 1, 2, 5, 8], 8)])
def test_virtual_sizes_of_the_fused_kernels_run_unfused(p, mv):
    # n = 1, TOP_BINS, MUSIC, a peak-only call: what a plain handle of 4 or 8 elements runs in one fused launch
    m, W, K = len(p), 64, 360
    blk = make(p, 1, 1024, K=K, mv=mv)
    Mv = blk.virtual_size
    assert Mv == (4 if mv == 0 else 8)
    x = windows(p, [63.0], W, 40 + m)
    out, launches = dev_call(blk, x, R=False)
    assert launches >= 3, launches
    full, _ = dev_call(blk, x)
    assert np.array_equal(out["bins"], full["bins"]) and np.array_equal(out["angles"], full["angles"])
    assert rel(full["R"], co.smoothed_batch(physical_R(x, m), p, Mv)) <= 1e-12
    table = blk.array_response_c64().astype(np.complex128)
    for w in range(W):
        G = np.linalg.eigh(full["R"][w])[1][:, : Mv - 1]
        P = 1.0 / np.sum(np.abs(table.conj() @ G) ** 2, axis=1)
        assert P[out["bins"][w, 0]] >= (1.0 - 1e-9) * np.max(P)
    blk.close()
    n = Mv - 1
    blk = make(p, n, 1024, K=3600, mv=mv, mode="esprit")
    x = windows(p, np.linspace(30.0, 150.0, n), 16, 41 + m)
    out, _ = dev_call(blk, x)
    for w in range(16):
        assert sorted_close(out["angles"][w], co.esprit(out["R"][w], STEP, LAM, 3600, n)["angles"], 1e-3)
    blk.close()


def test_virtual_table_is_the_plain_ula_table():
    blk = make(NESTED6, 3, 64, K=720)
    vpos = co.virtual_positions(STEP, 12)
    plain = music_doa(12, 1, 12 * 64, np.ones((720, 12), np.complex64), 720)
    plain.set_array_geometry(vpos, LAM)
    assert np.array_equal(blk.array_response_c64(), plain.array_response_c64())
    blk.set_array_geometry((0.3, 0.1), 0.8)
    plain.set_array_geometry(co.virtual_positions((0.3, 0.1), 12), 0.8)
    assert np.array_equal(blk.array_response_c64(), plain.array_response_c64())
    blk.close()
    plain.close()


# ---- calibration workflow -------------------------------------------------------------------------------------------------
def test_calibration_from_a_plain_handle():
    p, n, W, snaps, K = MRA4, 5, 24, 2048, 360
    g = helpers.random_gains(np.random.default_rng(8), 4)
    deg = np.linspace(30.0, 150.0, n) + 1.7
    x = helpers.corrupt(windows(p, deg, W, 81, snaps=snaps), g)
    blk = make(p, n, snaps, K=K, mode="esprit")
    raw, _ = dev_call(blk, x, R=False)
    assert max(co.worst_error(raw["angles"][w], deg) for w in range(W)) > 360.0 / K
    plain = music_doa(4, 1, 4 * snaps, np.ones((K, 4), np.complex64), K)
    plain.set_array_geometry(co.physical_positions(p, STEP), LAM)
    cal = helpers.corrupt(windows(p, [70.0], 16, 82, snaps=snaps), g)
    gains, _, _ = plain.calibrate(cal, 70.0)
    blk.set_calibration(gains)
    fixed, _ = dev_call(blk, x, R=False)
    assert max(co.worst_error(fixed["angles"][w], deg) for w in range(W)) <= 360.0 / K
    assert np.allclose(blk.calibration(), gains)
    blk.close()
    plain.close()


# ---- refusals and the retune ----------------------------------------------------------------------------------------------
def test_refusals():
    p, n, W, snaps = MRA4, 5, 8, 256
    x = windows(p, np.linspace(30.0, 150.0, n), W, 90, snaps=snaps)
    fresh = make(p, n, snaps, mode="esprit")
    ref, _ = dev_call(fresh, x, R=False)
    fresh.close()
    blk = make(p, n, snaps)
    E = _capi.MusicB200Error
    for first in ("esprit", "local_maxima"):
        blk.set_peak_mode(first)
        blk.set_refine(first == "local_maxima")
        for kind in ("mvdr", "bartlett", "iaa"):
            with pytest.raises(E):
                blk.set_estimator(kind, 0.1 if kind != "bartlett" else 0.0)
        blk.set_refine(False)
    for mode in ("dml", "wsf", "manifold"):
        with pytest.raises(E):
            blk.set_peak_mode(mode)
    for rule in ("mdl", "aic"):
        with pytest.raises(E):
            blk.set_source_rule(rule)
    with pytest.raises(E):
        blk.set_refine("joint")
    with pytest.raises(E):
        blk.set_beamformer("das")
    with pytest.raises(E):
        blk.set_tracking("crb")
    d_in = torch.from_numpy(x.view(np.float32)).to(DEV)
    f = lambda shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device=DEV).data_ptr()
    with pytest.raises(E):
        blk.process_device_crb(d_in.data_ptr(), W, f((W, n)), f((W, n)), stream=gh.stream())
    with pytest.raises(E):
        blk.process_device_beams(d_in.data_ptr(), W, f((W, n)), d_weights=f((W, n, 4, 2), torch.float64), stream=gh.stream())
    blk.set_tracking("fixed")
    with pytest.raises(E):
        blk.process_device_tracks(d_in.data_ptr(), W, f((W, n)), f((W, n), torch.int32), d_std=f((W, n)), stream=gh.stream())
    blk.set_tracking("off")
    with pytest.raises(E):
        blk.calib_reset()
    with pytest.raises(E):
        blk.calib_accumulate(x)
    with pytest.raises(E):
        blk.calib_accumulate_device(d_in.data_ptr(), W)
    with pytest.raises(E):
        blk.calib_solve(70.0)
    with pytest.raises(E):
        blk.calib_blind_reset()
    with pytest.raises(E):
        blk.calib_blind_accumulate(x, 1)
    with pytest.raises(E):
        blk.calib_blind_solve(1)
    with pytest.raises(E):
        blk.set_array_response(np.ones((360, 4), np.complex64))
    pos = np.ascontiguousarray(co.physical_positions(p, STEP))
    assert blk._lib.music_b200_set_geometry(blk._h, pos.ctypes.data, LAM, None) == _capi.EINVAL
    with pytest.raises(E):
        blk.gather_create(W)
    with pytest.raises(E):
        blk.process_device_sharded([d_in.data_ptr()], W, [f((W, n))])
    # the refusals left the handle as it was
    blk.set_peak_mode("esprit")
    got, _ = dev_call(blk, x, R=False)
    for k in ("angles", "levels", "bins"):
        assert np.array_equal(got[k], ref[k])
    blk.close()


def test_retune_resets_integration_and_tracks():
    p, n, W = MRA4, 5, 20
    x1 = windows(p, np.linspace(30.0, 150.0, n), W, 91, snaps=256)
    x2 = windows(p, np.linspace(35.0, 145.0, n), W, 92, snaps=256)
    fresh = make(p, n, 256, mode="esprit")
    fresh.set_integration(0.9)
    ref, _ = dev_call(fresh, x2)
    fresh.close()
    blk = make(p, n, 256, mode="esprit")
    blk.set_integration(0.9)
    blk.set_tracking("fixed")
    dev_call(blk, x1)
    d_in = torch.from_numpy(x1.view(np.float32)).to(DEV)
    st = torch.zeros((W, n), dtype=torch.int32, device=DEV)
    ang = torch.zeros((W, n), dtype=torch.float32, device=DEV)
    blk.process_device_tracks(d_in.data_ptr(), W, ang.data_ptr(), st.data_ptr(), stream=gh.stream())
    torch.cuda.synchronize()
    assert blk.tracks()[2] > 0
    blk.set_array_geometry(STEP, LAM)
    rows, _, nxt = blk.tracks()
    assert nxt == 0 and np.all(rows[:, 0] == -1)
    got, _ = dev_call(blk, x2)
    assert np.array_equal(got["R"], ref["R"])
    with pytest.raises(ValueError):
        make(p, 7, 256)  # n < Mv = 7
    with pytest.raises(_capi.MusicB200Error):
        blk.set_array_geometry((1.0, 0.0), LAM)  # |s| > lambda / 2
    blk.close()


# ---- the C++ block ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode, refine, calibrated", [(3, 0, 0), (1, 1, 1)])
def test_cpp_block(mode, refine, calibrated):
    p, n, W, snaps, K = NESTED6, 8, 24, 512, 720
    m = len(p)
    g = helpers.random_gains(np.random.default_rng(12), m)
    x = windows(p, np.linspace(30.0, 150.0, n), W, 93, snaps=snaps)
    blk = make(p, n, snaps, K=K, mode={3: "esprit", 1: "local_maxima"}[mode], refine=bool(refine))
    if calibrated:
        blk.set_calibration(g)
    ang, lvl, spec = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32), np.zeros((W, K), np.float32)
    blk.work(W, [x], [ang, lvl, spec])
    bins = blk.last_bins().copy()
    blk.close()
    header = struct.pack("<9I3d", m, n, m * snaps, W, K, 0, mode, refine, calibrated, STEP[0], STEP[1], LAM)
    gains = np.stack([g.real, g.imag], axis=1).astype(np.float64)
    out = gh.run_cpp_block("test_block_coarray", header, [np.asarray(p, np.int32), gains, x.view(np.float32)],
                           [("angles", np.float32, W * n), ("levels", np.float32, W * n), ("spectrum", np.float32, W * K),
                            ("bins", np.int32, W * n)])
    assert np.array_equal(out["angles"], ang.ravel())
    assert np.array_equal(out["levels"], lvl.ravel())
    assert np.array_equal(out["spectrum"], spec.ravel())
    assert np.array_equal(out["bins"], bins.ravel())
