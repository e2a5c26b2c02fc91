"""GPU: receiver calibration (music_b200_set_calibration, music_b200_calib_*) - the correction of R in every entry and
mode, and the gain estimate against its fp64 definition (tests/calibration_oracle.py) and against the truth."""
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200.music_doa_azel import music_doa_azel

import calibration_oracle as co
import gpu_harness as gh
import helpers
import refine_oracle as ro
from helpers import LAM, array_wl, corrupt, random_gains, ula

pytestmark = pytest.mark.gpu

ALL = ("levels", "bins", "spectrum", "P64", "R", "eigvals")
BEAMS = ("levels", "bins", "counts", "weights", "beams")


# ---- fixtures --------------------------------------------------------------------------------------------------------
def windows(pos, degs_per_window, seed, snaps, snr_db=20.0, azel=False):
    """complex64 windows [W][snaps * M]: unit complex noise plus independent sources at the given directions (degrees;
    (az, el) pairs when azel)"""
    rng = np.random.default_rng(seed)
    m = len(pos)
    xs = []
    for degs in degs_per_window:
        X = (rng.standard_normal((m, snaps)) + 1j * rng.standard_normal((m, snaps))) / math.sqrt(2.0)
        for t in degs:
            a = co.steering_azel(pos, LAM, *t) if azel else co.steering_1d(pos, LAM, t)
            s = (rng.standard_normal(snaps) + 1j * rng.standard_normal(snaps)) / math.sqrt(2.0)
            X += 10.0 ** (snr_db / 20.0) * a[:, None] * s[None, :]
        xs.append(X.T.reshape(-1))
    return np.ascontiguousarray(np.array(xs).astype(np.complex64))


def pow2_gains(rng, m):
    return rng.choice([-1.0, 1.0], m) * 2.0 ** rng.integers(-2, 3, m)


def handle(m, n, snaps, K, pos, mode="top_bins", rule="fixed", est=("music", 0.0), refine=False, devices=None):
    return gh.make_block(m, n, snaps, K, pos=pos, est=est, rule=rule, mode=mode, refine=refine, devices=devices)


def same(a, b, ctx):
    assert set(a) == set(b), ctx
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), (ctx, k)


# ---- 1. identity is a no-op --------------------------------------------------------------------------------------------
MODES = [  # (name, m, n, pos, handle kwargs)
    ("top_bins", 8, 2, array_wl("uca", 8), {}),
    ("local", 8, 2, array_wl("uca", 8), {"mode": "local_maxima"}),
    ("roots", 8, 2, ula(8, "x"), {"mode": "roots"}),
    ("esprit", 8, 2, ula(8, "x"), {"mode": "esprit"}),
    ("dml", 8, 2, array_wl("uca", 8), {"mode": "dml"}),
    ("mvdr", 8, 2, array_wl("uca", 8), {"est": ("mvdr", 0.01), "mode": "local_maxima"}),
    ("bartlett", 8, 2, array_wl("uca", 8), {"est": ("bartlett", 0.0), "mode": "local_maxima"}),
    ("mdl", 8, 3, array_wl("uca", 8), {"rule": "mdl", "mode": "local_maxima"}),
    ("refine", 8, 2, array_wl("uca", 8), {"refine": True, "mode": "local_maxima"}),
    ("m4", 4, 1, array_wl("uca", 4), {}),
    ("m5", 5, 2, array_wl("uca", 5), {}),
]


@pytest.mark.parametrize("name,m,n,pos,kw", MODES, ids=[c[0] for c in MODES])
def test_identity_is_a_no_op(name, m, n, pos, kw):
    """gains all (1, 0): every output of process_device_ex with d_R is byte-identical to an uncalibrated handle's"""
    K, snaps = 720, 256
    rng = np.random.default_rng(11)
    x = windows(pos, [rng.uniform(0, 360, 2) for _ in range(12)], 12, snaps)
    a, b = handle(m, n, snaps, K, pos, **kw), handle(m, n, snaps, K, pos, **kw)
    b.set_calibration(np.ones(m))
    assert np.array_equal(b.calibration(), np.ones(m))
    ra, _ = gh.device_call(a, x, ALL)
    rb, _ = gh.device_call(b, x, ALL)
    same(ra, rb, name)
    if name in ("top_bins", "m4"):
        # bins of the default (fused where the shape allows) call
        rd, _ = gh.device_call(a, x, ("levels", "bins"))
        assert np.array_equal(rd["bins"], rb["bins"])
    a.close()
    b.close()


# ---- 2. exact correction: real power-of-two gains ----------------------------------------------------------------------
@pytest.mark.parametrize("m,n,mode", [(4, 1, "top_bins"), (8, 1, "top_bins"), (8, 2, "local_maxima"), (5, 2, "top_bins"),
                                      (16, 2, "local_maxima"), (3, 1, "top_bins")])
def test_exact_correction_device(m, n, mode):
    """x_raw = g o x and R_raw = G R G^H are exact, and so is the correction: a calibrated handle on x_raw is
    byte-identical to an uncalibrated one on x (process_device_ex with d_R: both unfused)"""
    K, snaps = 720, 256
    pos = array_wl("uca", m)
    rng = np.random.default_rng(20 + m)
    x = windows(pos, [rng.uniform(0, 360, n) for _ in range(10)], 21 + m, snaps)
    g = pow2_gains(rng, m)
    a, b = handle(m, n, snaps, K, pos, mode=mode), handle(m, n, snaps, K, pos, mode=mode)
    b.set_calibration(g)
    ra, la = gh.device_call(a, x, ALL)
    rb, lb = gh.device_call(b, corrupt(x, g), ALL)
    same(ra, rb, (m, n, mode))
    assert lb == la + 1  # plus the apply kernel
    a.close()
    b.close()


def test_exact_correction_every_entry():
    """host, device, _counts, planar host / device and the default peak-only call (n = 2: unfused) agree byte for byte"""
    m, n, K, snaps, W = 8, 2, 720, 256, 24
    pos = array_wl("uca", m)
    rng = np.random.default_rng(31)
    x = windows(pos, [rng.uniform(0, 360, 2) for _ in range(W)], 32, snaps)
    g = pow2_gains(rng, m)
    xr = corrupt(x, g)
    a, b = handle(m, n, snaps, K, pos), handle(m, n, snaps, K, pos)
    b.set_calibration(g)

    def host(blk, xin):
        ang, lvl, spec = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32), np.zeros((W, K), np.float32)
        assert blk.work(W, [xin], [ang, lvl, spec]) == W
        return {"a": ang, "l": lvl, "s": spec, "b": blk.last_bins().copy()}

    def counts(blk, xin):
        return gh.device_call(blk, xin, ("levels", "bins", "counts"))[0]

    def planar_host(blk, xin):
        ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
        assert blk.work_planar(W, helpers.antenna_streams(xin, m), [ang, lvl]) == W
        return {"a": ang, "l": lvl, "b": blk.last_bins().copy()}

    def planar_device(blk, xin):
        return gh.planar_device_call(blk, helpers.antenna_streams(xin, m), snaps, W, ("levels", "bins"))[0]

    for f in (host, counts, planar_host, planar_device):
        same(f(a, x), f(b, xr), f.__name__)
    a.close()
    b.close()


def test_exact_correction_azel():
    """an az-el handle: calibrated on x_raw equals uncalibrated on x, host and device"""
    m, n, snaps, W = 8, 2, 256, 12
    pos = np.c_[array_wl("uca", m), np.r_[np.zeros(4), 0.3 * np.ones(4)]]
    rng = np.random.default_rng(41)
    x = windows(pos, [[(rng.uniform(0, 360), rng.uniform(0, 40)) for _ in range(2)] for _ in range(W)], 42, snaps, azel=True)
    g = pow2_gains(rng, m)
    blks = [music_doa_azel(m, n, m * snaps, 72, 9, (0.0, 80.0), pos, LAM) for _ in range(2)]
    for b in blks:
        b.set_peak_mode("local_maxima", 0)
    blks[1].set_calibration(g)
    outs = []
    for b, xin in zip(blks, (x, corrupt(x, g))):
        az, el, lv = (np.zeros((W, n), np.float32) for _ in range(3))
        sp = np.zeros((W, b.resolution), np.float32)
        assert b.work(W, [xin], [az, el, lv, sp]) == W
        outs.append({"az": az, "el": el, "lv": lv, "sp": sp, "b": b.last_bins().copy()})
    same(outs[0], outs[1], "azel")
    for b in blks:
        b.close()


def test_exact_correction_beams():
    """beams entries: the weights of the calibrated handle are c o w exactly and the beams are identical"""
    m, n, K, snaps, W = 8, 2, 720, 256, 12
    pos = array_wl("uca", m)
    rng = np.random.default_rng(51)
    x = windows(pos, [rng.uniform(0, 360, 2) for _ in range(W)], 52, snaps)
    g = pow2_gains(rng, m)
    for rule, loading in (("das", 0.0), ("mvdr", 0.01), ("lcmv", 0.01)):
        a, b = handle(m, n, snaps, K, pos, mode="local_maxima"), handle(m, n, snaps, K, pos, mode="local_maxima")
        for blk in (a, b):
            blk.set_beamformer(rule, loading)
        b.set_calibration(g)
        ra, la = gh.device_call(a, x, BEAMS)
        rb, lb = gh.device_call(b, corrupt(x, g), BEAMS)
        for k in ("angles", "levels", "bins", "counts", "beams"):
            assert ra[k].tobytes() == rb[k].tobytes(), (rule, k)
        c = co.inverse(g)
        assert np.array_equal(rb["weights"], ra["weights"] * c[None, None, :]), rule
        assert lb == la + 2  # the apply kernel and the weight correction
        a.close()
        b.close()


def test_multi_device_entries():
    """a multi-device handle over every GPU (sharded entry too, with two or more): same outputs as a single-device one"""
    G = torch.cuda.device_count()
    if G < 2:
        pytest.skip("needs two GPUs")
    m, n, K, snaps, W = 8, 2, 720, 256, 16
    pos = array_wl("uca", m)
    rng = np.random.default_rng(61)
    x = windows(pos, [rng.uniform(0, 360, 2) for _ in range(W)], 62, snaps)
    g = pow2_gains(rng, m)
    a = handle(m, n, snaps, K, pos)
    b = handle(m, n, snaps, K, pos, devices=list(range(G)))
    b.set_calibration(g)
    oa = [np.zeros((W, n), np.float32) for _ in range(2)]
    ob = [np.zeros((W, n), np.float32) for _ in range(2)]
    a.work(W, [x], oa)
    b.work(W, [corrupt(x, g)], ob)
    assert all(p.tobytes() == q.tobytes() for p, q in zip(oa, ob))
    a.close()
    b.close()


# ---- 3. complex gains --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [2, 4, 7, 16])
def test_complex_gains_correct_R(m):
    """d_R of a calibrated handle = C R_raw C^H from an uncalibrated call's d_R, to 1e-15 |R_ij| per entry"""
    K, snaps, W = 360, 128, 8
    pos = array_wl("uca", m) if m > 2 else ula(2, "x")
    rng = np.random.default_rng(70 + m)
    g = random_gains(rng, m)
    xr = corrupt(windows(pos, [rng.uniform(0, 360, 1) for _ in range(W)], 71, snaps), g)
    a, b = handle(m, 1, snaps, K, pos), handle(m, 1, snaps, K, pos)
    b.set_calibration(g)
    assert np.array_equal(b.calibration(), g)
    Ra = gh.device_call(a, xr, ALL)[0]["R"]
    Rb = gh.device_call(b, xr, ALL)[0]["R"]
    want = np.array([co.correct(R, g) for R in Ra])
    assert np.all(np.abs(Rb - want) <= 1e-15 * np.abs(want))
    a.close()
    b.close()


# ---- 4 / 5. the estimator against the oracle and against the truth -----------------------------------------------------
EST_CASES = [("ula2", ula(2, "x"), co.PHASE, 25.0), ("ula4", ula(4, "x"), co.GAIN_PHASE, 50.0),
             ("uca8", array_wl("uca", 8), co.GAIN_PHASE, 130.0), ("uca16", array_wl("uca", 16), co.GAIN_PHASE, 290.0)]
KINDS = {co.PHASE: "phase", co.GAIN_PHASE: "gain_phase"}


def truth_error(got, g, kind):
    want = co.normalised(g, kind)
    return float(np.max(np.abs(np.angle(got / want)))), float(np.max(np.abs(np.abs(got) / np.abs(want) - 1.0)))


@pytest.mark.parametrize("name,pos,kind,az", EST_CASES, ids=[c[0] for c in EST_CASES])
def test_estimator(name, pos, kind, az):
    """solve on seeded corrupted windows = the oracle on numpy's fp64 R-bar of the same bytes (gains 1e-9, sweeps +-1);
    host and device accumulation agree, so does a split over several calls; the error to the truth stays within 3x the
    oracle's own on the same seeds plus the rounding of R"""
    m, K, snaps, W = len(pos), 360, 1024, 16
    rng = np.random.default_rng(80 + m)
    g = random_gains(rng, m)
    xr = corrupt(windows(pos, [[az]] * W, 81 + m, snaps), g)
    blk = handle(m, 1, snaps, K, pos)
    got, rho, sweeps = blk.calibrate(xr, az, kind=KINDS[kind])
    Rbar = co.covariance(xr, m).mean(axis=0)
    a0 = co.steering_1d(pos, LAM, az)
    ref, rho_ref, sw_ref = co.solve(Rbar, a0, kind)
    assert np.max(np.abs(got - ref)) <= 1e-9 * np.max(np.abs(ref)), (got, ref)
    assert abs(sweeps - sw_ref) <= 1 and abs(rho - rho_ref) <= 1e-9
    # device accumulation, split over three calls
    blk.calib_reset()
    d_in = torch.from_numpy(xr.view(np.float32).reshape(-1)).to(gh.DEV)
    step = m * snaps * 2
    for lo, hi in ((0, 5), (5, 6), (6, W)):
        blk.calib_accumulate_device(d_in[lo * step:].data_ptr(), hi - lo, stream=gh.stream())
    gd, rho_d, sw_d = blk.calib_solve(az, 0.0, KINDS[kind])
    assert np.max(np.abs(gd - got)) <= 1e-12 * np.max(np.abs(got)) and abs(sw_d - sweeps) <= 1
    # the accumulator is kept: a second solve gives the same answer
    assert np.array_equal(blk.calib_solve(az, 0.0, KINDS[kind])[0], gd)
    ph, mag = truth_error(got, g, kind)
    ph_o, mag_o = truth_error(ref, g, kind)
    assert ph <= 3.0 * ph_o + 1e-9 and mag <= 3.0 * mag_o + 1e-9
    assert ph <= math.radians(0.5) and (kind == co.PHASE or mag <= 0.01)
    blk.close()


def test_estimator_azel():
    m, snaps, W = 8, 1024, 16
    pos = np.c_[array_wl("uca", m), np.r_[np.zeros(4), 0.3 * np.ones(4)]]
    rng = np.random.default_rng(91)
    g = random_gains(rng, m)
    az, el = 200.0, 25.0
    xr = corrupt(windows(pos, [[(az, el)]] * W, 92, snaps, azel=True), g)
    blk = music_doa_azel(m, 1, m * snaps, 72, 9, (0.0, 80.0), pos, LAM)
    got, rho, sweeps = blk.calibrate(xr, az, el)
    ref, _, sw_ref = co.solve(co.covariance(xr, m).mean(axis=0), co.steering_azel(pos, LAM, az, el), co.GAIN_PHASE)
    assert np.max(np.abs(got - ref)) <= 1e-9 * np.max(np.abs(ref)) and abs(sweeps - sw_ref) <= 1
    ph, mag = truth_error(got, g, co.GAIN_PHASE)
    assert ph <= math.radians(0.5) and mag <= 0.01
    blk.close()


# ---- 6. DOA restored -----------------------------------------------------------------------------------------------------
def rms_error(ang, bins, truth, axis_mirror):
    errs = []
    for w in range(len(truth)):
        for t in truth[w]:
            d = [ro.angle_error(a, t, "ula_x" if axis_mirror else "uca") for a, b in zip(ang[w], bins[w]) if b >= 0]
            errs.append(min(d) if d else 180.0)
    return float(np.sqrt(np.mean(np.square(errs))))


@pytest.mark.parametrize("case", ["uca8_local", "ula8_roots"])
def test_doa_restored(case):
    """uncalibrated errors on corrupted windows are large; with the estimated gains the RMS error is within 1.5x of the
    same handle on clean windows"""
    if case == "uca8_local":
        m, n, pos, mode, cal_az = 8, 2, array_wl("uca", 8), "local_maxima", 130.0
    else:
        m, n, pos, mode, cal_az = 8, 2, ula(8, "x"), "roots", 50.0
    K, snaps, W = 3600, 512, 40
    rng = np.random.default_rng(101)
    g = random_gains(rng, m)
    truth = []
    for _ in range(W):
        if case == "ula8_roots":
            t = rng.uniform(20.0, 75.0)
            truth.append([t, t + rng.uniform(40.0, 80.0)])
        else:
            t = rng.uniform(0, 360)
            truth.append([t, (t + rng.uniform(60.0, 180.0)) % 360.0])
    x = windows(pos, truth, 102, snaps)
    xr = corrupt(x, g)
    blk = handle(m, n, snaps, K, pos, mode=mode)
    mirror = case == "ula8_roots"

    def run(xin):
        ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
        blk.work(W, [xin], [ang, lvl])
        return rms_error(ang, blk.last_bins(), truth, mirror)

    clean, raw = run(x), run(xr)
    cal = corrupt(windows(pos, [[cal_az]] * 32, 103, snaps), g)
    gains, rho, _ = blk.calibrate(cal, cal_az)
    blk.set_calibration(gains)
    fixed = run(xr)
    assert raw > 5.0 * max(clean, 0.05), (clean, raw)
    assert fixed <= 1.5 * clean + 1e-3, (clean, raw, fixed)
    blk.close()


# ---- 7. errors and persistence -----------------------------------------------------------------------------------------
def test_errors_and_persistence():
    L = _capi.load()
    m, snaps, K = 4, 64, 360
    pos = array_wl("uca", m)
    blk = handle(m, 1, snaps, K, pos)
    EINVAL = _capi.EINVAL
    g = np.ones(2 * m)
    bad = [np.r_[0.0, 0.0, g[2:]], np.r_[np.nan, 0.0, g[2:]], np.r_[1.0, np.inf, g[2:]], np.r_[1e-300, 0.0, g[2:]]]
    blk.set_calibration(2.0 * np.ones(m))
    for b in bad:
        b = np.ascontiguousarray(b)
        assert L.music_b200_set_calibration(blk._h, b.ctypes.data) == EINVAL
    assert np.array_equal(blk.calibration(), 2.0 * np.ones(m))  # the old setting stays
    out = np.zeros(2 * m)
    st = np.zeros(2)
    # empty accumulator, unknown kind, GAIN_PHASE with m < 3, el != 0 on a 1-D handle
    blk.calib_reset()
    assert L.music_b200_calib_solve(blk._h, 0.0, 0.0, 2, out.ctypes.data, st.ctypes.data) == EINVAL
    x = windows(pos, [[10.0]] * 4, 5, snaps)
    blk.calib_accumulate(x)
    assert L.music_b200_calib_solve(blk._h, 10.0, 0.0, 3, out.ctypes.data, None) == EINVAL
    assert L.music_b200_calib_solve(blk._h, 10.0, 5.0, 2, out.ctypes.data, None) == EINVAL
    assert L.music_b200_calib_solve(blk._h, 10.0, 0.0, 2, out.ctypes.data, None) == _capi.OK
    small = handle(2, 1, snaps, K, ula(2, "x"))
    small.calib_accumulate(windows(ula(2, "x"), [[10.0]] * 2, 6, snaps))
    assert L.music_b200_calib_solve(small._h, 10.0, 0.0, 2, out.ctypes.data, None) == EINVAL
    assert L.music_b200_calib_solve(small._h, 10.0, 0.0, 1, out.ctypes.data, None) == _capi.OK
    small.close()
    # all-zero accumulator, a dead channel
    blk.calib_reset()
    blk.calib_accumulate(np.zeros((3, m * snaps), np.complex64))
    assert L.music_b200_calib_solve(blk._h, 0.0, 0.0, 2, out.ctypes.data, None) == EINVAL
    blk.calib_reset()
    blk.calib_accumulate(corrupt(x, np.r_[1.0, 0.0, 1.0, 1.0]))
    assert L.music_b200_calib_solve(blk._h, 10.0, 0.0, 2, out.ctypes.data, None) == EINVAL
    # the setting survives set_table / set_geometry; solve on a set_table() table is refused
    blk.set_array_response(np.ones((K, m), np.complex64))
    assert np.array_equal(blk.calibration(), 2.0 * np.ones(m))
    blk.calib_reset()
    blk.calib_accumulate(x)
    assert L.music_b200_calib_solve(blk._h, 10.0, 0.0, 2, out.ctypes.data, None) == EINVAL
    blk.set_array_geometry(pos, LAM)
    assert np.array_equal(blk.calibration(), 2.0 * np.ones(m))
    blk.set_calibration(None)
    assert np.array_equal(blk.calibration(), np.ones(m))
    blk.close()
    # a multi-device handle reaches every child (single GPU: one child)
    multi = handle(m, 1, snaps, K, pos, devices=list(range(torch.cuda.device_count())))
    multi.set_calibration(2.0 * np.ones(m))
    a = handle(m, 1, snaps, K, pos)
    o1, o2 = np.zeros((4, 1), np.float32), np.zeros((4, 1), np.float32)
    multi.work(4, [corrupt(x, 2.0 * np.ones(m))], [o1])
    a.work(4, [x], [o2])
    assert np.array_equal(o1, o2)
    multi.close()
    a.close()


# ---- 8. C++ block --------------------------------------------------------------------------------------------------------
def test_cpp_block():
    """calibrate() armed on the C++ block, corrupted items over several work() calls: the gains it applies equal the
    Python block's estimate on the same items, and its later DOA outputs equal the Python block's with those gains"""
    m, n, K, snaps, C, W, chunk = 8, 2, 720, 256, 12, 10, 5
    pos = array_wl("uca", m)
    rng = np.random.default_rng(111)
    g = random_gains(rng, m)
    cal = corrupt(windows(pos, [[70.0]] * C, 112, snaps), g)
    x = corrupt(windows(pos, [rng.uniform(0, 360, 2) for _ in range(W)], 113, snaps), g)
    c = gh.run_cpp_block("test_block_calibration", struct.pack("<9I", m, n, m * snaps, K, C, W, 1, 2, chunk) +
                         struct.pack("<2d", 70.0, LAM), [np.ascontiguousarray(pos, np.float64), cal, x],
                         [("g", np.complex128, m), ("rho", np.float64, 1), ("a", np.float32, W * n), ("b", np.int32, W * n)])
    cg, crho, ca, cb = c["g"], c["rho"][0], c["a"], c["b"]
    blk = handle(m, n, snaps, K, pos, mode="local_maxima")
    blk.calib_reset()
    for lo in range(0, C, chunk):  # the same split over accumulate calls as the block's work() calls
        blk.calib_accumulate(cal[lo:lo + chunk])
    pg, prho, _ = blk.calib_solve(70.0)
    assert np.array_equal(cg, pg) and crho == prho
    blk.set_calibration(pg)
    ang, lvl = np.zeros((W, n), np.float32), np.zeros((W, n), np.float32)
    blk.work(W, [x], [ang, lvl])
    assert np.array_equal(ca, ang.ravel()) and np.array_equal(cb, blk.last_bins().ravel())
    assert np.max(np.abs(np.angle(pg / co.normalised(g, co.GAIN_PHASE)))) <= math.radians(1.0)
    blk.close()
