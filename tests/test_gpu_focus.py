"""GPU: the COHERENT combine of a channel handle (focusing matrices, focused covariance, one plain problem per window)
against tests/focus_oracle.py and composed_oracle.work_R: the matrices and errors, R_foc, every accepted mode
combination on the GPU's own R_foc, the two-path case, the entry points and blocks, the launch plan and the refusals."""
import ctypes
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200._capi import MusicB200Error
from gr_baz_b200.music_doa_channels import TAPERS, music_doa_channels

import channels_oracle as ch
import composed_oracle as cmp
import focus_oracle as fo
import gpu_harness as gh
import helpers

pytestmark = pytest.mark.gpu

FC, FS = 400e6, 56e6
LAM0 = ch.C0 / FC
P_RTOL = 1e-5
FLIP = 1e-9  # decisions the oracle sees this close to flipping may go either way
PEAK_NAMES = {"top": "top_bins", "local": "local_maxima", "roots": "roots", "esprit": "esprit", "dml": "dml"}
ESTS = {"music": 0.0, "mvdr": 1e-3, "bartlett": 0.0}


def planar_pos(m, seed):
    return np.random.default_rng(seed).uniform(-0.6, 0.6, (m, 2)) * LAM0


def make(m, n, snaps, K, F, first, C, pos, combine="coherent", taper="hann", fc=FC, fs=FS):
    return music_doa_channels(m, n, m * snaps, K, F, (first, C), taper, combine, pos, 1.0, fc, fs)


def lams(blk, fc=FC, fs=FS):
    return ch.wavelengths(blk.nfft, blk.chan_first, blk.chan_count, fc, fs)


def device_call(blk, x, outputs=("levels", "bins")):
    """one process_device call asking for the angles and `outputs`; R is (W, m, m) under coherent, (C, W, m, m) otherwise"""
    W, r, n, m, K, C = x.shape[0], blk.rows, blk.n, blk.m, blk.resolution, blk.chan_count
    f32, i32 = torch.float32, torch.int32
    rshape = (W, m, m, 2) if blk.combine == "coherent" else (C, W, m, m, 2)
    shapes = {"angles": ((r, W, n), f32), "levels": ((r, W, n), f32), "spectrum": ((r, W, K), f32), "bins": ((r, W, n), i32),
              "counts": ((r, W), i32), "R": (rshape, torch.float64)}
    o = {k: torch.full(shapes[k][0], gh.SENTINEL, dtype=shapes[k][1], device=gh.DEV) for k in ("angles",) + tuple(outputs)}
    p = lambda k: o[k].data_ptr() if k in o else None
    d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
    l0 = blk.launch_count()
    blk.process_device(d_in.data_ptr(), W, p("angles"), p("levels"), p("spectrum"), p("bins"), p("counts"), p("R"), stream=gh.stream())
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    if "R" in out:
        out["R"] = out["R"].view(np.complex128)[..., 0]
    return out, blk.launch_count() - l0


def noise_windows(W, m, snaps, seed):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((W, snaps * m)) + 1j * rng.standard_normal((W, snaps * m))) / math.sqrt(2.0)).astype(np.complex64)


def path_windows(W, pos, N, seed, degs=(40.0, 110.0), noise=0.3):
    rng = np.random.default_rng(seed)
    return np.stack([fo.two_paths(rng, pos, N, degs=degs, noise=noise, fc=FC, fs=FS) for _ in range(W)])


def check_focusing(blk, pos, fc=FC, first=0, count=None):
    T, err = blk.focusing()
    Tr, er = fo.focusing(pos, lams(blk, fc), blk.resolution, first, count)
    ref = fo.ref_channel(blk.chan_count)
    assert np.array_equal(T[ref], np.eye(blk.m)) and err[ref] == 0.0
    assert np.max(np.abs(T - Tr)) <= 1e-10
    assert np.all(np.abs(err - er) <= 1e-9 * er)


@pytest.mark.parametrize("C", [1, 7, 64])
@pytest.mark.parametrize("m", [2, 4, 8, 16])
def test_focusing_matrices_match_the_oracle(m, C):
    K, F = 180, 64
    first = (F - C // 2) % F
    pos = planar_pos(m, 3 * m + C)
    blk = make(m, 1, F, K, F, first, C, pos)
    check_focusing(blk, pos)
    blk.set_focusing(K - 20, 70)  # a sector that wraps through bin 0
    check_focusing(blk, pos, first=K - 20, count=70)
    blk.set_array_geometry(pos, 1.3 * FC, FS)  # a retune keeps the sector
    check_focusing(blk, pos, fc=1.3 * FC, first=K - 20, count=70)
    blk.set_focusing(0, K)
    check_focusing(blk, pos, fc=1.3 * FC)
    blk.close()


SHAPES = [(4, 16, 8, 0, 16), (7, 8, 9, 6, 4), (16, 64, 4, 40, 30), (8, 256, 2, 250, 12), (3, 8, 3, 0, 2)]  # m, F, J, first, C


@pytest.mark.parametrize("m,F,J,first,C", SHAPES)
def test_focused_covariance_matches_the_oracle(m, F, J, first, C):
    K, W = 120, 9
    pos = planar_pos(m, 7 * m + F)
    x = noise_windows(W, m, F * J, 10 * m + C)
    x[2] *= 1e3
    sep = make(m, 1, F * J, K, F, first, C, pos, "separate")
    R_c, _ = device_call(sep, x, ("R",))
    sep.close()
    blk = make(m, 1, F * J, K, F, first, C, pos)
    T, _ = blk.focusing()
    got, _ = device_call(blk, x, ("R",))
    for w in range(W):
        ref = fo.focus(R_c["R"][:, w], T)
        assert np.max(np.abs(got["R"][w] - ref)) <= 1e-12 * np.max(np.abs(ref)), w
    assert np.array_equal(got["R"], np.conj(np.swapaxes(got["R"], 1, 2)))
    again, _ = device_call(blk, x, ("R",))
    head, _ = device_call(blk, x[:4], ("R",))
    tail, _ = device_call(blk, x[4:], ("R",))
    bits = lambda a: a.view(np.uint8)
    assert np.array_equal(bits(got["R"]), bits(again["R"]))
    assert np.array_equal(bits(got["R"]), bits(np.concatenate([head["R"], tail["R"]])))
    blk.close()


def test_a_call_larger_than_one_sub_batch():
    """m = 16 with all 256 channels: the workspace and the channel buffer hold 376 windows, so 400 run as 376 + 24; R_foc
    and every output do not depend on the split"""
    m, K, F, W = 16, 360, 256, 400
    pos = planar_pos(m, 8)
    blk = make(m, 1, F, K, F, 0, F, pos, taper="rect")
    x = noise_windows(W, m, F, 21)
    every = ("levels", "bins", "counts", "spectrum", "R")
    got, launches = device_call(blk, x, every)
    assert launches == 2 * 4 + 1  # per sub-batch filter bank, focus, eigensolver, scan (with the arg-max); the counts fill once
    head, _ = device_call(blk, x[:200], every)
    tail, _ = device_call(blk, x[200:], every)
    axis = lambda k: 0 if k == "R" else 1
    for k in got:
        assert np.array_equal(got[k].view(np.uint8), np.concatenate([head[k], tail[k]], axis=axis(k)).view(np.uint8)), k
    sep = make(m, 1, F, K, F, 0, F, pos, "separate", taper="rect")
    R_c, _ = device_call(sep, x[375:377], ("R",))
    sep.close()
    T, _ = blk.focusing()
    for i, w in enumerate((375, 376)):
        ref = fo.focus(R_c["R"][:, i], T)
        assert np.max(np.abs(got["R"][w] - ref)) <= 1e-12 * np.max(np.abs(ref))
    blk.close()


def test_one_channel_is_separate():
    m, n, K, F, J, W = 4, 2, 180, 16, 16, 7
    pos = planar_pos(m, 2)
    x = path_windows(W, pos, F * J, 12)
    every = ("levels", "bins", "counts", "spectrum", "R")
    outs = []
    for combine in ("separate", "coherent"):
        blk = make(m, n, F * J, K, F, 3, 1, pos, combine)
        blk.set_source_rule("mdl")
        blk.set_peak_mode("local_maxima", 2)
        o, _ = device_call(blk, x, every)
        outs.append(o)
        blk.close()
    for k in every:
        assert np.array_equal(outs[0][k].reshape(-1).view(np.uint8), outs[1][k].reshape(-1).view(np.uint8)), k


def ulps(a, b):
    return helpers.circ(a, b) / float(np.spacing(np.float32(max(abs(float(a)), abs(float(b)), 1e-3))))


def combos():
    rows = []
    for peak in ("top", "local", "roots", "esprit", "dml"):
        for est in ("music", "mvdr", "bartlett"):
            for rule in ("fixed", "mdl", "aic"):
                for refine in (False, True):
                    if peak in ("roots", "esprit", "dml") and (est != "music" or refine):
                        continue
                    rows.append((peak, est, rule, refine))
    return rows


@pytest.mark.parametrize("peak,est,rule,refine", combos())
def test_every_accepted_combination_matches_the_composed_oracle(peak, est, rule, refine):
    m, n, K, F, J, first, C, W = 6, 2, 360, 16, 8, 12, 8, 6
    lam_ref = ch.wavelengths(F, first, C, FC, FS)[fo.ref_channel(C)]
    gridless = peak in ("roots", "esprit")
    pos = np.stack([np.arange(m) * lam_ref / 2.0, np.zeros(m)], axis=1) if gridless else fo.uca(m, lam_ref)
    blk = make(m, n, F * J, K, F, first, C, pos)
    blk.set_estimator(est, ESTS[est])
    blk.set_source_rule(rule)
    excl = 3 if peak == "local" else 0
    blk.set_peak_mode(PEAK_NAMES[peak], excl)
    blk.set_refine(refine)
    x = path_windows(W, pos, F * J, 400 + len(peak) + 7 * refine, degs=(35.0, 120.0) if gridless else (40.0, 110.0))
    x[0] = noise_windows(1, m, F * J, 5)[0]
    got, _ = device_call(blk, x, ("levels", "bins", "counts", "R"))
    tab = blk.array_response_c64(fo.ref_channel(C))
    md = cmp.modes(peak=peak, exclusion=excl, est=est, loading=ESTS[est], rule=rule, refine=refine)
    checked = 0
    for w in range(W):
        R = got["R"][w]
        r = cmp.work_R(R, md, tab, (pos, lam_ref), n, J * C)
        ctx = (w,)
        if r["margin"] > 1e-6:
            assert got["counts"][0, w] == r["count"], ctx
        elif got["counts"][0, w] != r["count"]:
            continue
        gb, ga, gl = got["bins"][0, w], got["angles"][0, w], got["levels"][0, w]
        if not np.array_equal(gb, r["bins"]):
            i = int(np.nonzero(gb != r["bins"])[0][0])
            b, rb = int(gb[i]), int(r["bins"][i])
            P = r["P"]
            tie = r["flip"][i] <= FLIP or (peak in ("top", "local") and b >= 0 and rb >= 0 and abs(P[b] - P[rb]) <= 1e-12 * P[rb])
            if gridless and not tie:  # an angle on a bin boundary may round either way
                tie = b >= 0 and np.array_equal(np.delete(gb, i), np.delete(r["bins"], i)) and ulps(ga[i], r["angles"][i]) <= 2.0
            assert tie, (ctx, gb, r["bins"])
            if not gridless:
                continue
        for i in range(n):
            rb = int(r["bins"][i])
            if i >= r["count"] or rb < 0:
                assert ga[i] == 0.0 and gl[i] == 0.0 and gb[i] == -1, (ctx, i)
                continue
            ra, rl = r["angles"][i], r["levels"][i]
            if refine or gridless:
                if r["flip"][i] <= FLIP and ulps(ga[i], ra) > 2.0:
                    continue
                if refine and est != "music":
                    assert helpers.circ(ga[i], ra) <= 1e-4, (ctx, i, ga, r["angles"])
                else:
                    assert ulps(ga[i], ra) <= 2.0, (ctx, i, ga, r["angles"])
            else:
                assert ga[i] == ra, (ctx, i, ga, r["angles"])
            if peak == "dml":
                tol = max(float(np.spacing(np.abs(np.float32(rl)))), 1e-10 * float(np.real(np.trace(R))))
                assert abs(float(gl[i]) - float(rl)) <= tol, (ctx, i, gl, r["levels"])
            else:
                assert abs(float(gl[i]) - float(rl)) <= P_RTOL * abs(float(rl)), (ctx, i, gl, r["levels"])
        checked += 1
    assert checked >= W - 2
    blk.close()


def test_two_paths_are_resolved_on_the_device():
    """the motivating case: one wideband signal and its one-sample-late reflection on a UCA of 8"""
    W = 20
    pos, _, x = fo.scenario(W, 7)
    counts = {}
    for combine in ("coherent", "incoherent"):
        blk = music_doa_channels(8, 2, 8 * fo.F * fo.J, fo.K, fo.F, (fo.FIRST, fo.C), "rect", combine, pos, 1.0, fo.FC, fo.FS)
        blk.set_peak_mode("local_maxima", 0)
        got, _ = device_call(blk, x, ())
        counts[combine] = sum(fo.resolved(got["angles"][0, w]) for w in range(W))
        blk.close()
    assert counts["coherent"] >= 18 and counts["incoherent"] <= 2, counts


def test_entries_and_blocks_agree():
    """outputs do not depend on which are requested; host entry = device entry byte for byte; the Python block and the
    C++ block hand out the same items"""
    m, n, K, F, J, first, C, W = 4, 2, 120, 16, 12, 13, 6, 7
    pos = planar_pos(m, 6)
    blk = make(m, n, F * J, K, F, first, C, pos)
    blk.set_source_rule("mdl")
    blk.set_peak_mode("local_maxima", 2)
    blk.set_focusing(100, 60)
    x = path_windows(W, pos, F * J, 99)
    every = ("levels", "bins", "spectrum", "counts", "R")
    full, _ = device_call(blk, x, every)
    for subset in ((), ("bins",), ("levels", "spectrum"), ("R",), ("counts",)):
        part, _ = device_call(blk, x, subset)
        for k, v in part.items():
            assert np.array_equal(v.view(np.uint8), full[k].view(np.uint8)), (subset, k)
    host = blk.process_host(x, W, levels=True, spectrum=True, bins=True, counts=True, R=True)
    for k, v in host.items():
        assert np.array_equal(np.ascontiguousarray(v).view(np.uint8), full[k].view(np.uint8)), k
    ports = [np.zeros((W, n), np.float32), np.zeros((W, n), np.float32), np.zeros((W, K), np.float32)]
    assert blk.work(W, [x], ports) == W
    assert np.array_equal(ports[0], full["angles"][0]) and np.array_equal(ports[1], full["levels"][0])
    assert np.array_equal(ports[2], full["spectrum"][0])
    assert np.array_equal(blk.last_bins().reshape(W, n), full["bins"][0])
    assert np.array_equal(blk.last_counts().reshape(W), full["counts"][0])
    header = struct.pack("<15I3d", m, n, m * F * J, K, F, first, C, TAPERS["hann"], W, 1, 2, 1, 0, 100, 60, 0.0, FC, FS)
    layout = [("angles", np.float32, W * n), ("levels", np.float32, W * n), ("spectrum", np.float32, W * K),
              ("bins", np.int32, W * n), ("counts", np.int32, W), ("err", np.float64, C)]
    cpp = gh.run_cpp_block("test_block_focus", header, [pos.astype(np.float64), x.view(np.float32)], layout)
    for k in ("angles", "levels", "spectrum", "bins"):
        assert np.array_equal(cpp[k].reshape(W, -1), ports[["angles", "levels", "spectrum"].index(k)] if k != "bins" else full["bins"][0]), k
    assert np.array_equal(cpp["counts"], full["counts"][0])
    assert np.array_equal(cpp["err"], blk.focusing()[1])
    blk.close()


@pytest.mark.parametrize("est,peak,rule,n", [("music", "top", "fixed", 1), ("music", "local", "mdl", 2), ("mvdr", "top", "aic", 2),
                                             ("music", "dml", "fixed", 2), ("bartlett", "local", "fixed", 1)])
def test_launch_count_does_not_grow_with_the_channels(est, peak, rule, n):
    """per sub-batch: filter bank, focus, then the plain plan (eigensolver, count, MVDR preparation, scan, peak rule)
    once; the same for C = 1 and C = 64"""
    m, K, F, J, W = 4, 90, 64, 8, 11
    pos = fo.uca(m, LAM0)
    music, fixed = est == "music", rule == "fixed"
    argmax = n == 1 and peak == "top"
    per = 2 + ((music and peak != "dml") or not fixed) + (not fixed) + (est == "mvdr") + (peak != "dml") + (not argmax)
    for outs in (("bins",), ("levels", "counts")):
        want = per + (fixed and "counts" in outs)
        got = []
        for C in (1, 64):
            blk = make(m, n, F * J, K, F, (F - C // 2) % F, C, pos)
            blk.set_estimator(est, ESTS[est])
            blk.set_source_rule(rule)
            blk.set_peak_mode(PEAK_NAMES[peak], 0)
            got.append(device_call(blk, noise_windows(W, m, F * J, 5), outs)[1])
            blk.close()
        assert got == [want, want], (outs, got, want)


def einval(call, *args, **kw):
    with pytest.raises(MusicB200Error) as e:
        call(*args, **kw)
    assert e.value.code == _capi.EINVAL


def test_refusals_leave_the_handle_usable():
    m, n, K, F, J, first, C, W = 4, 2, 90, 8, 8, 0, 4, 3
    pos = planar_pos(m, 1)
    x = noise_windows(W, m, F * J, 3)
    lib = _capi.load()
    buf = np.zeros(1 << 16, np.float32)
    blk = make(m, n, F * J, K, F, first, C, pos)
    before, _ = device_call(blk, x)
    T0 = blk.focusing()
    for kind in ("das", "mvdr", "lcmv"):
        einval(blk.set_beamformer, kind, 0.0 if kind == "das" else 1e-3)
    einval(blk.set_calibration, np.ones(m, np.complex128))
    einval(blk.calib_reset)
    einval(blk.calib_accumulate, x)
    einval(blk.gather_create, W)
    einval(blk.set_array_response, helpers.random_table(m, K, 1))
    for first_bin, count in ((0, 0), (0, K + 1), (K, 1)):
        einval(blk.set_focusing, first_bin, count)
    einval(blk.set_peak_mode, "roots")  # a planar array is no ULA
    h, p = blk._h, buf.ctypes.data
    entries = [
        lambda: lib.music_b200_process_planar_host(h, p, 1, W, p, None, None, None),
        lambda: lib.music_b200_process_planar_device(h, p, 1, W, p, None, None, None, None),
        lambda: lib.music_b200_process_device_sharded(h, p, W, p, None, None, None),
        lambda: lib.music_b200_process_azel_host(h, x.ctypes.data, W, p, p, None, None, None, None),
        lambda: lib.music_b200_set_geometry(h, pos.ctypes.data, LAM0, None),
        lambda: lib.music_b200_set_geometry_azel(h, pos.ctypes.data, LAM0),
        lambda: lib.music_b200_process_host(h, x.ctypes.data, W, p, None, None, None),
    ]
    for i, entry in enumerate(entries):
        assert entry() == _capi.EINVAL, i
    after, _ = device_call(blk, x)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    T1 = blk.focusing()
    assert np.array_equal(T0[0], T1[0]) and np.array_equal(T0[1], T1[1])
    blk.close()
    # set_focusing / get_focusing need a COHERENT handle; get_focusing needs a geometry
    for combine in ("separate", "incoherent"):
        other = make(m, n, F * J, K, F, first, C, pos, combine)
        einval(other.set_focusing, 0, K)
        einval(other.focusing)
        other.close()
    raw = ctypes.c_void_p()
    assert lib.music_b200_create_channels(ctypes.byref(raw), m, 1, m * F * J, K, F, 0, C, 0, 2, 0) == _capi.OK
    assert lib.music_b200_get_focusing(raw, None, buf.ctypes.data) == _capi.EINVAL
    assert lib.music_b200_set_focusing(raw, 10, 20) == _capi.OK  # kept for the first geometry
    assert lib.music_b200_set_geometry_channels(raw, np.ascontiguousarray(pos).ctypes.data, FC, FS) == _capi.OK
    err = np.zeros(C)
    assert lib.music_b200_get_focusing(raw, None, err.ctypes.data) == _capi.OK
    assert np.all(np.abs(err - fo.focusing(pos, ch.wavelengths(F, 0, C, FC, FS), K, 10, 20)[1]) <= 1e-9 * err)
    lib.music_b200_destroy(raw)
