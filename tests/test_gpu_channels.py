"""GPU: the frequency-channelised modes (music_b200_create_channels) against tests/channels_oracle.py: the filter bank's
per-channel covariances, every accepted estimator x peak rule x source rule per channel on the GPU's own R_c and table c,
the incoherent combine, the entry points and blocks, the refusals and the launch plan."""
import ctypes
import math
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi
from gr_baz_b200._capi import MusicB200Error
from gr_baz_b200.music_doa_channels import COMBINES, TAPERS, music_doa_channels

import channels_oracle as ch
import composed_oracle as cmp
import gpu_harness as gh
import helpers

pytestmark = pytest.mark.gpu

FC, FS = 400e6, 56e6
LAM0 = ch.C0 / FC
P_RTOL = 1e-5
SCAN_B = 8  # windows per scan CTA: sub-batches are whole multiples of it


def planar_pos(m, seed):
    """m elements scattered over about a wavelength: no mirror symmetry, so no two table rows tie"""
    return np.random.default_rng(seed).uniform(-0.6, 0.6, (m, 2)) * LAM0


def make(m, n, snaps, K, F, first, C, taper="hann", combine="separate", pos=None, est=None, rule=None, mode=None, excl=0):
    pos = planar_pos(m, 5 * m + F) if pos is None else pos
    blk = music_doa_channels(m, n, m * snaps, K, F, (first, C), taper, combine, pos, 1.0, FC, FS)
    if est is not None:
        blk.set_estimator(*est)
    if rule is not None:
        blk.set_source_rule(rule)
    if mode is not None:
        blk.set_peak_mode(mode, excl)
    return blk


def device_call(blk, x, outputs=("levels", "bins"), fill=gh.SENTINEL):
    """One process_device call on the windows x asking for the angles and `outputs` (levels, spectrum, bins, counts, R), in
    the channel-major layout.  Returns (numpy outputs, kernel launches); R as complex128 (C, W, m, m)."""
    W, r, n, m, K, C = x.shape[0], blk.rows, blk.n, blk.m, blk.resolution, blk.chan_count
    f32, i32 = torch.float32, torch.int32
    shapes = {"angles": ((r, W, n), f32), "levels": ((r, W, n), f32), "spectrum": ((r, W, K), f32), "bins": ((r, W, n), i32),
              "counts": ((r, W), i32), "R": ((C, W, m, m, 2), torch.float64)}
    o = {k: torch.full(shapes[k][0], fill, dtype=shapes[k][1], device=gh.DEV) for k in ("angles",) + tuple(outputs)}
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


def scene_windows(W, pos, F, snaps, first, C, seed, noise=0.1):
    """windows with two emitters each, in two channels of the range (first, C) (the same channel when C = 1)"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(W):
        cs = [(first + int(c)) % F for c in rng.choice(C, size=2, replace=C < 2)]
        degs = rng.uniform(0.0, 360.0, 2)
        out.append(ch.two_emitters(rng, pos, FC, FS, F, snaps, cs, degs, amps=rng.uniform(0.5, 2.0, 2), noise=noise))
    return np.stack(out)


def oracle_R(x, blk, taper):
    return np.stack([ch.covariances(w, blk.m, blk.nfft, blk.chan_first, blk.chan_count, taper) for w in x], axis=1)  # (C, W, m, m)


SHAPES = [  # m, F, J, first, C, taper
    (2, 8, 1, 0, 1, "rect"), (2, 8, 5, 0, 8, "hann"), (4, 64, 8, 0, 64, "hann"), (4, 64, 8, 0, 64, "rect"),
    (7, 8, 9, 6, 4, "hann"), (8, 64, 3, 60, 10, "rect"), (16, 256, 1, 0, 256, "rect"), (16, 64, 20, 0, 64, "hann"),
    (4, 256, 2, 250, 12, "hann"), (7, 64, 1, 33, 1, "rect"),
]


@pytest.mark.parametrize("m,F,J,first,C,taper", SHAPES)
def test_channel_covariances_match_the_definition(m, F, J, first, C, taper):
    W = 5
    blk = make(m, 1, F * J, 90, F, first, C, taper)
    x = noise_windows(W, m, F * J, 1000 + m + F + C)
    x[1] *= 1e3
    got, _ = device_call(blk, x, ("R",))
    ref = oracle_R(x, blk, taper)
    for c in range(C):
        for w in range(W):
            assert np.max(np.abs(got["R"][c, w] - ref[c, w])) <= 1e-12 * np.max(np.abs(ref[c, w])), (c, w)
    assert np.array_equal(got["R"], np.conj(np.swapaxes(got["R"], 2, 3)))  # Hermitian exactly
    again, _ = device_call(blk, x, ("R",))
    assert np.array_equal(got["R"].view(np.float64), again["R"].view(np.float64))
    blk.close()


@pytest.mark.parametrize("m,F,J,taper", [(4, 64, 4, "hann"), (16, 256, 1, "rect"), (7, 16, 3, "rect")])
def test_a_channels_covariance_does_not_depend_on_the_range(m, F, J, taper):
    W = 4
    x = noise_windows(W, m, F * J, 31 * m + F)
    full = make(m, 1, F * J, 90, F, 0, F, taper)
    R_full, _ = device_call(full, x, ("R",))
    full.close()
    for first, C in ((3, 2), (F - 2, 5), (F // 2, 1)):
        sub = make(m, 1, F * J, 90, F, first, C, taper)
        R_sub, _ = device_call(sub, x, ("R",))
        sub.close()
        for c in range(C):
            assert np.array_equal(R_sub["R"][c].view(np.float64), R_full["R"][(first + c) % F].view(np.float64)), (first, c)


def test_channel_tables_are_the_plain_tables_of_each_wavelength():
    m, K, F, first, C = 5, 360, 16, 14, 4
    pos = planar_pos(m, 3)
    blk = make(m, 1, F * 2, K, F, first, C, pos=pos)
    f = blk.channel_frequencies()
    assert np.array_equal(f, ch.offsets(F, first, C, FS))
    tabs = blk.array_response_c64()
    for c in range(C):
        plain = gh.make_block(m, 1, F * 2, K=K, pos=pos, lam=299792458.0 / (FC + f[c]))
        assert np.array_equal(tabs[c].view(np.float32), plain.array_response_c64().view(np.float32)), c
        plain.close()
    # one measured table for every channel
    t = helpers.random_table(m, K, 9)
    blk.set_array_response(t)
    assert all(np.array_equal(blk.array_response_c64(c), t) for c in range(C))
    blk.close()


def check_separate(blk, x, md, J):
    """every channel of every window against composed_oracle.work_R on the GPU's own R_c and table c"""
    got, _ = device_call(blk, x, ("levels", "bins", "counts", "spectrum", "R"))
    tabs = blk.array_response_c64()
    W = x.shape[0]
    for c in range(blk.chan_count):
        for w in range(W):
            r = cmp.work_R(got["R"][c, w], md, tabs[c], None, blk.n, J)
            ctx = (c, w)
            if r["margin"] > 1e-6:
                assert got["counts"][c, w] == r["count"], ctx
            elif got["counts"][c, w] != r["count"]:
                continue
            P = r["P"]
            assert helpers.rel_err(got["spectrum"][c, w], P) <= P_RTOL, ctx
            for i, (g, b) in enumerate(zip(got["bins"][c, w], r["bins"])):
                if g != b:  # only where the oracle sees a tie inside fp64 noise
                    assert g >= 0 and b >= 0 and abs(P[g] - P[b]) <= 1e-12 * P[b], ctx + (i, g, b)
                    continue
                if b < 0:
                    assert got["angles"][c, w, i] == 0.0 and got["levels"][c, w, i] == 0.0, ctx
                else:
                    assert got["angles"][c, w, i] == r["angles"][i], ctx
                    assert abs(got["levels"][c, w, i] - r["levels"][i]) <= P_RTOL * abs(r["levels"][i]), ctx
    return got


ESTS = {"music": ("music", 0.0), "mvdr": ("mvdr", 1e-3), "bartlett": ("bartlett", 0.0)}
PEAKS = {"top": ("top_bins", 0), "local": ("local_maxima", 3)}


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("rule", cmp.RULES)
@pytest.mark.parametrize("peak", sorted(PEAKS))
@pytest.mark.parametrize("est", sorted(ESTS))
def test_separate_matches_the_composed_oracle_per_channel(est, peak, rule, n):
    m, K, F, J, first, C, W = 4, 360, 16, 32, 14, 5, 6
    pos = planar_pos(m, 17)
    blk = make(m, n, F * J, K, F, first, C, "hann", "separate", pos, ESTS[est], rule, *PEAKS[peak])
    x = scene_windows(W, pos, F, F * J, first, C, 4000 + n)
    x[0] = noise_windows(1, m, F * J, 8)[0] * 0.1  # every channel empty
    md = cmp.modes(peak=peak, exclusion=PEAKS[peak][1], est=est, loading=ESTS[est][1], rule=rule)
    got = check_separate(blk, x, md, J)
    if rule == "fixed":
        assert np.all(got["counts"] == n)
    blk.close()


@pytest.mark.parametrize("m,n,F,J,first,C,est,peak,rule", [
    (7, 3, 8, 16, 5, 6, "music", "local", "mdl"), (16, 2, 8, 24, 0, 8, "mvdr", "top", "aic"), (16, 1, 64, 18, 40, 30, "music", "top", "fixed"),
    (8, 1, 256, 9, 0, 3, "music", "top", "mdl"), (2, 1, 8, 4, 7, 2, "bartlett", "top", "fixed"), (8, 3, 64, 1, 0, 4, "bartlett", "local", "fixed"),
])
def test_separate_on_other_shapes(m, n, F, J, first, C, est, peak, rule):
    K, W = 180, 3
    pos = planar_pos(m, 23)
    loading = 1e-2 if est == "mvdr" else 0.0
    blk = make(m, n, F * J, K, F, first, C, "rect", "separate", pos, (est, loading), rule, *PEAKS[peak])
    x = scene_windows(W, pos, F, F * J, first, C, 77 + m)
    check_separate(blk, x, cmp.modes(peak=peak, exclusion=PEAKS[peak][1], est=est, loading=loading, rule=rule), J)
    blk.close()


@pytest.mark.parametrize("m,n,F,J,first,C,peak", [(4, 1, 16, 16, 10, 11, "top"), (4, 2, 16, 16, 0, 16, "local"), (7, 2, 8, 10, 6, 3, "top"),
                                                  (16, 3, 64, 20, 0, 64, "local")])
def test_incoherent_matches_the_oracle(m, n, F, J, first, C, peak):
    K, W = 360, 4
    pos = planar_pos(m, 41)
    blk = make(m, n, F * J, K, F, first, C, "hann", "incoherent", pos, mode=PEAKS[peak][0], excl=PEAKS[peak][1])
    rng = np.random.default_rng(m + C)
    x = np.stack([ch.white_source(rng, pos, FC, FS, F * J, rng.uniform(0, 360)) for _ in range(W)])
    got, _ = device_call(blk, x, ("levels", "bins", "spectrum", "R"))
    tabs = blk.array_response_c64()
    assert got["angles"].shape == (1, W, n)
    for w in range(W):
        P, (ang, lvl, bins) = ch.incoherent(got["R"][:, w], tabs, n, peak, PEAKS[peak][1])
        assert helpers.rel_err(got["spectrum"][0, w], P) <= P_RTOL, w
        for i, (g, b) in enumerate(zip(got["bins"][0, w], bins)):
            if g != b:
                assert g >= 0 and b >= 0 and abs(P[g] - P[b]) <= 1e-12 * P[b], (w, i, g, b)
            elif b >= 0:
                assert got["angles"][0, w, i] == np.float32(ang[i]), (w, i)
                assert abs(got["levels"][0, w, i] - lvl[i]) <= P_RTOL * abs(lvl[i]), (w, i)
    blk.close()


def test_incoherent_with_one_channel_is_that_channel():
    m, n, K, F, J, W = 4, 2, 360, 16, 16, 5
    pos = planar_pos(m, 2)
    x = scene_windows(W, pos, F, F * J, 3, 1, 12)
    sep = make(m, n, F * J, K, F, 3, 1, "hann", "separate", pos)
    inc = make(m, n, F * J, K, F, 3, 1, "hann", "incoherent", pos)
    a, _ = device_call(sep, x, ("levels", "bins", "spectrum"))
    b, _ = device_call(inc, x, ("levels", "bins", "spectrum"))
    assert np.array_equal(a["bins"], b["bins"]) and np.array_equal(a["angles"], b["angles"])
    assert helpers.rel_err(b["levels"], a["levels"]) <= 1e-6 and helpers.rel_err(b["spectrum"], a["spectrum"]) <= 1e-6
    sep.close()
    inc.close()


@pytest.mark.parametrize("combine,rule,n", [("separate", "mdl", 2), ("separate", "fixed", 1), ("incoherent", "fixed", 2)])
def test_entries_and_blocks_agree(combine, rule, n):
    """outputs do not depend on which are requested; host entry = device entry byte for byte; the Python block and the
    C++ block hand out the transposed C-ABI results"""
    m, K, F, J, first, C, W = 4, 120, 16, 12, 13, 6, 7
    pos = planar_pos(m, 6)
    blk = make(m, n, F * J, K, F, first, C, "hann", combine, pos, rule=rule)
    x = scene_windows(W, pos, F, F * J, first, C, 99)
    sep = combine == "separate"
    every = ("levels", "bins", "spectrum", "R") + (("counts",) if sep else ())
    full, _ = device_call(blk, x, every)
    for subset in ((), ("bins",), ("levels", "spectrum"), ("R",)):
        part, _ = device_call(blk, x, subset)
        for k, v in part.items():
            assert np.array_equal(v.view(np.uint8), full[k].view(np.uint8)), (subset, k)
    host = blk.process_host(x, W, levels=True, spectrum=True, bins=True, counts=sep, R=True)
    for k, v in host.items():
        assert np.array_equal(np.ascontiguousarray(v).view(np.uint8), full[k].view(np.uint8)), k
    # the Python block: window-major items
    r = blk.rows
    ports = [np.zeros((W, r * n), np.float32), np.zeros((W, r * n), np.float32), np.zeros((W, r * K), np.float32)]
    assert blk.work(W, [x], ports) == W
    items = lambda a: np.ascontiguousarray(np.swapaxes(a, 0, 1)).reshape(W, -1)
    assert np.array_equal(ports[0], items(full["angles"])) and np.array_equal(ports[1], items(full["levels"]))
    assert np.array_equal(ports[2], items(full["spectrum"]))
    assert np.array_equal(blk.last_bins().reshape(W, -1), items(full["bins"]))
    if sep:
        assert np.array_equal(blk.last_counts(), full["counts"].T)
    # the C++ block
    rules = {"fixed": 0, "mdl": 1, "aic": 2}
    header = struct.pack("<14I3d", m, n, m * F * J, K, F, first, C, TAPERS["hann"], COMBINES[combine], W, 0, 0, rules[rule], 0, 0.0, FC, FS)
    layout = [("angles", np.float32, W * r * n), ("levels", np.float32, W * r * n), ("spectrum", np.float32, W * r * K),
              ("bins", np.int32, W * r * n), ("counts", np.int32, W * C if sep else 0), ("freqs", np.float64, C)]
    cpp = gh.run_cpp_block("test_block_channels", header, [pos.astype(np.float64), x.view(np.float32)], layout)
    for k in ("angles", "levels", "spectrum", "bins"):
        assert np.array_equal(cpp[k].reshape(W, -1), items(full[k])), k
    if sep:
        assert np.array_equal(cpp["counts"].reshape(W, C), full["counts"].T)
    assert np.array_equal(cpp["freqs"], blk.channel_frequencies())
    blk.close()


def sub_windows(blk, p64, counts):
    """Python restatement of the workspace bound: windows per sub-batch"""
    m, K, n, C = blk.m, blk.resolution, blk.n, blk.chan_count
    per = m * m * 2 * 8 * 2 + m * 8 + (K * 8 if p64 else 0) + (4 if counts else 0)
    c = (384 << 20) // (per * C)
    return max(SCAN_B, min(c, 1 << 20)) // SCAN_B * SCAN_B


def planned_launches(blk, W, est, peak, rule, counts_asked):
    """Python restatement of the plan: per sub-batch 1 filter bank + eigensolver [+ count] [+ MVDR preparation] + one scan
    per channel + the peak stage (separate: one launch per channel unless the scan takes the arg-max; incoherent: the
    combine and one peak launch), plus the fill of the counts under FIXED"""
    sep = blk.combine == "separate"
    argmax = sep and blk.n == 1 and peak == "top"
    p64 = not argmax
    sub = min((W + SCAN_B - 1) // SCAN_B * SCAN_B, sub_windows(blk, p64, rule != "fixed"))
    nsub = (W + sub - 1) // sub
    per = 1 + (1 if est == "music" or rule != "fixed" else 0) + (1 if rule != "fixed" else 0) + (1 if est == "mvdr" else 0) + blk.chan_count
    per += (0 if argmax else blk.chan_count) if sep else 2
    return nsub * per + (1 if rule == "fixed" and counts_asked else 0), nsub


@pytest.mark.parametrize("combine,est,peak,rule,n", [
    ("separate", "music", "top", "fixed", 1), ("separate", "music", "top", "mdl", 1), ("separate", "mvdr", "local", "aic", 2),
    ("separate", "bartlett", "top", "fixed", 2), ("incoherent", "music", "top", "fixed", 1), ("incoherent", "music", "local", "fixed", 2),
])
def test_launch_counts_follow_the_plan(combine, est, peak, rule, n):
    m, K, F, J, first, C, W = 4, 90, 8, 8, 6, 5, 11
    blk = make(m, n, F * J, K, F, first, C, "rect", combine, None, ESTS[est], rule, *PEAKS[peak])
    x = noise_windows(W, m, F * J, 5)
    for outs in (("bins",), ("levels", "bins", "counts") if combine == "separate" else ("levels", "spectrum")):
        _, launches = device_call(blk, x, outs)
        assert launches == planned_launches(blk, W, est, peak, rule, "counts" in outs)[0], outs
    blk.close()


def test_a_call_larger_than_one_sub_batch():
    """m = 16 with all 256 channels: 136 windows fill the workspace, so 150 windows run as 136 + 14, and every block of
    the channel-major outputs is written in place"""
    m, n, K, F, J, W = 16, 2, 360, 256, 1, 150
    pos = planar_pos(m, 8)
    blk = make(m, n, F * J, K, F, 0, F, "rect", "separate", pos)
    x = noise_windows(W, m, F * J, 21)
    want, nsub = planned_launches(blk, W, "music", "top", "fixed", True)
    assert nsub == 2 and sub_windows(blk, True, False) == 136
    every = ("levels", "bins", "counts", "spectrum", "R")
    got, launches = device_call(blk, x, every)
    assert launches == want
    head, _ = device_call(blk, x[:136], every)
    tail, _ = device_call(blk, x[136:], every)
    for k in got:
        assert np.array_equal(got[k][:, :136].view(np.uint8), head[k].view(np.uint8)), k
        assert np.array_equal(got[k][:, 136:].view(np.uint8), tail[k].view(np.uint8)), k
    ref = oracle_R(x[140:142], blk, "rect")
    assert np.max(np.abs(got["R"][:, 140:142] - ref)) <= 1e-12 * np.max(np.abs(ref))
    blk.close()


def einval(call, *args, **kw):
    with pytest.raises(MusicB200Error) as e:
        call(*args, **kw)
    assert e.value.code == _capi.EINVAL


def test_what_is_not_built_is_refused_and_the_handle_stays_usable():
    m, n, K, F, J, first, C, W = 4, 2, 90, 8, 8, 0, 4, 3
    pos = planar_pos(m, 1)
    x = noise_windows(W, m, F * J, 3)
    lib = _capi.load()
    buf = np.zeros(1 << 16, np.float32)
    for combine in ("separate", "incoherent"):
        blk = make(m, n, F * J, K, F, first, C, "hann", combine, pos)
        before, _ = device_call(blk, x)
        for mode in ("roots", "esprit", "dml"):
            einval(blk.set_peak_mode, mode)
        einval(blk.set_refine, True)
        for kind in ("das", "mvdr", "lcmv"):
            einval(blk.set_beamformer, kind, 0.0 if kind == "das" else 1e-3)
        einval(blk.set_calibration, np.ones(m, np.complex128))
        einval(blk.calib_reset)
        einval(blk.calib_accumulate, x)
        einval(blk.gather_create, W)
        h, p = blk._h, buf.ctypes.data
        plain_entries = [
            lambda: lib.music_b200_process_host(h, x.ctypes.data, W, p, None, None, None),
            lambda: lib.music_b200_process_host_counts(h, x.ctypes.data, W, p, None, None, None, None),
            lambda: lib.music_b200_process_device(h, p, W, p, None, None, None, None),
            lambda: lib.music_b200_process_device_ex(h, p, W, p, None, None, None, None, None, None, None),
            lambda: lib.music_b200_process_azel_host(h, x.ctypes.data, W, p, p, None, None, None, None),
            lambda: lib.music_b200_process_planar_host(h, p, 1, W, p, None, None, None),
            lambda: lib.music_b200_process_planar_device(h, p, 1, W, p, None, None, None, None),
            lambda: lib.music_b200_process_device_sharded(h, p, W, p, None, None, None),
            lambda: lib.music_b200_set_geometry(h, pos.ctypes.data, LAM0, None),
            lambda: lib.music_b200_set_geometry_azel(h, pos.ctypes.data, LAM0),
            lambda: lib.music_b200_get_table(h, p),
            lambda: lib.music_b200_get_table_channel(h, C, p),
            lambda: lib.music_b200_set_geometry_channels(h, pos.ctypes.data, FS / 2, FS),
        ]
        for i, entry in enumerate(plain_entries):
            assert entry() == _capi.EINVAL, i
        if combine == "incoherent":
            einval(blk.set_estimator, "mvdr", 1e-3)
            einval(blk.set_estimator, "bartlett")
            einval(blk.set_source_rule, "mdl")
            einval(blk.set_source_rule, "aic")
            d = torch.zeros(W * n * 4, dtype=torch.float32, device=gh.DEV)
            d_in = torch.from_numpy(x.view(np.float32)).to(gh.DEV)
            einval(blk.process_device, d_in.data_ptr(), W, d.data_ptr(), d_counts=d.data_ptr())
        after, _ = device_call(blk, x)
        for k in before:
            assert np.array_equal(before[k], after[k]), k
        blk.close()
    # the segments are the looks: J = 2 <= m refuses MDL, AIC and unloaded MVDR although N = 16 > m
    blk = make(m, 1, F * 2, K, F, 0, 2)
    einval(blk.set_source_rule, "mdl")
    einval(blk.set_estimator, "mvdr", 0.0)
    blk.set_estimator("mvdr", 1e-2)
    blk.close()
    # a channel entry on a plain handle
    plain = gh.make_block(m, 1, F * J, K=K)
    assert lib.music_b200_process_channels_host(plain._h, x.ctypes.data, W, buf.ctypes.data, None, None, None, None, None) == _capi.EINVAL
    assert lib.music_b200_process_channels_device(plain._h, buf.ctypes.data, W, buf.ctypes.data, None, None, None, None, None, None) == _capi.EINVAL
    assert lib.music_b200_set_geometry_channels(plain._h, pos.ctypes.data, FC, FS) == _capi.EINVAL
    assert lib.music_b200_channel_frequencies(plain._h, buf.ctypes.data) == _capi.EINVAL
    assert lib.music_b200_get_table_channel(plain._h, 0, buf.ctypes.data) == _capi.EINVAL
    plain.close()


@pytest.mark.parametrize("args", [
    dict(nfft=4), dict(nfft=512), dict(nfft=24), dict(snaps=100), dict(channels=(0, 0)), dict(channels=(0, 17)), dict(channels=(16, 1)),
    dict(n=4), dict(m=17, n=1),
])
def test_invalid_shapes_are_rejected_on_the_host(args):
    a = dict(m=4, n=1, snaps=64, nfft=16, channels=(0, 16))
    a.update(args)
    with pytest.raises(ValueError):
        music_doa_channels(a["m"], a["n"], a["m"] * a["snaps"], 90, a["nfft"], a["channels"], "rect", "separate",
                           np.zeros((a["m"], 2)), 1.0, FC, FS)


def test_no_table_no_call():
    """create_channels() installs no table: a call before set_geometry_channels() / set_table() is refused"""
    lib = _capi.load()
    h = ctypes.c_void_p()
    assert lib.music_b200_create_channels(ctypes.byref(h), 4, 1, 4 * 64, 90, 16, 0, 4, 0, 0, 0) == _capi.OK
    x = noise_windows(2, 4, 64, 1)
    out = np.zeros(4 * 2, np.float32)
    assert lib.music_b200_process_channels_host(h, x.ctypes.data, 2, out.ctypes.data, None, None, None, None, None) == _capi.EINVAL
    assert lib.music_b200_channel_frequencies(h, out.ctypes.data) == _capi.EINVAL
    table = np.ascontiguousarray(helpers.random_table(4, 90, 1))
    assert lib.music_b200_set_table(h, table.ctypes.data) == _capi.OK
    assert lib.music_b200_process_channels_host(h, x.ctypes.data, 2, out.ctypes.data, None, None, None, None, None) == _capi.OK
    lib.music_b200_destroy(h)


def test_two_emitters_are_separated_on_the_device():
    """the motivating case end to end: each channel reports its own emitter, MDL reports the empty channels empty"""
    m, F, J, K, W = 4, 64, 64, 360, 8
    pos = ch.ula_pos(m, LAM0)
    chans, degs = (6, 58), (50.0, 120.0)
    x = np.stack([ch.two_emitters(np.random.default_rng(300 + s), pos, FC, FS, F, F * J, chans, degs, noise=0.1, walk=0.002) for s in range(W)])
    blk = make(m, 1, F * J, K, F, 0, F, "hann", "separate", pos, rule="mdl")
    got, _ = device_call(blk, x, ("levels", "bins", "counts"))
    for c, deg in zip(chans, degs):
        assert np.all(got["counts"][c] == 1) and np.all(np.abs(got["angles"][c, :, 0] - deg) <= 1.0), c
    near = {(c + d) % F for c in chans for d in (-1, 0, 1)}
    empty = [c for c in range(F) if c not in near]
    assert np.mean(got["counts"][empty] == 0) >= 0.95  # MDL from 64 looks has a small false-alarm rate
    assert np.all(got["bins"][got["counts"] == 0] == -1)
    blk.close()


def test_wideband_source_on_the_device():
    """one source white across a 14 % band near end-fire: the incoherent spectrum over per-channel tables finds it; one
    centre-frequency table for every channel (set_array_response) is biased at the band edge"""
    m, F, J, K, W, deg = 4, 16, 256, 1440, 6, 20.0
    pos = ch.ula_pos(m, ch.C0 / (FC + FS / 2))
    first, C = F // 2 + 2, F - 3
    x = np.stack([ch.white_source(np.random.default_rng(500 + s), pos, FC, FS, F * J, deg) for s in range(W)])
    inc = make(m, 1, F * J, K, F, first, C, "hann", "incoherent", pos)
    got, _ = device_call(inc, x)
    assert np.all(np.abs(got["angles"][0, :, 0] - deg) <= 0.75)
    inc.close()
    sep = make(m, 1, F * J, K, F, first, C, "hann", "separate", pos)
    own, _ = device_call(sep, x)
    sep.set_array_response(ch.table(pos, LAM0, K))
    centre, _ = device_call(sep, x)
    edge = [0, C - 1]
    assert np.max(np.abs(own["angles"][edge, :, 0].mean(axis=1) - deg)) <= 0.75
    assert np.min(np.abs(centre["angles"][edge, :, 0].mean(axis=1) - deg)) >= 5.0
    sep.close()
