"""GPU: (azimuth, elevation) MUSIC (music_b200_create_azel) against its fp64 definition (tests/azel_oracle.py), through
every entry point, and its refusals.

The oracle runs on the device table read back with get_table (the table itself is checked to one float32 ulp), so what
is compared is the pipeline: flat scan, both peak rules, the decode and the 2-D refinement."""
import os
import struct
import subprocess

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, build
from gr_baz_b200.music_doa_azel import music_doa_azel
from oracle import music_oracle as mo

import azel_oracle as ao

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1.0
SNAPS = 256
W = 4
EXCL = 2
SENTINEL = -7
TIE = 1e-12      # bins may differ where the oracle's strengths at the two bins agree to this
FLIP = 1e-9      # refinement decisions this close to flipping may go either way
L_RTOL = 1e-5
D_FLOOR = 1e-12  # per antenna: below this D is rounding noise of the fp64 sums

GEOMETRIES = {
    "uca": (lambda m: ao.uca_xyz(m, LAM), (0.0, 90.0)),
    "uca_z": (lambda m: ao.uca_xyz(m, LAM, alternate_z=True), (-90.0, 90.0)),
    "ura": (lambda m: ao.ura_xyz(4, 4, LAM), (0.0, 90.0)),
}
MATRIX = [(m, g) for m in (3, 4, 8, 16) for g in ("uca", "uca_z")] + [(16, "ura")]


def handle(m, n, grid, pos, snaps=SNAPS):
    return music_doa_azel(m, n, m * snaps, grid.n_az, grid.n_el, (grid.el_lo, grid.el_hi), pos, LAM)


def dev_call(blk, x, n, K, spectrum=True, bins=True, levels=True, counts=True):
    dev = torch.device("cuda:0")
    Wn = x.shape[0]
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)
    o = {"azimuth": torch.full((Wn, n), SENTINEL, dtype=torch.float32, device=dev),
         "elevation": torch.full((Wn, n), SENTINEL, dtype=torch.float32, device=dev)}
    if levels:
        o["levels"] = torch.full((Wn, n), SENTINEL, dtype=torch.float32, device=dev)
    if spectrum:
        o["spectrum"] = torch.full((Wn, K), SENTINEL, dtype=torch.float32, device=dev)
    if bins:
        o["bins"] = torch.full((Wn, n), SENTINEL, dtype=torch.int32, device=dev)
    if counts:
        o["counts"] = torch.full((Wn,), SENTINEL, dtype=torch.int32, device=dev)
    p = lambda k: o[k].data_ptr() if k in o else None
    l0 = blk.launch_count()
    blk.process_device(d_in.data_ptr(), Wn, p("azimuth"), p("elevation"), p("levels"), p("spectrum"), p("bins"), p("counts"),
                       stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}, blk.launch_count() - l0


def ulps_apart(a, b, circular=True):
    d = abs(float(a) - float(b))
    if circular:
        d = min(d, 360.0 - d)
    return d / float(np.spacing(np.float32(max(abs(a), abs(b), 1e-30))))


def check_table(dev_table, pos, grid):
    """each component within one float32 ulp of the fp64 definition (absolute 1e-14 at zero crossings, where the
    value is the rounding error of the phase)"""
    ref = ao.table(pos, LAM, grid)
    for part in ("real", "imag"):
        a, b = getattr(dev_table, part).ravel().astype(np.float64), getattr(ref, part).ravel()
        ok = np.abs(a - b) <= np.spacing(np.abs(b).astype(np.float32)).astype(np.float64) + 1e-14
        assert ok.all(), np.argwhere(~ok)[:5]


@pytest.mark.parametrize("m,geometry", MATRIX, ids=lambda v: str(v))
def test_parity_with_oracle(m, geometry):
    pos_of, el_range = GEOMETRIES[geometry]
    pos = pos_of(m)
    near = slots = 0
    for gi, (n_az, n_el) in enumerate(((36, 10), (360, 46))):
        grid = ao.Grid(n_az, n_el, *el_range)
        for n in (1, 2):
            blk = handle(m, n, grid, pos)
            T = blk.array_response_c64()
            check_table(T, pos, grid)
            T = T.reshape(grid.K, m)
            for rule in ("fixed", "mdl"):
                n_of = [n] * W if rule == "fixed" else [w % (n + 1) for w in range(W)]
                x, _ = ao.windows(pos, LAM, n_of, 1000 * m + 10 * gi + n + (0 if rule == "fixed" else 5), SNAPS, el_range)
                blk.set_source_rule(rule)
                for peak in ("top", "local"):
                    ctx = (m, geometry, n_az, n_el, n, rule, peak)
                    blk.set_peak_mode("top_bins" if peak == "top" else "local_maxima", EXCL)
                    blk.set_refine(False)
                    off, _ = dev_call(blk, x, n, grid.K)
                    blk.set_refine(True)
                    on, _ = dev_call(blk, x, n, grid.K)
                    for k in ("bins", "spectrum", "counts"):
                        assert np.array_equal(on[k].view(np.int32), off[k].view(np.int32)), (ctx, k)
                    for w in range(W):
                        r = ao.work(x[w], m, n, T, grid, peak, EXCL, None if rule == "fixed" else rule)
                        assert off["counts"][w] == r["count"], (ctx, w)
                        P = r["P"]
                        rel = np.abs(off["spectrum"][w].astype(np.float64) - P) / P
                        assert np.nanmax(rel) <= L_RTOL, (ctx, w)
                        for i in range(n):
                            gb, ob = int(off["bins"][w, i]), int(r["bins"][i])
                            if gb != ob:
                                assert gb >= 0 and ob >= 0 and abs(P[gb] - P[ob]) <= TIE * P[ob], (ctx, w, i, gb, ob)
                                break  # later slots depend on this pick
                            if gb < 0:
                                assert off["azimuth"][w, i] == 0 and off["elevation"][w, i] == 0 and off["levels"][w, i] == 0
                                assert on["azimuth"][w, i] == 0 and on["elevation"][w, i] == 0 and on["levels"][w, i] == 0
                                continue
                            assert off["azimuth"][w, i] == r["azimuth"][i] and off["elevation"][w, i] == r["elevation"][i], (ctx, w, i)
                            assert abs(float(off["levels"][w, i]) - float(r["levels"][i])) <= L_RTOL * float(r["levels"][i])
                            # refinement of the same grid bin with the oracle's noise subspace
                            slots += 1
                            G = r["G"]
                            q = ao.refine_slot(G, pos, LAM, gb, grid)
                            ga, ge, gl = on["azimuth"][w, i], on["elevation"][w, i], on["levels"][w, i]
                            assert 0.0 <= ga < 360.0 and grid.el_lo - 1e-4 <= ge <= grid.el_hi + 1e-4, (ctx, w, i, ga, ge)
                            if ulps_apart(ga, q["azimuth"]) > 1.0 or ulps_apart(ge, q["elevation"], False) > 1.0:
                                assert q["margin"] <= FLIP, (ctx, w, i, (ga, ge), q)
                                near += 1
                                continue
                            if q["Dx"] <= D_FLOOR * m:
                                # D reached its rounding floor (a one-vector noise subspace has exact zeros in 2-D):
                                # the level 1 / D is rounding noise, so D itself is compared
                                assert 1.0 / float(gl) <= 2 * D_FLOOR * m, (ctx, w, i, gl, q["Dx"])
                                continue
                            assert abs(float(gl) - float(q["level"])) <= L_RTOL * float(q["level"]), (ctx, w, i, gl, q["level"])
            blk.close()
    assert slots > 0
    assert near <= max(1, slots // 50), (near, slots)


def test_refinement_beats_the_half_step_at_20db():
    m, n = 8, 1
    pos = ao.uca_xyz(m, LAM)
    grid = ao.Grid(360, 46, 0.0, 90.0)
    x, truth = ao.windows(pos, LAM, [1] * 64, 4242, 1024, (10.0, 70.0))
    blk = handle(m, n, grid, pos, snaps=1024)
    err = {}
    for refine in (False, True):
        blk.set_refine(refine)
        o, _ = dev_call(blk, x, n, grid.K, spectrum=False)
        ea = [abs((float(o["azimuth"][w, 0]) - truth[w][0][0] + 180.0) % 360.0 - 180.0) for w in range(len(x))]
        ee = [abs(float(o["elevation"][w, 0]) - truth[w][0][1]) for w in range(len(x))]
        err[refine] = (float(np.sqrt(np.mean(np.square(ea)))), float(np.sqrt(np.mean(np.square(ee)))))
    blk.close()
    print("RMS (az, el) error in degrees: grid %s, refined %s" % (err[False], err[True]))
    assert err[True][0] < 0.5 and err[True][1] < 1.0  # half of the 1 deg / 2 deg steps
    assert err[True][0] < err[False][0] and err[True][1] < err[False][1]


def test_host_and_device_entries_agree():
    m, n = 4, 2
    pos = ao.uca_xyz(m, LAM)
    for (n_az, n_el), Wn, snaps in (((36, 10), 24, SNAPS), ((360, 181), 2000, 64)):
        grid = ao.Grid(n_az, n_el, 0.0, 90.0)
        x, _ = ao.windows(pos, LAM, [w % 3 for w in range(Wn)], 77 + n_el, snaps)
        blk = handle(m, n, grid, pos, snaps=snaps)
        blk.set_source_rule("mdl")
        blk.set_peak_mode("local_maxima", EXCL)
        blk.set_refine(True)
        spec = Wn * grid.K * 4 < (1 << 30)
        ref, launches = dev_call(blk, x, n, grid.K, spectrum=spec)
        if n_el == 181:
            assert launches > 2 * 6, launches  # more than one workspace sub-batch
        outs = [np.zeros((Wn, n), np.float32) for _ in range(3)] + ([np.zeros((Wn, grid.K), np.float32)] if spec else [])
        blk.work(Wn, [x], outs)
        names = ["azimuth", "elevation", "levels"] + (["spectrum"] if spec else [])
        for k, o in zip(names, outs):
            assert np.array_equal(o.view(np.int32), ref[k].view(np.int32)), (n_el, k)
        assert np.array_equal(blk.last_bins(), ref["bins"]) and np.array_equal(blk.last_counts(), ref["counts"])
        # fewer ports and no bins on the device entry: the workspace holds the bins
        a2, e2 = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32)
        blk.work(Wn, [x], [a2, e2])
        assert np.array_equal(a2, ref["azimuth"]) and np.array_equal(e2, ref["elevation"])
        nb, _ = dev_call(blk, x, n, grid.K, spectrum=False, bins=False, levels=False, counts=False)
        assert np.array_equal(nb["azimuth"], ref["azimuth"]) and np.array_equal(nb["elevation"], ref["elevation"])
        blk.close()


def test_fused_kernels_never_run():
    for m in (4, 8):
        pos = ao.uca_xyz(m, LAM)
        grid = ao.Grid(36, 10, 0.0, 90.0)
        blk = handle(m, 1, grid, pos, snaps=1024)
        x, _ = ao.windows(pos, LAM, [1] * 16, 5, 1024)
        _, launches = dev_call(blk, x, 1, grid.K, spectrum=False, levels=True, bins=False, counts=False)
        assert launches == 4, launches  # covariance + eigenvectors + peak scan + decode
        blk.set_refine(True)
        _, launches = dev_call(blk, x, 1, grid.K, spectrum=False, levels=True, bins=False, counts=False)
        assert launches == 5, launches
        blk.close()


def test_settable_table_stage_timing_and_reducers():
    m, n = 8, 1
    pos = ao.uca_xyz(m, LAM)
    grid = ao.Grid(36, 10, 0.0, 90.0)
    blk = handle(m, n, grid, pos)
    x, _ = ao.windows(pos, LAM, [1] * 8, 9, SNAPS)
    geo, _ = dev_call(blk, x, n, grid.K)
    T = blk.array_response_c64()
    assert T.shape == (grid.n_el, grid.n_az, m)
    blk.set_array_response(T)  # the same manifold as a measured table: same grid results
    tab, _ = dev_call(blk, x, n, grid.K)
    for k in geo:
        assert np.array_equal(geo[k].view(np.int32), tab[k].view(np.int32)), k
    with pytest.raises(_capi.MusicB200Error) as e:
        blk.set_refine(True)  # no geometry behind a set table
    assert e.value.code == _capi.EINVAL
    blk.set_array_geometry(pos, LAM)
    blk.set_refine(True)
    blk.set_stage_timing(True)
    dev_call(blk, x, n, grid.K)
    ms, chunks = blk.stage_times_ms()
    assert chunks == 1 and all(v > 0 for v in ms)
    mean, res, wsum = blk.reduce_angles(geo["azimuth"], geo["levels"])
    assert mean.shape == (n,) and wsum[0] == 8
    assert blk.reduce_spectrum(geo["spectrum"]).shape == (grid.K,)
    blk.close()


def test_einval_cases():
    L = _capi.load()
    m, n = 4, 1
    pos = ao.uca_xyz(m, LAM)
    grid = ao.Grid(36, 10, 0.0, 90.0)
    az = handle(m, n, grid, pos)
    one = music_oracle_handle(m, n)
    dev = torch.device("cuda:0")
    d_in = torch.zeros((4, m * SNAPS * 2), dtype=torch.float32, device=dev)
    d_o = torch.zeros((4, n), dtype=torch.float32, device=dev)
    p2 = np.zeros((m, 2))
    # 1-D entries on an az-el handle
    assert L.music_b200_process_device(az._h, d_in.data_ptr(), 4, d_o.data_ptr(), None, None, None, None) == _capi.EINVAL
    assert L.music_b200_process_device_counts(az._h, d_in.data_ptr(), 4, d_o.data_ptr(), None, None, None, None, None) == _capi.EINVAL
    h_in, h_o = np.zeros((4, m * SNAPS), np.complex64), np.zeros((4, n), np.float32)
    assert L.music_b200_process_host(az._h, h_in.ctypes.data, 4, h_o.ctypes.data, None, None, None) == _capi.EINVAL
    assert L.music_b200_process_host_counts(az._h, h_in.ctypes.data, 4, h_o.ctypes.data, None, None, None, None) == _capi.EINVAL
    assert L.music_b200_set_geometry(az._h, p2.ctypes.data, LAM, None) == _capi.EINVAL
    streams = (np.ctypeslib.ctypes.c_void_p * m)(*([h_in.ctypes.data] * m))
    assert L.music_b200_process_planar_host(az._h, streams, SNAPS, 1, h_o.ctypes.data, None, None, None) == _capi.EINVAL
    dstreams = (np.ctypeslib.ctypes.c_void_p * m)(*([d_in.data_ptr()] * m))
    assert L.music_b200_process_planar_device(az._h, dstreams, SNAPS, 1, d_o.data_ptr(), None, None, None, None) == _capi.EINVAL
    buf = (np.ctypeslib.ctypes.c_ubyte * 128)()
    assert L.music_b200_gather_create(az._h, 4, buf) == _capi.EINVAL
    assert L.music_b200_gather_attach(az._h, 1, 0, buf) == _capi.EINVAL
    assert L.music_b200_process_device_sharded(az._h, None, 4, None, None, None, None) == _capi.EINVAL
    # az-el entries on a 1-D handle
    assert L.music_b200_set_geometry_azel(one._h, pos.ctypes.data, LAM) == _capi.EINVAL
    assert L.music_b200_process_azel_device(one._h, d_in.data_ptr(), 4, d_o.data_ptr(), d_o.data_ptr(), None, None, None, None, None) == _capi.EINVAL
    assert L.music_b200_process_azel_host(one._h, h_in.ctypes.data, 4, h_o.ctypes.data, h_o.ctypes.data, None, None, None, None) == _capi.EINVAL
    # missing elevation output, bad geometry on retune, refinement on a set table
    assert L.music_b200_process_azel_device(az._h, d_in.data_ptr(), 4, d_o.data_ptr(), None, None, None, None, None, None) == _capi.EINVAL
    assert L.music_b200_process_azel_host(az._h, h_in.ctypes.data, 4, h_o.ctypes.data, None, None, None, None, None) == _capi.EINVAL
    bad = pos.copy()
    bad[0, 2] = np.inf
    assert L.music_b200_set_geometry_azel(az._h, bad.ctypes.data, LAM) == _capi.EINVAL
    assert L.music_b200_set_geometry_azel(az._h, pos.ctypes.data, -1.0) == _capi.EINVAL
    assert L.music_b200_set_peak_mode(az._h, 1, grid.K) == _capi.EINVAL
    az.set_refine(True)
    az.set_array_response(az.array_response_c64())
    with pytest.raises(_capi.MusicB200Error) as e:
        az.work(4, [h_in], [h_o, h_o.copy()])
    assert e.value.code == _capi.EINVAL
    az.close()
    one.close()


def music_oracle_handle(m, n):
    from gr_baz_b200.music_doa import music_doa

    K = 360
    return music_doa(m, n, m * SNAPS, mo.steering_table_c64([[0.5 * e, 0.0] for e in range(m)], K, LAM), K)


def test_cpp_block_azel(tmp_path):
    build.build_cuda()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "lib"), "-s"])
    m, n, Wn = 8, 2, 12
    pos = ao.uca_xyz(m, LAM, alternate_z=True)
    grid = ao.Grid(72, 19, -90.0, 90.0)
    x, _ = ao.windows(pos, LAM, [n] * Wn, 55, SNAPS, (-90.0, 90.0))
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(struct.pack("<10I", m, n, m * SNAPS, grid.n_az, grid.n_el, Wn, 1, EXCL, 1, 1))
        f.write(struct.pack("<3d", grid.el_lo, grid.el_hi, LAM))
        f.write(np.ascontiguousarray(pos).tobytes())
        f.write(x.view(np.float32).tobytes())
    r = subprocess.run([os.path.join(ROOT, "lib", "_build", "test_block_azel"), str(fin), str(fout)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(fout, dtype=np.float32)
    o, got = 0, {}
    for k, size in (("azimuth", n), ("elevation", n), ("levels", n), ("spectrum", grid.K), ("bins", n), ("counts", 1)):
        got[k] = raw[o:o + Wn * size].reshape(Wn, size)
        o += Wn * size
    assert o == raw.size
    py = handle(m, n, grid, pos)
    py.set_peak_mode("local_maxima", EXCL)
    py.set_source_rule("mdl")
    py.set_refine(True)
    outs = [np.zeros((Wn, n), np.float32) for _ in range(3)] + [np.zeros((Wn, grid.K), np.float32)]
    py.work(Wn, [x], outs)
    for k, v in zip(("azimuth", "elevation", "levels", "spectrum"), outs):
        assert np.array_equal(got[k], v), k
    assert np.array_equal(got["bins"].view(np.int32), py.last_bins())
    assert np.array_equal(got["counts"].view(np.int32).ravel(), py.last_counts())
    py.close()
