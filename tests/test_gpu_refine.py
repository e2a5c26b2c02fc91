"""GPU: off-grid peak refinement (music_b200_set_refine) against its fp64 definition (tests/refine_oracle.py), against
a 1000x finer grid, and through every entry point.

The oracle refines the GPU's own grid bins with LAPACK noise eigenvectors, so what is compared here is the refinement
itself; the grid bins are compared with the same handle with refinement off (byte for byte) and, elsewhere in the
suite, with the C oracle."""
import struct

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, synth
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_helper import music_doa_helper
from oracle import music_oracle as mo

import gpu_harness as gh
import refine_oracle as ro
from helpers import LAM, offgrid_windows, positions

pytestmark = pytest.mark.gpu

N = 256
W = 6
EXCL = 3
FLIP = 1e-9      # decisions the oracle sees this close to flipping may go either way
L_RTOL = 1e-5
ALL = ("levels", "bins", "spectrum", "counts")
PEAKS = ("levels", "bins")


def windows(pos, n_of, seed, snaps=N):
    return offgrid_windows(pos, n_of, seed, snaps)


def handle(m, n, K, pos, snaps=N, devices=None):
    return gh.make_block(m, n, snaps, K, pos=pos, devices=devices)


def ulps_apart(a, b):
    """float32 angles a, b in [0, 360): distance in units of the float32 spacing at the larger one (circular at 0)"""
    d = abs(float(a) - float(b))
    d = min(d, 360.0 - d)
    return d / float(np.spacing(np.float32(max(a, b, 1e-30))))


PARITY = [(m, n) for m in (2, 3, 4, 5, 8, 12, 16) for n in (1, 2, 3) if n < m]


@pytest.mark.parametrize("m,n", PARITY, ids=lambda v: str(v))
def test_parity_with_oracle(m, n):
    """every geometry, K, peak rule and source rule: angles within 1 float32 ulp and levels within 1e-5 of the oracle,
    the same kept-grid decisions except within FLIP of a flip, and grid outputs byte-identical to refinement off"""
    near_flip = slots = 0
    for gi, geometry in enumerate(("ula_x", "ula_y", "uca")):
        pos = positions(geometry, m)
        for K in (360, 3600):
            blk = handle(m, n, K, pos)
            for rule in ("fixed", "mdl"):
                n_of = [n] * W if rule == "fixed" else [w % (n + 1) for w in range(W)]
                x, _ = windows(pos, n_of, 1000 * m + 100 * n + 10 * gi + K % 7)
                blk.set_source_rule(rule)
                for peak in ("top", "local"):
                    ctx = (m, n, geometry, K, rule, peak)
                    blk.set_peak_mode("top_bins" if peak == "top" else "local_maxima", EXCL)
                    blk.set_refine(False)
                    off, _ = gh.device_call(blk, x, ALL)
                    blk.set_refine(True)
                    on, _ = gh.device_call(blk, x, ALL)
                    for k in ("bins", "spectrum", "counts"):
                        assert np.array_equal(on[k].view(np.int32), off[k].view(np.int32)), (ctx, k)
                    for w in range(W):
                        d = int(on["counts"][w])
                        _, V = np.linalg.eigh(mo.covariance(x[w], m))
                        G = V[:, : m - d]
                        for i in range(n):
                            b = int(on["bins"][w, i])
                            if b < 0:
                                assert on["angles"][w, i] == 0.0 and on["levels"][w, i] == 0.0, (ctx, w, i)
                                continue
                            slots += 1
                            r = ro.refine_slot(G, pos, LAM, b, K)
                            ga, gl = on["angles"][w, i], on["levels"][w, i]
                            assert 0.0 <= ga < 360.0, (ctx, w, i, ga)
                            # a refined level is never below the analytic level at the grid angle
                            assert gl >= (1.0 - L_RTOL) * (1.0 / r["Db"]), (ctx, w, i)
                            if ulps_apart(ga, r["angle"]) > 1.0:
                                # only a kept-grid decision the oracle sees on the edge may differ
                                gpu_kept = ga == np.float32(b * 360.0 / K)
                                assert gpu_kept != r["kept"] and ro.flip_margin(r) <= FLIP, (ctx, w, i, ga, r)
                                near_flip += 1
                                continue
                            assert abs(float(gl) - float(r["level"])) <= L_RTOL * float(r["level"]), (ctx, w, i, gl, r["level"])
            blk.close()
    assert slots > 0
    assert near_flip <= max(1, slots // 100), (near_flip, slots)


def test_off_means_off_on_every_entry():
    """a handle switched on and then off gives the bytes of a fresh handle on every entry point, and M = 4 / n = 1
    returns to the fused kernel"""
    for m, n, K in ((4, 1, 3600), (8, 2, 720)):
        pos = positions("uca", m)
        x, _ = windows(pos, [n] * 16, 77 + m)
        fresh, used = handle(m, n, K, pos), handle(m, n, K, pos)
        used.set_refine(True)
        gh.device_call(used, x, ALL)
        used.set_refine(False)
        assert not used.refine
        a, la = gh.device_call(fresh, x, PEAKS)
        b, lb = gh.device_call(used, x, PEAKS)
        assert la == lb and (m != 4 or la == 1), (la, lb)
        for k in a:
            assert np.array_equal(a[k].view(np.int32), b[k].view(np.int32)), (m, k)
        outs = []
        for blk in (fresh, used):
            ang, lvl, spec = np.zeros((16, n), np.float32), np.zeros((16, n), np.float32), np.zeros((16, K), np.float32)
            blk.work(16, [x], [ang, lvl, spec])
            xs = x.reshape(16, N, m)
            streams = [np.ascontiguousarray(xs[:, :, r].reshape(-1)) for r in range(m)]
            pa, pl = np.zeros((16, n), np.float32), np.zeros((16, n), np.float32)
            blk.work_planar(16, streams, [pa, pl])
            outs.append([ang, lvl, spec, blk.last_bins().copy(), pa, pl])
        for u, v in zip(*outs):
            assert np.array_equal(u.view(np.int32), v.view(np.int32)), m
        fresh.close()
        used.close()


@pytest.mark.parametrize("cid", [2, 4])
def test_against_a_1000x_finer_grid(cid):
    """refined angles at K = 360 against the arg-max of a K = 360 000 handle on the same windows.  The fine handle scans
    the float32-rounded table, and P is conditioned about 4000x, so its arg-max can sit more than one fine bin away from
    the analytic optimum; the tolerance is one fine bin plus the largest such distance, computed here on the CPU with
    the numpy scan of the same rounded table and LAPACK eigenvectors"""
    cfg = synth.config(cid, snapshots=1024)
    m, Kc, Kf, Wc = cfg["m"], 360, 360000, 8
    pos = positions(cfg["geometry"], m)
    x = synth.gen_windows_numpy(cfg, 2718 + cid, 0, Wc)
    coarse = handle(m, 1, Kc, pos, snaps=1024)
    coarse.set_refine(True)
    rc, _ = gh.device_call(coarse, x, ("levels", "bins", "counts"))
    fine = handle(m, 1, Kf, pos, snaps=1024)
    rf, _ = gh.device_call(fine, x, ("levels", "bins", "counts"))
    table_f = fine.array_response_c64().astype(np.complex128)
    coarse.close()
    fine.close()
    fine_deg = 360.0 / Kf
    dist = lambda a, b: float(ro.angle_error(a, b, cfg["geometry"]))
    worst_cpu = 0.0
    for w in range(Wc):
        _, V = np.linalg.eigh(mo.covariance(x[w], m))
        G = V[:, : m - 1]
        P = 1.0 / np.sum(np.abs(table_f @ G.conj()) ** 2, axis=1)
        kf = int(np.argmax(P))
        r = ro.refine_slot(G, pos, LAM, int(rc["bins"][w, 0]), Kc)
        worst_cpu = max(worst_cpu, dist(kf * fine_deg, np.degrees(r["theta"])))
    tol = fine_deg + worst_cpu
    print("K = 360 000 arg-max vs analytic optimum on the CPU: up to %.2e deg; tolerance %.2e deg" % (worst_cpu, tol))
    for w in range(Wc):
        assert dist(rc["angles"][w, 0], rf["bins"][w, 0] * fine_deg) <= tol, (w, rc["angles"][w, 0], rf["bins"][w, 0])


def test_edges():
    m, n, K = 8, 1, 360
    pos = positions("uca", m)
    blk = handle(m, n, K, pos)
    blk.set_refine(True)
    # sources just either side of 0 degrees: outputs in [0, 360)
    rng = np.random.default_rng(5)
    xs = []
    for t in (0.05, 359.95, 0.05, 359.95):
        a = ro.steering(pos, LAM, np.deg2rad(t))[0]
        X = a[:, None] * np.exp(2j * np.pi * rng.uniform(0, 1, N))[None, :]
        X += 0.01 * (rng.standard_normal((m, N)) + 1j * rng.standard_normal((m, N)))
        xs.append(X.T.reshape(-1))
    x = np.array(xs).astype(np.complex64)
    got, _ = gh.device_call(blk, x, ALL)
    assert np.all(got["angles"] >= 0.0) and np.all(got["angles"] < 360.0), got["angles"]
    err = ro.angle_error(got["angles"][:, 0], np.array([0.05, 359.95, 0.05, 359.95]), "uca")
    assert np.all(err < 0.02), err
    # NaN windows (both rules), all-zero and noise-only windows under MDL: (0, 0, -1)
    xe, _ = windows(pos, [1, 1, 0, 1], 9)
    xe[0] = 0
    xe[1, 5] = np.nan
    for rule in ("fixed", "mdl"):
        blk.set_source_rule(rule)
        got, _ = gh.device_call(blk, xe, ALL)
        empty = [1] if rule == "fixed" else [0, 1, 2]
        for w in empty:
            assert got["bins"][w, 0] == -1 and got["angles"][w, 0] == 0.0 and got["levels"][w, 0] == 0.0, (rule, w)
        assert got["bins"][3, 0] >= 0 and got["levels"][3, 0] > 0.0
    blk.close()


def test_entries_agree():
    """work(), process_device, planar host / device, the helper, multi-device handles on device 0 and on every GPU"""
    m, n, K, Wn = 8, 2, 720, 24
    pos = positions("uca", m)
    x, _ = windows(pos, [n] * Wn, 31)
    blk = handle(m, n, K, pos)
    blk.set_peak_mode("local_maxima", EXCL)
    blk.set_refine(True)
    assert blk.refine
    ref, _ = gh.device_call(blk, x, PEAKS)
    # the device entry without bins, angles only
    nb, _ = gh.device_call(blk, x)
    assert np.array_equal(nb["angles"], ref["angles"])
    blk.close()

    def make(devices=None):
        b = handle(m, n, K, pos, devices=devices)
        b.set_peak_mode("local_maxima", EXCL)
        b.set_refine(True)
        return b

    # planar device without bins: the workspace holds them
    e = gh.entry_outputs(make, x, planar_outputs=("levels",))
    ang, lvl = e["host"]["angles"], e["host"]["levels"]
    assert np.array_equal(ang, ref["angles"]) and np.array_equal(lvl, ref["levels"]) and np.array_equal(e["host"]["bins"], ref["bins"])
    assert not np.array_equal(ang, (ref["bins"] * (360.0 / K)).astype(np.float32))  # refined, not grid angles
    pa, pl = e["planar_host"]["angles"], e["planar_host"]["levels"]
    assert np.array_equal(pa, ref["angles"]) and np.array_equal(pl, ref["levels"])
    da, dl = e["planar_device"]["angles"], e["planar_device"]["levels"]
    assert np.array_equal(da, ref["angles"]) and np.array_equal(dl, ref["levels"])
    for devices in ([0], list(range(torch.cuda.device_count()))):
        a2, l2 = e["multi_host%s" % devices]["angles"], e["multi_host%s" % devices]["levels"]
        assert np.array_equal(a2, ref["angles"]) and np.array_equal(l2, ref["levels"]), devices
        g = e["multi_device%s" % devices]
        assert np.array_equal(g["angles"], ref["angles"]) and np.array_equal(g["bins"], ref["bins"]), devices
    # the helper installs the geometry and keeps refining across a retune
    cfg = synth.config(4, snapshots=N, resolution=K)
    hx = synth.gen_windows_numpy(cfg, 99, 0, 8)
    hp = music_doa_helper(m, 1, m * N, K, synth.FREQUENCY, synth.SPACING, cfg["antenna_array"], refine=True)
    assert hp.impl.refine
    plain = handle(m, 1, K, positions("uca", m))
    plain.set_refine(True)
    pr, _ = gh.device_call(plain, hx, PEAKS)
    plain.close()
    ha, hl = np.zeros((8, 1), np.float32), np.zeros((8, 1), np.float32)
    hp.work(8, [hx], [ha, hl])
    assert np.array_equal(ha, pr["angles"]) and np.array_equal(hl, pr["levels"])
    hp.set_frequency(synth.FREQUENCY * 1.01)
    hp.work(8, [hx], [ha, hl])
    assert hp.impl.refine and np.all(hp.impl.last_bins() >= 0)
    hp.impl.close()


def test_sharded_entry():
    G = torch.cuda.device_count()
    if G < 2:
        pytest.skip("process_device_sharded needs two or more GPUs")
    m, n, K, Wn = 8, 1, 720, 40
    pos = positions("uca", m)
    x, _ = windows(pos, [n] * Wn, 41)
    blk = handle(m, n, K, pos)
    blk.set_refine(True)
    ref, _ = gh.device_call(blk, x, PEAKS)
    blk.close()
    mb = handle(m, n, K, pos, devices=list(range(G)))
    mb.set_refine(True)
    for g, sh in enumerate(gh.sharded_call(mb, x)):
        assert np.array_equal(sh["angles"], ref["angles"][g::G]), g
        assert np.array_equal(sh["bins"], ref["bins"]), g
    mb.close()


def test_launch_counts_and_sub_batches():
    # M = 4 / n = 1 leaves the fused kernel: cov4_tma + eig + scan_peak1 + refine
    pos = positions("ula_x", 4)
    x, _ = windows(pos, [1] * 8, 3)
    blk = handle(4, 1, 3600, pos)
    _, l_off = gh.device_call(blk, x, PEAKS)
    blk.set_refine(True)
    _, l_on = gh.device_call(blk, x, PEAKS)
    assert (l_off, l_on) == (1, 4)
    blk.close()
    # several sub-batches: one extra launch in each, and the whole call equals two calls over its halves
    m, n, Nb, Kb, Wb = 4, 2, 64, 36000, 3000
    pos = positions("uca", m)
    x, _ = windows(pos, [w % 3 for w in range(Wb)], 808, snaps=Nb)
    blk = handle(m, n, Kb, pos, snaps=Nb)
    dev = torch.device("cuda:0")
    d_in = torch.from_numpy(x.view(np.float32)).to(dev)

    def run(w0, nw, o):
        l0 = blk.launch_count()
        blk.process_device(d_in[w0].data_ptr(), nw, o[0][w0].data_ptr(), o[1][w0].data_ptr(), None, o[2][w0].data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return blk.launch_count() - l0

    outs = lambda: [torch.full((Wb, n), gh.SENTINEL, dtype=torch.float32, device=dev), torch.full((Wb, n), gh.SENTINEL, dtype=torch.float32, device=dev),
                    torch.full((Wb, n), gh.SENTINEL, dtype=torch.int32, device=dev)]
    per_sub = 4  # cov4_tma + eig + scan + top-n
    l_off = run(0, Wb, outs())
    assert l_off % per_sub == 0 and l_off // per_sub >= 2
    blk.set_refine(True)
    whole = outs()
    l_on = run(0, Wb, whole)
    assert l_on % (per_sub + 1) == 0 and l_on // (per_sub + 1) >= 2, (l_off, l_on)
    assert run(0, 8, outs()) == per_sub + 1
    halves = outs()
    run(0, Wb // 2, halves)
    run(Wb // 2, Wb - Wb // 2, halves)
    for a, b in zip(whole, halves):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    blk.close()


def test_errors():
    L = _capi.load()
    m, K = 4, 360
    pos = positions("uca", m)
    blk = music_doa(m, 1, m * N, np.ones((K, m), np.complex64), K)
    for mode in (-1, 2, 7):
        assert L.music_b200_set_refine(blk._h, mode) == _capi.EINVAL
    assert L.music_b200_set_refine(blk._h, 1) == _capi.EINVAL  # table only: no geometry
    with pytest.raises(_capi.MusicB200Error):
        blk.set_refine(True)
    assert not blk.refine and L.music_b200_set_refine(blk._h, 0) == _capi.OK
    blk.set_array_geometry(pos, LAM)
    blk.set_refine(True)
    x, _ = windows(pos, [1] * 4, 13)
    gh.device_call(blk, x, ALL)
    blk.set_array_response(np.ones((K, m), np.complex64))  # a table without geometry: the next call must fail
    with pytest.raises(_capi.MusicB200Error) as e:
        gh.device_call(blk, x, ALL)
    assert e.value.code == _capi.EINVAL
    with pytest.raises(_capi.MusicB200Error) as e:
        blk.work(4, [x], [np.zeros((4, 1), np.float32)])
    assert e.value.code == _capi.EINVAL
    blk.set_refine(False)
    gh.device_call(blk, x, ALL)
    blk.close()


def test_cpp_block_refine():
    m, n, K, Wn = 8, 2, 720, 12
    pos = positions("uca", m)
    x, _ = windows(pos, [n] * Wn, 55)
    table = np.ones((K, m), np.complex64)
    geometry = np.ascontiguousarray(pos).tobytes() + struct.pack("<d", LAM)
    c = gh.run_cpp_block("test_block", struct.pack("<5I", m, n, m * N, K, Wn), [table, table, x],
                         [("a", np.float32, Wn * n), ("l", np.float32, Wn * n), ("s", np.float32, Wn * K),
                          ("b", np.int32, Wn * n), ("c", np.int32, Wn)], args=("0", geometry))
    ang, lvl, spec = c["a"].reshape(Wn, n), c["l"].reshape(Wn, n), c["s"].reshape(Wn, K)
    bins, counts = c["b"].reshape(Wn, n), c["c"]
    assert np.all(counts == n)
    py = handle(m, n, K, pos)
    py.set_refine(True)
    pa, pl, ps = np.zeros((Wn, n), np.float32), np.zeros((Wn, n), np.float32), np.zeros((Wn, K), np.float32)
    py.work(Wn, [x], [pa, pl, ps])
    assert np.array_equal(ang, pa) and np.array_equal(lvl, pl) and np.array_equal(spec, ps) and np.array_equal(bins, py.last_bins())
    py.close()
