"""GPU: a handle whose tables, workspace and host staging have been replaced or grown gives bit for bit what a freshly
created handle in the same final state gives.  Each table sequence retunes at least three times, so that a table slot is
refilled after it has been current; the workspace and the staging buffers grow, shrink and grow past their old size
while the outputs a call asks for change."""
import numpy as np
import pytest

from gr_baz_b200.music_doa_azel import music_doa_azel
from gr_baz_b200.music_doa_channels import music_doa_channels

import gpu_harness as gh
import helpers

pytestmark = pytest.mark.gpu

LAM = helpers.LAM
FC, FS = 400e6, 56e6
LAM0 = 299792458.0 / FC


def same(got, ref, ctx):
    """the same keys with byte-identical values"""
    assert got.keys() == ref.keys(), ctx
    for k in ref:
        if ref[k] is None:
            assert got[k] is None, (ctx, k)
        else:
            a, b = np.asarray(got[k]), np.asarray(ref[k])
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), (ctx, k)


def outputs_1d(blk, x):
    """the fused and the unfused plans through the device entry, the host entry, and the table"""
    out = {"table": blk.array_response_c64()}
    for name, o in (("peaks", ("levels", "bins", "counts")), ("spectrum", ("levels", "spectrum", "bins")),
                    ("unfused", ("levels", "spectrum", "bins", "P64"))):
        for k, v in gh.device_call(blk, x, o)[0].items():
            out[name + "." + k] = v
    for k, v in gh.host_call(blk, x, spectrum=True).items():
        out["host." + k] = v
    return out


@pytest.fixture
def unregistered(monkeypatch):
    """Handles that do not register caller memory (MUSIC_B200_HOSTREG=0).  Two handles here read the same input, and a
    registration rounds the input out to whole pages, which other arrays may share; the results do not depend on it."""
    monkeypatch.setenv("MUSIC_B200_HOSTREG", "0")


@pytest.mark.parametrize("m", [4, 8])
def test_1d_retunes_match_a_fresh_handle(m, unregistered):
    """set_geometry, set_table, set_geometry: the fused screen layout (M = 4) is rebuilt in each refilled slot"""
    K, snaps, W = 360, 256, 96
    p1, p2 = helpers.array_wl("uca", m) * LAM, helpers.array_wl("random", m, seed=3) * LAM
    t0, t1 = helpers.random_table(m, K, 5), helpers.random_table(m, K, 6)
    x = helpers.angle_windows(p1 / LAM, [[40.0 + w] for w in range(W)], False, W, seed=11, snaps=snaps)
    blk = gh.make_block(m, 1, snaps, table=t0)
    steps = [("set_geometry p1", lambda b: b.set_array_geometry(p1, LAM), dict(table=t0, pos=p1)),
             ("set_table t1", lambda b: b.set_array_response(t1), dict(table=t1)),
             ("set_geometry p2", lambda b: b.set_array_geometry(p2, LAM), dict(table=t1, pos=p2))]
    for ctx, step, fresh_state in steps:
        step(blk)
        fresh = gh.make_block(m, 1, snaps, **fresh_state)
        same(outputs_1d(blk, x), outputs_1d(fresh, x), ctx)
        fresh.close()
    blk.close()


def test_azel_retunes_match_a_fresh_handle(unregistered):
    m, n, snaps, W = 6, 2, 128, 48
    rng = np.random.default_rng(21)
    geos = [rng.uniform(-1.0, 1.0, (m, 3)) * LAM for _ in range(3)]
    x = helpers.angle_windows(geos[0][:, :2] / LAM, [[30.0, 140.0]] * W, False, W, seed=12, snaps=snaps)
    make = lambda pos: music_doa_azel(m, n, m * snaps, 72, 9, (0.0, 60.0), pos, LAM)

    def outputs(blk):
        out = {"table": blk.array_response_c64()}
        for k, v in gh.device_call(blk, x, ("levels", "spectrum", "bins", "counts"))[0].items():
            out["device." + k] = v
        for k, v in gh.host_call(blk, x, spectrum=True).items():
            out["host." + k] = v
        return out

    blk = make(geos[0])
    for i in (1, 2, 1):
        blk.set_array_geometry(geos[i], LAM)
        fresh = make(geos[i])
        same(outputs(blk), outputs(fresh), "set_geometry_azel %d" % i)
        fresh.close()
    blk.close()


def make_channels(combine, pos, fc=FC):
    return music_doa_channels(4, 1, 4 * 256, 90, 16, (14, 5), "hann", combine, pos, 1.0, fc, FS)


def outputs_channels(blk, x):
    out = {"tables": blk.array_response_c64()}
    if blk.combine == "coherent":
        out["T"], out["err"] = blk.focusing()
    for k, v in blk.process_host(x, x.shape[0], spectrum=True, counts=True, R=True).items():
        out["host." + k] = v
    return out


def test_channel_retunes_match_a_fresh_handle():
    """separate: set_geometry_channels, set_table (one table for every channel), set_geometry_channels at another centre
    frequency"""
    p1, p2 = helpers.array_wl("uca", 4) * LAM0, helpers.array_wl("random", 4, seed=7) * LAM0
    table = helpers.random_table(4, 90, 8)
    x = helpers.angle_windows(p1 / LAM0, [[50.0]] * 24, False, 24, seed=13, snaps=256)
    blk = make_channels("separate", p1)

    def fresh_table():
        f = make_channels("separate", p2)
        f.set_array_response(table)
        return f

    steps = [("set_geometry_channels p2", lambda b: b.set_array_geometry(p2, FC, FS), lambda: make_channels("separate", p2)),
             ("set_table", lambda b: b.set_array_response(table), fresh_table),
             ("set_geometry_channels p1 at fc + 20 MHz", lambda b: b.set_array_geometry(p1, FC + 20e6, FS),
              lambda: make_channels("separate", p1, FC + 20e6))]
    for ctx, step, fresh_of in steps:
        step(blk)
        fresh = fresh_of()
        same(outputs_channels(blk, x), outputs_channels(fresh, x), ctx)
        fresh.close()
    blk.close()


def test_coherent_retunes_match_a_fresh_handle():
    """coherent: set_geometry_channels, set_focusing (the current tables with new matrices), set_geometry_channels at
    another centre frequency, which keeps the sector"""
    p1, p2 = helpers.array_wl("uca", 4) * LAM0, helpers.array_wl("uca", 4) * LAM0 * 1.1
    x = helpers.angle_windows(p1 / LAM0, [[60.0, 150.0]] * 24, True, 24, seed=14, snaps=256)
    blk = make_channels("coherent", p1)

    def fresh_of(pos, fc, sector):
        f = make_channels("coherent", pos, fc)
        if sector:
            f.set_focusing(*sector)
        return f

    sector = (20, 60)
    steps = [("set_geometry_channels p2", lambda b: b.set_array_geometry(p2, FC, FS), (p2, FC, None)),
             ("set_focusing", lambda b: b.set_focusing(*sector), (p2, FC, sector)),
             ("set_geometry_channels p1 at fc - 30 MHz", lambda b: b.set_array_geometry(p1, FC - 30e6, FS), (p1, FC - 30e6, sector))]
    for ctx, step, state in steps:
        step(blk)
        fresh = fresh_of(*state)
        same(outputs_channels(blk, x), outputs_channels(fresh, x), ctx)
        fresh.close()
    blk.close()


def test_workspace_growth_matches_a_fresh_handle():
    """the unfused workspace grows, shrinks and grows past its old capacity while the spectrum, counts, P64 and beam
    outputs are switched on and off"""
    m, n, snaps, K = 8, 2, 64, 180
    pos = helpers.array_wl("uca", m) * LAM
    settings = dict(K=None, table=helpers.table_wl(pos / LAM, K), pos=pos, rule="mdl", beamformer=("mvdr", 1e-3))
    calls = [(40, ("levels", "bins")),
             (300, ("levels", "spectrum", "counts")),
             (24, ("beams",)),
             (900, ("levels", "spectrum", "bins", "counts", "weights", "beams")),
             (100, ("P64", "bins")),
             (1500, ("levels", "weights")),
             (1500, ("P64",))]
    x_all = helpers.angle_windows(pos / LAM, [[35.0, 120.0]] * 1500, False, 1500, seed=15, snaps=snaps)
    blk = gh.make_block(m, n, snaps, **settings)
    for W, outs in calls:
        fresh = gh.make_block(m, n, snaps, **settings)
        got, ref = gh.device_call(blk, x_all[:W], outs), gh.device_call(fresh, x_all[:W], outs)
        same(got[0], ref[0], (W, outs))
        assert got[1] == ref[1], (W, outs, got[1], ref[1])
        fresh.close()
    blk.close()


def test_host_staging_growth_matches_a_fresh_handle(unregistered):
    """work() with W growing, the spectrum port connected later and the beamformer switched on later"""
    m, n, snaps, K = 4, 1, 512, 360
    pos = helpers.array_wl("uca", m) * LAM
    x_all = helpers.angle_windows(pos / LAM, [[75.0]] * 1200, False, 1200, seed=16, snaps=snaps)
    calls = [(10, False, None), (300, True, None), (600, True, ("das", 0.0)), (1200, True, ("das", 0.0)), (50, False, None)]
    blk = gh.make_block(m, n, snaps, table=helpers.table_wl(pos / LAM, K), pos=pos)
    for W, spectrum, beamformer in calls:
        blk.set_beamformer(*(beamformer or ("off", 0.0)))
        fresh = gh.make_block(m, n, snaps, table=helpers.table_wl(pos / LAM, K), pos=pos, beamformer=beamformer)
        same(gh.host_call(blk, x_all[:W], spectrum), gh.host_call(fresh, x_all[:W], spectrum), (W, spectrum, beamformer))
        fresh.close()
    blk.close()
