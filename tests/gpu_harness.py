"""The plumbing the GPU tests share: build a block, call its device and host entries, run the same windows through every
entry point, and run a C++ block driver of lib/.  Nothing here asserts what a result should be (apart from a driver's
exit code and file size); the comparisons stay in the test modules."""
import contextlib
import os
import subprocess
import tempfile

import numpy as np
import torch

from gr_baz_b200 import build
from gr_baz_b200.music_doa import music_doa
from gr_baz_b200.music_doa_azel import music_doa_azel

import helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = -7
DEV = torch.device("cuda:0")


def stream():
    return torch.cuda.current_stream().cuda_stream


@contextlib.contextmanager
def _environment(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def make_block(m, n, snaps, K=None, table=None, pos=None, lam=helpers.LAM, est=None, rule=None, mode=None, excl=0,
               refine=False, beamformer=None, calibration=None, devices=None, env=None):
    """a 1-D block of m elements, n slots and `snaps` snapshots per window on `table` (default: K all-ones rows), with
    the geometry `pos` installed and then each given setting applied in this order: estimator (kind, loading), source
    rule, peak mode (with `excl` exclusion bins), refinement, beamformer (kind, loading), calibration gains.  `env`:
    environment switches read when the block is created."""
    table = np.ones((K, m), np.complex64) if table is None else table
    with _environment(env or {}):
        blk = music_doa(m, n, m * snaps, table, len(table), devices=devices)
    if pos is not None:
        blk.set_array_geometry(pos, lam)
    if est is not None:
        blk.set_estimator(*est)
    if rule is not None:
        blk.set_source_rule(rule)
    if mode is not None:
        blk.set_peak_mode(mode, excl)
    if refine:
        blk.set_refine(True)
    if beamformer is not None:
        blk.set_beamformer(*beamformer)
    if calibration is not None:
        blk.set_calibration(calibration)
    return blk


def _output_shapes(blk, W):
    m, n, K = blk.m, blk.n, blk.resolution
    N = blk.nsamples // m
    f32, f64, i32 = torch.float32, torch.float64, torch.int32
    return {"angles": ((W, n), f32), "azimuth": ((W, n), f32), "elevation": ((W, n), f32), "levels": ((W, n), f32),
            "spectrum": ((W, K), f32), "bins": ((W, n), i32), "counts": ((W,), i32), "P64": ((W, K), f64),
            "R": ((W, m, m, 2), f64), "eigvals": ((W, m), f64), "weights": ((W, n, m, 2), f64), "beams": ((W, n, N, 2), f32)}


def device_call(blk, x, outputs=(), fill=SENTINEL):
    """One device call on the windows x (complex64 [W][nsamples], host memory) asking for the angles (azimuth and
    elevation on an az-el block) and `outputs`, a subset of levels, spectrum, bins, counts, P64, R, eigvals, weights,
    beams.  The entry is the one these outputs select: process_device_beams with weights or beams, the az-el
    process_device on an az-el block, else process_device_counts with counts and process_device_ex without.  Outputs
    start filled with `fill`.  Returns (numpy outputs, kernel launches); R and weights as complex128, beams as
    complex64."""
    W = x.shape[0]
    azel = isinstance(blk, music_doa_azel)
    shapes = _output_shapes(blk, W)
    keys = (("azimuth", "elevation") if azel else ("angles",)) + tuple(outputs)
    o = {k: torch.full(shapes[k][0], fill, dtype=shapes[k][1], device=DEV) for k in keys}
    p = lambda k: o[k].data_ptr() if k in o else None
    d_in = torch.from_numpy(x.view(np.float32)).to(DEV)
    l0 = blk.launch_count()
    if "weights" in o or "beams" in o:
        blk.process_device_beams(d_in.data_ptr(), W, p("angles"), p("levels"), p("spectrum"), p("bins"), p("counts"),
                                 p("weights"), p("beams"), stream=stream())
    elif azel:
        blk.process_device(d_in.data_ptr(), W, p("azimuth"), p("elevation"), p("levels"), p("spectrum"), p("bins"),
                           p("counts"), stream=stream())
    else:
        blk.process_device(d_in.data_ptr(), W, p("angles"), p("levels"), p("spectrum"), p("bins"), stream=stream(),
                           d_P64=p("P64"), d_R=p("R"), d_eigvals=p("eigvals"), d_counts=p("counts"))
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    for k in ("R", "weights", "beams"):
        if k in out:
            out[k] = out[k][..., 0] + 1j * out[k][..., 1]
    if "beams" in out:
        out["beams"] = out["beams"].astype(np.complex64)
    return out, blk.launch_count() - l0


def host_call(blk, x, spectrum=False):
    """One work() call on all windows of x with the angle and level ports (and the spectrum port): angles (azimuth and
    elevation on an az-el block), levels, spectrum, bins, counts, beams and weights (None while no beamformer is set)."""
    W = x.shape[0]
    azel = isinstance(blk, music_doa_azel)
    names = (["azimuth", "elevation"] if azel else ["angles"]) + ["levels"]
    ports = [np.zeros((W, blk.n), np.float32) for _ in names]
    if spectrum:
        names.append("spectrum")
        ports.append(np.zeros((W, blk.resolution), np.float32))
    blk.work(W, [x], ports)
    return dict(zip(names, ports), bins=blk.last_bins().copy(), counts=blk.last_counts().copy(), beams=blk.last_beams(),
                weights=blk.last_weights())


def sharded_call(blk, x, levels=False):
    """process_device_sharded over every device of a multi-device block, window w on device w % G: per device the
    angles (and levels) of its shard and the peak bins of all windows"""
    G = blk.device_count()
    W, n = x.shape[0], blk.n
    ins, angs, lvls, bins_all = [], [], [], []
    for g in range(G):
        d = torch.device("cuda", g)
        ins.append(torch.from_numpy(np.ascontiguousarray(x[g::G]).view(np.float32)).to(d))
        angs.append(torch.full((len(x[g::G]), n), SENTINEL, dtype=torch.float32, device=d))
        lvls.append(torch.full((len(x[g::G]), n), SENTINEL, dtype=torch.float32, device=d))
        bins_all.append(torch.full((W, n), SENTINEL, dtype=torch.int32, device=d))
    ptrs = lambda ts: [t.data_ptr() for t in ts]
    blk.process_device_sharded(ptrs(ins), W, ptrs(angs), ptrs(lvls) if levels else None, ptrs(bins_all))
    for g in range(G):
        torch.cuda.synchronize(g)
    return [{"angles": angs[g].cpu().numpy(), "bins": bins_all[g].cpu().numpy(),
             **({"levels": lvls[g].cpu().numpy()} if levels else {})} for g in range(G)]


def planar_device_call(blk, streams, hop, W, outputs=()):
    """process_planar_device on the antenna streams (host memory) asking for the angles and `outputs` (levels,
    spectrum, bins); returns (numpy outputs, kernel launches)"""
    shapes = _output_shapes(blk, W)
    o = {k: torch.full(shapes[k][0], SENTINEL, dtype=shapes[k][1], device=DEV) for k in ("angles",) + tuple(outputs)}
    p = lambda k: o[k].data_ptr() if k in o else None
    d_streams = [torch.from_numpy(s.view(np.float32)).to(DEV) for s in streams]
    l0 = blk.launch_count()
    blk.process_planar_device([s.data_ptr() for s in d_streams], hop, W, p("angles"), p("levels"), p("spectrum"), p("bins"),
                              stream=stream())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}, blk.launch_count() - l0


def entry_outputs(make, x, spectrum=False, planar_outputs=(), device_outputs=("levels", "bins"), multi_device=True):
    """The windows x through every entry point of blocks from `make(devices=None)`, each entry as a dict of numpy
    outputs: "host" (host_call, with the spectrum port when `spectrum`), "planar_host" (work_planar, hop = N: angles,
    levels, bins), "planar_device" (angles and `planar_outputs`, with "planar_launches"), and for multi-device blocks
    on device 0 and on every device "multi_host[devices]" and (with `multi_device`) "multi_device[devices]"
    (device_call with `device_outputs`); "sharded" (sharded_call, one dict per device) when two or more devices
    exist."""
    W, blk = x.shape[0], make()
    out = {"host": host_call(blk, x, spectrum)}
    streams = helpers.antenna_streams(x, blk.m)
    pa, pl = np.zeros((W, blk.n), np.float32), np.zeros((W, blk.n), np.float32)
    blk.work_planar(W, streams, [pa, pl])
    out["planar_host"] = {"angles": pa, "levels": pl, "bins": blk.last_bins().copy()}
    out["planar_device"], out["planar_launches"] = planar_device_call(blk, streams, blk.nsamples // blk.m, W, planar_outputs)
    blk.close()
    G = torch.cuda.device_count()
    for devices in ([0], list(range(G))):
        mb = make(devices=devices)
        out["multi_host%s" % devices] = host_call(mb, x)
        if multi_device:
            out["multi_device%s" % devices] = device_call(mb, x, device_outputs)[0]
        mb.close()
    if G > 1:
        mb = make(devices=list(range(G)))
        out["sharded"] = sharded_call(mb, x)
        mb.close()
    return out


_lib_built = False


def run_cpp_block(driver, header, payload, layout, args=()):
    """Run the C++ block driver lib/_build/<driver> on an input file of `header` (bytes) followed by each array or
    bytes of `payload`; the driver's output file is read back as `layout`, a sequence of (name, dtype, count), and
    must hold exactly that.  Items of `args` that are bytes are written to a file whose path is passed instead.
    Builds the CUDA extension and lib/ on the first call.  Returns {name: 1-D array}."""
    global _lib_built
    if not _lib_built:
        build.build_cuda()
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "lib"), "-s"])
        _lib_built = True
    with tempfile.TemporaryDirectory() as tdir:
        fin, fout = os.path.join(tdir, "in.bin"), os.path.join(tdir, "out.bin")
        with open(fin, "wb") as f:
            f.write(header)
            for a in payload:
                f.write(a if isinstance(a, bytes) else np.ascontiguousarray(a).tobytes())
        argv = []
        for i, a in enumerate(args):
            if isinstance(a, bytes):
                path = os.path.join(tdir, "arg%d.bin" % i)
                with open(path, "wb") as f:
                    f.write(a)
                a = path
            argv.append(str(a))
        r = subprocess.run([os.path.join(ROOT, "lib", "_build", driver), fin, fout] + argv, capture_output=True, text=True)
        assert r.returncode == 0, (driver, r.returncode, r.stderr)
        raw = open(fout, "rb").read()
    out, o = {}, 0
    for name, dtype, count in layout:
        size = np.dtype(dtype).itemsize * count
        out[name] = np.frombuffer(raw[o:o + size], dtype)
        o += size
    assert o == len(raw), (driver, o, len(raw))
    return out
