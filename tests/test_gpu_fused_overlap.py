"""GPU: back-to-back calls of the fused M = 4 kernel, which run side by side on every SM (programmatic dependent launch,
two half-SM CTAs per SM) and stage their results until the previous call on the stream has written its own.  Every call's
outputs must be what the same call computes alone after a synchronise, and land in stream order."""
import numpy as np
import pytest
import torch

from gr_baz_b200 import synth
from gr_baz_b200.music_doa import music_doa

import helpers

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def block(cfg):
    return music_doa(cfg["m"], cfg["n"], cfg["nsamples"], helpers.table_for(cfg), cfg["resolution"])


def outputs(W):
    return (torch.full((W, 1), float("nan"), device=DEV), torch.full((W, 1), float("nan"), device=DEV),
            torch.full((W, 1), -7, dtype=torch.int32, device=DEV))


def call(blk, x, W, out, spec=None):
    a, l, b = out
    blk.process_device(x.data_ptr(), W, a.data_ptr(), l.data_ptr(), None if spec is None else spec.data_ptr(), b.data_ptr(),
                       stream=torch.cuda.current_stream().cuda_stream)


def alone(blk, x, W, spec=None):
    torch.cuda.synchronize()
    out = outputs(W)
    call(blk, x, W, out, spec)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out]


def same(out, ref):
    got = [t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in out]
    for g, r in zip(got, ref):
        assert g.tobytes() == r.tobytes()


def windows(cfg, seed, W):
    return synth.gen_windows_torch(cfg, synth.BASE_SEED + seed, 0, W, DEV)


def test_eight_back_to_back_calls_match_each_call_alone():
    cfg = synth.config(2)
    W = 3000
    blk = block(cfg)
    xs = [windows(cfg, 100 + i, W) for i in range(8)]
    refs = [alone(blk, x, W) for x in xs]
    # distinct output buffers: each call's outputs are byte-equal to the call run alone
    outs = [outputs(W) for _ in xs]
    torch.cuda.synchronize()
    l0 = blk.launch_count()
    for x, o in zip(xs, outs):
        call(blk, x, W, o)
    assert blk.launch_count() - l0 == len(xs)  # one launch per call
    torch.cuda.synchronize()
    for o, r in zip(outs, refs):
        same(o, r)
    # one shared output buffer: it ends holding the last call's result
    shared = outputs(W)
    for x in xs:
        call(blk, x, W, shared)
    torch.cuda.synchronize()
    same(shared, refs[-1])


@pytest.mark.parametrize("W", [1, 7, 131, 10000, 40000])
def test_window_counts_back_to_back(W):
    cfg = synth.config(2, snapshots=256)  # short windows keep 40 000 of them small; still the fused kernel
    blk = block(cfg)
    xa, xb = windows(cfg, 7, W), windows(cfg, 8, W)
    ra, rb = alone(blk, xa, W), alone(blk, xb, W)
    assert (ra[2] >= 0).all() and np.isfinite(ra[0]).all()
    out = outputs(W)
    torch.cuda.synchronize()
    for x in (xb, xa, xb, xa):  # the last call's results must win in every window
        call(blk, x, W, out)
    torch.cuda.synchronize()
    same(out, ra)
    out_b = outputs(W)
    call(blk, xa, W, out)
    call(blk, xb, W, out_b)
    torch.cuda.synchronize()
    same(out, ra)
    same(out_b, rb)


def test_two_handles_with_different_tables_interleaved():
    c1 = synth.config(2)
    c2 = synth.config(2, geometry="uca", resolution=720)
    W = 2000
    b1, b2 = block(c1), block(c2)
    x1, x2 = windows(c1, 21, W), windows(c2, 22, W)
    r1, r2 = alone(b1, x1, W), alone(b2, x2, W)
    o1, o2 = outputs(W), outputs(W)
    torch.cuda.synchronize()
    for _ in range(3):
        call(b1, x1, W, o1)
        call(b2, x2, W, o2)
    torch.cuda.synchronize()
    same(o1, r1)
    same(o2, r2)


def test_torch_op_reads_outputs_right_after_the_call():
    cfg = synth.config(2)
    W = 5000
    blk = block(cfg)
    xs = [windows(cfg, 31 + i, W) for i in range(3)]
    refs = [alone(blk, x, W) for x in xs]
    out = outputs(W)
    torch.cuda.synchronize()
    copies = []
    for x in xs:
        call(blk, x, W, out)
        copies.append([t.clone() for t in out])  # stream-ordered after the call
    torch.cuda.synchronize()
    for c, r in zip(copies, refs):
        same(c, r)


def test_spectrum_port_and_planar_path_back_to_back():
    cfg = synth.config(2, snapshots=1024, resolution=720)
    W, N = 600, 1024
    blk = block(cfg)
    x = windows(cfg, 41, W)
    spec = torch.zeros((W, cfg["resolution"]), device=DEV)
    ref_spec_out = alone(blk, x, W, spec)
    ref_spec = spec.cpu().numpy()
    ref_peak = alone(blk, x, W)
    # planar: the same windows as four antenna streams, hop = N
    streams = [x.view(W, N, 4, 2)[:, :, r, :].contiguous().view(-1) for r in range(4)]
    ptrs = [s.data_ptr() for s in streams]

    def planar(out):
        a, l, b = out
        blk.process_planar_device(ptrs, N, W, a.data_ptr(), l.data_ptr(), None, b.data_ptr(),
                                  stream=torch.cuda.current_stream().cuda_stream)

    torch.cuda.synchronize()
    ref_planar = outputs(W)
    planar(ref_planar)
    torch.cuda.synchronize()
    same(ref_planar, ref_peak)
    spec2 = torch.zeros_like(spec)
    o1, o2, o3, o4 = outputs(W), outputs(W), outputs(W), outputs(W)
    l0 = blk.launch_count()
    call(blk, x, W, o1)
    call(blk, x, W, o2, spec2)
    planar(o3)
    call(blk, x, W, o4)
    assert blk.launch_count() - l0 == 4
    torch.cuda.synchronize()
    same(o1, ref_peak)
    same(o2, ref_spec_out)
    assert spec2.cpu().numpy().tobytes() == ref_spec.tobytes()
    same(o3, ref_peak)
    same(o4, ref_peak)
