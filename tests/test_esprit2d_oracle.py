"""CPU: 2-D ESPRIT on az-el handles.  The library's lattice hook (music_b200_azel_lattice_host) against the oracle's
lattice condition on every accepted and refused family; the oracle (tests/esprit2d_oracle.py) against the truth of
noiseless windows; the kernel's emulation (tools/emulate_esprit2d_warp.py) against the oracle; planted defects
failing the checker; and the numpy model that sets the GPU test's accuracy thresholds."""
import ctypes
import math
import os
import sys
import zlib

import numpy as np
import pytest

from gr_baz_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import emulate_esprit2d_warp as e2  # noqa: E402

import azel_oracle as ao  # noqa: E402
import esprit2d_oracle as eo  # noqa: E402

LAM = 0.5
H = 0.5 * LAM
TRUTH_DEG = 1e-3


def hook(pos, lam=LAM):
    L = _capi.load()
    pos = np.ascontiguousarray(pos, np.float64)
    mx, my, s = ctypes.c_int(), ctypes.c_int(), np.zeros(4)
    rc = L.music_b200_azel_lattice_host(pos.ctypes.data, pos.shape[0], lam, ctypes.byref(mx), ctypes.byref(my), s.ctypes.data)
    return (mx.value, my.value, s[:2].copy(), s[2:].copy()) if rc == _capi.OK else None


def rot(t):
    c, s = math.cos(math.radians(t)), math.sin(math.radians(t))
    return lambda v: (c * v[0] - s * v[1], s * v[0] + c * v[1])


def accepted():
    """name -> positions of the lattices the condition accepts"""
    out = {}
    for mx, my in ((2, 2), (2, 3), (3, 2), (2, 4), (4, 2), (3, 3), (3, 4), (4, 3), (4, 4), (2, 8), (8, 2), (3, 5), (5, 3)):
        out["ura%dx%d" % (mx, my)] = eo.lattice_xyz(mx, my, (H, 0.0), (0.0, H))
    r = rot(27.0)
    out["rotated3x3"] = eo.lattice_xyz(3, 3, r((H, 0.0)), r((0.0, H)))
    out["triangular4x4"] = eo.lattice_xyz(4, 4, (H, 0.0), (0.5 * H, math.sqrt(3.0) / 2.0 * H))
    out["skew_rot3x4"] = eo.lattice_xyz(3, 4, r((0.9 * H, 0.0)), r((0.3 * H, 0.8 * H)))
    out["offset2x4"] = eo.lattice_xyz(2, 4, (H, 0.0), (0.0, 0.8 * H), p0=(3.1, -2.2, 0.7))
    out["column_major3x4"] = eo.lattice_xyz(3, 4, (0.0, H), (H, 0.0))
    out["fine4x4"] = eo.lattice_xyz(4, 4, (0.8 * H, 0.0), (0.0, 0.9 * H))
    out["ura_centred3x4"] = ao.ura_xyz(4, 3, LAM)
    return out


def refused():
    out = {}
    out["collinear8"] = eo.lattice_xyz(8, 1, (H, 0.0), (0.0, H))
    out["collinear_2x4"] = np.array([[i * H, 0.0, 0.0] for i in range(8)])
    out["uca8"] = ao.uca_xyz(8, LAM)
    out["uca16"] = ao.uca_xyz(16, LAM)
    tilt = eo.lattice_xyz(3, 3, (H, 0.0), (0.0, H))
    tilt[:, 2] = 0.3 * tilt[:, 1]
    out["tilted3x3"] = tilt
    out["vertical2x4"] = np.array([[i * H, 0.0, k * H] for k in range(4) for i in range(2)])
    out["stacked2x2x2"] = np.array([[i * H, k * H, z * H] for z in range(2) for k in range(2) for i in range(2)])
    rng = np.random.default_rng(3)
    out["shuffled3x3"] = eo.lattice_xyz(3, 3, (H, 0.0), (0.0, H))[rng.permutation(9)]
    moved = eo.lattice_xyz(4, 4, (H, 0.0), (0.0, H))
    moved[9, 0] += 1e-4 * H
    out["moved4x4"] = moved
    out["wide3x3"] = eo.lattice_xyz(3, 3, (0.6 * LAM, 0.0), (0.0, H))
    out["prime7"] = np.array([[i * H, 0.0, 0.0] for i in range(7)])
    out["coincident4"] = np.zeros((4, 3))
    return out


@pytest.mark.parametrize("name", sorted(accepted()))
def test_lattice_hook_accepts(name):
    pos = accepted()[name]
    got, want = hook(pos), eo.lattice(pos, LAM)
    assert want is not None and got is not None, name
    assert got[:2] == want[:2] and np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3]), (got, want)


@pytest.mark.parametrize("name", sorted(refused()))
def test_lattice_hook_refuses(name):
    pos = refused()[name]
    assert eo.lattice(pos, LAM) is None and hook(pos) is None, name


def test_lattice_hook_arguments():
    L = _capi.load()
    pos = eo.lattice_xyz(2, 2, (H, 0.0), (0.0, H))
    mx, my, s = ctypes.c_int(), ctypes.c_int(), np.zeros(4)
    assert L.music_b200_azel_lattice_host(pos.ctypes.data, 4, 0.0, ctypes.byref(mx), ctypes.byref(my), s.ctypes.data) == _capi.EINVAL
    assert L.music_b200_azel_lattice_host(None, 4, LAM, ctypes.byref(mx), ctypes.byref(my), s.ctypes.data) == _capi.EINVAL
    bad = pos.copy()
    bad[1, 0] = np.nan
    assert hook(bad) is None
    # the column-major order passes with the steps swapped
    cm = hook(accepted()["column_major3x4"])
    assert cm[0] == 3 and np.allclose(cm[2], (0.0, H)) and np.allclose(cm[3], (H, 0.0))


def random_dirs(rng, d, el_range=(0.0, 85.0)):
    return [(rng.uniform(0.0, 360.0), rng.uniform(*el_range)) for _ in range(d)]


def check_truth(res, dirs, d, tol=TRUTH_DEG):
    got = [(float(a), float(e)) for a, e in zip(res["az"][:d], res["el"][:d])]
    assert np.all(res["bins"][:d] >= 0), res
    used = set()
    for t in dirs:
        errs = [(ao.direction_error(g[0], g[1], *t), j) for j, g in enumerate(got) if j not in used]
        e, j = min(errs)
        assert e <= tol, (t, got)
        used.add(j)


@pytest.mark.parametrize("name", sorted(accepted()))
def test_noiseless_truth(name):
    """every accepted lattice, d = 1 .. d_max: the oracle within 1e-3 degrees of the truth"""
    pos = accepted()[name]
    mx, my, _, _ = eo.lattice(pos, LAM)
    grid = ao.Grid(360, 91, 0.0, 90.0)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    for d in range(1, eo.d_max(mx, my) + 1):
        if d >= pos.shape[0]:
            break
        for _ in range(3):
            dirs = random_dirs(rng, d)
            res = eo.work_V(eo.noiseless_V(pos, LAM, dirs), d, pos, LAM, grid, d)
            check_truth(res, dirs, d)


def pairing_families():
    """name -> (positions, directions): the cases a pairing must get right"""
    ura = eo.lattice_xyz(4, 4, (H, 0.0), (0.0, H))
    rect = eo.lattice_xyz(3, 3, (H, 0.0), (0.0, H))
    tri = accepted()["triangular4x4"]
    fam = {}
    # equal s1 . u: ux equal, so Psi_1 alone has a double eigenvalue
    fam["equal_s1u"] = (ura, [(math.degrees(math.atan2(0.2, 0.5)), math.degrees(math.acos(math.hypot(0.5, 0.2)))),
                              (math.degrees(math.atan2(-0.6, 0.5)), math.degrees(math.acos(math.hypot(0.5, 0.6))))])
    fam["equal_s2u"] = (ura, [(math.degrees(math.atan2(0.4, 0.3)), math.degrees(math.acos(0.5))),
                              (math.degrees(math.atan2(0.4, -0.7)), math.degrees(math.acos(math.hypot(0.7, 0.4))))])
    # mirror images across the lattice diagonal: (ux, uy) and (uy, ux) tie for gamma = 1
    fam["diagonal_mirror"] = (rect, [(math.degrees(math.atan2(0.6, 0.2)), math.degrees(math.acos(math.hypot(0.2, 0.6)))),
                                     (math.degrees(math.atan2(0.2, 0.6)), math.degrees(math.acos(math.hypot(0.2, 0.6))))])
    fam["zenith"] = (ura, [(0.0, 90.0), (120.0, 30.0)])
    fam["horizon"] = (ura, [(40.0, 0.5), (250.0, 2.0)])
    fam["triangular_three"] = (tri, [(10.0, 20.0), (130.0, 45.0), (250.0, 70.0)])
    return fam


@pytest.mark.parametrize("name", sorted(pairing_families()))
def test_pairing_families(name):
    pos, dirs = pairing_families()[name]
    d = len(dirs)
    res = eo.work_V(eo.noiseless_V(pos, LAM, dirs), d, pos, LAM, ao.Grid(360, 91, 0.0, 90.0), d)
    check_truth(res, dirs, d, tol=1e-3 if name != "zenith" else 2e-3)


def _emu_sources(V, d, pos, grid):
    mx, my, s1, s2 = eo.lattice(pos, LAM)
    f1, f2, steps = e2.window(V, d, mx, my)
    if f1 is None:
        return None, steps
    return sorted(eo.direction(a, b, s1, s2, LAM, grid.el_hi) for a, b in zip(f1, f2)), steps


def chord_deg(a, b):
    """|u(a) - u(b)| in degrees: the great-circle angle without acos's loss near 0"""
    u = lambda t: np.array([math.cos(math.radians(t[1])) * math.cos(math.radians(t[0])),
                            math.cos(math.radians(t[1])) * math.sin(math.radians(t[0])), math.sin(math.radians(t[1]))])
    return math.degrees(float(np.linalg.norm(u(a) - u(b))))


def _same(a, b, tol):
    return len(a) == len(b) and all(chord_deg(x, y) <= tol for x, y in zip(a, b))


@pytest.mark.parametrize("name", sorted(pairing_families()) + ["random"])
def test_emulation_matches_oracle(name):
    """the kernel's sequence (Householder with Z, whole-row QR, back-substitution) converges and gives the oracle's
    directions: on the pairing families, on noisy windows, and on random subspaces"""
    grid = ao.Grid(360, 91, 0.0, 90.0)
    rng = np.random.default_rng(17)
    cases = []
    if name == "random":
        for pos in (accepted()["ura4x4"], accepted()["triangular4x4"], accepted()["ura2x4"], accepted()["rotated3x3"]):
            mx, my, _, _ = eo.lattice(pos, LAM)
            for d in range(1, eo.d_max(mx, my) + 1):
                if d >= pos.shape[0]:
                    break
                Q, _ = np.linalg.qr(rng.standard_normal((pos.shape[0],) * 2) + 1j * rng.standard_normal((pos.shape[0],) * 2))
                cases.append((pos, Q, d))
                dirs = random_dirs(rng, d)
                x, _ = ao.windows(pos, LAM, [0], 1, 64)  # shapes only
                A = np.stack([ao.steering(pos, LAM, *t) for t in dirs], 1)
                X = A @ (rng.standard_normal((d, 256)) + 1j * rng.standard_normal((d, 256))) + 0.1 * (
                    rng.standard_normal((pos.shape[0], 256)) + 1j * rng.standard_normal((pos.shape[0], 256)))
                _, V = np.linalg.eigh(X @ X.conj().T / 256)
                cases.append((pos, V, d))
    else:
        pos, dirs = pairing_families()[name]
        cases.append((pos, eo.noiseless_V(pos, LAM, dirs), len(dirs)))
    for pos, V, d in cases:
        got, steps = _emu_sources(V, d, pos, grid)
        ref = eo.work_V(V, d, pos, LAM, grid, d)
        want = sorted((s[1], s[2]) for s in ref["sources"])
        assert got is not None and steps <= 40, (name, d, steps)
        assert _same(got, want, 1e-6), (name, d, got, want)


def _planted_fails(defect):
    """True when the defect makes the checker fail on some pairing family or noiseless lattice window"""
    grid = ao.Grid(360, 91, 0.0, 90.0)
    for name, (pos, dirs) in sorted(pairing_families().items()):
        d = len(dirs)
        V = eo.noiseless_V(pos, LAM, dirs)
        try:
            if defect == "schur_ranges":
                got, _ = _emu_sources(V, d, pos, grid)
                if got is None:
                    return True
                res = {"az": np.array([g[0] for g in got], np.float32), "el": np.array([g[1] for g in got], np.float32),
                       "bins": np.zeros(d, np.int32)}
                mx, my, s1, s2 = eo.lattice(pos, LAM)
                f1, f2, _ = e2.window(V, d, mx, my, schur_ranges=False)
                if f1 is None:
                    return True
                bad = [eo.direction(a, b, s1, s2, LAM, 90.0) for a, b in zip(f1, f2)]
                if any(x is None for x in bad):
                    return True
                res = {"az": np.array([b[0] for b in bad], np.float32), "el": np.array([b[1] for b in bad], np.float32),
                       "bins": np.zeros(d, np.int32)}
            else:
                kw = {"gamma": 0.0} if defect == "gamma0" else {defect: True}
                res = eo.work_V(V, d, pos, LAM, grid, d, **kw)
            check_truth(res, dirs, d)
        except AssertionError:
            return True
    return False


@pytest.mark.parametrize("defect", ["gamma0", "swap", "no_conj", "schur_ranges"])
def test_planted_defects_fail(defect):
    """pairing from Psi_1's eigenvectors alone, a swapped doublet order, a missing conjugate in C_j and the
    eigenvalues-only QR ranges in the Schur form each fail the checker"""
    assert _planted_fails(defect), defect


def test_accuracy_model():
    """The numpy model behind the GPU test's thresholds: 4 x 4 URA, two sources at 20 dB per element, 512 snapshots,
    el in [5, 80] degrees, a 360 x 46 grid over el [0, 90] (2 degree elevation step).  ESPRIT's RMS direction error is
    below TOP_BINS's and within eo.RMS_FACTOR of grid + NEWTON's; tests/test_gpu_esprit2d.py asserts the same two
    bounds on the device."""
    pos = eo.lattice_xyz(4, 4, (H, 0.0), (0.0, H))
    r = eo.rms_model(pos, LAM, ao.Grid(360, 46, 0.0, 90.0), 2, 40, seed=5)
    print(r)
    assert r["esprit"] < r["top_bins"], r
    assert r["esprit"] <= eo.RMS_FACTOR * r["newton"], r
