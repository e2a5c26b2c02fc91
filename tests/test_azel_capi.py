"""CPU: the az-el C ABI checks its arguments before it looks for a device, and fails loudly without one; the C++ block
builds into the same library as the 1-D block."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from gr_baz_b200 import _capi, build
from gr_baz_b200.music_doa_azel import music_doa_azel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build.build_cuda()
    return _capi.load()


def _pos(m):
    return np.ascontiguousarray([[0.5 * e, 0.0, 0.1 * e] for e in range(m)], dtype=np.float64)


GOOD = dict(m=4, n=1, nsamples=512, n_az=36, n_el=10, el_lo=0.0, el_hi=90.0, lam=1.0)
BAD = [
    dict(m=0), dict(m=17, nsamples=17 * 4), dict(n=0), dict(n=4), dict(nsamples=0), dict(nsamples=510),
    dict(n_az=0), dict(n_el=0), dict(n_az=1024, n_el=1025), dict(el_lo=-91.0), dict(el_hi=90.5), dict(el_lo=30.0, el_hi=20.0),
    dict(el_lo=10.0, el_hi=10.0), dict(el_lo=float("nan")), dict(lam=0.0), dict(lam=-1.0), dict(lam=float("inf")),
    dict(lam=float("nan")), dict(pos="nan"), dict(pos="null"),
]


def _create(lib, **over):
    a = dict(GOOD, **over)
    pos = _pos(max(a["m"], 1))
    if a.get("pos") == "nan":
        pos[1, 2] = np.nan
    h = ctypes.c_void_p()
    p = None if a.get("pos") == "null" else pos.ctypes.data
    rc = lib.music_b200_create_azel(ctypes.byref(h), a["m"], a["n"], a["nsamples"], a["n_az"], a["n_el"], a["el_lo"], a["el_hi"],
                                    p, a["lam"], 0)
    return rc, h


@pytest.mark.parametrize("over", BAD, ids=lambda d: ",".join("%s=%s" % kv for kv in d.items()))
def test_create_azel_rejects_bad_arguments(lib, over):
    rc, h = _create(lib, **over)
    assert rc == _capi.EINVAL and not h
    assert lib.music_b200_last_error(None)


def test_single_elevation_step_allows_an_equal_range(lib):
    # n_el = 1 only needs el_lo <= el_hi; the argument checks pass and only the device check remains
    rc, h = _create(lib, n_el=1, el_lo=10.0, el_hi=10.0)
    assert rc in (_capi.OK, _capi.ENODEVICE)
    if h:
        lib.music_b200_destroy(h)
    rc, h = _create(lib, n_az=1024, n_el=1024)  # exactly 2^20 bins
    assert rc in (_capi.OK, _capi.ENODEVICE)
    if h:
        lib.music_b200_destroy(h)


def test_null_handle_and_python_argument_checks(lib):
    assert lib.music_b200_set_geometry_azel(None, _pos(4).ctypes.data, 1.0) == _capi.EINVAL
    assert lib.music_b200_process_azel_host(None, None, 1, None, None, None, None, None, None) == _capi.EINVAL
    assert lib.music_b200_process_azel_device(None, None, 1, None, None, None, None, None, None, None) == _capi.EINVAL
    with pytest.raises(ValueError):
        music_doa_azel(4, 1, 512, 36, 10, (0.0, 90.0), [[0.0, 0.0]] * 4, 1.0)  # [x, y] only
    with pytest.raises(ValueError):
        music_doa_azel(4, 4, 512, 36, 10, (0.0, 90.0), _pos(4), 1.0)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_device_is_enodevice(lib):
    rc, h = _create(lib)
    assert rc == _capi.ENODEVICE and not h
    with pytest.raises(_capi.MusicB200Error) as e:
        music_doa_azel(4, 1, 512, 36, 10, (0.0, 90.0), _pos(4), 1.0)
    assert e.value.code == _capi.ENODEVICE


def test_cpp_blocks_build_into_one_library():
    build.build_cuda()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "lib"), "-s"])
    so = os.path.join(ROOT, "lib", "_build", "libgnuradio-baz-music.so")
    syms = subprocess.run(["nm", "-D", "-C", so], capture_output=True, text=True, check=True).stdout
    assert "baz_make_music_doa_azel" in syms and "baz_make_music_doa(" in syms
    assert os.access(os.path.join(ROOT, "lib", "_build", "test_block_azel"), os.X_OK)
    assert os.access(os.path.join(ROOT, "lib", "_build", "test_block"), os.X_OK)
