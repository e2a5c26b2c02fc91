"""Sparse linear arrays through the difference co-array: the Python block of ``music_b200_create_coarray``
(include/music_b200.h has the definition).

    blk = music_doa_coarray(m, n, nsamples, resolution, positions, step_xy, wavelength, mv=0)
    produced = blk.work(noutput_items, [in_items], [angles(, levels(, spectrum))])

The m physical elements sit at the integer ``positions`` (p_0 = 0 < p_1 < ...) times the step ``step_xy`` (metres, at
most half the wavelength long); each input item holds nsamples / m snapshots of the m channels, as on a ``music_doa``
block.  Every window's covariance is mapped to the smoothed covariance of the virtual uniform linear array of
``virtual_size`` elements at l * step_xy that the lags of the array fill, and MUSIC, root-MUSIC or ESPRIT run on it:
up to ``virtual_size - 1`` mutually uncorrelated sources, n may exceed m.  ``set_calibration`` takes the m physical
gains; estimate them on a plain ``music_doa`` block of the same receivers (``calibrate``), which this block does not do.
Refused settings raise as on the other blocks.
"""
from __future__ import annotations

import ctypes
import sys

import numpy as np

from . import _capi
from .music_doa import _uid, _uid_lock, music_doa


class music_doa_coarray(music_doa):
    def __init__(self, m, n, nsamples, resolution, positions, step_xy, wavelength, mv=0, device=0):
        self._lib = _capi.load()
        self._h = ctypes.c_void_p()
        self.m, self.n, self.nsamples, self.resolution = int(m), int(n), int(nsamples), int(resolution)
        p = np.ascontiguousarray(np.asarray(positions, dtype=np.int64))
        if p.shape != (self.m,) or np.any(np.abs(p) > 2 ** 31 - 1):
            raise ValueError("positions must hold m = %d int32 element positions" % self.m)
        self.positions = p.astype(np.int32)
        step = self._step(step_xy)
        rc = self._lib.music_b200_create_coarray(ctypes.byref(self._h), self.m, self.n, self.nsamples, self.resolution,
                                                 self.positions.ctypes.data, step.ctypes.data, float(wavelength), int(mv),
                                                 int(device))
        if rc == _capi.EINVAL:
            raise ValueError(self._lib.music_b200_last_error(None).decode())
        _capi.check(rc)
        with _uid_lock:
            _uid[0] += 1
            self._unique_id = _uid[0]
        sys.stderr.write("[%s<%i>] MUSIC DOA co-array: M: %d, virtual M: %d, N: %d, # samples: %d, angular resolution: %d\n"
                         % (self.name(), self._unique_id, self.m, self.virtual_size, self.n, self.nsamples, self.resolution))

    @staticmethod
    def _step(step_xy):
        s = np.ascontiguousarray(np.asarray(step_xy, dtype=np.float64))
        if s.shape != (2,):
            raise ValueError("step_xy must be [s_x, s_y] in metres")
        return s

    def name(self):
        return "music_doa_coarray"

    @property
    def virtual_size(self):
        """Mv, the elements of the virtual uniform linear array (what mv = 0 resolved to)"""
        mv = ctypes.c_uint32(0)
        _capi.check(self._lib.music_b200_coarray_size(self._h, ctypes.byref(mv)), self._h)
        return int(mv.value)

    def set_array_geometry(self, step_xy, l):
        """Retune (after an LO change): the step [s_x, s_y] in metres and the wavelength ``l``; the virtual table is
        rebuilt on the device.  Resets the integration and the tracks."""
        _capi.check(self._lib.music_b200_set_geometry_coarray(self._h, self._step(step_xy).ctypes.data, float(l)), self._h)

    def array_response_c64(self):
        """The virtual table in use, complex64 (resolution, virtual_size)."""
        out = np.empty((self.resolution, self.virtual_size), np.complex64)
        _capi.check(self._lib.music_b200_get_table(self._h, out.ctypes.data), self._h)
        return out
