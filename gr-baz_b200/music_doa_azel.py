"""(azimuth, elevation) MUSIC over a 3-D array geometry: the Python block of ``music_b200_create_azel``
(include/music_b200.h has the definition).

    blk = music_doa_azel(m, n, nsamples, n_az, n_el, (el_lo, el_hi), antenna_array_xyz, wavelength)
    produced = blk.work(noutput_items, [in_items], [azimuth, elevation(, levels(, spectrum))])

The grid has n_az azimuth steps k * 360 / n_az and n_el elevation steps from el_lo to el_hi degrees (elevation measured
from the xy-plane); the spectrum port carries n_el * n_az floats per window, elevation-major.  The setters, reducers,
``last_bins`` / ``last_counts`` and ``close`` are those of :class:`music_doa`; ``last_bins`` holds flat bins
b = i * n_az + k.  For a planar array use el_lo >= 0: +el and -el have identical steering vectors there.
``set_peak_mode("esprit")`` selects 2-D ESPRIT on a planar lattice array (a uniform rectangular array, or any other
Mx x My lattice in row-major element order): gridless (azimuth, elevation) pairs with no grid scan (the spectrum port
still gets the grid spectrum when it is connected).
"""
from __future__ import annotations

import ctypes
import sys

import numpy as np

from . import _capi
from .music_doa import _uid, _uid_lock, music_doa


class music_doa_azel(music_doa):
    def __init__(self, m, n, nsamples, n_az, n_el, el_range, antenna_array_xyz, wavelength, device=0):
        self._lib = _capi.load()
        self._h = ctypes.c_void_p()
        self.m, self.n, self.nsamples = int(m), int(n), int(nsamples)
        self.n_az, self.n_el = int(n_az), int(n_el)
        self.el_range = (float(el_range[0]), float(el_range[1]))
        if self.m <= 0 or self.n_az <= 0 or self.n_el <= 0:
            raise ValueError("m, n_az and n_el must be > 0")
        self.resolution = self.n_az * self.n_el
        pos = self._positions(antenna_array_xyz)
        rc = self._lib.music_b200_create_azel(ctypes.byref(self._h), self.m, self.n, self.nsamples, self.n_az, self.n_el,
                                              self.el_range[0], self.el_range[1], pos.ctypes.data, float(wavelength), int(device))
        if rc == _capi.EINVAL:
            raise ValueError(self._lib.music_b200_last_error(None).decode())
        _capi.check(rc)
        with _uid_lock:
            _uid[0] += 1
            self._unique_id = _uid[0]
        sys.stderr.write("[%s<%i>] MUSIC DOA az-el: M: %d, N: %d, # samples: %d, azimuth steps: %d, elevation steps: %d (%g .. %g deg)\n"
                         % (self.name(), self._unique_id, self.m, self.n, self.nsamples, self.n_az, self.n_el, *self.el_range))

    def _positions(self, antenna_array_xyz):
        pos = np.ascontiguousarray(np.asarray(antenna_array_xyz, dtype=np.float64))
        if pos.shape != (self.m, 3):
            raise ValueError("antenna_array_xyz must hold m = %d [x, y, z] positions" % self.m)
        return pos

    def name(self):
        return "music_doa_azel"

    def _azel(self):
        return True

    def output_signature(self):
        """(min, max, [item sizes]): azimuth, elevation, level (n floats each), spectrum (n_el * n_az floats)"""
        return (2, 4, [self.n * 4, self.n * 4, self.n * 4, self.resolution * 4])

    def set_array_geometry(self, antenna_array_xyz, l):
        """Retune: element positions [[x, y, z], ...] in metres and the wavelength ``l``; the table is built on the
        device.  Refinement (``set_refine``) needs a table installed this way."""
        pos = self._positions(antenna_array_xyz)
        _capi.check(self._lib.music_b200_set_geometry_azel(self._h, pos.ctypes.data, float(l)), self._h)

    def set_array_response(self, array_response):
        """A measured or calibrated manifold, complex [n_el][n_az][m] (rounded to complex64)."""
        t = np.asarray(array_response, dtype=np.complex128)
        if t.shape != (self.n_el, self.n_az, self.m):
            raise ValueError("array_response must be [n_el=%d][n_az=%d][m=%d], got %s" % (self.n_el, self.n_az, self.m, t.shape))
        super().set_array_response(t.reshape(self.resolution, self.m))

    def array_response_c64(self):
        """The table in use, complex64 (n_el, n_az, m)."""
        return super().array_response_c64().reshape(self.n_el, self.n_az, self.m)

    def work(self, noutput_items, input_items, output_items):
        """input_items[0]: complex64 (noutput_items, nsamples); output_items: 2..4 float32 arrays (azimuth (., n),
        elevation (., n), levels (., n), spectrum (., n_el * n_az)).  Returns items produced."""
        W = int(noutput_items)
        if W <= 0:
            return 0
        x = input_items[0]
        if x.dtype != np.complex64 or not x.flags["C_CONTIGUOUS"] or x.size < W * self.nsamples:
            raise ValueError("input_items[0] must be C-contiguous complex64 with >= noutput_items*nsamples elements")
        outs = list(output_items)
        if not 2 <= len(outs) <= 4:
            raise ValueError("2 to 4 output ports")
        for o, s in zip(outs, [self.n, self.n, self.n, self.resolution]):
            if o.dtype != np.float32 or not o.flags["C_CONTIGUOUS"] or o.size < W * s:
                raise ValueError("output buffers must be C-contiguous float32 of the port's item size")
        ptr = lambda i: outs[i].ctypes.data if len(outs) > i else None
        self._last_bins = np.empty((W, self.n), np.int32)
        self._last_counts = np.empty(W, np.int32)
        self._last_crb = None
        trk = self._track_buffers(W)
        if self.crb():
            self._last_crb = np.empty((W, self.n, 3), np.float32)
        if trk is not None:
            rc = self._lib.music_b200_process_azel_host_tracks(self._h, x.ctypes.data, W, ptr(0), ptr(1), ptr(2), ptr(3),
                                                               self._last_bins.ctypes.data, self._last_counts.ctypes.data,
                                                               self._last_crb.ctypes.data if self.crb() else None, *trk)
        elif self.crb():
            rc = self._lib.music_b200_process_azel_host_crb(self._h, x.ctypes.data, W, ptr(0), ptr(1), ptr(2), ptr(3),
                                                            self._last_bins.ctypes.data, self._last_counts.ctypes.data,
                                                            self._last_crb.ctypes.data)
        else:
            rc = self._lib.music_b200_process_azel_host(self._h, x.ctypes.data, W, ptr(0), ptr(1), ptr(2), ptr(3),
                                                        self._last_bins.ctypes.data, self._last_counts.ctypes.data)
        _capi.check(rc, self._h)
        return W

    def process_device(self, d_in, nwindows, d_azimuth, d_elevation, d_levels=None, d_spectrum=None, d_bins=None,
                       d_counts=None, stream=None):
        """Raw device-pointer entry (ints); buffers stay resident in HBM."""
        rc = self._lib.music_b200_process_azel_device(self._h, d_in, int(nwindows), d_azimuth, d_elevation, d_levels,
                                                      d_spectrum, d_bins, d_counts, stream)
        _capi.check(rc, self._h)

    def process_device_crb(self, d_in, nwindows, d_azimuth, d_elevation, d_crb, d_levels=None, d_spectrum=None, d_bins=None,
                           d_counts=None, stream=None):
        """Raw device-pointer entry (ints): the outputs of ``process_device`` plus ``d_crb`` (float32
        [nwindows][n][3], required)."""
        rc = self._lib.music_b200_process_azel_device_crb(self._h, d_in, int(nwindows), d_azimuth, d_elevation, d_levels,
                                                          d_spectrum, d_bins, d_counts, d_crb, stream)
        _capi.check(rc, self._h)

    def process_device_tracks(self, d_in, nwindows, d_azimuth, d_elevation, d_slot_track, d_levels=None, d_spectrum=None,
                              d_bins=None, d_counts=None, d_crb=None, d_track_ids=None, d_track_state=None, stream=None):
        """Raw device-pointer entry (ints): the outputs of ``process_device_crb`` (``d_crb`` may be None) plus
        ``d_slot_track`` (int32 [nwindows][n], required), ``d_track_ids`` (int32 [nwindows][T]) and ``d_track_state``
        (float32 [nwindows][T][6]), the last two both or neither."""
        rc = self._lib.music_b200_process_azel_device_tracks(self._h, d_in, int(nwindows), d_azimuth, d_elevation, d_levels,
                                                             d_spectrum, d_bins, d_counts, d_crb, d_slot_track, d_track_ids,
                                                             d_track_state, stream)
        _capi.check(rc, self._h)
