"""Frequency-channelised direction finding: the Python block of ``music_b200_create_channels`` (include/music_b200.h has
the definition).

    blk = music_doa_channels(m, n, nsamples, resolution, nfft, (first, count), taper, combine,
                             antenna_array, spacing, centre_frequency, sample_rate)
    produced = blk.work(noutput_items, [in_items], [angles, levels(, spectrum)])

Each window is cut into nsamples / m / nfft segments, an nfft-point FFT filter bank runs over them and every channel
(FFT bin (first + c) mod nfft, c < count) gets its own covariance and its own steering table, built for that channel's
wavelength.  ``combine="separate"``: one direction-finding problem per channel; an output item holds the channels of one
window, ``count * n`` angles, ``count * n`` levels and optionally ``count * resolution`` spectrum floats, channel by
channel.  ``combine="incoherent"``: one incoherent wideband MUSIC spectrum per window; items as for :class:`music_doa`.
``combine="coherent"``: every channel's covariance is focused onto the centre channel's frequency and summed, and each
window is one ordinary problem on that sum and the centre channel's table; items as for :class:`music_doa`, and the
root-MUSIC, ESPRIT, DML, WSF and NEWTON refinement setters work (JOINT refinement raises).  ``set_focusing`` chooses the sector of grid bins the focusing
matrices fit, ``focusing`` returns them and their errors.
``antenna_array`` holds m [x, y] positions in units of ``spacing`` metres.  Peak mode, estimator and source rule setters,
the reducers, ``last_bins`` / ``last_counts`` and ``close`` are those of :class:`music_doa`; the modes that are not
built for channels (beams, calibration, planar input, and under "separate" / "incoherent" root-MUSIC, ESPRIT, DML, WSF
and refinement) raise.
"""
from __future__ import annotations

import ctypes
import sys

import numpy as np

from . import _capi
from .music_doa import _table_c64, _uid, _uid_lock, music_doa

TAPERS = {"rect": 0, "hann": 1}
COMBINES = {"separate": 0, "incoherent": 1, "coherent": 2}


class music_doa_channels(music_doa):
    def __init__(self, m, n, nsamples, resolution, nfft, channels, taper, combine, antenna_array, spacing, centre_frequency,
                 sample_rate, device=0):
        self._lib = _capi.load()
        self._h = ctypes.c_void_p()
        self.m, self.n, self.nsamples, self.resolution = int(m), int(n), int(nsamples), int(resolution)
        self.nfft = int(nfft)
        self.chan_first, self.chan_count = int(channels[0]), int(channels[1])
        if taper not in TAPERS or combine not in COMBINES:
            raise ValueError("taper must be one of %s and combine one of %s" % (sorted(TAPERS), sorted(COMBINES)))
        if self.m <= 0 or self.resolution <= 0 or self.chan_first < 0 or self.chan_count <= 0 or self.nfft <= 0:
            raise ValueError("m, resolution, nfft and the channel count must be > 0, the first channel >= 0")
        self.taper, self.combine = taper, combine
        rc = self._lib.music_b200_create_channels(ctypes.byref(self._h), self.m, self.n, self.nsamples, self.resolution, self.nfft,
                                                  self.chan_first, self.chan_count, TAPERS[taper], COMBINES[combine], int(device))
        if rc == _capi.EINVAL:
            raise ValueError(self._lib.music_b200_last_error(None).decode())
        _capi.check(rc)
        with _uid_lock:
            _uid[0] += 1
            self._unique_id = _uid[0]
        sys.stderr.write("[%s<%i>] MUSIC DOA channels: M: %d, N: %d, # samples: %d, angular resolution: %d, FFT: %d, channels: %d from bin %d, %s, %s\n"
                         % (self.name(), self._unique_id, self.m, self.n, self.nsamples, self.resolution, self.nfft,
                            self.chan_count, self.chan_first, taper, combine))
        self.set_array_geometry(np.asarray(antenna_array, dtype=np.float64) * float(spacing), centre_frequency, sample_rate)

    def name(self):
        return "music_doa_channels"

    @property
    def rows(self):
        """channel blocks per output item: the channel count under "separate", 1 under "incoherent" and "coherent" """
        return self.chan_count if self.combine == "separate" else 1

    def output_signature(self):
        r = self.rows
        return (1, 3, [r * self.n * 4, r * self.n * 4, r * self.resolution * 4])

    def set_array_geometry(self, antenna_array, centre_frequency, sample_rate):
        """Retune: element positions [[x, y], ...] in metres, the centre frequency and the sample rate in Hz; one table
        per channel is built on the device, for the wavelength c0 / (centre_frequency + channel offset)."""
        pos = np.ascontiguousarray(np.asarray(antenna_array, dtype=np.float64))
        if pos.shape != (self.m, 2):
            raise ValueError("antenna_array must hold m = %d [x, y] positions" % self.m)
        _capi.check(self._lib.music_b200_set_geometry_channels(self._h, pos.ctypes.data, float(centre_frequency), float(sample_rate)),
                    self._h)

    def set_array_response(self, array_response):
        """One measured table [resolution][m] for every channel (the narrowband assumption)."""
        table = _table_c64(array_response, self.resolution, self.m)
        _capi.check(self._lib.music_b200_set_table(self._h, table.ctypes.data), self._h)

    def set_focusing(self, first_bin, bin_count):
        """coherent: fit the focusing matrices on grid bins (first_bin + i) mod resolution, i < bin_count"""
        _capi.check(self._lib.music_b200_set_focusing(self._h, int(first_bin), int(bin_count)), self._h)

    def focusing(self):
        """coherent: (T complex128 (count, m, m), err float64 (count,)), the focusing matrices and their errors"""
        T = np.empty((self.chan_count, self.m, self.m), np.complex128)
        err = np.empty(self.chan_count, np.float64)
        _capi.check(self._lib.music_b200_get_focusing(self._h, T.ctypes.data, err.ctypes.data), self._h)
        return T, err

    def channel_frequencies(self):
        """float64 (count,): each channel's frequency offset from the centre frequency in Hz"""
        f = np.empty(self.chan_count, np.float64)
        _capi.check(self._lib.music_b200_channel_frequencies(self._h, f.ctypes.data), self._h)
        return f

    def array_response_c64(self, channel=None):
        """The tables in use, complex64 (count, resolution, m), or channel ``channel``'s (resolution, m)."""
        chans = range(self.chan_count) if channel is None else [int(channel)]
        out = np.empty((len(chans), self.resolution, self.m), np.complex64)
        for i, c in enumerate(chans):
            _capi.check(self._lib.music_b200_get_table_channel(self._h, c, out[i].ctypes.data), self._h)
        return out if channel is None else out[0]

    def set_crb(self, enable):
        """The CRB of every slot is not built for channel handles (include/music_b200.h): enabling it raises, as the C
        entry points refuse a channel handle."""
        if enable:
            raise ValueError("the CRB is not built for channel handles")

    def set_tracking(self, variance="off", **kwargs):
        """Per-channel tracking is not built (include/music_b200.h): music_b200_set_tracking refuses a channel handle,
        so this raises whatever the variance."""
        rc = self._lib.music_b200_set_tracking(self._h, self.TRACK_VARIANCES.get(variance, -1), 0.01, 1.0, 0.5, 1.0, 9.0, 3, 5, 5, 8)
        _capi.check(rc, self._h)

    def process_host(self, x, nwindows, levels=True, spectrum=False, bins=True, counts=False, R=False):
        """The host entry on complex64 windows x, results in the C ABI's channel-major layout: a dict of angles / levels /
        bins (rows, W, n), counts (rows, W), spectrum (rows, W, resolution), R (count, W, m, m) complex128, under
        "coherent" the focused covariances (W, m, m)."""
        W, r, n, m = int(nwindows), self.rows, self.n, self.m
        if x.dtype != np.complex64 or not x.flags["C_CONTIGUOUS"] or x.size < W * self.nsamples:
            raise ValueError("x must be C-contiguous complex64 with >= nwindows*nsamples elements")
        out = {"angles": np.zeros((r, W, n), np.float32)}
        if levels:
            out["levels"] = np.zeros((r, W, n), np.float32)
        if spectrum:
            out["spectrum"] = np.zeros((r, W, self.resolution), np.float32)
        if bins:
            out["bins"] = np.zeros((r, W, n), np.int32)
        if counts:
            out["counts"] = np.zeros((r, W), np.int32)
        if R:
            out["R"] = np.zeros((W, m, m) if self.combine == "coherent" else (self.chan_count, W, m, m), np.complex128)
        p = lambda k: out[k].ctypes.data if k in out else None
        rc = self._lib.music_b200_process_channels_host(self._h, x.ctypes.data, W, p("angles"), p("levels"), p("spectrum"), p("bins"),
                                                        p("counts"), p("R"))
        _capi.check(rc, self._h)
        return out

    def work(self, noutput_items, input_items, output_items):
        """input_items[0]: complex64 (noutput_items, nsamples); output_items: 1..3 float32 arrays of the item sizes of
        ``output_signature``.  The library's channel-major results are transposed into window-major items here (small
        arrays on the PCIe-bound path).  Returns items produced."""
        W = int(noutput_items)
        if W <= 0:
            return 0
        outs = list(output_items)
        if not 1 <= len(outs) <= 3:
            raise ValueError("1 to 3 output ports")
        r = self.rows
        for o, s in zip(outs, [r * self.n, r * self.n, r * self.resolution]):
            if o.dtype != np.float32 or not o.flags["C_CONTIGUOUS"] or o.size < W * s:
                raise ValueError("output buffers must be C-contiguous float32 of the port's item size")
        res = self.process_host(input_items[0], W, levels=len(outs) > 1, spectrum=len(outs) > 2, counts=self.combine != "incoherent")
        for o, k in zip(outs, ["angles", "levels", "spectrum"]):
            a = res[k]
            o.reshape(-1)[: a.size].reshape(W, r, a.shape[2])[...] = a.transpose(1, 0, 2)
        self._last_bins = np.ascontiguousarray(res["bins"].transpose(1, 0, 2))          # (W, rows, n)
        self._last_counts = np.ascontiguousarray(res["counts"].T) if "counts" in res else None  # (W, rows)
        return W

    def process_device(self, d_in, nwindows, d_angles, d_levels=None, d_spectrum=None, d_bins=None, d_counts=None, d_R=None,
                       stream=None):
        """Raw device-pointer entry (ints); buffers stay resident in HBM, outputs in the channel-major layout."""
        rc = self._lib.music_b200_process_channels_device(self._h, d_in, int(nwindows), d_angles, d_levels, d_spectrum, d_bins,
                                                          d_counts, d_R, stream)
        _capi.check(rc, self._h)
