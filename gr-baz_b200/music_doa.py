"""Python mirror of the reference block ``baz.music_doa`` (SWIG name,
/root/reference/swig/baz_swig.i:562-572; C++ class /root/reference/lib/baz_music_doa.h:38-60).

Same constructor arguments, ``set_array_response`` and ``work`` contract:

    blk = music_doa(m, n, nsamples, array_response, resolution)
    produced = blk.work(noutput_items, [in_items], [angles, levels(, spectrum)])

``array_response`` is the nested list ``[resolution][m]`` of complex the helper builds; it is
rounded to complex64 exactly as SWIG does when filling ``std::vector<std::vector<gr_complex>>``.
``work`` takes numpy arrays in the GNU Radio item layouts (input items of ``nsamples``
complex64; output items of ``n`` / ``n`` / ``resolution`` float32) and, unlike the reference
(which returns 1, lib/baz_music_doa.cc:160), consumes all ``noutput_items`` windows per call -
legal for a gr::sync_block and the only way a GPU gets a batch; per-window results are the
reference's.  All compute happens in the CUDA library behind include/music_b200.h.
"""
from __future__ import annotations

import ctypes
import sys
import threading

import numpy as np

from . import _capi

_uid = [0]
_uid_lock = threading.Lock()


def _table_c64(array_response, resolution, m):
    t = np.asarray(array_response, dtype=np.complex128)
    if t.ndim != 2 or t.shape[0] != resolution or t.shape[1] != m:
        # reference: assert(array_response.size() == resolution); assert(array_response[0].size() == m)
        raise ValueError("array_response must be [resolution=%d][m=%d], got %s" % (resolution, m, t.shape))
    return np.ascontiguousarray(t.astype(np.complex64))


class music_doa(object):
    def __init__(self, m, n, nsamples, array_response, resolution, device=0, devices=None):
        """``devices`` (extension): a list of CUDA device ordinals - the block then owns one engine per GPU and
        ``work()`` deals its windows round-robin to them (``music_b200_create_multi``); the C++ block reads the same
        list from the environment variable BAZ_MUSIC_DOA_DEVICES so that flowgraph parameters do not change."""
        self._lib = _capi.load()
        self._h = ctypes.c_void_p()
        self.m, self.n, self.nsamples, self.resolution = int(m), int(n), int(nsamples), int(resolution)
        if self.m <= 0 or self.resolution <= 0:
            raise ValueError("m and resolution must be > 0")
        table = _table_c64(array_response, self.resolution, self.m)
        if devices is not None:
            devs = (ctypes.c_int * len(devices))(*[int(d) for d in devices])
            rc = self._lib.music_b200_create_multi(ctypes.byref(self._h), self.m, self.n, self.nsamples, self.resolution,
                                                   table.ctypes.data, devs, len(devices))
        else:
            rc = self._lib.music_b200_create(ctypes.byref(self._h), self.m, self.n, self.nsamples, self.resolution,
                                             table.ctypes.data, int(device))
        if rc == _capi.EINVAL:
            raise ValueError(self._lib.music_b200_last_error(None).decode())
        _capi.check(rc)
        with _uid_lock:
            _uid[0] += 1
            self._unique_id = _uid[0]
        # banner, reference lib/baz_music_doa.cc:52
        sys.stderr.write("[%s<%i>] MUSIC DOA: M: %d, N: %d, # samples: %d, angular resolution: %d\n"
                         % (self.name(), self._unique_id, self.m, self.n, self.nsamples, self.resolution))

    # -- gr::basic_block look-alikes used by the banner ---------------------------------
    def name(self):
        return "music_doa"

    def unique_id(self):
        return self._unique_id

    def input_signature(self):
        """(min, max, [item sizes]) - reference lib/baz_music_doa.cc:37"""
        return (1, 1, [self.nsamples * 8])

    def output_signature(self):
        """reference lib/baz_music_doa.cc:38 (make3(1, 3, n*4, n*4, resolution*4))"""
        return (1, 3, [self.n * 4, self.n * 4, self.resolution * 4])

    # -- reference API ------------------------------------------------------------------
    def set_array_response(self, array_response):
        table = _table_c64(array_response, self.resolution, self.m)
        sys.stderr.write("[%s<%i>] Updating array response\n" % (self.name(), self._unique_id))  # :65
        _capi.check(self._lib.music_b200_set_table(self._h, table.ctypes.data), self._h)

    # -- extension (SURVEY.md section 8(f) rank 1): retune on the device ---------------------
    def set_array_geometry(self, antenna_array, l):
        """Device-side equivalent of ``set_array_response(calculate_antenna_array_response(
        antenna_array, resolution, l))`` (/root/reference/python/music_doa_helper.py:32-46,
        :100-103): ``antenna_array`` = element positions [[x, y], ...] in metres (already scaled by
        the spacing, :56), ``l`` = wavelength.  Returns the number of entries the library
        re-evaluated with the host libm to keep the table bit-identical to the Python helper's."""
        pos = np.ascontiguousarray(np.asarray(antenna_array, dtype=np.float64))
        if pos.shape != (self.m, 2):
            raise ValueError("antenna_array must hold m = %d [x, y] positions" % self.m)
        guarded = ctypes.c_uint32(0)
        _capi.check(self._lib.music_b200_set_geometry(self._h, pos.ctypes.data, float(l), ctypes.byref(guarded)), self._h)
        return int(guarded.value)

    # -- extension (SURVEY.md section 8(f) rank 3): opt-in local-maximum peak rule --------------
    def set_peak_mode(self, mode="top_bins", exclusion_bins=0):
        """``"top_bins"`` (default) = the reference's rule (/root/reference/lib/baz_music_doa.cc:129-141);
        ``"local_maxima"`` = the n largest circular local maxima more than ``exclusion_bins`` apart;
        ``"roots"`` = root-MUSIC: gridless angles from the roots of the noise-subspace polynomial, for a uniform linear
        array with spacing <= lambda / 2 installed with ``set_array_geometry`` (include/music_b200.h).  It needs
        ``exclusion_bins`` = 0, the "music" estimator and refinement off."""
        modes = {"top_bins": 0, "local_maxima": 1, "roots": 2}
        if mode not in modes:
            raise ValueError("mode must be one of %s" % sorted(modes))
        _capi.check(self._lib.music_b200_set_peak_mode(self._h, modes[mode], int(exclusion_bins)), self._h)

    # -- extension: per-window estimate of the number of sources ---------------------------------
    SOURCE_RULES = {"fixed": 0, "mdl": 1, "aic": 2}

    def set_source_rule(self, rule="fixed"):
        """``"fixed"`` (default): every window has the n sources given at construction.  ``"mdl"`` / ``"aic"``: n is
        the maximum, and each window's count d in [0, n] is estimated from its covariance eigenvalues (Wax-Kailath
        MDL / AIC, include/music_b200.h); the peak rule fills the first d slots, the rest stay (0, 0, bin -1).
        Needs more snapshots than antennas (nsamples / m > m)."""
        if rule not in self.SOURCE_RULES:
            raise ValueError("rule must be one of %s" % sorted(self.SOURCE_RULES))
        _capi.check(self._lib.music_b200_set_source_rule(self._h, self.SOURCE_RULES[rule]), self._h)
        self._source_rule = rule

    def source_rule(self):
        return getattr(self, "_source_rule", "fixed")

    def last_counts(self):
        """int32 (W,) number of sources of each window of the last work() call (all n under the "fixed" rule)."""
        return self._last_counts

    # -- extension: off-grid peak refinement -------------------------------------------------------
    def set_refine(self, enable):
        """True: every reported peak is refined off the grid by safeguarded Newton steps on the exact fp64 MUSIC
        spectrum of the array geometry (include/music_b200.h); angles and levels change, bins and the spectrum stay the
        grid results.  Needs a table installed with ``set_array_geometry``; False (default) reports grid angles."""
        _capi.check(self._lib.music_b200_set_refine(self._h, 1 if enable else 0), self._h)
        self._refine = bool(enable)

    @property
    def refine(self):
        return getattr(self, "_refine", False)

    # -- extension: the spectrum estimator -----------------------------------------------------------
    ESTIMATORS = {"music": 0, "mvdr": 1, "bartlett": 2}

    def set_estimator(self, kind="music", loading=0.0):
        """``"music"`` (default): P = 1 / ||G^H a||^2.  ``"bartlett"``: the delay-and-sum beamscan,
        P = a^H R a / (a^H a)^2.  ``"mvdr"``: the Capon spectrum P = 1 / (a^H (R + delta I)^-1 a) with the diagonal
        loading delta = loading * tr(R) / m; loading 0 needs more snapshots than antennas.  Both new spectra are power
        estimates (include/music_b200.h); the peak rule, ``n`` slots, the source rule and the refinement apply to them
        unchanged.  ``loading`` must be 0 for "music" and "bartlett"."""
        if kind not in self.ESTIMATORS:
            raise ValueError("kind must be one of %s" % sorted(self.ESTIMATORS))
        _capi.check(self._lib.music_b200_set_estimator(self._h, self.ESTIMATORS[kind], float(loading)), self._h)
        self._estimator = (kind, float(loading))

    @property
    def estimator(self):
        """(kind, loading) in use"""
        return getattr(self, "_estimator", ("music", 0.0))

    # -- extension (SURVEY.md section 8(f) rank 4): GUI-rate reducers -----------------------------
    def reduce_angles(self, angles, levels=None, weighted=False):
        """Circular mean (degrees), mean resultant length and total weight per angle slot over the
        windows of ``angles`` (W, n) float32 - what a compass-type sink
        (/root/reference/python/doa_compass_control.py:102-108) consumes.  ``levels`` (W, n) marks
        unfilled slots (level 0) and, with ``weighted``, weights the windows."""
        a = np.ascontiguousarray(angles, dtype=np.float32).reshape(-1, self.n)
        l = None if levels is None else np.ascontiguousarray(levels, dtype=np.float32).reshape(-1, self.n)
        if l is not None and l.shape != a.shape:
            raise ValueError("levels must have the shape of angles")
        mean = np.empty(self.n, np.float32)
        res = np.empty(self.n, np.float32)
        wsum = np.empty(self.n, np.float32)
        rc = self._lib.music_b200_reduce_angles_host(self._h, a.ctypes.data, None if l is None else l.ctypes.data, a.shape[0],
                                                     1 if weighted else 0, mean.ctypes.data, res.ctypes.data, wsum.ctypes.data)
        _capi.check(rc, self._h)
        return mean, res, wsum

    def reduce_spectrum(self, spectrum):
        """Mean pseudospectrum over the windows of ``spectrum`` (W, resolution) float32."""
        sp = np.ascontiguousarray(spectrum, dtype=np.float32).reshape(-1, self.resolution)
        mean = np.empty(self.resolution, np.float32)
        _capi.check(self._lib.music_b200_reduce_spectrum_host(self._h, sp.ctypes.data, sp.shape[0], mean.ctypes.data), self._h)
        return mean

    def array_response_c64(self):
        """The table in use, as complex64 (resolution, m) - what the block holds after the SWIG
        conversion (swig/baz_swig.i:564)."""
        out = np.empty((self.resolution, self.m), np.complex64)
        _capi.check(self._lib.music_b200_get_table(self._h, out.ctypes.data), self._h)
        return out

    def work(self, noutput_items, input_items, output_items):
        """input_items[0]: complex64 (noutput_items, nsamples); output_items: 1..3 float32 arrays
        (angles (., n), levels (., n), spectrum (., resolution)).  Returns items produced."""
        W = int(noutput_items)
        if W <= 0:
            return 0
        x = input_items[0]
        if x.dtype != np.complex64 or not x.flags["C_CONTIGUOUS"] or x.size < W * self.nsamples:
            raise ValueError("input_items[0] must be C-contiguous complex64 with >= noutput_items*nsamples elements")
        outs = list(output_items)
        if not 1 <= len(outs) <= 3:
            raise ValueError("1 to 3 output ports")
        sizes = [self.n, self.n, self.resolution]
        for o, s in zip(outs, sizes):
            if o.dtype != np.float32 or not o.flags["C_CONTIGUOUS"] or o.size < W * s:
                raise ValueError("output buffers must be C-contiguous float32 of the port's item size")
        ang = outs[0]
        lvl = outs[1] if len(outs) > 1 else None
        spec = outs[2] if len(outs) > 2 else None
        self._last_bins = np.empty((W, self.n), np.int32)
        lvl_p, spec_p = lvl.ctypes.data if lvl is not None else None, spec.ctypes.data if spec is not None else None
        if self.source_rule() == "fixed":
            rc = self._lib.music_b200_process_host(self._h, x.ctypes.data, W, ang.ctypes.data, lvl_p, spec_p, self._last_bins.ctypes.data)
            self._last_counts = np.full(W, self.n, np.int32)
        else:
            self._last_counts = np.empty(W, np.int32)
            rc = self._lib.music_b200_process_host_counts(self._h, x.ctypes.data, W, ang.ctypes.data, lvl_p, spec_p,
                                                          self._last_bins.ctypes.data, self._last_counts.ctypes.data)
        _capi.check(rc, self._h)
        return W

    # -- extras (not in the reference) ---------------------------------------------------
    def last_bins(self):
        """int32 (W, n) peak-bin indices of the last work() call (-1 = unfilled slot)."""
        return self._last_bins

    def process_device(self, d_in, nwindows, d_angles, d_levels=None, d_spectrum=None, d_bins=None,
                       stream=None, d_P64=None, d_R=None, d_eigvals=None, d_counts=None):
        """Raw device-pointer entry (ints); buffers stay resident in HBM.  ``d_counts``: int32 [nwindows] device
        array that receives the per-window source counts (music_b200_process_device_counts; no fp64 internals)."""
        if d_counts is not None:
            if d_P64 is not None or d_R is not None or d_eigvals is not None:
                raise ValueError("d_counts cannot be combined with d_P64 / d_R / d_eigvals")
            rc = self._lib.music_b200_process_device_counts(
                self._h, d_in, int(nwindows), d_angles, d_levels, d_spectrum, d_bins, d_counts, stream)
            _capi.check(rc, self._h)
            return
        rc = self._lib.music_b200_process_device_ex(
            self._h, d_in, int(nwindows), d_angles, d_levels, d_spectrum, d_bins, d_P64, d_R, d_eigvals, stream)
        _capi.check(rc, self._h)

    # -- extension (SURVEY.md section 8(f) rank 2): planar antenna streams, windows by pointer arithmetic
    def work_planar(self, noutput_items, input_items, output_items, hop=None):
        """``input_items``: m C-contiguous complex64 1-D arrays, one per antenna, each holding at least
        ``(noutput_items - 1) * hop + N`` samples (N = nsamples / m); window w is
        ``x_w(r, c) = input_items[r][w * hop + c]``.  ``hop`` defaults to N (back-to-back vectors, what
        interleave + stream_to_vector feed the reference block); ``hop < N`` slides the window like
        /root/reference/lib/baz_overlap.cc:107-129 without copying the overlap.  Outputs as in work()."""
        W = int(noutput_items)
        if W <= 0:
            return 0
        N = self.nsamples // self.m
        hop = N if hop is None else int(hop)
        if hop < 1:
            raise ValueError("hop must be >= 1")
        if len(input_items) != self.m:
            raise ValueError("one input stream per antenna (m = %d)" % self.m)
        need = (W - 1) * hop + N
        for x in input_items:
            if x.dtype != np.complex64 or x.ndim != 1 or not x.flags["C_CONTIGUOUS"] or x.size < need:
                raise ValueError("each antenna stream must be a C-contiguous 1-D complex64 array of >= %d samples" % need)
        outs = list(output_items)
        if not 1 <= len(outs) <= 3:
            raise ValueError("1 to 3 output ports")
        sizes = [self.n, self.n, self.resolution]
        for o, sz in zip(outs, sizes):
            if o.dtype != np.float32 or not o.flags["C_CONTIGUOUS"] or o.size < W * sz:
                raise ValueError("output buffers must be C-contiguous float32 of the port's item size")
        ptrs = (ctypes.c_void_p * self.m)(*[x.ctypes.data for x in input_items])
        self._last_bins = np.empty((W, self.n), np.int32)
        rc = self._lib.music_b200_process_planar_host(
            self._h, ptrs, hop, W, outs[0].ctypes.data, outs[1].ctypes.data if len(outs) > 1 else None,
            outs[2].ctypes.data if len(outs) > 2 else None, self._last_bins.ctypes.data)
        _capi.check(rc, self._h)
        return W

    def process_planar_device(self, d_streams, hop, nwindows, d_angles, d_levels=None, d_spectrum=None, d_bins=None, stream=None):
        """Raw device-pointer entry: ``d_streams`` = m device addresses (ints) of the antenna streams."""
        if len(d_streams) != self.m:
            raise ValueError("one device stream per antenna (m = %d)" % self.m)
        ptrs = (ctypes.c_void_p * self.m)(*[int(p) for p in d_streams])
        rc = self._lib.music_b200_process_planar_device(self._h, ptrs, int(hop), int(nwindows), d_angles, d_levels, d_spectrum, d_bins, stream)
        _capi.check(rc, self._h)

    # -- extension (SURVEY.md section 8e): sharded device entry / fused all-gather of the peak bins ------------
    def device_count(self):
        return int(self._lib.music_b200_device_count(self._h))

    def process_device_sharded(self, d_in, nwindows_total, d_angles, d_levels=None, d_bins_all=None, streams=None):
        """Multi-device handle, inputs resident: ``d_in[g]`` / ``d_angles[g]`` / ``d_levels[g]`` are device addresses
        (ints) on device g holding the shard w = i*G + g; ``d_bins_all[p]`` is an int32 [nwindows_total][n] array on
        device p that receives EVERY shard's peak bins in stream order (stored by the scan epilogues over NVLink)."""
        G = self.device_count()
        arr = lambda v: None if v is None else (ctypes.c_void_p * G)(*[None if x is None else int(x) for x in v])
        a_in, a_ang, a_lvl, a_bins, a_st = arr(d_in), arr(d_angles), arr(d_levels), arr(d_bins_all), arr(streams)
        _capi.check(self._lib.music_b200_process_device_sharded(self._h, a_in, int(nwindows_total), a_ang, a_lvl, a_bins, a_st), self._h)

    def gather_create(self, total_windows):
        """One rank per process: allocate this rank's stream-ordered gather buffer; returns the 128 bytes of CUDA IPC
        handles to exchange with the other ranks (see include/music_b200.h)."""
        buf = (ctypes.c_ubyte * 128)()
        _capi.check(self._lib.music_b200_gather_create(self._h, int(total_windows), buf), self._h)
        return bytes(buf)

    def gather_attach(self, nranks, rank, all_handles):
        raw = b"".join(all_handles)
        if len(raw) != 128 * int(nranks):
            raise ValueError("need 128 bytes of IPC handles per rank")
        buf = (ctypes.c_ubyte * len(raw)).from_buffer_copy(raw)
        _capi.check(self._lib.music_b200_gather_attach(self._h, int(nranks), int(rank), buf), self._h)

    def gather_wait(self, stream=None):
        _capi.check(self._lib.music_b200_gather_wait(self._h, stream), self._h)

    def gather_read(self, total_windows):
        """Host copy (int32 (total_windows, n), stream order) of this rank's gather buffer."""
        out = np.empty((int(total_windows), self.n), np.int32)
        _capi.check(self._lib.music_b200_gather_read(self._h, out.ctypes.data, out.size), self._h)
        return out

    def gather_buffer_ptr(self):
        return int(self._lib.music_b200_gather_buffer(self._h) or 0)

    def set_stage_timing(self, enable):
        _capi.check(self._lib.music_b200_set_stage_timing(self._h, 1 if enable else 0), self._h)

    def stage_times_ms(self):
        """(ms[4] = cov, eig, scan, topn accumulated since the last call; chunks)"""
        ms = (ctypes.c_double * 4)()
        ch = ctypes.c_uint64(0)
        _capi.check(self._lib.music_b200_get_stage_times(self._h, ms, ctypes.byref(ch)), self._h)
        return list(ms), int(ch.value)

    def fused8_stats(self):
        """(windows solved by squaring, windows solved by the Jacobi fallback) of the fused M = 8 kernel so far."""
        v = (ctypes.c_uint64 * 2)()
        _capi.check(self._lib.music_b200_debug_fused8_stats(self._h, v), self._h)
        return int(v[0]), int(v[1])

    def launch_count(self):
        return int(self._lib.music_b200_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.music_b200_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
