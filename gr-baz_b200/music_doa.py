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

CALIB_MAX_SEGMENTS = 1024  # MUSIC_B200_CALIB_MAX_SEGMENTS

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
        ``exclusion_bins`` = 0, the "music" estimator and refinement off;
        ``"esprit"`` = LS-ESPRIT: gridless angles from the eigenvalues of the signal subspace's shift-invariance matrix,
        for the same arrays and with the same restrictions as ``"roots"``.  On a ``music_doa_azel`` block it is 2-D
        ESPRIT instead: gridless (azimuth, elevation) pairs for a planar lattice array (Mx x My elements in row-major
        order, one z, steps <= lambda / 2) installed with ``set_array_geometry``, with no grid scan or 2-D peak pick;
        it needs n <= min((Mx - 1) My, Mx (My - 1)) besides the restrictions of ``"roots"``;
        ``"dml"`` = deterministic maximum likelihood by alternating projection: the n table rows whose span captures the
        most power of the covariance, so coherent sources (multipath) are resolved, on any table; levels are
        least-squares source powers.  It needs ``exclusion_bins`` = 0, the "music" estimator and refinement off or "joint"; use the
        "fixed" source rule for coherent sources;
        ``"wsf"`` = weighted subspace fitting: DML's search on the eigenvalue-weighted signal subspace, whose
        large-sample variance is the stochastic CRB; coherent sources need no smoothing.  It has the restrictions of
        ``"dml"`` and also takes ``set_refine("joint")``;
        ``"manifold"`` = root-MUSIC on any planar array by manifold separation: gridless angles over the whole 360
        degrees from the roots of one polynomial per window, for a geometry installed with ``set_array_geometry``
        spanning about 4.4 wavelengths or less.  It has the restrictions of ``"roots"``; on a line array every source
        also has a mirror root, so use ``"roots"`` or ``"esprit"`` there."""
        modes = {"top_bins": 0, "local_maxima": 1, "roots": 2, "esprit": 3, "dml": 4, "manifold": 5, "wsf": 6}
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
    REFINE_MODES = {"off": 0, "newton": 1, "joint": 2}

    def set_refine(self, enable):
        """True or ``"newton"``: every reported peak is refined off the grid by safeguarded Newton steps on the exact
        fp64 MUSIC spectrum of the array geometry (include/music_b200.h); angles and levels change, bins and the spectrum
        stay the grid results.  ``"joint"`` (the "dml" and "wsf" peak modes only): all slots of a window are refined
        together by Gauss-Newton steps on the peak mode's own criterion.  Both need a table installed with
        ``set_array_geometry``; False or ``"off"`` (default) reports grid angles."""
        if isinstance(enable, str):
            if enable not in self.REFINE_MODES:
                raise ValueError("refine must be True, False or one of %s" % sorted(self.REFINE_MODES))
            mode = self.REFINE_MODES[enable]
        else:
            mode = 1 if enable else 0
        _capi.check(self._lib.music_b200_set_refine(self._h, mode), self._h)
        self._refine = mode

    @property
    def refine(self):
        """The refine mode as its C code: 0 = off, 1 = Newton, 2 = joint (false only when off)."""
        return getattr(self, "_refine", 0)

    # -- extension: the spectrum estimator -----------------------------------------------------------
    ESTIMATORS = {"music": 0, "mvdr": 1, "bartlett": 2, "iaa": 4}

    def set_estimator(self, kind="music", loading=0.0):
        """``"music"`` (default): P = 1 / ||G^H a||^2.  ``"bartlett"``: the delay-and-sum beamscan,
        P = a^H R a / (a^H a)^2.  ``"mvdr"``: the Capon spectrum P = 1 / (a^H (R + delta I)^-1 a) with the diagonal
        loading delta = loading * tr(R) / m; loading 0 needs more snapshots than antennas.  Both new spectra are power
        estimates (include/music_b200.h); the peak rule, ``n`` slots, the source rule and the refinement apply to them
        unchanged.  ``loading`` must be 0 for "music" and "bartlett".
        ``"iaa"``: the iterative adaptive approach (Yardibi et al. 2010), a weighted-least-squares power spectrum that
        starts from Bartlett and re-weights it ``set_iaa_iterations`` times (default 15) with the loading
        delta = loading * tr(R) / m (any loading >= 0; 0 works for any snapshot count).  It needs no source count,
        works with fewer snapshots than antennas and resolves coherent sources (multipath) on every block kind and
        table; its level at a peak is the source's power.  It takes refinement off and the grid peak modes only.  It
        does not replace "music" for closely spaced uncorrelated sources with plenty of snapshots, which MUSIC resolves
        and IAA does not."""
        if kind not in self.ESTIMATORS:
            raise ValueError("kind must be one of %s" % sorted(self.ESTIMATORS))
        _capi.check(self._lib.music_b200_set_estimator(self._h, self.ESTIMATORS[kind], float(loading)), self._h)
        self._estimator = (kind, float(loading))

    @property
    def estimator(self):
        """(kind, loading) in use"""
        return getattr(self, "_estimator", ("music", 0.0))

    def set_iaa_iterations(self, n=15):
        """The iteration count of the "iaa" estimator: 1 .. 64, default 15 (read only under "iaa")."""
        _capi.check(self._lib.music_b200_set_iaa_iterations(self._h, int(n)), self._h)
        self._iaa_iterations = int(n)

    @property
    def iaa_iterations(self):
        return getattr(self, "_iaa_iterations", 15)

    # -- extension: beamformed source signals ------------------------------------------------------------
    BEAMFORMERS = {"off": 0, "das": 1, "mvdr": 2, "lcmv": 3}

    def set_beamformer(self, kind="off", loading=0.0):
        """Receive every reported source: ``"das"`` (delay-and-sum, w = a / a^H a), ``"mvdr"`` (distortionless,
        minimum output power on R + delta I, delta = loading * tr(R) / m) or ``"lcmv"`` (unit gain on its own source,
        a null on every other filled slot of the window).  While it is not ``"off"`` (default), ``work()`` also returns
        the beams and weights of its windows through ``last_beams()`` / ``last_weights()`` (include/music_b200.h).
        ``loading`` must be 0 for "off" and "das"; loading 0 under "mvdr" / "lcmv" needs more snapshots than antennas.
        With coherent sources (the "dml" peak mode) MVDR and LCMV beams cancel the signal: use "das" there."""
        if kind not in self.BEAMFORMERS:
            raise ValueError("kind must be one of %s" % sorted(self.BEAMFORMERS))
        _capi.check(self._lib.music_b200_set_beamformer(self._h, self.BEAMFORMERS[kind], float(loading)), self._h)
        self._beamformer = (kind, float(loading))

    def beamformer(self):
        """(kind, loading) in use"""
        return getattr(self, "_beamformer", ("off", 0.0))

    def last_beams(self):
        """complex64 (W, n, N) beams of the last work() call (N = nsamples / m), zeros for unfilled slots; None while the
        beamformer is off."""
        return getattr(self, "_last_beams", None)

    def last_weights(self):
        """complex128 (W, n, m) beam weights of the last work() call; None while the beamformer is off."""
        return getattr(self, "_last_weights", None)

    def process_device_beams(self, d_in, nwindows, d_angles, d_levels=None, d_spectrum=None, d_bins=None, d_counts=None,
                             d_weights=None, d_beams=None, stream=None):
        """Raw device-pointer entry (ints): the outputs of ``process_device(..., d_counts=...)`` plus ``d_weights``
        (complex fp64 [nwindows][n][m]) and ``d_beams`` (complex64 [nwindows][n][N]); one of the two may be None."""
        rc = self._lib.music_b200_process_device_beams(self._h, d_in, int(nwindows), d_angles, d_levels, d_spectrum, d_bins,
                                                        d_counts, d_weights, d_beams, stream)
        _capi.check(rc, self._h)

    # -- extension: covariance integration across windows ----------------------------------------------------
    def set_integration(self, alpha):
        """Integrate the covariance across windows with forgetting factor ``alpha`` (0 <= alpha < 1; 0, the default, is
        off): each window's estimators read Rbar_j = S_j / c_j, S_j = alpha S_{j-1} + R_j, c_j = alpha c_{j-1} + 1, over
        the windows since the last reset, across calls (include/music_b200.h).  MDL / AIC count with N_eff.  Resets the
        carry; so do ``reset_integration``, ``set_array_response``, ``set_array_geometry`` and ``set_calibration``."""
        _capi.check(self._lib.music_b200_set_integration(self._h, float(alpha)), self._h)

    def reset_integration(self):
        """Restart the integration at the next window (the next window's covariance is its own)."""
        _capi.check(self._lib.music_b200_reset_integration(self._h), self._h)

    # -- extension: the stochastic Cramer-Rao bound of every reported direction ------------------------------------
    def set_crb(self, enable):
        """True: ``work()`` also returns, through ``last_crb()``, the stochastic Cramer-Rao bound on the standard deviation
        of every reported angle, in degrees, evaluated on the device at the window's covariance and reported angles
        (include/music_b200.h).  It is the bound for Gaussian sources in white noise, the same whatever peak mode found
        the angle, not that estimator's own variance.  Needs a table installed with ``set_array_geometry``.  Under the
        "top_bins" peak mode with n >= 2 the slots are neighbouring bins of one peak, and their finite values mean
        nothing: use "local_maxima" or a gridless mode there."""
        self._crb = bool(enable)

    def crb(self):
        return getattr(self, "_crb", False)

    def last_crb(self):
        """float32 (W, n) bound of the last work() call in degrees (0 for unfilled slots, NaN where the window's bound
        does not exist); None while ``set_crb`` is off.  On a ``music_doa_azel`` block (W, n, 3): std of the azimuth,
        std of the elevation (degrees) and their correlation."""
        return getattr(self, "_last_crb", None)

    def process_device_crb(self, d_in, nwindows, d_angles, d_std, d_levels=None, d_spectrum=None, d_bins=None, d_counts=None,
                           d_weights=None, d_beams=None, stream=None):
        """Raw device-pointer entry (ints): the outputs of ``process_device_beams`` plus ``d_std`` (float32
        [nwindows][n], required); ``d_weights`` and ``d_beams`` may both be None, and otherwise need a beamformer."""
        rc = self._lib.music_b200_process_device_crb(self._h, d_in, int(nwindows), d_angles, d_levels, d_spectrum, d_bins,
                                                      d_counts, d_weights, d_beams, d_std, stream)
        _capi.check(rc, self._h)

    # -- extension: angle tracking across windows ---------------------------------------------------------
    TRACK_VARIANCES = {"off": 0, "fixed": 1, "crb": 2}

    def set_tracking(self, variance="off", q=0.01, rate_std0=1.0, floor_deg=0.5, crb_scale=1.0, gate=9.0, confirm_hits=3,
                     confirm_window=5, max_misses=5, max_tracks=8):
        """Track every source across windows and calls on the device: one constant-velocity Kalman filter per track
        (angles in degrees, time in windows: ``q`` is the white-acceleration density in deg^2 / window^3), global
        nearest-neighbour assignment inside the chi-square ``gate``, confirmation after ``confirm_hits`` hits within
        ``confirm_window`` windows, deletion after ``max_misses`` consecutive misses, at most ``max_tracks`` (<= 32)
        tracks (include/music_b200.h).  ``variance``: "fixed" (measurement std ``floor_deg``), "crb" (``crb_scale`` times
        the slot's Cramer-Rao bound plus ``floor_deg``, which needs a table installed with ``set_array_geometry``) or
        "off" (default).  While it is on, ``work()`` also returns ``last_tracks()``.  Resets the tracks; so do
        ``reset_tracks``, ``set_array_response`` and ``set_array_geometry``.  Use the "local_maxima" or a gridless peak
        mode: "top_bins" with n >= 2 puts two slots, and so two tracks, on one source."""
        if variance not in self.TRACK_VARIANCES:
            raise ValueError("variance must be one of %s" % sorted(self.TRACK_VARIANCES))
        _capi.check(self._lib.music_b200_set_tracking(self._h, self.TRACK_VARIANCES[variance], float(q), float(rate_std0),
                                                      float(floor_deg), float(crb_scale), float(gate), int(confirm_hits),
                                                      int(confirm_window), int(max_misses), int(max_tracks)), self._h)
        self._tracking = (variance, int(max_tracks))

    def tracking(self):
        """the variance in use ("off", "fixed" or "crb")"""
        return getattr(self, "_tracking", ("off", 0))[0]

    def reset_tracks(self):
        """Drop every track: the next window starts from no tracks and ids restart at 0."""
        _capi.check(self._lib.music_b200_reset_tracks(self._h), self._h)

    def tracks(self):
        """The tracker's carry after the last tracking call: (rows int32 (T, 5) = id, status (0 empty, 1 tentative, 2
        confirmed), age, hits, consecutive misses; state float64 (T, 2D + (2D)^2) = x then P row-major, D = 1 (2 on a
        ``music_doa_azel`` block); next_id)."""
        T = getattr(self, "_tracking", ("off", 0))[1]
        D = 2 if self._azel() else 1
        rows = np.zeros((T, 5), np.int32)
        state = np.zeros((T, 2 * D + 4 * D * D), np.float64)
        nxt = ctypes.c_uint32(0)
        ptr = lambda a: a.ctypes.data if T else None  # no rows asked for before set_tracking()
        _capi.check(self._lib.music_b200_get_tracks(self._h, ptr(rows), ptr(state), ctypes.byref(nxt)), self._h)
        return rows, state, int(nxt.value)

    def last_tracks(self):
        """(slot_track int32 (W, n): the track each slot's measurement updated or started, -1 for none; track_ids int32
        (W, T): the confirmed track of every row, -1 for none; track_state float32 (W, T, 3): angle, rate (degrees per
        window) and std of the angle of those rows, (W, T, 6) on a ``music_doa_azel`` block: az, rate, el, rate, std az,
        std el) of the last work() call; None while tracking is off."""
        return getattr(self, "_last_tracks", None)

    def _azel(self):
        return False

    def _track_buffers(self, W):
        """the tracker's outputs of a work() call of W windows (None while tracking is off)"""
        self._last_tracks = None
        if self.tracking() == "off":
            return None
        T = self._tracking[1]
        self._last_tracks = (np.empty((W, self.n), np.int32), np.empty((W, T), np.int32),
                             np.empty((W, T, 6 if self._azel() else 3), np.float32))
        return [a.ctypes.data for a in self._last_tracks]

    def process_device_tracks(self, d_in, nwindows, d_angles, d_slot_track, d_levels=None, d_spectrum=None, d_bins=None,
                              d_counts=None, d_weights=None, d_beams=None, d_std=None, d_track_ids=None, d_track_state=None,
                              stream=None):
        """Raw device-pointer entry (ints): the outputs of ``process_device_crb`` (``d_std`` may be None) plus
        ``d_slot_track`` (int32 [nwindows][n], required), ``d_track_ids`` (int32 [nwindows][T]) and ``d_track_state``
        (float32 [nwindows][T][3]), the last two both or neither."""
        rc = self._lib.music_b200_process_device_tracks(self._h, d_in, int(nwindows), d_angles, d_levels, d_spectrum, d_bins,
                                                         d_counts, d_weights, d_beams, d_std, d_slot_track, d_track_ids,
                                                         d_track_state, stream)
        _capi.check(rc, self._h)

    # -- extension: receiver calibration -----------------------------------------------------------------
    CALIBRATIONS = {"phase": 1, "gain_phase": 2}

    def set_calibration(self, gains=None):
        """Correct every element's receiver gain on the device: ``gains`` = complex (m,) g_m, the chain of element m
        multiplies its signal by g_m; every later call works on the covariance corrected by c_m = 1 / g_m, in every mode
        (include/music_b200.h).  ``None`` clears it.  The setting survives ``set_array_response`` and
        ``set_array_geometry``; beam weights are returned for the raw input."""
        if gains is None:
            _capi.check(self._lib.music_b200_set_calibration(self._h, None), self._h)
            return
        g = np.asarray(gains, dtype=np.complex128).reshape(-1)
        if g.size != self.m:
            raise ValueError("gains must hold m = %d complex values" % self.m)
        g = np.ascontiguousarray(g)
        _capi.check(self._lib.music_b200_set_calibration(self._h, g.ctypes.data), self._h)

    def calibration(self):
        """complex128 (m,) gains in use, all 1 when none is set"""
        g = np.empty(self.m, np.complex128)
        _capi.check(self._lib.music_b200_get_calibration(self._h, g.ctypes.data), self._h)
        return g

    def calib_reset(self):
        _capi.check(self._lib.music_b200_calib_reset(self._h), self._h)

    def calib_accumulate(self, windows):
        """adds the raw covariance of ``windows`` (complex64 (W, nsamples), host memory) to the calibration accumulator"""
        x = np.ascontiguousarray(windows, dtype=np.complex64).reshape(-1, self.nsamples)
        _capi.check(self._lib.music_b200_calib_accumulate_host(self._h, x.ctypes.data, x.shape[0]), self._h)

    def calib_accumulate_device(self, d_in, nwindows, stream=None):
        """raw device-pointer form of ``calib_accumulate`` (enqueued on ``stream``)"""
        _capi.check(self._lib.music_b200_calib_accumulate_device(self._h, d_in, int(nwindows), stream), self._h)

    def calib_solve(self, angle_deg, el_deg=0.0, kind="gain_phase"):
        """the gains fitted to the accumulated windows of one source at (``angle_deg``, ``el_deg``): (complex128 (m,)
        gains, residual, sweeps).  The accumulator is kept; nothing is applied."""
        if kind not in self.CALIBRATIONS:
            raise ValueError("kind must be one of %s" % sorted(self.CALIBRATIONS))
        g = np.empty(self.m, np.complex128)
        st = np.empty(2, np.float64)
        _capi.check(self._lib.music_b200_calib_solve(self._h, float(angle_deg), float(el_deg), self.CALIBRATIONS[kind], g.ctypes.data,
                                                     st.ctypes.data), self._h)
        return g, float(st[0]), int(st[1])

    def calibrate(self, windows, angle_deg, el_deg=0.0, kind="gain_phase"):
        """Estimate the receiver gains from ``windows`` (complex64 (W, nsamples)) of one dominant source at the known
        direction (``angle_deg``, ``el_deg``; el 0 on a 1-D block): reset, accumulate and solve on the device.  Returns
        (gains, residual, sweeps); apply the gains with ``set_calibration`` once the residual looks right.  ``kind``:
        "gain_phase" (m >= 3) or "phase".  Needs a table installed with ``set_array_geometry``."""
        self.calib_reset()
        self.calib_accumulate(windows)
        return self.calib_solve(angle_deg, el_deg, kind)

    # -- extension: receiver self-calibration without a known source ------------------------------------------------
    def calib_blind_reset(self):
        _capi.check(self._lib.music_b200_calib_blind_reset(self._h), self._h)

    def calib_blind_accumulate(self, windows, segment):
        """adds the segments of ``windows`` (complex64 (W, nsamples), host memory; W a multiple of ``segment``): every
        ``segment`` consecutive windows form one segment covariance"""
        x = np.ascontiguousarray(windows, dtype=np.complex64).reshape(-1, self.nsamples)
        _capi.check(self._lib.music_b200_calib_blind_accumulate_host(self._h, x.ctypes.data, x.shape[0], int(segment)), self._h)

    def calib_blind_accumulate_device(self, d_in, nwindows, segment, stream=None):
        """raw device-pointer form of ``calib_blind_accumulate`` (enqueued on ``stream``)"""
        _capi.check(self._lib.music_b200_calib_blind_accumulate_device(self._h, d_in, int(nwindows), int(segment), stream),
                    self._h)

    def calib_blind_solve(self, nsources, kind="gain_phase", starts=32, seed=0):
        """the gains fitted to the accumulated segments, each holding ``nsources`` unknown sources: (complex128 (m,)
        gains, float64 (S, nsources) angles in degrees (NaN where a segment had fewer local minima), stats) with stats a
        dict of the misfit (small when calibrated), the polish iterations and the winning start.  The segments are
        kept; nothing is applied."""
        if kind not in self.CALIBRATIONS:
            raise ValueError("kind must be one of %s" % sorted(self.CALIBRATIONS))
        d = int(nsources)
        g = np.empty(self.m, np.complex128)
        st = np.empty(4, np.float64)
        ang = np.empty((CALIB_MAX_SEGMENTS, max(d, 0)), np.float64)  # room for every segment the handle can hold
        _capi.check(self._lib.music_b200_calib_blind_solve(self._h, d, self.CALIBRATIONS[kind], int(starts), int(seed),
                                                           g.ctypes.data, ang.ctypes.data, st.ctypes.data), self._h)
        S = int(st[3])
        return g, ang[:S].copy(), {"misfit": float(st[0]), "polish": int(st[1]), "start": int(st[2])}

    def calibrate_blind(self, windows, nsources, segment, kind="gain_phase", starts=32, seed=0):
        """Estimate the receiver gains from ``windows`` (complex64 (W, nsamples)) of unknown emitters, ``nsources`` in
        every segment of ``segment`` consecutive windows, without a known direction: reset, accumulate and solve on the
        device.  Returns (gains, angles, stats) as ``calib_blind_solve``; apply the gains with ``set_calibration`` once
        the misfit looks right.  Needs m >= 3 elements off one line and a table installed with ``set_array_geometry``."""
        self.calib_blind_reset()
        self.calib_blind_accumulate(windows, segment)
        return self.calib_blind_solve(nsources, kind, starts, seed)

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
        self._last_beams = self._last_weights = self._last_crb = None
        beams = self.beamformer()[0] != "off"
        if beams:
            N = self.nsamples // self.m
            self._last_weights = np.empty((W, self.n, self.m), np.complex128)
            self._last_beams = np.empty((W, self.n, N), np.complex64)
        wts_p = self._last_weights.ctypes.data if beams else None
        beams_p = self._last_beams.ctypes.data if beams else None
        trk = self._track_buffers(W)
        if trk is not None:
            # one call for the tracks, the bound and the beams: two would advance the integration and track carries twice
            self._last_counts = np.empty(W, np.int32)
            if self.crb():
                self._last_crb = np.empty((W, self.n), np.float32)
            crb_p = self._last_crb.ctypes.data if self.crb() else None
            rc = self._lib.music_b200_process_host_tracks(self._h, x.ctypes.data, W, ang.ctypes.data, lvl_p, spec_p,
                                                          self._last_bins.ctypes.data, self._last_counts.ctypes.data, wts_p, beams_p,
                                                          crb_p, *trk)
        elif self.crb():
            # one call for the bound and the beams: two would advance the integration carry twice
            self._last_counts = np.empty(W, np.int32)
            self._last_crb = np.empty((W, self.n), np.float32)
            rc = self._lib.music_b200_process_host_crb(self._h, x.ctypes.data, W, ang.ctypes.data, lvl_p, spec_p,
                                                       self._last_bins.ctypes.data, self._last_counts.ctypes.data, wts_p, beams_p,
                                                       self._last_crb.ctypes.data)
        elif beams:
            self._last_counts = np.empty(W, np.int32)
            rc = self._lib.music_b200_process_host_beams(self._h, x.ctypes.data, W, ang.ctypes.data, lvl_p, spec_p,
                                                         self._last_bins.ctypes.data, self._last_counts.ctypes.data, wts_p, beams_p)
        elif self.source_rule() == "fixed":
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
