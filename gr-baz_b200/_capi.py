"""ctypes binding of the C ABI in include/music_b200.h (libmusic_b200.so).

This is the stand-in for the SWIG layer of the reference (swig/baz_swig.i:560-574): SWIG is
not available in this image, so the Python mirror of ``baz.music_doa`` talks to the same
C ABI that lib/baz_music_doa.cc (the GNU Radio block) calls.  There is no fallback: if the
library is missing or no sm_90 device is present, this raises.
"""
from __future__ import annotations

import ctypes
import os

from . import build as _build

_lib = None

OK, EINVAL, ECUDA, ENODEVICE, ENOMEM = 0, -1, -2, -3, -4


class MusicB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("music_b200 error %d: %s" % (code, msg))
        self.code = code


def lib_path() -> str:
    return _build.LIB


def load():
    """Load libmusic_b200.so (must have been built by __graft_entry__.build())."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.exists(path):
            raise ImportError(
                "CUDA library %s is missing - run `python -c 'import __graft_entry__ as g; g.build()'`; "
                "there is no CPU fallback" % path)
        L = ctypes.CDLL(path)
        vp, u32, fp = ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p
        L.music_b200_version.restype = ctypes.c_int
        L.music_b200_create.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, fp, ctypes.c_int]
        L.music_b200_create.restype = ctypes.c_int
        L.music_b200_create_multi.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, fp, ctypes.POINTER(ctypes.c_int), ctypes.c_int]
        L.music_b200_create_multi.restype = ctypes.c_int
        L.music_b200_device_count.argtypes = [vp]
        L.music_b200_device_count.restype = ctypes.c_int
        L.music_b200_process_device_sharded.argtypes = [vp, fp, u32, fp, fp, fp, fp]
        L.music_b200_process_device_sharded.restype = ctypes.c_int
        L.music_b200_gather_create.argtypes = [vp, u32, fp]
        L.music_b200_gather_create.restype = ctypes.c_int
        L.music_b200_gather_attach.argtypes = [vp, ctypes.c_int, ctypes.c_int, fp]
        L.music_b200_gather_attach.restype = ctypes.c_int
        L.music_b200_gather_wait.argtypes = [vp, vp]
        L.music_b200_gather_wait.restype = ctypes.c_int
        L.music_b200_gather_buffer.argtypes = [vp]
        L.music_b200_gather_buffer.restype = ctypes.c_void_p
        L.music_b200_gather_read.argtypes = [vp, fp, u32]
        L.music_b200_gather_read.restype = ctypes.c_int
        L.music_b200_set_table.argtypes = [vp, fp]
        L.music_b200_set_table.restype = ctypes.c_int
        L.music_b200_process_planar_host.argtypes = [vp, fp, u32, u32, fp, fp, fp, fp]
        L.music_b200_process_planar_host.restype = ctypes.c_int
        L.music_b200_process_planar_device.argtypes = [vp, fp, u32, u32, fp, fp, fp, fp, vp]
        L.music_b200_process_planar_device.restype = ctypes.c_int
        L.music_b200_reduce_angles_device.argtypes = [vp, fp, fp, u32, ctypes.c_int, fp, fp, fp, vp]
        L.music_b200_reduce_angles_device.restype = ctypes.c_int
        L.music_b200_reduce_spectrum_device.argtypes = [vp, fp, u32, fp, vp]
        L.music_b200_reduce_spectrum_device.restype = ctypes.c_int
        L.music_b200_reduce_angles_host.argtypes = [vp, fp, fp, u32, ctypes.c_int, fp, fp, fp]
        L.music_b200_reduce_angles_host.restype = ctypes.c_int
        L.music_b200_reduce_spectrum_host.argtypes = [vp, fp, u32, fp]
        L.music_b200_reduce_spectrum_host.restype = ctypes.c_int
        L.music_b200_set_peak_mode.argtypes = [vp, ctypes.c_int, u32]
        L.music_b200_set_peak_mode.restype = ctypes.c_int
        L.music_b200_set_source_rule.argtypes = [vp, ctypes.c_int]
        L.music_b200_set_source_rule.restype = ctypes.c_int
        L.music_b200_set_refine.argtypes = [vp, ctypes.c_int]
        L.music_b200_set_refine.restype = ctypes.c_int
        L.music_b200_set_estimator.argtypes = [vp, ctypes.c_int, ctypes.c_double]
        L.music_b200_set_estimator.restype = ctypes.c_int
        L.music_b200_set_iaa_iterations.argtypes = [vp, ctypes.c_int]
        L.music_b200_set_iaa_iterations.restype = ctypes.c_int
        L.music_b200_set_geometry.argtypes = [vp, fp, ctypes.c_double, ctypes.POINTER(u32)]
        L.music_b200_set_geometry.restype = ctypes.c_int
        L.music_b200_steer_entry_host.argtypes = [fp, ctypes.c_double, u32, u32, u32, fp]
        L.music_b200_steer_entry_host.restype = None
        L.music_b200_manifold_coeffs_host.argtypes = [fp, u32, ctypes.c_double, ctypes.POINTER(u32), fp]
        L.music_b200_manifold_coeffs_host.restype = ctypes.c_int
        L.music_b200_azel_lattice_host.argtypes = [fp, u32, ctypes.c_double, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int), fp]
        L.music_b200_azel_lattice_host.restype = ctypes.c_int
        L.music_b200_get_table.argtypes = [vp, fp]
        L.music_b200_get_table.restype = ctypes.c_int
        L.music_b200_process_host.argtypes = [vp, fp, u32, fp, fp, fp, fp]
        L.music_b200_process_host.restype = ctypes.c_int
        L.music_b200_process_device.argtypes = [vp, fp, u32, fp, fp, fp, fp, vp]
        L.music_b200_process_device.restype = ctypes.c_int
        L.music_b200_process_device_ex.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_device_ex.restype = ctypes.c_int
        L.music_b200_process_host_counts.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp]
        L.music_b200_process_host_counts.restype = ctypes.c_int
        L.music_b200_process_device_counts.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_device_counts.restype = ctypes.c_int
        dbl = ctypes.c_double
        L.music_b200_set_beamformer.argtypes = [vp, ctypes.c_int, ctypes.c_double]
        L.music_b200_set_beamformer.restype = ctypes.c_int
        L.music_b200_process_device_beams.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_device_beams.restype = ctypes.c_int
        L.music_b200_process_host_beams.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp]
        L.music_b200_process_host_beams.restype = ctypes.c_int
        L.music_b200_set_calibration.argtypes = [vp, fp]
        L.music_b200_set_calibration.restype = ctypes.c_int
        L.music_b200_get_calibration.argtypes = [vp, fp]
        L.music_b200_get_calibration.restype = ctypes.c_int
        L.music_b200_calib_reset.argtypes = [vp]
        L.music_b200_calib_reset.restype = ctypes.c_int
        L.music_b200_calib_accumulate_device.argtypes = [vp, fp, u32, vp]
        L.music_b200_calib_accumulate_device.restype = ctypes.c_int
        L.music_b200_calib_accumulate_host.argtypes = [vp, fp, u32]
        L.music_b200_calib_accumulate_host.restype = ctypes.c_int
        L.music_b200_calib_solve.argtypes = [vp, dbl, dbl, ctypes.c_int, fp, fp]
        L.music_b200_calib_solve.restype = ctypes.c_int
        L.music_b200_calib_blind_reset.argtypes = [vp]
        L.music_b200_calib_blind_reset.restype = ctypes.c_int
        L.music_b200_calib_blind_accumulate_device.argtypes = [vp, fp, u32, u32, vp]
        L.music_b200_calib_blind_accumulate_device.restype = ctypes.c_int
        L.music_b200_calib_blind_accumulate_host.argtypes = [vp, fp, u32, u32]
        L.music_b200_calib_blind_accumulate_host.restype = ctypes.c_int
        L.music_b200_calib_blind_solve.argtypes = [vp, u32, ctypes.c_int, u32, ctypes.c_uint64, fp, fp, fp]
        L.music_b200_calib_blind_solve.restype = ctypes.c_int
        L.music_b200_set_integration.argtypes = [vp, dbl]
        L.music_b200_set_integration.restype = ctypes.c_int
        L.music_b200_reset_integration.argtypes = [vp]
        L.music_b200_reset_integration.restype = ctypes.c_int
        L.music_b200_process_device_crb.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_device_crb.restype = ctypes.c_int
        L.music_b200_process_host_crb.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, fp]
        L.music_b200_process_host_crb.restype = ctypes.c_int
        L.music_b200_process_azel_device_crb.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_azel_device_crb.restype = ctypes.c_int
        L.music_b200_process_azel_host_crb.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp]
        L.music_b200_process_azel_host_crb.restype = ctypes.c_int
        L.music_b200_set_tracking.argtypes = [vp, ctypes.c_int, dbl, dbl, dbl, dbl, dbl, u32, u32, u32, u32]
        L.music_b200_set_tracking.restype = ctypes.c_int
        L.music_b200_reset_tracks.argtypes = [vp]
        L.music_b200_reset_tracks.restype = ctypes.c_int
        L.music_b200_get_tracks.argtypes = [vp, fp, fp, ctypes.POINTER(u32)]
        L.music_b200_get_tracks.restype = ctypes.c_int
        L.music_b200_process_device_tracks.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_device_tracks.restype = ctypes.c_int
        L.music_b200_process_host_tracks.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp]
        L.music_b200_process_host_tracks.restype = ctypes.c_int
        L.music_b200_process_azel_device_tracks.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_azel_device_tracks.restype = ctypes.c_int
        L.music_b200_process_azel_host_tracks.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp]
        L.music_b200_process_azel_host_tracks.restype = ctypes.c_int
        L.music_b200_create_azel.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, u32, dbl, dbl, fp, dbl, ctypes.c_int]
        L.music_b200_create_azel.restype = ctypes.c_int
        L.music_b200_set_geometry_azel.argtypes = [vp, fp, dbl]
        L.music_b200_set_geometry_azel.restype = ctypes.c_int
        L.music_b200_process_azel_host.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp]
        L.music_b200_process_azel_host.restype = ctypes.c_int
        L.music_b200_process_azel_device.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_azel_device.restype = ctypes.c_int
        L.music_b200_create_channels.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, u32, u32, u32, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.music_b200_create_channels.restype = ctypes.c_int
        L.music_b200_set_geometry_channels.argtypes = [vp, fp, dbl, dbl]
        L.music_b200_set_geometry_channels.restype = ctypes.c_int
        L.music_b200_channel_frequencies.argtypes = [vp, fp]
        L.music_b200_channel_frequencies.restype = ctypes.c_int
        L.music_b200_get_table_channel.argtypes = [vp, u32, fp]
        L.music_b200_get_table_channel.restype = ctypes.c_int
        L.music_b200_set_focusing.argtypes = [vp, u32, u32]
        L.music_b200_set_focusing.restype = ctypes.c_int
        L.music_b200_get_focusing.argtypes = [vp, fp, fp]
        L.music_b200_get_focusing.restype = ctypes.c_int
        L.music_b200_process_channels_device.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp, vp]
        L.music_b200_process_channels_device.restype = ctypes.c_int
        L.music_b200_process_channels_host.argtypes = [vp, fp, u32, fp, fp, fp, fp, fp, fp]
        L.music_b200_process_channels_host.restype = ctypes.c_int
        L.music_b200_create_coarray.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, fp, fp, dbl, u32, ctypes.c_int]
        L.music_b200_create_coarray.restype = ctypes.c_int
        L.music_b200_set_geometry_coarray.argtypes = [vp, fp, dbl]
        L.music_b200_set_geometry_coarray.restype = ctypes.c_int
        L.music_b200_coarray_size.argtypes = [vp, ctypes.POINTER(u32)]
        L.music_b200_coarray_size.restype = ctypes.c_int
        L.music_b200_launch_count.argtypes = [vp]
        L.music_b200_launch_count.restype = ctypes.c_uint64
        L.music_b200_set_stage_timing.argtypes = [vp, ctypes.c_int]
        L.music_b200_set_stage_timing.restype = ctypes.c_int
        L.music_b200_get_stage_times.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint64)]
        L.music_b200_get_stage_times.restype = ctypes.c_int
        L.music_b200_debug_fused_trace.argtypes = [vp, ctypes.c_void_p, ctypes.c_int]
        L.music_b200_debug_fused_trace.restype = ctypes.c_int
        L.music_b200_debug_fused8_stats.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64)]
        L.music_b200_debug_fused8_stats.restype = ctypes.c_int
        L.music_b200_last_error.argtypes = [vp]
        L.music_b200_last_error.restype = ctypes.c_char_p
        L.music_b200_destroy.argtypes = [vp]
        L.music_b200_destroy.restype = None
        _lib = L
    return _lib


EXPORTS = [
    "music_b200_version", "music_b200_create", "music_b200_create_multi", "music_b200_device_count",
    "music_b200_process_device_sharded", "music_b200_gather_create", "music_b200_gather_attach", "music_b200_gather_wait",
    "music_b200_gather_buffer", "music_b200_gather_read", "music_b200_set_table", "music_b200_set_geometry", "music_b200_set_peak_mode", "music_b200_set_source_rule", "music_b200_set_refine", "music_b200_set_estimator", "music_b200_set_iaa_iterations", "music_b200_reduce_angles_device",
    "music_b200_reduce_spectrum_device", "music_b200_reduce_angles_host", "music_b200_reduce_spectrum_host",
    "music_b200_get_table", "music_b200_steer_entry_host", "music_b200_manifold_coeffs_host", "music_b200_process_host",
    "music_b200_process_device", "music_b200_process_device_ex", "music_b200_process_host_counts",
    "music_b200_process_device_counts", "music_b200_process_planar_host",
    "music_b200_process_planar_device", "music_b200_launch_count",
    "music_b200_set_stage_timing", "music_b200_get_stage_times", "music_b200_debug_fused_trace", "music_b200_debug_fused8_stats",
    "music_b200_last_error", "music_b200_destroy",
    "music_b200_create_azel", "music_b200_set_geometry_azel", "music_b200_process_azel_host", "music_b200_process_azel_device",
    "music_b200_azel_lattice_host",
    "music_b200_set_beamformer", "music_b200_process_device_beams", "music_b200_process_host_beams",
    "music_b200_set_calibration", "music_b200_get_calibration", "music_b200_calib_reset", "music_b200_calib_accumulate_device",
    "music_b200_calib_accumulate_host", "music_b200_calib_solve", "music_b200_calib_blind_reset", "music_b200_calib_blind_accumulate_device",
    "music_b200_calib_blind_accumulate_host", "music_b200_calib_blind_solve", "music_b200_set_integration", "music_b200_reset_integration",
    "music_b200_process_device_crb", "music_b200_process_host_crb", "music_b200_process_azel_device_crb",
    "music_b200_process_azel_host_crb", "music_b200_set_tracking", "music_b200_reset_tracks", "music_b200_get_tracks",
    "music_b200_process_device_tracks", "music_b200_process_host_tracks", "music_b200_process_azel_device_tracks",
    "music_b200_process_azel_host_tracks",
    "music_b200_create_channels", "music_b200_set_geometry_channels", "music_b200_channel_frequencies",
    "music_b200_get_table_channel", "music_b200_process_channels_device", "music_b200_process_channels_host",
    "music_b200_set_focusing", "music_b200_get_focusing",
    "music_b200_create_coarray", "music_b200_set_geometry_coarray", "music_b200_coarray_size",
]


def check(rc, handle=None):
    if rc != OK:
        msg = load().music_b200_last_error(handle)
        raise MusicB200Error(rc, msg.decode() if msg else "?")
