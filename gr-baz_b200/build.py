"""In-tree build of the sm_90a (H100) CUDA library (libmusic_b200.so) with nvcc.

nvcc cross-compiles without a GPU; the built .so sits next to the sources
(gr-baz_b200/csrc/), where the package loads it from.
"""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libmusic_b200.so")
SOURCES = ["music_b200.cu"]
DEPS = ["music_b200.cu", "music_kernels.cuh", "music_fused.cuh", "music_eig4p.cuh", "music_covn.cuh", "music_fused8.cuh", "music_steer.cuh", "music_planar.cuh", "music_reduce.cuh", "music_sources.cuh", "music_refine.cuh", "music_azel.cuh", "music_estimators.cuh", "music_warp_la.cuh", "music_roots.cuh", "music_manifold.cuh", "music_esprit.cuh", "music_esprit2d.cuh", "music_dml.cuh", "music_wsf.cuh", "music_iaa.cuh", "music_beams.cuh", "music_calib.cuh", "music_calib_blind.cuh", "music_integrate.cuh", "music_crb.cuh", "music_track.cuh", "music_channels.cuh", "music_focus.cuh", "music_coarray.cuh", os.path.join("..", "..", "include", "music_b200.h")]

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "-ldl",
]


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found; the CUDA library cannot be built")
    return p


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


def build_cuda(force: bool = False, verbose: bool = False) -> str:
    if force or needs_build():
        cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + SOURCES
        subprocess.check_call(cmd, cwd=CSRC)
    return LIB


if __name__ == "__main__":
    print(build_cuda(force=True, verbose=True))
