"""Deterministic synthetic multi-antenna stream for the MUSIC DOA path (SURVEY.md section 8d).

Produces the block's input item layout - one vector of ``nsamples = M*N`` complex64 per
window, antennas sample-interleaved (``x(r, c) = in[c*M + r]``,
/root/reference/lib/baz_music_doa.cc:82-84) - from a counter-based integer hash, so any
window can be regenerated independently on the host (numpy) or on the device (torch) and
the two are BIT-IDENTICAL: every floating-point step is a single correctly rounded
fp32 operation (int->float, one multiply, adds) and no transcendental is evaluated on the
device (per-window steering phasors are computed on the host in fp64 and uploaded).

Signal model (helper's sign convention, /root/reference/python/music_doa_helper.py:40-41):
    x[:, c] = sum_s amp * a(phi_s) * sym_s[c] + noise[:, c]
    a(phi)[ant] = exp(-j 2 pi <p_ant, u(phi)> / lambda),  sym in {1, j, -1, -j},
    noise = Irwin-Hall(4 bytes) per component scaled to the requested SNR.
"""
from __future__ import annotations

import math

import numpy as np

C_LIGHT = 299792458.0
FREQUENCY = 299792458.0  # lambda = 1 m
SPACING = 0.5  # lambda / 2
M32 = 0xFFFFFFFF
BASE_SEED = 0x62617A00  # "baz\0"

# BASELINE.json configs (SURVEY.md section 8): (M, snapshots N, angles K, sources n)
CONFIGS = {
    1: dict(m=4, snapshots=1024, resolution=360, n=1, geometry="ula_x", windows=1),
    2: dict(m=4, snapshots=4096, resolution=3600, n=1, geometry="ula_x", windows=10000),
    3: dict(m=8, snapshots=8192, resolution=7200, n=1, geometry="uca", windows=100000),
    4: dict(m=8, snapshots=4096, resolution=3600, n=1, geometry="uca", windows=1000000),
    5: dict(m=16, snapshots=4096, resolution=3600, n=2, geometry="uca", windows=1000000,
            fixed_sources=(15.0, 345.0)),
}


def config(cfg_id: int, **over):
    c = dict(CONFIGS[cfg_id])
    c["id"] = cfg_id
    c["snr_db"] = 20.0
    c.update(over)
    c["nsamples"] = c["m"] * c["snapshots"]
    c["antenna_array"] = antenna_array(c["geometry"], c["m"])
    return c


def antenna_array(geometry: str, m: int):
    """Element coordinates in units of ``array_spacing`` (what the GRC 'Array' parameter
    holds, /root/reference/grc/baz_music_doa.xml:55)."""
    if geometry == "ula_x":
        return [[float(i), 0.0] for i in range(m)]
    if geometry == "ula_y":
        return [[0.0, float(i)] for i in range(m)]
    if geometry == "uca":
        # radius such that adjacent elements are one spacing unit apart
        r = 0.5 / math.sin(math.pi / m)
        return [[r * math.cos(2 * math.pi * i / m), r * math.sin(2 * math.pi * i / m)] for i in range(m)]
    raise ValueError(geometry)


def steering(antenna_array_units, phi_deg, spacing=SPACING, frequency=FREQUENCY):
    """a(phi) in fp64/complex128 for angles phi_deg (any shape) -> (..., M)."""
    lam = C_LIGHT / frequency
    pos = np.asarray(antenna_array_units, dtype=np.float64) * spacing  # (M, 2)
    phi = np.deg2rad(np.asarray(phi_deg, dtype=np.float64))[..., None]
    proj = pos[:, 0] * np.cos(phi) + pos[:, 1] * np.sin(phi)
    return np.exp(-1j * 2.0 * np.pi * proj / lam)


# ---- 32-bit integer hash evaluated in int64 (identical in numpy and torch) -------------
def _h32(x):
    """lowbias-style mixer; x holds values in [0, 2^32) stored as int64.  Multipliers are
    < 2^27 so products stay below 2^63 (no int64 overflow, shifts are on non-negatives)."""
    x = ((x >> 16) ^ x) * 0x45D9F3B & M32
    x = ((x >> 16) ^ x) * 0x45D9F3B & M32
    x = (x >> 16) ^ x
    return x


def _h32_int(x: int) -> int:
    x = ((x >> 16) ^ x) * 0x45D9F3B & M32
    x = ((x >> 16) ^ x) * 0x45D9F3B & M32
    return (x >> 16) ^ x


def _window_keys(seed: int, w):
    """Per-window stream keys from window indices w (numpy int64 array)."""
    s = _h32_int(seed & M32)
    k_noise = _h32((w & M32) ^ s)
    k_sym = _h32(k_noise ^ 0x5BD1E995)
    k_ang = _h32(k_noise ^ 0x2545F491)
    return k_noise, k_sym, k_ang


_FRACS = np.array([0.1, 0.15, 0.2, 0.25, 0.3, 0.35, 0.4, 0.6, 0.65, 0.7, 0.75, 0.8, 0.85, 0.9])


def _windex(w0, W, indices):
    if indices is not None:
        return np.asarray(indices, dtype=np.int64)
    return np.arange(w0, w0 + W, dtype=np.int64)


def window_params(cfg, seed: int, w0: int = 0, W: int = 0, indices=None):
    """Host-side (numpy) per-window parameters: true source angles in degrees (W, S) and
    the fp32 rotated-phasor table rot[w, ant, sym, comp] = (amp * a_s(phi) * j^sym).
    Windows are w0..w0+W-1, or the explicit global window numbers in ``indices``."""
    w = _windex(w0, W, indices)
    _, _, k_ang = _window_keys(seed, w)
    K = cfg["resolution"]
    h1 = _h32(k_ang)
    h2 = _h32(k_ang ^ 0x68E31DA4)
    frac = _FRACS[(h2 % len(_FRACS))]
    if cfg.get("fixed_sources"):
        dbin = (h1 % 41) - 20
        jitter = (dbin + frac) * 360.0 / K
        ang = np.stack([(b + jitter) % 360.0 for b in cfg["fixed_sources"]], axis=1)
    else:
        S = cfg["n"]
        cols = []
        for s in range(S):
            hb = _h32(h1 ^ (0x9E3779B1 * (s + 1) & M32))
            cols.append(((hb % K) + frac) * 360.0 / K)
        ang = np.stack(cols, axis=1) if S else np.zeros((len(w), 0))  # n = 0: noise-only windows
    a = steering(cfg["antenna_array"], ang)  # (W, S, M) c128, unit power per source
    jpow = np.array([1, 1j, -1, -1j], dtype=np.complex128)
    rot = a[..., None] * jpow  # (W, S, M, 4)
    rot32 = np.stack([rot.real, rot.imag], axis=-1).astype(np.float32)  # (W, S, M, 4, 2)
    return ang, rot32


def _noise_scale(cfg) -> np.float32:
    sigma2 = 10.0 ** (-cfg["snr_db"] / 10.0)  # total complex noise power, signal power 1
    ih_std = math.sqrt(4.0 * (256.0 ** 2 - 1.0) / 12.0)
    return np.float32(math.sqrt(sigma2 / 2.0) / ih_std)


def gen_windows_numpy(cfg, seed: int, w0: int = 0, W: int = 0, indices=None):
    """(W, nsamples) complex64, host reference generator."""
    M, N = cfg["m"], cfg["snapshots"]
    w = _windex(w0, W, indices)
    W = len(w)
    _, rot32 = window_params(cfg, seed, indices=w)
    S = rot32.shape[1]
    k_noise, k_sym, _ = _window_keys(seed, w)
    idx = np.arange(N * M * 2, dtype=np.int64)
    hn = _h32((k_noise[:, None] + idx[None, :]) & M32)
    u = (hn & 255) + ((hn >> 8) & 255) + ((hn >> 16) & 255) + ((hn >> 24) & 255) - 510
    x = u.astype(np.float32) * _noise_scale(cfg)  # (W, N*M*2)
    x = x.reshape(W, N, M, 2)
    cidx = np.arange(N, dtype=np.int64)
    sig = None
    for s in range(S):
        hs = _h32((k_sym[:, None] + (cidx[None, :] * S + s)) & M32)
        sym = (hs >> 13) & 3  # (W, N)
        rs = np.ascontiguousarray(rot32[:, s].transpose(0, 2, 1, 3))  # (W, 4, M, 2)
        term = rs[np.arange(W)[:, None], sym]  # (W, N, M, 2)
        sig = term if sig is None else sig + term
    if sig is not None:
        x = sig + x
    return np.ascontiguousarray(x.reshape(W, N * M * 2)).view(np.complex64)


def gen_windows_torch(cfg, seed: int, w0: int, W: int, device, out=None, chunk: int = 64, indices=None):
    """Same stream generated with torch ops on ``device``; returns float32 (W, nsamples*2)
    (interleaved re, im).  Bit-identical to gen_windows_numpy (tests/test_synth.py)."""
    import torch

    M, N = cfg["m"], cfg["snapshots"]
    wall = _windex(w0, W, indices)
    W = len(wall)
    if out is None:
        out = torch.empty((W, N * M * 2), dtype=torch.float32, device=device)
    scale = torch.tensor(float(_noise_scale(cfg)), dtype=torch.float32, device=device)
    idx = torch.arange(N * M * 2, dtype=torch.int64, device=device)
    cidx = torch.arange(N, dtype=torch.int64, device=device)
    for c0 in range(0, W, chunk):
        cw = min(chunk, W - c0)
        w = wall[c0 : c0 + cw]
        _, rot32 = window_params(cfg, seed, indices=w)
        S = rot32.shape[1]
        k_noise, k_sym, _ = _window_keys(seed, w)
        k_noise = torch.from_numpy(k_noise).to(device)
        k_sym = torch.from_numpy(k_sym).to(device)
        rot = torch.from_numpy(rot32).to(device)  # (cw, S, M, 4, 2)
        hn = _h32((k_noise[:, None] + idx[None, :]) & M32)
        u = (hn & 255) + ((hn >> 8) & 255) + ((hn >> 16) & 255) + ((hn >> 24) & 255) - 510
        x = u.to(torch.float32) * scale
        x = x.reshape(cw, N, M, 2)
        ar = torch.arange(cw, device=device)[:, None]
        sig = None
        for s in range(S):
            hs = _h32((k_sym[:, None] + (cidx[None, :] * S + s)) & M32)
            sym = (hs >> 13) & 3
            rs = rot[:, s].permute(0, 2, 1, 3).contiguous()  # (cw, 4, M, 2)
            term = rs[ar, sym]  # (cw, N, M, 2)
            sig = term if sig is None else sig + term
        if sig is not None:
            x = sig + x
        out[c0 : c0 + cw] = x.reshape(cw, N * M * 2)
    return out


def true_bins(cfg, seed: int, w0: int = 0, W: int = 0, indices=None):
    """Nearest grid bin of each true source angle (diagnostic; the parity gate is the
    oracle's bins, not these)."""
    ang, _ = window_params(cfg, seed, w0, W, indices)
    K = cfg["resolution"]
    return np.rint(ang * K / 360.0).astype(np.int64) % K
