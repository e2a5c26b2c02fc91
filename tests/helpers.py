"""Shared helpers for the test-suite (oracle-side: allowed to import oracle/)."""
import glob
import hashlib
import os
import re

import numpy as np

from gr_baz_b200 import synth
from oracle import music_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

_table_cache = {}


def table_for(cfg):
    key = (cfg["geometry"], cfg["m"], cfg["resolution"])
    if key not in _table_cache:
        arr = mo.scaled_antenna_array(synth.SPACING, cfg["antenna_array"])
        _table_cache[key] = mo.steering_table_c64(arr, cfg["resolution"], synth.C_LIGHT / synth.FREQUENCY)
    return _table_cache[key]


def golden_files():
    return sorted(glob.glob(os.path.join(GOLDEN, "*.npz")))


def load_golden(path):
    """Returns (cfg, seed, table, list of per-window dicts incl. regenerated input)."""
    g = np.load(path)
    cfg = synth.config(int(g["base"]), m=int(g["m"]), n=int(g["n"]), snapshots=int(g["snapshots"]),
                       resolution=int(g["resolution"]), geometry=str(g["geometry"]), snr_db=float(g["snr_db"]))
    seed = int(g["seed"])
    table = g["table"] if "table" in g.files else table_for(cfg)
    wins = []
    for i, w in enumerate(g["windows"]):
        x = g["in_%d" % i] if ("in_%d" % i) in g.files else synth.gen_windows_numpy(cfg, seed, int(w), 1)[0]
        d = {k: g["%s_%d" % (k, i)] for k in ("R", "eigvals", "noise_projector", "P", "spectrum", "bins", "angles", "levels")}
        d["in"] = x
        d["in_sha256"] = str(g["in_sha256_%d" % i])
        d["w"] = int(w)
        wins.append(d)
    return cfg, seed, table, wins, str(g["table_sha256"])


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b) / np.abs(b)))


def grc_signature(root):
    """What a flowgraph depends on in a GRC block descriptor (xml.etree root): key, import, make, callback, params, ports."""
    return [root.findtext("key"), root.findtext("import"), root.findtext("make"), root.findtext("callback"),
            [[p.findtext("key"), p.findtext("value"), p.findtext("type")] for p in root.findall("param")],
            [[s.findtext("name"), s.findtext("type"), s.findtext("vlen")] for s in root.findall("sink")],
            [[s.findtext("name"), s.findtext("type"), s.findtext("vlen"), s.findtext("optional")] for s in root.findall("source")]]


def normalized_declarations(text):
    """C++ source without comments, whitespace collapsed and removed around & * ( ) , - for substring checks."""
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    return re.sub(r"\s*([&*(),])\s*", r"\1", re.sub(r"\s+", " ", text))


# the C++ surface of lib/baz_music_doa.h a gr-baz user compiles against
CPP_SURFACE = [
    "class baz_music_doa : public gr::sync_block",
    "typedef boost::shared_ptr<baz_music_doa> baz_music_doa_sptr;",
    "typedef std::vector<gr_complex> antenna_response_t;",
    "typedef std::vector<antenna_response_t> array_response_t;",
    "baz_music_doa_sptr baz_make_music_doa(unsigned int m, unsigned int n, unsigned int nsamples, const array_response_t& array_response, unsigned int resolution);",
    "int work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items);",
    "void set_array_response(const array_response_t& array_response);",
]
# gr-baz's grc/baz_music_doa.xml signature and the CPP_SURFACE lines its lib/baz_music_doa.h declares
REFERENCE_INTERFACE = os.path.join(GOLDEN, "reference", "interface.json")


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---- outputs of the reference's own work() (tests/golden/reference/work.npz) ---------------------------------------
# lib/baz_music_doa.cc of gr-baz, compiled unmodified against stand-in GNU Radio / Armadillo headers (oracle/Makefile
# target `ref`) and run on the inputs below; tests/golden/reference/make_reference_golden.py regenerates the file.  Angles and
# levels are stored in full, each spectrum at the columns listed in "bins" (a seeded sample plus every window's top bins
# and their neighbours).
REFERENCE_GOLDEN = os.path.join(GOLDEN, "reference", "work.npz")

# (base config, overrides, windows) of tests/test_ref_shim.py: the oracles against the reference on seeded windows
ORACLE_CASES = [
    (1, {}, 12), (1, {"n": 2}, 8), (1, {"n": 3}, 8), (1, {"geometry": "ula_y"}, 6),
    (2, {"snapshots": 512}, 6), (4, {"snapshots": 256, "n": 3}, 5), (5, {"snapshots": 256, "resolution": 720}, 4),
    (1, {"m": 6, "geometry": "uca", "n": 2}, 5),
]
ORACLE_SEED = 2024
# tests/test_gpu_zz_reference_source.py: the CUDA path against it, incl. the BASELINE shapes at full size (configs[1..4]:
# C2 4x4096x3600, C3 8x8192x7200, C4 8x4096x3600, C5 16x4096x3600 n=2)
GPU_CASES = [
    (1, {}, 24), (1, {"n": 2}, 12), (2, {"snapshots": 1024}, 12), (4, {"snapshots": 512}, 10),
    (5, {"snapshots": 512, "resolution": 1800}, 8), (1, {"m": 6, "geometry": "uca", "n": 2}, 8),
    (2, {}, 16), (3, {}, 8), (4, {}, 8), (5, {}, 8),
]
GPU_SEED = 606
MIRROR_CASE = (1, {"n": 2}, 10, 77)  # base, overrides, windows, seed of the mirror-tie test


def case_key(kind, i):
    return "%s%d" % (kind, i)


def case_windows(base, over, W, seed):
    cfg = synth.config(base, **over)
    return cfg, table_for(cfg), synth.gen_windows_numpy(cfg, seed + base, 0, W)


def random_small_shapes():
    """The sweep of small shapes of tests/test_ref_shim.py (m 2..9, every valid n, odd grids, single-snapshot windows,
    strong / weak / no signal): yields (trial, m, n, snaps, K, table, x)."""
    rng = np.random.default_rng(20260922)
    for trial in range(60):
        m = int(rng.integers(2, 10))
        n = int(rng.integers(1, m))
        snaps = int(rng.choice([1, 2, 3, 7, 16, 33, 64]))
        K = int(rng.choice([7, 12, 45, 90, 360, 721]))
        W = 3
        pos = rng.uniform(-1.5, 1.5, (m, 2))
        lam = float(rng.uniform(0.5, 2.0))
        table = mo.steering_table_c64(pos.tolist(), K, lam)
        kind = trial % 3
        x = (rng.standard_normal((W, snaps, m)) + 1j * rng.standard_normal((W, snaps, m))) * (1.0 if kind else 1e-3)
        if kind == 1:  # plus sources on grid rows
            for w in range(W):
                for s in range(n):
                    a = table[int(rng.integers(0, K))].astype(np.complex128)
                    x[w] += 5.0 * a[None, :] * (rng.standard_normal((snaps, 1)) + 1j * rng.standard_normal((snaps, 1)))
        yield trial, m, n, snaps, K, table, x.reshape(W, snaps * m).astype(np.complex64)


def random_wide_shapes():
    """The same kind of sweep for the wide arrays (m 10..16, every n from 1 to m - 1, snapshots 16 / 33 / 64 / 256,
    strong / weak / no signal): yields (trial, m, n, snaps, K, table, x)."""
    rng = np.random.default_rng(20261015)
    trial = 0
    for m in range(10, 17):
        for n in range(1, m):
            snaps = int(rng.choice([16, 33, 64, 256]))
            K = int(rng.choice([7, 12, 45, 90, 360, 721]))
            W = 3
            pos = rng.uniform(-1.5, 1.5, (m, 2))
            lam = float(rng.uniform(0.5, 2.0))
            table = mo.steering_table_c64(pos.tolist(), K, lam)
            kind = trial % 3
            x = (rng.standard_normal((W, snaps, m)) + 1j * rng.standard_normal((W, snaps, m))) * (1.0 if kind else 1e-3)
            if kind == 1:  # plus sources on grid rows
                for w in range(W):
                    for s in range(n):
                        a = table[int(rng.integers(0, K))].astype(np.complex128)
                        x[w] += 5.0 * a[None, :] * (rng.standard_normal((snaps, 1)) + 1j * rng.standard_normal((snaps, 1)))
            yield trial, m, n, snaps, K, table, x.reshape(W, snaps * m).astype(np.complex64)
            trial += 1


def assert_bins_equal_up_to_exact_ties(got, ref):
    """Bit-exact bins, except where the oracle itself sees a tie inside fp64 noise.  On the x-axis ULA the broadside
    mirror pair (90 / 270 degrees) has table rows that differ only in imaginary parts of ~1e-16, so P at the two
    bins agrees to ~1e-14; P is conditioned ~4000x w.r.t. R (DESIGN.md section 3), i.e. any fp64 implementation
    (the reference's LAPACK path included) carries ~1e-12 of rounding noise in P, and which of the two bins wins
    depends on the summation order of R.  Seen when a source sits at broadside or a window straddles two sources."""
    bad = np.nonzero(np.any(got != ref["bins"], axis=1))[0]
    assert len(bad) <= 0.01 * len(got)
    for w in bad:
        P = ref["P"][w]
        for g, r in zip(got[w], ref["bins"][w]):
            assert abs(P[g] - P[r]) <= 1e-12 * P[r], (w, g, r, P[g], P[r])
    return len(bad)


# ---- arbitrary array-response tables (set_array_response): tests/test_gpu_tables.py, tests/test_ref_tables.py --------
def planar_table(m, K, seed):
    """[K][m] complex64 steering table of a random planar array (positions in wavelengths), theta_k = k * 360 / K"""
    pos = np.random.default_rng(seed).uniform(-1.5, 1.5, (m, 2))
    th = np.arange(K) * (2.0 * np.pi / K)
    return np.exp(-2j * np.pi * (np.outer(np.cos(th), pos[:, 0]) + np.outer(np.sin(th), pos[:, 1]))).astype(np.complex64)


def calibrated_table(table, seed):
    """a geometric table as a calibration would leave it: a fixed gain (0.5 .. 2) and phase error per element, a
    power-of-two factor 2^j per row (j in [-20, 20]) and a small complex perturbation of every entry"""
    rng = np.random.default_rng(seed)
    K, m = table.shape
    gain = rng.uniform(0.5, 2.0, m) * np.exp(1j * rng.uniform(-0.3, 0.3, m))
    row = 2.0 ** rng.integers(-20, 21, K)
    eps = 1e-3 * (rng.standard_normal((K, m)) + 1j * rng.standard_normal((K, m)))
    return ((table.astype(np.complex128) * gain[None, :] + eps) * row[:, None]).astype(np.complex64)


def random_table(m, K, seed):
    """i.i.d. complex Gaussian rows: a spectrum with a local maximum at about every third bin"""
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal((K, m)) + 1j * rng.standard_normal((K, m))) / np.sqrt(2.0)).astype(np.complex64)


def source_windows(rng, vectors, m, N, amp=5.0):
    """one window per entry of `vectors` (each None or a list of complex (m,) source directions): unit complex noise
    plus sources of amplitude `amp` along the directions, each normalised to ||a||^2 = m; (W, N * m) complex64"""
    W = len(vectors)
    x = (rng.standard_normal((W, N, m)) + 1j * rng.standard_normal((W, N, m))) / np.sqrt(2.0)
    for w, vs in enumerate(vectors):
        for a in vs or []:
            a = np.asarray(a, np.complex128)
            a = a * np.sqrt(m) / np.linalg.norm(a)
            x[w] += amp * a[None, :] * (rng.standard_normal((N, 1)) + 1j * rng.standard_normal((N, 1)))
    return x.reshape(W, N * m).astype(np.complex64)


# reference outputs on these tables: tests/golden/reference/tables.npz (make_reference_tables_golden.py)
REFERENCE_TABLES = os.path.join(GOLDEN, "reference", "tables.npz")
TABLE_ZERO_ROWS = (5, 200, 201)
TABLE_DUPLICATES = ((37, 100), (0, 399))  # (row copied, row overwritten)


def table_golden_cases():
    """(key, m, n, table, x) of the small batches stored with the reference's outputs: M = 4, K = 400, tables scaled by
    2^63 and 2^-70, calibrated, with duplicated rows (a strong source along the duplicated row) and with zero rows"""
    m, K, N, W = 4, 400, 64, 4
    base = planar_table(m, K, 4040)
    rng = np.random.default_rng(4041)
    dup = base.copy()
    for src, dst in TABLE_DUPLICATES:
        dup[dst] = dup[src]
    zero = base.copy()
    zero[list(TABLE_ZERO_ROWS)] = 0
    tables = {"scaled63": (base.astype(np.complex128) * 2.0 ** 63).astype(np.complex64),
              "scaled-70": (base.astype(np.complex128) * 2.0 ** -70).astype(np.complex64),
              "calibrated": calibrated_table(base, 4042), "duplicate": dup, "zero": zero}
    for name, t in tables.items():
        srcs = [[t[37]], [t[37], t[250]], [t[0]], None] if name == "duplicate" else \
               [[base[int(k)]] for k in rng.integers(0, K, W - 1)] + [None]
        x = source_windows(rng, srcs, m, N, amp=20.0 if name == "duplicate" else 5.0)
        for n in (1, 2):
            yield "%s_n%d" % (name, n), m, n, t, x


def table_reference_outputs(key, x, table):
    """the reference's angles, levels and full spectrum of table_golden_cases() entry `key`, after checking that x and
    the table are the ones it was computed from"""
    g = np.load(REFERENCE_TABLES)
    assert str(g[key + "/in_sha256"]) == sha256(x), key
    assert str(g[key + "/table_sha256"]) == sha256(table), key
    return {f: g[key + "/" + f] for f in ("angles", "levels", "spectrum")}


def assert_float32_close(got, ref, rtol, ctx):
    """non-finite values (NaN included) and zeros bit-equal, the rest within rtol"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    exact = ~np.isfinite(ref) | (ref == 0)
    assert np.array_equal(got[exact], ref[exact], equal_nan=True), ctx
    if np.any(~exact):
        assert rel_err(got[~exact], ref[~exact]) <= rtol, ctx


_reference_golden = None


def reference_outputs(key, x=None):
    """The reference's angles, levels and sampled spectrum ("spectrum" at the columns "bins") stored under `key`, and
    whether all its levels and spectrum values were finite; with `x`, first checks that these are the inputs they were
    computed from."""
    global _reference_golden
    if _reference_golden is None:
        g = np.load(REFERENCE_GOLDEN)
        shape = g["shape"]
        offs = {f: np.concatenate([[0], np.cumsum(size)]) for f, size in (
            ("angles", shape[:, 0] * shape[:, 1]), ("spectrum", shape[:, 0] * shape[:, 2]), ("bins", shape[:, 2]))}
        _reference_golden = {}
        for i, k in enumerate(g["keys"]):
            W, n, c = (int(v) for v in shape[i])
            a0, s0, b0 = offs["angles"][i], offs["spectrum"][i], offs["bins"][i]
            _reference_golden[str(k)] = {
                "in_sha256": str(g["in_sha256"][i]), "finite": bool(g["finite"][i]),
                "angles": g["angles"][a0:a0 + W * n].reshape(W, n), "levels": g["levels"][a0:a0 + W * n].reshape(W, n),
                "spectrum": g["spectrum"][s0:s0 + W * c].reshape(W, c), "bins": g["bins"][b0:b0 + c]}
    ref = _reference_golden[key]
    if x is not None:
        assert sha256(x) == ref["in_sha256"], "%s: the inputs differ from those the reference was run on" % key
    return ref
