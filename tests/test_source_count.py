"""CPU tests of the per-window source count (MDL / AIC, music_b200_set_source_rule): the definition in
tests/source_count_oracle.py on a hand-computed case and on seeded synthetic windows, noise-only synthetic streams, and
the C++ block's new entry point."""
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from gr_baz_b200 import build, synth
from oracle import c_oracle as co
from oracle import music_oracle as mo

import source_count_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(m, N) for m in (4, 5, 8, 12, 16) for N in (256, 4096)]
SEED = 100


def eigvals_of(x, m):
    return np.linalg.eigvalsh(mo.covariance(x, m))


def test_hand_computed_case():
    """l = (1, 1, 1, 10), N = 100, M = 4: L(0) = 100 (4 log(13/4) - log 10), L(d >= 1) = 0"""
    lam, N, M = [1.0, 1.0, 1.0, 10.0], 100, 4
    L0 = 100.0 * (4.0 * math.log(13.0 / 4.0) - math.log(10.0))
    mdl = [L0, 0.5 * 7 * math.log(100.0), 0.5 * 12 * math.log(100.0), 0.5 * 15 * math.log(100.0)]
    aic = [2.0 * L0, 14.0, 24.0, 30.0]
    d, c = so.estimate_source_count(lam, N, 3, "mdl")
    assert d == 1 and np.allclose(c, mdl, rtol=1e-15, atol=1e-12)
    d, c = so.estimate_source_count(lam, N, 3, "aic")
    assert d == 1 and np.allclose(c, aic, rtol=1e-15, atol=1e-12)
    # n_max caps the search: with n_max = 0 only d = 0 is a candidate
    assert so.estimate_source_count(lam, N, 0, "mdl")[0] == 0
    assert abs(L0 - 241.2035) < 1e-3


def test_ties_go_to_the_smaller_count_and_bad_windows_to_zero():
    # all eigenvalues equal: L(d) = 0 for every d, AIC / MDL grow with d -> 0; equal criteria -> smallest d
    assert so.estimate_source_count([2.0] * 6, 50, 5, "aic")[0] == 0
    assert so.estimate_source_count([0.0, 1.0, 2.0, 3.0], 50, 3, "mdl")[0] == 0  # l_0 <= 0
    assert so.estimate_source_count([-1e-30, 1.0, 2.0, 3.0], 50, 3, "mdl")[0] == 0
    assert so.estimate_source_count([1.0, np.nan, 2.0, 3.0], 50, 3, "mdl")[0] == 0
    assert so.estimate_source_count([1.0, 2.0, 3.0, np.inf], 50, 3, "aic")[0] == 0


def test_aic_never_below_mdl():
    """AIC's penalty per parameter (2) is below MDL's (log N) whenever log N > 2, so d_AIC >= d_MDL"""
    rng = np.random.default_rng(2026)
    for trial in range(200):
        m = int(rng.integers(3, 17))
        N = int(rng.choice([16, 33, 64, 256, 1024]))
        if N <= m:
            continue
        n_max = int(rng.integers(1, m))
        x = rng.standard_normal((N, m)) + 1j * rng.standard_normal((N, m))
        for _ in range(int(rng.integers(0, m))):
            a = np.exp(2j * np.pi * rng.uniform(size=m))
            x += rng.uniform(0.1, 3.0) * a[None, :] * (rng.standard_normal((N, 1)) + 1j * rng.standard_normal((N, 1)))
        ev = eigvals_of(x.reshape(-1).astype(np.complex64), m)
        assert math.log(N) > 2
        assert so.estimate_source_count(ev, N, n_max, "aic")[0] >= so.estimate_source_count(ev, N, n_max, "mdl")[0], trial


def test_mdl_is_zero_on_noise_only_windows():
    hits = total = 0
    for m, N in SHAPES:
        cfg = synth.config(4, m=m, n=0, snapshots=N, resolution=360, geometry="uca")
        x = synth.gen_windows_numpy(cfg, 4242 + m, 0, 20)
        for w in range(len(x)):
            hits += so.estimate_source_count(eigvals_of(x[w], m), N, m - 1, "mdl")[0] == 0
            total += 1
    assert hits >= 0.95 * total, (hits, total)


def test_mdl_finds_the_true_count_on_the_mixed_sets():
    """every window at N = 4096; the hit rate at N = 256 is reported (it is what the criterion gives, not a gate)"""
    rates = {}
    for m, N in SHAPES:
        _, x, truth = so.mixed_windows(m, N, 360, SEED + m)
        d = np.array([so.estimate_source_count(eigvals_of(x[w], m), N, 3, "mdl")[0] for w in range(len(x))])
        rates[(m, N)] = float(np.mean(d == truth))
        if N == 4096:
            assert np.array_equal(d, truth), (m, d, truth)
    print("MDL hit rate at N = 256:", {m: rates[(m, 256)] for m, N in SHAPES if N == 256})
    assert min(rates[(m, 256)] for m, N in SHAPES if N == 256) >= 0.75


def test_jacobi_and_lapack_eigenvalues_give_the_same_count():
    for m, N in SHAPES:
        _, x, _ = so.mixed_windows(m, N, 360, SEED + m)
        for w in range(len(x)):
            R = mo.covariance(x[w], m)
            lj = np.sort(co.herm_eig(R)[0])
            ll = np.linalg.eigvalsh(R)
            for rule in so.RULES:
                assert so.estimate_source_count(lj, N, 3, rule)[0] == so.estimate_source_count(ll, N, 3, rule)[0], (m, N, w, rule)


def test_noise_only_synth_streams():
    """n = 0 generates noise-only windows, identically on the host and with torch"""
    cfg = synth.config(4, n=0, snapshots=64)
    ang, rot = synth.window_params(cfg, 9, 0, 5)
    assert ang.shape == (5, 0) and rot.shape[:2] == (5, 0)
    x = synth.gen_windows_numpy(cfg, 9, 0, 5)
    y = synth.gen_windows_torch(cfg, 9, 0, 5, torch.device("cpu"))
    assert np.array_equal(y.numpy().view(np.complex64), x)
    # same noise as a one-source stream of the same seed, without the source
    x1 = synth.gen_windows_numpy(synth.config(4, n=1, snapshots=64), 9, 0, 5)
    assert not np.array_equal(x, x1) and np.std(x) < np.std(x1)


def test_cpp_block_exports_set_source_rule():
    build.build_cuda()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "lib"), "-s"])
    so_path = os.path.join(ROOT, "lib", "_build", "libgnuradio-baz-music.so")
    out = subprocess.check_output(["nm", "-DC", so_path], text=True)
    assert "baz_music_doa::set_source_rule(int)" in out
    undefined = subprocess.check_output(["nm", "-D", "--undefined-only", so_path], text=True)
    assert "music_b200_process_host_counts" in undefined and "music_b200_set_source_rule" in undefined
    assert "void set_source_rule(int rule);" in open(os.path.join(ROOT, "swig", "baz_music_doa.i")).read()
