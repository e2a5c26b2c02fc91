"""GPU: every Hermitian eigensolver path against the mpmath reference of tests/eig_oracle.py on adversarial spectra.

Unfused rows (eig_kernel<4, true>, eig_kernel<8, false>, eig_kernel<MAXM, false>, eig_coop_kernel<8 / 12 / 16>) read d_R,
d_eigvals and d_P64 on the probe table (rows e_i, e_i + e_j, e_i + i e_j), rebuild the GPU's noise projector from
1 / P64 and hold the eigenvalues and the projector to the bounds of eig_oracle (projector only where its bound is below
PROJ_CHECKED; those skipped are counted and reported).  Exact diagonal windows must give the sorted diagonal and the
exact projector bit for bit, and exact windows scaled by 2^-140 / 2^96 the same P64 bits.  The launch count of each call
proves which branch ran.

Fused rows (eig4_principal_coop and herm_eig4_coop at M = 4, eig8_principal_warp and eig_coop_warp at M = 8) run one
window per call on a table built for that window's R (taken from the unfused path, which the fused Jacobi matches bit for
bit): probe rows and sensitive rows a = u + eta v, on which an eigenvector error delta moves the float32 strength by
~2 delta / eta.  They assert that the inputs drive each principal solver both to its answer and to its Jacobi fallback.
The channel handle runs the same unfused eigensolvers over its pseudo-windows and is not repeated here."""
import numpy as np
import pytest

import eig_oracle as eo
import gpu_harness as gh

pytestmark = pytest.mark.gpu

N = eo.EXACT_N

# path, M, base launches of an unfused call with P64 + R + eigenvalues (covariance + eig + scan; + 1 top-n for n >= 2)
UNFUSED = [
    ("eig_kernel<4,true>", 4, 3),
    ("eig_kernel<8,false> M=3", 3, 3),
    ("eig_kernel<8,false> M=7", 7, 3),
    ("eig_kernel<MAXM,false> M=9", 9, 3),
    ("eig_kernel<MAXM,false> M=13", 13, 3),
    ("eig_coop_kernel<8>", 8, 3),
    ("eig_coop_kernel<12>", 12, 4),
    ("eig_coop_kernel<16>", 16, 3),
]


def windows(M, n, seed):
    """[(family, x [N][M] complex64, kind)], kind in exact / diagonal / rounded / zero / nan / inf"""
    rng = np.random.default_rng(seed)
    out = [(name, x, "exact") for name, x, _, _ in eo.exact_family(M, n, rng)]
    out += [("diagonal " + name, x, "diagonal") for name, x, _, _ in eo.exact_family(M, n, rng, diagonal=True)]
    Q = eo.unitary(M, rng)
    out += [(name, eo.spectrum_window(lam, Q, N), "rounded") for name, lam in eo.prescribed_spectra(M, n)]
    if M >= 3:
        out += [("top pair %g" % r, eo.spectrum_window(eo.top_pair_spectrum(M, r), Q, N), "rounded") for r in eo.top_pair_ratios()]
    out.append(("imaginary", eo.imaginary_window(M, N, rng), "rounded"))
    out.append(("rank one f32", eo.rank_one_window(M, N, rng), "rounded"))
    z = np.zeros((N, M), np.complex64)
    out.append(("zero", z, "zero"))
    nan = eo.spectrum_window(np.linspace(1, 2, M), Q, N)
    nan[3, M // 2] = np.nan
    out.append(("nan", nan, "nan"))
    inf = eo.spectrum_window(np.linspace(1, 2, M), Q, N)
    inf[5, 0] = np.inf
    out.append(("inf", inf, "inf"))
    return out


def unfused_call(M, n, xs, launches):
    table = eo.probe_table(M)
    blk = gh.make_block(M, n, N, table=table)
    x = np.stack([w.reshape(-1) for w in xs])
    got, nl = gh.device_call(blk, x, ("levels", "bins", "P64", "R", "eigvals"))
    blk.close()
    assert nl == launches, ("launches", nl, launches)
    for k in ("angles", "levels", "bins", "P64", "R", "eigvals"):
        assert not np.any(got[k] == gh.SENTINEL), k
    return got


@pytest.mark.parametrize("path,M,base", UNFUSED, ids=[u[0] for u in UNFUSED])
@pytest.mark.parametrize("nsel", ["n=1", "n=M/2"])
def test_unfused_eigensolver_within_bounds(path, M, base, nsel):
    n = 1 if nsel == "n=1" or M < 4 else M // 2
    launches = base + (1 if n >= 2 else 0)
    fam = windows(M, n, 7000 + 31 * M + n)
    got = unfused_call(M, n, [x for _, x, _ in fam], launches)
    worst_e, worst_p, skipped, checked = 0.0, 0.0, [], 0
    for w, (name, x, kind) in enumerate(fam):
        ctx = (path, n, name)
        R, ev, P = got["R"][w], got["eigvals"][w], got["P64"][w]
        if kind in ("nan", "inf"):
            if kind == "nan":
                assert np.all(np.isnan(P)) and got["bins"][w, 0] == -1, ctx  # NaN in -> NaN out, no peak
            continue
        if kind == "zero":
            assert np.all(ev == 0.0) and np.all(R == 0.0), ctx
            continue
        assert np.all(np.isfinite(ev)), ctx
        Pi_hat = eo.projector_from_P(P, M)
        if kind == "diagonal":
            d = np.diag(R).real
            assert np.count_nonzero(R - np.diag(d)) == 0, ctx
            order = np.argsort(d, kind="stable")
            assert np.array_equal(ev, d[order]), ctx
            Pi = np.zeros((M, M), np.complex128)
            Pi[order[:M - n], order[:M - n]] = 1.0
            assert np.array_equal(Pi_hat, Pi), ctx
            continue
        ref = eo.reference(R, n)
        e, p = eo.check(M, n, ref, ev, Pi_hat, readout=eo.C_SCAN * M * eo.EPS)
        worst_e = max(worst_e, e)
        assert e <= 1.0, (ctx, "eigenvalues", e)
        if p is None:
            skipped.append(name)
            continue
        checked += 1
        worst_p = max(worst_p, p)
        assert p <= 1.0, (ctx, "projector", p)
    print("%s n=%d: worst eigenvalue error %.3g of its bound, projector %.3g; %d checked, ill-conditioned splits skipped: %s"
          % (path, n, worst_e, worst_p, checked, skipped))
    assert checked >= len(fam) // 2, skipped


@pytest.mark.parametrize("path,M,base", UNFUSED, ids=[u[0] for u in UNFUSED])
def test_unfused_scaled_exact_windows_are_bit_identical(path, M, base):
    n = max(1, M // 3)
    launches = base + (1 if n >= 2 else 0)
    rng = np.random.default_rng(900 + M)
    xs = [x for _, x, _, _ in eo.exact_family(M, n, rng)] + [x for _, x, _, _ in eo.exact_family(M, n, rng, diagonal=True)]
    base_out = unfused_call(M, n, xs, launches)
    for e in (-140, 96):
        ys = [(x.astype(np.complex128) * 2.0 ** e).astype(np.complex64) for x in xs]
        for x, y in zip(xs, ys):
            assert np.array_equal(y.astype(np.complex128) * 2.0 ** -e, x.astype(np.complex128))
        got = unfused_call(M, n, ys, launches)
        assert np.array_equal(got["P64"], base_out["P64"]), e
        assert np.array_equal(got["eigvals"], base_out["eigvals"] * 2.0 ** (2 * e)), e
        assert np.array_equal(got["bins"], base_out["bins"]), e


# ---- fused M = 4 and M = 8 ------------------------------------------------------------------------------------------
TRACE_WORDS, TRACE_CTAS, TRACE_LAUNCHES = 40, 1024, 32  # music_fused.cuh: FZ_TRACE, FZ_TRACE_CTAS, FZ_TRACE_LAUNCHES


def jacobi_rounds(blk, launch):
    """Jacobi rounds the fused M = 4 kernel ran in the handle's `launch`-th call (per-CTA trace word 19)"""
    ring = np.zeros(TRACE_LAUNCHES * TRACE_CTAS * TRACE_WORDS, np.int64)
    assert blk._lib.music_b200_debug_fused_trace(blk._h, ring.ctypes.data, TRACE_LAUNCHES * TRACE_CTAS) == 0
    rows = ring.reshape(TRACE_LAUNCHES, TRACE_CTAS, TRACE_WORDS)[launch % TRACE_LAUNCHES]
    return int(rows[rows[:, 31] != 0, 19].sum())


def fused_windows(M, seed):
    fam = [(name, x) for name, x, kind in windows(M, 1, seed) if kind in ("exact", "rounded", "zero")]
    return fam


@pytest.mark.parametrize("M,eig", [(4, "power"), (4, "jacobi"), (8, "power"), (8, "jacobi")])
def test_fused_eigensolver_on_sensitive_rows(M, eig):
    fam = fused_windows(M, 8100 + M)
    # the GPU's own R of every window, from the unfused path
    R = gh.device_call(gh.make_block(M, 1, N, K=M * M), np.stack([x.reshape(-1) for _, x in fam]), ("P64", "R"))[0]["R"]
    probe = eo.probe_table(M) if M == 4 else np.zeros((0, M), np.complex64)
    K = len(probe) + 2 * (M - 1)
    env = {"MUSIC_B200_EIG": eig, "MUSIC_B200_TRACE": "1"}
    blk = gh.make_block(M, 1, N, K=K, env=env)
    outs = ("levels", "bins", "spectrum") if M == 4 else ("levels", "bins")
    principal, fallback, skipped, checked = 0, 0, [], 0
    for w, (name, x) in enumerate(fam):
        ctx = (M, eig, name)
        ref = eo.reference(R[w], 1) if np.any(R[w] != 0) else None
        rows = eo.sensitive_rows(ref, 1) if ref is not None else np.ones((2 * (M - 1), M), np.complex64)
        table = np.concatenate([probe, rows]).astype(np.complex64)
        blk.set_array_response(table)
        got, nl = gh.device_call(blk, x.reshape(1, -1), outs)
        assert nl == 1, (ctx, "launches", nl)
        for k in outs:
            assert not np.any(got[k] == gh.SENTINEL), (ctx, k)
        if M == 4:
            rounds = jacobi_rounds(blk, w)
            principal += rounds == 0
            fallback += rounds > 0
            if eig == "jacobi":
                assert rounds > 0, ctx
        if ref is None:
            continue
        if not eo.proj_bound(M, ref["norm"], ref["gap"]) <= eo.PROJ_CHECKED:
            skipped.append(name)
            continue
        checked += 1
        Pref, _, _ = eo.strength_ref(ref, table)
        tol = eo.strength_tol(ref, table, M)
        if M == 4:
            err = np.abs(got["spectrum"][0].astype(np.float64) - Pref) / Pref
            assert np.all(err <= tol), (ctx, float(np.max(err / tol)))
        b = int(got["bins"][0, 0])
        best = int(np.argmax(Pref))
        assert b == best or Pref[b] >= Pref[best] * (1 - 2 * tol[best]), (ctx, b, best)
        assert abs(float(got["levels"][0, 0]) - Pref[b]) <= tol[b] * Pref[b], ctx
    if M == 8:
        principal, fallback = blk.fused8_stats()
        if eig == "jacobi":
            assert principal == 0 and fallback == len(fam)
    blk.close()
    print("fused M=%d %s: %d windows solved by the principal solver, %d by the Jacobi fallback; %d checked, skipped: %s"
          % (M, eig, principal, fallback, checked, skipped))
    if eig == "power":
        assert principal > 0 and fallback > 0, (principal, fallback)  # both outcomes of the principal solver
    assert checked >= len(fam) // 2, skipped
