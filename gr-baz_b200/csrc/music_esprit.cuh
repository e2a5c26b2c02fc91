// music_esprit.cuh - LS-ESPRIT for uniform linear arrays (opt-in peak mode MUSIC_B200_PEAKS_ESPRIT).
//
// On a ULA the steering vectors of the d sources satisfy A_2 = A_1 diag(z0_k) (A_1 / A_2 = rows 0 .. M-2 / 1 .. M-1,
// z0 = exp(-j 2 pi (s.u) / lambda)), and the d signal eigenvectors E_s span the columns of A.  So with E1 / E2 the
// same row blocks of E_s, Psi = (E1^H E1)^-1 E1^H E2 is similar to diag(z0_k): its d eigenvalues give the d directions
// with no grid, no polynomial and no root selection.  E_s is orthonormal, so E1^H E1 = I - r^H r with r = the last row
// of E_s, and Sherman-Morrison gives the inverse I + r^H r / (1 - |r|^2) without a factorisation.  The eigenvalues of
// Psi come from a Householder reduction to Hessenberg form and single-shift complex QR steps (Wilkinson shifts, an
// exceptional shift at the 10th and 20th step without a deflation, deflation on a negligible subdiagonal).  The full
// definition (angles, levels, bins, slot order) is in include/music_b200.h and is restated by tests/esprit_oracle.py.
//
// One warp per window; Psi (d x d, d <= 15) lives in the warp's shared memory, lane j <-> column j (or row j) in each
// update.  Everything is fp64.
#pragma once
#include "music_roots.cuh"

namespace music {

constexpr int ESPRIT_WARPS = 4;
constexpr int ESPRIT_LD = MAXM;                       // row stride of the per-warp matrix
constexpr int ESPRIT_MAX_IT = 30;                     // QR steps allowed between two deflations
constexpr double ESPRIT_EPS = 2.220446049250313e-16;  // 2^-52: a subdiagonal this small (relative) is negligible
constexpr int ESPRIT_EXC_EVERY = 10;                  // exceptional shifts at the 10th and 20th step without a deflation
constexpr double ESPRIT_EXC_SCALE = 0.75;             // their size, in units of the subdiagonal (zlahqr's dat1);
                                                      // anchored at h_hi,hi at step 10 and at h_l,l at step 20
// their direction: the unit vector (0.6, 0.8), whose angle is no rational multiple of pi, so that no arrangement of
// roots of unity around the diagonal entry is equally far from it
constexpr double ESPRIT_EXC_RE = 0.6, ESPRIT_EXC_IM = 0.8;

__device__ __forceinline__ double cabs2(double2 a) { return a.x * a.x + a.y * a.y; }
__device__ __forceinline__ double2 cconj(double2 a) { return make_double2(a.x, -a.y); }
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double2 cscale(double2 a, double s) { return make_double2(a.x * s, a.y * s); }

// Eigenvalues of the d x d matrix A (row stride ESPRIT_LD, overwritten) into ev[0 .. d-1], by the whole warp; v and g
// (d entries each) are scratch.  Returns false when a QR step count exceeds ESPRIT_MAX_IT between deflations.
// SCHUR: also the complex Schur form A = Z S Z^H (LAPACK zlahqr's wantt and wantz): every QR step updates the whole
// rows l .. hi (columns k .. d-1) and columns l .. hi (rows 0 .. hi), so A ends upper triangular (its entries below the
// diagonal are the negligible subdiagonals the QR deflated on, not zeroed), and Z (row stride ESPRIT_LD, the identity
// on entry) accumulates every Householder reflection and Givens rotation.  Without SCHUR only the active block is kept.
template <bool SCHUR = false>
__device__ bool esprit_eigvals(double2 *A, double2 *v, double2 *g, double2 *ev, int d, int lane, double2 *Z = nullptr)
{
    // Householder reduction to upper Hessenberg form: H = I - tau v v^H zeroes column k below row k + 1
    for (int k = 0; k + 2 < d; ++k) {
        const double2 x0 = A[(k + 1) * ESPRIT_LD + k];
        double sigma = 0.0;
        for (int i = k + 2; i < d; ++i) sigma += cabs2(A[i * ESPRIT_LD + k]);
        __syncwarp();
        if (sigma == 0.0) continue;  // uniform: every lane read the same column
        const double ax0 = sqrt(cabs2(x0)), nrm = sqrt(ax0 * ax0 + sigma);
        const double2 ph = ax0 > 0.0 ? cscale(x0, 1.0 / ax0) : make_double2(1.0, 0.0);
        const double2 v0 = cadd(x0, cscale(ph, nrm));  // x - alpha e_1 with alpha = -phase(x0) |x|: no cancellation
        const double tau = 2.0 / (cabs2(v0) + sigma);
        if (lane > k && lane < d) v[lane] = lane == k + 1 ? v0 : A[lane * ESPRIT_LD + k];
        __syncwarp();
        if (lane >= k && lane < d) {  // H A: column `lane`
            double2 s = make_double2(0.0, 0.0);
            for (int i = k + 1; i < d; ++i) s = cadd(s, cmul(cconj(v[i]), A[i * ESPRIT_LD + lane]));
            s = cscale(s, tau);
            for (int i = k + 1; i < d; ++i) A[i * ESPRIT_LD + lane] = csub(A[i * ESPRIT_LD + lane], cmul(v[i], s));
        }
        __syncwarp();
        if (lane < d) {  // (H A) H: row `lane`
            double2 s = make_double2(0.0, 0.0);
            for (int j = k + 1; j < d; ++j) s = cadd(s, cmul(A[lane * ESPRIT_LD + j], v[j]));
            s = cscale(s, tau);
            for (int j = k + 1; j < d; ++j) A[lane * ESPRIT_LD + j] = csub(A[lane * ESPRIT_LD + j], cmul(s, cconj(v[j])));
        }
        if constexpr (SCHUR) {
            if (lane < d) {  // Z H: row `lane`
                double2 s = make_double2(0.0, 0.0);
                for (int j = k + 1; j < d; ++j) s = cadd(s, cmul(Z[lane * ESPRIT_LD + j], v[j]));
                s = cscale(s, tau);
                for (int j = k + 1; j < d; ++j) Z[lane * ESPRIT_LD + j] = csub(Z[lane * ESPRIT_LD + j], cmul(s, cconj(v[j])));
            }
        }
        __syncwarp();
    }
    // shifted QR on the active block l .. hi; every lane takes the same decisions from the same shared values
    int hi = d - 1, its = 0;
    while (hi >= 0) {
        int l = hi;
        for (; l > 0; --l) {
            const double h = sqrt(cabs2(A[l * ESPRIT_LD + l - 1]));
            const double t = sqrt(cabs2(A[(l - 1) * ESPRIT_LD + l - 1])) + sqrt(cabs2(A[l * ESPRIT_LD + l]));
            if (h <= ESPRIT_EPS * t) break;
        }
        if (l == hi) {  // a 1 x 1 block has deflated
            ev[hi] = A[hi * ESPRIT_LD + hi];
            --hi;
            its = 0;
            continue;
        }
        if (++its > ESPRIT_MAX_IT) return false;
        double2 mu;
        if (its % ESPRIT_EXC_EVERY == 0 && its < ESPRIT_MAX_IT) {
            // exceptional shift (after LAPACK zlahqr, which anchors them the other way round): Wilkinson shifts stall on
            // a Psi whose trailing eigenvalues are all equally far from the shift, e.g. the phase-weighted cyclic
            // permutation of equally spaced sources
            const int k = its == ESPRIT_EXC_EVERY ? hi : l;
            const double h = sqrt(cabs2(k == hi ? A[hi * ESPRIT_LD + hi - 1] : A[(l + 1) * ESPRIT_LD + l]));
            mu = cadd(A[k * ESPRIT_LD + k], cscale(make_double2(ESPRIT_EXC_RE, ESPRIT_EXC_IM), ESPRIT_EXC_SCALE * h));
        } else {
            // Wilkinson shift: the eigenvalue of the trailing 2 x 2 block [a b; c e] nearer to e, e - bc / (p +- sqrt(p^2 + bc))
            const double2 a = A[(hi - 1) * ESPRIT_LD + hi - 1], b = A[(hi - 1) * ESPRIT_LD + hi];
            const double2 c = A[hi * ESPRIT_LD + hi - 1], e = A[hi * ESPRIT_LD + hi];
            const double2 p = cscale(csub(a, e), 0.5), bc = cmul(b, c), q = cadd(cmul(p, p), bc);
            const double qa = sqrt(cabs2(q)), ar = atan2(q.y, q.x) * 0.5;
            double sr, cr;
            sincos(ar, &sr, &cr);
            double2 sq = make_double2(sqrt(qa) * cr, sqrt(qa) * sr);
            if (p.x * sq.x + p.y * sq.y < 0.0) sq = cscale(sq, -1.0);
            const double2 den = cadd(p, sq);
            mu = cabs2(den) > 0.0 ? csub(e, cdiv(bc, den)) : e;
        }
        __syncwarp();
        if (lane >= l && lane <= hi) A[lane * ESPRIT_LD + lane] = csub(A[lane * ESPRIT_LD + lane], mu);
        __syncwarp();
        // Q^H (A - mu I) = R by Givens rotations G_k = [conj(c) conj(s); -s c] on rows k, k + 1; then R Q
        for (int k = l; k < hi; ++k) {
            const double2 x = A[k * ESPRIT_LD + k], y = A[(k + 1) * ESPRIT_LD + k];
            const double nr = sqrt(cabs2(x) + cabs2(y));
            const double2 gc = nr > 0.0 ? cscale(x, 1.0 / nr) : make_double2(1.0, 0.0);
            const double2 gs = nr > 0.0 ? cscale(y, 1.0 / nr) : make_double2(0.0, 0.0);
            __syncwarp();
            if (lane >= k && lane <= (SCHUR ? d - 1 : hi)) {
                const double2 u = A[k * ESPRIT_LD + lane], w = A[(k + 1) * ESPRIT_LD + lane];
                A[k * ESPRIT_LD + lane] = cadd(cmul(cconj(gc), u), cmul(cconj(gs), w));
                A[(k + 1) * ESPRIT_LD + lane] = csub(cmul(gc, w), cmul(gs, u));
            }
            if (lane == 0) v[k] = gc, g[k] = gs;
            __syncwarp();
        }
        for (int k = l; k < hi; ++k) {
            const double2 gc = v[k], gs = g[k];
            if (lane >= (SCHUR ? 0 : l) && lane <= hi) {  // columns k, k + 1 times G_k^H = [c -conj(s); s conj(c)]
                const double2 u = A[lane * ESPRIT_LD + k], w = A[lane * ESPRIT_LD + k + 1];
                A[lane * ESPRIT_LD + k] = cadd(cmul(u, gc), cmul(w, gs));
                A[lane * ESPRIT_LD + k + 1] = csub(cmul(w, cconj(gc)), cmul(u, cconj(gs)));
            }
            if constexpr (SCHUR) {
                if (lane < d) {  // the same columns of Z
                    const double2 u = Z[lane * ESPRIT_LD + k], w = Z[lane * ESPRIT_LD + k + 1];
                    Z[lane * ESPRIT_LD + k] = cadd(cmul(u, gc), cmul(w, gs));
                    Z[lane * ESPRIT_LD + k + 1] = csub(cmul(w, cconj(gc)), cmul(u, cconj(gs)));
                }
            }
            __syncwarp();
        }
        if (lane >= l && lane <= hi) A[lane * ESPRIT_LD + lane] = cadd(A[lane * ESPRIT_LD + lane], mu);
        __syncwarp();
    }
    return true;
}

// Vt: per window M * M complex doubles, eigenvector j contiguous, ascending eigenvalues; counts (may be null): the
// per-window source count d (else d = n).  The signal subspace is eigenvectors M - d .. M - 1, the noise subspace (the
// level's D) eigenvectors 0 .. M - d - 1, as in the scan.
__global__ void __launch_bounds__(ESPRIT_WARPS * 32) esprit_kernel(const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                                  int M, int n, int K, int W, const RefineGeom geo, const UlaGeom ula,
                                                                  PeakOut out)
{
    __shared__ double2 sA[ESPRIT_WARPS][MAXM * ESPRIT_LD];
    __shared__ double2 sv[ESPRIT_WARPS][MAXM], sev[ESPRIT_WARPS][MAXM], sq[ESPRIT_WARPS][MAXM];
    const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * ESPRIT_WARPS + wi;
    if (w >= W) return;
    const int d = counts ? counts[w] : n;
    const int p = M - d;
    const double2 *G = reinterpret_cast<const double2 *>(Vt) + (size_t)w * M * M;
    const double2 *Es = G + (size_t)p * M;  // Es[a * M + i] = row i of signal eigenvector a
    double2 *A = sA[wi], *v = sv[wi], *ev = sev[wi], *q = sq[wi];

    // r = the last row of E_s, 1 - |r|^2 (> 0 iff E1^H E1 is positive definite)
    double nr = 0.0;
    for (int a = 0; a < d; ++a) nr += cabs2(Es[a * M + M - 1]);
    const double den = 1.0 - nr;
    bool ok = d > 0 && den > 0.0;
    if (ok) {
        // B = E1^H E2, then q = r B and Psi = B + r^H q / (1 - |r|^2)
        for (int e = lane; e < d * d; e += 32) {
            const int a = e / d, b = e - a * d;
            double2 s = make_double2(0.0, 0.0);
            for (int i = 0; i + 1 < M; ++i) s = cadd(s, cmul(cconj(Es[a * M + i]), Es[b * M + i + 1]));
            A[a * ESPRIT_LD + b] = s;
        }
        __syncwarp();
        if (lane < d) {
            double2 s = make_double2(0.0, 0.0);
            for (int a = 0; a < d; ++a) s = cadd(s, cmul(Es[a * M + M - 1], A[a * ESPRIT_LD + lane]));
            q[lane] = cscale(s, 1.0 / den);
        }
        __syncwarp();
        bool fin = true;
        for (int e = lane; e < d * d; e += 32) {
            const int a = e / d, b = e - a * d;
            const double2 t = cadd(A[a * ESPRIT_LD + b], cmul(cconj(Es[a * M + M - 1]), q[b]));
            A[a * ESPRIT_LD + b] = t;
            fin = fin && isfinite(t.x) && isfinite(t.y);
        }
        ok = __all_sync(0xffffffffu, fin);
        __syncwarp();
    }
    if (ok) ok = esprit_eigvals(A, v, q, ev, d, lane);
    __syncwarp();

    // lane k < d: eigenvalue k -> direction, level; a zero eigenvalue has no direction
    double tdeg = 0.0, lvl = 0.0, D = 0.0;
    bool filled = false;
    if (ok && lane < d) {
        const double2 z = ev[lane];
        filled = isfinite(z.x) && isfinite(z.y) && (z.x != 0.0 || z.y != 0.0);
        if (filled) {
            tdeg = ula_direction(z, geo, ula);
            double D1, D2;
            refine_eval(geo, G, M, p, tdeg * STEER_DEG2RAD, &D, &D1, &D2);
            lvl = 1.0 / D;
        }
    }
    ok = ok && __all_sync(0xffffffffu, lane >= d || !isnan(lvl));
    filled = filled && ok;
    // slot = rank in descending fp64 level, ties to the lower angle, then the lower eigenvalue index
    int r = 0;
    for (int s = 0; s < d; ++s) {
        const bool fs = __shfl_sync(0xffffffffu, filled, s);
        const double ls = __shfl_sync(0xffffffffu, lvl, s), ts = __shfl_sync(0xffffffffu, tdeg, s);
        if (fs && (ls > lvl || (ls == lvl && (ts < tdeg || (ts == tdeg && s < lane))))) ++r;
    }
    const int f = __popc(__ballot_sync(0xffffffffu, filled));
    if (filled) ula_store_slot(out, (size_t)w * n + r, tdeg, D, K);
    if (lane >= f && lane < n) peak_write(out, (size_t)w * n + lane, -1, 0.0, K);
}

}  // namespace music
