// music_estimators.cuh - the MVDR (Capon) and Bartlett beamscan spectra (opt-in, music_b200_set_estimator).
//
// Both are full-rank quadratic forms of the window's covariance R (ws.R) in the steering vector a = a_k:
//   BARTLETT  P[k] = (a^H R a) / (a^H a)^2                         the output power of the unit-gain beam a / ||a||^2;
//   MVDR      P[k] = 1 / (a^H R_L^-1 a),  R_L = R + delta I,  delta = loading * tr(R) / M
//                                                              the output power of the distortionless beam.
// MVDR is evaluated as a sum of squares: mvdr_prep_kernel factors R_L = L L^H (Cholesky) and writes the rows of L^-1,
// conjugated, into the window's ws.Vt slot as g_j = conj(row j of L^-1), so that
//     a^H R_L^-1 a = ||L^-1 a||^2 = sum_j |g_j^H a|^2,
// which cannot cancel and is the form the refinement kernels already evaluate (music_refine.cuh, with p = M vectors).
// The grid scan is scan_kernel (music_kernels.cuh) with FORM = EST_MVDR or EST_BARTLETT.  The full definition is in
// include/music_b200.h and is restated literally by tests/estimator_oracle.py.
#pragma once
#include "music_kernels.cuh"
#include "music_warp_la.cuh"

namespace music {

// ---- MVDR preparation: one warp per window, the matrix in shared memory --------------------------------------------
// A 16 x 16 complex fp64 matrix is 4 KiB: too large for one thread's registers, so each window gets a warp and two
// shared-memory copies (the factor and its inverse).  About 1.4 k complex flops per window at M = 16, next to the
// covariance's N * M^2.
constexpr int PREP_WARPS = 4;

// R [W][M][M] (re, im) -> Vt [W][M][M] (re, im): Vt[w][j][m] = conj((L^-1)[j][m]) for m <= j, 0 for m > j.  A pivot
// that is not > 0 (NaN included) makes every entry of the window NaN, so its whole spectrum is NaN and the peak rules
// report no peak.
__global__ void __launch_bounds__(PREP_WARPS * 32) mvdr_prep_kernel(const double *__restrict__ R, double *__restrict__ Vt, int M, int W,
                                                                    double loading)
{
    __shared__ double2 sA[PREP_WARPS][MAXM * MAXM];  // R_L, overwritten by L (lower triangle, row-major)
    __shared__ double2 sI[PREP_WARPS][MAXM * MAXM];  // L^-1 (row-major)
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int w = blockIdx.x * PREP_WARPS + wid;
    if (w >= W) return;
    double2 *A = sA[wid], *I = sI[wid];
    const int MM = M * M;
    const double2 *Rw = reinterpret_cast<const double2 *>(R) + (size_t)w * MM;
    double2 *Gw = reinterpret_cast<double2 *>(Vt) + (size_t)w * MM;
    for (int e = lane; e < MM; e += 32) A[e] = Rw[e];
    __syncwarp();
    warp_load_diagonal(A, M, M, loading, lane);
    const bool ok = warp_cholesky(A, M, lane, [](int, double d) { return d > 0.0; });
    if (!ok) {
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        for (int e = lane; e < MM; e += 32) Gw[e] = make_double2(nan, nan);
        return;
    }
    tril_inverse(A, M, I, M, M, lane);  // L^-1, column c by lane c
    __syncwarp();
    for (int e = lane; e < MM; e += 32) {
        const double2 v = I[e];
        Gw[e] = make_double2(v.x, -v.y);
    }
}

// ---- the strengths of the quadratic-form scan (scan_kernel) --------------------------------------------------------
// MVDR: a^H R_L^-1 a = sum_j |g_j^H a|^2 over the triangular g (M (M + 1) / 2 complex MACs)
template <int MT>
__device__ __forceinline__ double mvdr_form(const double *ar, const double *ai, const double *g, int M)
{
    constexpr int MA = MT ? MT : MAXM;
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < MA; ++j) {
        if (!MT && j >= M) break;
        double cr = 0.0, ci = 0.0;
#pragma unroll
        for (int i = 0; i <= j; ++i) {
            const double2 e = *reinterpret_cast<const double2 *>(g + 2 * (j * M + i));
            cr = fma(e.x, ar[i], fma(e.y, ai[i], cr));
            ci = fma(e.x, ai[i], fma(-e.y, ar[i], ci));
        }
        acc = fma(cr, cr, fma(ci, ci, acc));
    }
    return acc;
}

// Bartlett: a^H R a = sum_i (R_ii |a_i|^2 + 2 Re(conj(a_i) sum_{j > i} R_ij a_j)), from the upper triangle of R
template <int MT>
__device__ __forceinline__ double bartlett_form(const double *ar, const double *ai, const double *R, int M)
{
    constexpr int MA = MT ? MT : MAXM;
    double acc = 0.0;
#pragma unroll
    for (int i = 0; i < MA; ++i) {
        if (!MT && i >= M) break;
        double ur = 0.0, ui = 0.0;
#pragma unroll
        for (int j = i + 1; j < MA; ++j) {
            if (!MT && j >= M) break;
            const double2 r = *reinterpret_cast<const double2 *>(R + 2 * (i * M + j));
            ur = fma(r.x, ar[j], fma(-r.y, ai[j], ur));
            ui = fma(r.x, ai[j], fma(r.y, ar[j], ui));
        }
        const double rii = R[2 * (i * M + i)];
        acc = fma(rii, fma(ar[i], ar[i], ai[i] * ai[i]), acc);
        acc = fma(2.0, fma(ar[i], ur, ai[i] * ui), acc);
    }
    return acc;
}

}  // namespace music
