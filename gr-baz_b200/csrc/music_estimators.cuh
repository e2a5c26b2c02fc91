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
// scan_quad_kernel is scan_kernel (music_kernels.cuh) with the strength replaced by one of the two forms.  The full
// definition is in include/music_b200.h and is restated literally by tests/estimator_oracle.py.
#pragma once
#include "music_kernels.cuh"

namespace music {

constexpr int QUAD_MVDR = 1;      // MUSIC_B200_ESTIMATOR_MVDR
constexpr int QUAD_BARTLETT = 2;  // MUSIC_B200_ESTIMATOR_BARTLETT

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
    double tr = 0.0;  // every lane sums the diagonal in the same order
    for (int i = 0; i < M; ++i) tr += A[i * M + i].x;
    const double delta = loading * tr / (double)M;
    __syncwarp();
    if (lane < M) A[lane * M + lane].x += delta;
    __syncwarp();
    // right-looking Cholesky on the lower triangle; the pivot test reads the same value in every lane, so the warp
    // leaves the loop together
    bool ok = true;
    for (int k = 0; k < M; ++k) {
        const double d = A[k * M + k].x;
        if (!(d > 0.0)) { ok = false; break; }
        const double l = sqrt(d);
        __syncwarp();
        if (lane == k) A[k * M + k] = make_double2(l, 0.0);
        if (lane > k && lane < M) {
            const double2 v = A[lane * M + k];
            A[lane * M + k] = make_double2(v.x / l, v.y / l);
        }
        __syncwarp();
        const int r = M - 1 - k;  // trailing block: A[i][j] -= L[i][k] conj(L[j][k]) for k < j <= i
        for (int e = lane; e < r * r; e += 32) {
            const int i = k + 1 + e / r, j = k + 1 + e % r;
            if (j > i) continue;
            const double2 a = A[i * M + k], b = A[j * M + k];
            double2 &t = A[i * M + j];
            t.x -= a.x * b.x + a.y * b.y;
            t.y -= a.y * b.x - a.x * b.y;
        }
        __syncwarp();
    }
    if (!ok) {
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        for (int e = lane; e < MM; e += 32) Gw[e] = make_double2(nan, nan);
        return;
    }
    // column c of L^-1 by forward substitution (lane c): x_c = 1 / L_cc, x_i = -(sum_{c <= q < i} L_iq x_q) / L_ii
    if (lane < M) {
        const int c = lane;
        for (int i = 0; i < c; ++i) I[i * M + c] = make_double2(0.0, 0.0);
        I[c * M + c] = make_double2(1.0 / A[c * M + c].x, 0.0);
        for (int i = c + 1; i < M; ++i) {
            double sr = 0.0, si = 0.0;
            for (int q = c; q < i; ++q) {
                const double2 l = A[i * M + q], x = I[q * M + c];
                sr += l.x * x.x - l.y * x.y;
                si += l.x * x.y + l.y * x.x;
            }
            const double li = A[i * M + i].x;
            I[i * M + c] = make_double2(-sr / li, -si / li);
        }
    }
    __syncwarp();
    for (int e = lane; e < MM; e += 32) {
        const double2 v = I[e];
        Gw[e] = make_double2(v.x, -v.y);
    }
}

// ---- the quadratic-form scan ------------------------------------------------------------------------------------------
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

// scan_kernel with P[k] of the chosen form.  Q: per window M*M complex doubles, the g_j of mvdr_prep_kernel (MVDR) or
// R itself (BARTLETT), staged in shared memory for SCAN_B windows; thread <-> bin.  ARGMAX: n == 1 fused peak pick
// (P desc, bin asc, P > 0 strictly, NaN never).  counts (may be null, music_sources.cuh): with ARGMAX a window with
// count 0 reports no peak; the spectrum itself does not depend on the count.
template <int MT, int FORM, bool ARGMAX, bool WRITE_P64, bool WRITE_SPEC>
__global__ void __launch_bounds__(TILE) scan_quad_kernel(const double *__restrict__ soa, const double *__restrict__ Q, int Mrt, int K,
                                                         int W, PeakOut out, float *__restrict__ spectrum, double *__restrict__ P64,
                                                         const int32_t *__restrict__ counts)
{
    constexpr int MA = MT ? MT : MAXM;
    const int M = MT ? MT : Mrt;
    extern __shared__ __align__(16) double smem[];
    const int w0 = blockIdx.x * SCAN_B;
    const int nb = min(SCAN_B, W - w0);
    const int vsz = M * M * 2;
    for (int i = threadIdx.x; i < nb * vsz; i += blockDim.x) smem[i] = Q[(size_t)w0 * vsz + i];
    __syncthreads();

    double best[SCAN_B];
    int bestk[SCAN_B];
#pragma unroll
    for (int b = 0; b < SCAN_B; ++b) { best[b] = 0.0; bestk[b] = -1; }

    const int ntiles = (K + TILE - 1) / TILE;
    for (int tile = 0; tile < ntiles; ++tile) {
        const int k = tile * TILE + threadIdx.x;
        const double *tb = soa + (size_t)tile * (2 * M + 1) * TILE + threadIdx.x;
        double ar[MA], ai[MA];
#pragma unroll
        for (int i = 0; i < MA; ++i) {
            if (!MT && i >= M) break;
            ar[i] = tb[(size_t)(2 * i) * TILE];
            ai[i] = tb[(size_t)(2 * i + 1) * TILE];
        }
        const double na = tb[(size_t)(2 * M) * TILE];
        if (k < K) {
#pragma unroll
            for (int b = 0; b < SCAN_B; ++b) {
                if (b < nb) {
                    const double *q = smem + b * vsz;
                    const double P = FORM == QUAD_MVDR ? 1.0 / mvdr_form<MT>(ar, ai, q, M) : bartlett_form<MT>(ar, ai, q, M) / (na * na);
                    if (WRITE_SPEC) spectrum[(size_t)(w0 + b) * K + k] = (float)P;
                    if (WRITE_P64) P64[(size_t)(w0 + b) * K + k] = P;
                    if (ARGMAX) {
                        if (P > best[b]) { best[b] = P; bestk[b] = k; }  // k ascending per thread: strict > keeps the lower bin
                    }
                }
            }
        }
    }
    if (ARGMAX) {
        __shared__ double rP[SCAN_B][TILE / 32];
        __shared__ int rk[SCAN_B][TILE / 32];
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
        for (int b = 0; b < SCAN_B; ++b) {
            int kk = bestk[b];
            double P = best[b];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double Po = __shfl_xor_sync(0xffffffffu, P, o);
                const int ko = __shfl_xor_sync(0xffffffffu, kk, o);
                if (peak_better(Po, ko, P, kk)) { P = Po; kk = ko; }
            }
            if (lane == 0) { rP[b][wid] = P; rk[b][wid] = kk; }
        }
        __syncthreads();
        if (threadIdx.x < nb) {
            const int b = threadIdx.x;
            double P = rP[b][0];
            int kk = rk[b][0];
            for (int q = 1; q < TILE / 32; ++q)
                if (peak_better(rP[b][q], rk[b][q], P, kk)) { P = rP[b][q]; kk = rk[b][q]; }
            const size_t o = (size_t)(w0 + b);  // n == 1
            if (counts && counts[o] == 0) kk = -1;
            if (kk >= 0) {
                out.angles[o] = (float)((double)kk * 360.0 / (double)K);
                if (out.levels) out.levels[o] = (float)P;
            } else {
                out.angles[o] = 0.f;
                if (out.levels) out.levels[o] = 0.f;
            }
            peak_store_bin(out, o, kk);
        }
    }
}

}  // namespace music
