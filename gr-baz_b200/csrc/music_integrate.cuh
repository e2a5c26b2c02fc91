// music_integrate.cuh - covariance integration across windows (opt-in, music_b200_set_integration).
//
// Every estimate is made from one window's N snapshots unless the covariance is integrated over the recent past.  With a
// forgetting factor 0 < alpha < 1 the windows j = 0, 1, 2, ... of a handle since its last reset (in stream order, across
// calls) give
//     S_j = alpha S_{j-1} + R_j,   c_j = alpha c_{j-1} + 1,   Rbar_j = S_j / c_j      (S_{-1} = 0, c_{-1} = 0),
// and every stage after the covariance kernel (and the calibration) reads Rbar_j instead of R_j.  The full definition
// is in include/music_b200.h and is restated literally by tests/integration_oracle.py.
//
// This is a first-order linear recurrence with a constant coefficient over the W windows of a sub-batch; a loop over the
// windows would leave the GPU idle (at M = 4 a window has 32 doubles).  It runs as a three-phase scan in which a thread
// owns one double e < E = 2 M^2 of R (real and imaginary parts alike, so R's exact Hermitian symmetry, a mirrored lower
// triangle and a real diagonal, is kept bit for bit) over a tile of INTEG_T consecutive windows:
//   integ_tiles_kernel   the tile aggregate a_t = R_first, then a_t <- alpha a_t + R_i over the tile (Horner order);
//   integ_carry_kernel   one CTA per entry: the carry into every tile, a block scan of the affine maps
//                        x -> alpha^len_t x + a_t applied to the handle's carry S; the carry-ins overwrite the aggregates,
//                        the carry out of the last tile becomes S, and the window count since the reset advances by W;
//   integ_apply_kernel   per tile from its carry-in: S <- alpha S + R_i (the first window after a reset takes S = R_i
//                        itself), R_i <- S / c_i in place.  c_i takes the closed form (1 - alpha^(n+1)) / (1 - alpha) at
//                        the tile's first window (n: its count since the reset; integ_one_minus_pow keeps it accurate as
//                        alpha nears 1) and the recurrence after it.
// The carry (S and the count) lives in the handle's device buffers, read at the start of each sub-batch and written at its
// end; the handle orders consecutive sub-batches, on whichever streams they run, with one event.
// Bytes per window: the tile pass reads R and the apply pass reads and writes it, 16 M^2 bytes each way per pass.
//
// The source count (music_sources.cuh) then uses N_eff,j = N c_j^2 / q_j, q_j = alpha^2 q_{j-1} + 1, in place of N:
// source_count_neff_kernel derives it per window from the count the carry kernel left in the sub-batch's workspace slot.
#pragma once
#include "music_kernels.cuh"
#include "music_sources.cuh"

namespace music {

constexpr int INTEG_T = 32;             // windows per tile
constexpr int INTEG_THREADS = 256;      // tile and apply kernels
constexpr int INTEG_SCAN_THREADS = 256; // carry kernel: one CTA per entry

// 1 - a^k for 0 < a < 1 and k >= 1, without the cancellation of 1 - pow(a, k) as a nears 1 (there 1 - pow(a, k) loses
// all but about -log2(1 - a^k) of its bits): -expm1(k log a), with log a = log1p(a - 1) for a >= 1/2, where a - 1 is
// exact (Sterbenz), so every step keeps its own few-ulp relative error.
__device__ __forceinline__ double integ_one_minus_pow(double a, double k)
{
    return -expm1(k * (a >= 0.5 ? log1p(a - 1.0) : log(a)));
}

// c_n = sum_{k <= n} alpha^k, the closed form of c_j = alpha c_{j-1} + 1 at count n since the reset (c_0 = 1 exactly)
__device__ __forceinline__ double integ_c(double alpha, unsigned long long n)
{
    if (n == 0) return 1.0;
    return integ_one_minus_pow(alpha, (double)n + 1.0) / (1.0 - alpha);
}

// N_eff,n = N c_n^2 / q_n, q_n = sum_{k <= n} alpha^(2k): N at n = 0, tending to N (1 + alpha) / (1 - alpha).  q takes
// 1 - alpha^2 as (1 - alpha)(1 + alpha), and 1 - alpha^(2k) as d (2 - d) with d = 1 - alpha^k: no difference of two
// rounded numbers near 1.
__device__ __forceinline__ double integ_neff(double alpha, unsigned long long n, double N)
{
    if (n == 0) return N;
    const double k = (double)n + 1.0, d = integ_one_minus_pow(alpha, k), c = d / (1.0 - alpha);
    const double q = d * (2.0 - d) / ((1.0 - alpha) * (1.0 + alpha));
    return N * c * c / q;
}

// agg [ntiles][E]: the aggregate of tile t over windows [t T, min(W, (t + 1) T)) of R [W][E]
__global__ void __launch_bounds__(INTEG_THREADS) integ_tiles_kernel(const double *__restrict__ R, double *__restrict__ agg, int E, int W,
                                                                   double alpha)
{
    const size_t g = (size_t)blockIdx.x * INTEG_THREADS + threadIdx.x;
    const int ntiles = (W + INTEG_T - 1) / INTEG_T;
    if (g >= (size_t)ntiles * E) return;
    const int t = (int)(g / E), e = (int)(g - (size_t)t * E);
    const int w0 = t * INTEG_T, len = min(W - w0, INTEG_T);
    const double *p = R + (size_t)w0 * E + e;
    double r[INTEG_T];  // every load of the tile issued before the recurrence waits on the first
#pragma unroll
    for (int i = 0; i < INTEG_T; ++i)
        if (i < len) r[i] = p[(size_t)i * E];
    double a = r[0];
#pragma unroll
    for (int i = 1; i < INTEG_T; ++i)
        if (i < len) a = fma(alpha, a, r[i]);
    agg[g] = a;
}

// One CTA per entry e: in agg [ntiles][E] the aggregates are replaced by the carry into each tile, S[e] becomes the carry
// out of the last tile; *n0 <- *cnt (the count at this sub-batch's first window, in the sub-batch's workspace slot, where
// the later stages of the same sub-batch read it while the next sub-batch may already advance *cnt), *cnt += W.
// aT = alpha^INTEG_T, alast = alpha^(length of the last tile).
__global__ void __launch_bounds__(INTEG_SCAN_THREADS) integ_carry_kernel(double *__restrict__ agg, double *__restrict__ S,
                                                                        unsigned long long *__restrict__ cnt,
                                                                        unsigned long long *__restrict__ n0, int E, int W, double aT,
                                                                        double alast)
{
    __shared__ double wA[INTEG_SCAN_THREADS / 32], wB[INTEG_SCAN_THREADS / 32];
    const int e = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ntiles = (W + INTEG_T - 1) / INTEG_T;
    const int chunk = (ntiles + INTEG_SCAN_THREADS - 1) / INTEG_SCAN_THREADS;
    const int t0 = min(ntiles, tid * chunk), t1 = min(ntiles, t0 + chunk);
    // this thread's tiles as one map x -> A x + B
    double A = 1.0, B = 0.0;
    for (int t = t0; t < t1; ++t) {
        const double a = t == ntiles - 1 ? alast : aT;
        B = fma(a, B, agg[(size_t)t * E + e]);
        A *= a;
    }
    // inclusive scan of the maps within the warp (the later map applied after the earlier one)
    for (int off = 1; off < 32; off *= 2) {
        const double Ao = __shfl_up_sync(0xffffffffu, A, off), Bo = __shfl_up_sync(0xffffffffu, B, off);
        if (lane >= off) {
            B = fma(A, Bo, B);
            A *= Ao;
        }
    }
    if (lane == 31) {
        wA[warp] = A;
        wB[warp] = B;
    }
    __syncthreads();
    // the warps before this one, composed in order
    double pA = 1.0, pB = 0.0;
    for (int v = 0; v < warp; ++v) {
        pB = fma(wA[v], pB, wB[v]);
        pA *= wA[v];
    }
    // exclusive map within the warp, then after the earlier warps'
    double eA = __shfl_up_sync(0xffffffffu, A, 1), eB = __shfl_up_sync(0xffffffffu, B, 1);
    if (lane == 0) {
        eA = 1.0;
        eB = 0.0;
    }
    const double xA = eA * pA, xB = fma(eA, pB, eB);
    double x = fma(xA, S[e], xB);  // the carry into tile t0
    for (int t = t0; t < t1; ++t) {
        const double a = t == ntiles - 1 ? alast : aT;
        const double v = agg[(size_t)t * E + e];
        agg[(size_t)t * E + e] = x;
        x = fma(a, x, v);
    }
    __syncthreads();  // every thread has read S[e]
    if (t0 < t1 && t1 == ntiles) S[e] = x;
    if (e == 0 && tid == 0) {
        *n0 = *cnt;
        *cnt += (unsigned long long)W;
    }
}

// R [W][E] in place: R_i <- S_i / c_i from the carry-ins cin [ntiles][E]; *n0: the count at window 0
__global__ void __launch_bounds__(INTEG_THREADS) integ_apply_kernel(double *__restrict__ R, const double *__restrict__ cin,
                                                                   const unsigned long long *__restrict__ n0p, int E, int W, double alpha)
{
    const size_t g = (size_t)blockIdx.x * INTEG_THREADS + threadIdx.x;
    const int ntiles = (W + INTEG_T - 1) / INTEG_T;
    if (g >= (size_t)ntiles * E) return;
    const int t = (int)(g / E), e = (int)(g - (size_t)t * E);
    const int w0 = t * INTEG_T, len = min(W - w0, INTEG_T);
    double *p = R + (size_t)w0 * E + e;
    double r[INTEG_T];  // the tile's loads first: the stores below go to the same array
#pragma unroll
    for (int i = 0; i < INTEG_T; ++i)
        if (i < len) r[i] = p[(size_t)i * E];
    const unsigned long long n0 = *n0p + (unsigned long long)w0;
    double x = cin[g], c = integ_c(alpha, n0);
#pragma unroll
    for (int i = 0; i < INTEG_T; ++i) {
        if (i >= len) break;
        if (i > 0) c = fma(alpha, c, 1.0);
        x = (n0 == 0 && i == 0) ? r[i] : fma(alpha, x, r[i]);  // the first window after a reset is its own R, exactly
        p[(size_t)i * E] = x / c;
    }
}

// source_count_kernel with the per-window N_eff of an integrated covariance in place of N (*n0: the count at window 0)
__global__ void __launch_bounds__(128) source_count_neff_kernel(const double *__restrict__ ev, int M, int nmax, int N, int rule, int W,
                                                                double alpha, const unsigned long long *__restrict__ n0,
                                                                int32_t *__restrict__ counts, int32_t *__restrict__ counts_out)
{
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    const int best = source_count_window(ev + (size_t)w * M, M, nmax, integ_neff(alpha, *n0 + (unsigned long long)w, (double)N), rule);
    counts[w] = best;
    if (counts_out) counts_out[w] = best;
}

}  // namespace music
