// music_iaa.cuh - the iterative adaptive approach (IAA) spectrum estimator (opt-in, music_b200_set_estimator with
// MUSIC_B200_ESTIMATOR_IAA; Yardibi, Li, Stoica, Xue & Baggeroer 2010).
//
// A nonparametric weighted-least-squares power spectrum on the grid, from the window's covariance Rh (ws.R) alone:
//   p0_k = a_k^H Rh a_k / nu_k^2                                (the Bartlett spectrum),  nu_k = ||a_k||^2
//   R_i  = sum_k p(i-1)_k a_k a_k^H + delta I,  delta = loading tr(Rh) / M,  R_i = L L^H,  S_i = R_i^-1
//   p(i)_k = (a_k^H S_i Rh S_i a_k) / (a_k^H S_i a_k)^2                       for i = 1 .. I,   P = p(I)
// Rows with nu_k = 0 have p_k = 0.  With y = L^-1 a the two forms are
//   a^H S a = ||y||^2  (a sum of squares: cannot cancel, as MVDR)   and   a^H S Rh S a = y^H B y,  B = L^-1 Rh L^-H,
// so a pass needs L^-1 and B per window.  The full definition is in include/music_b200.h and is restated literally by
// tests/iaa_oracle.py.
//
// iaa_kernel: a CTA owns T windows and makes I + 1 passes over the SoA steering table.  Pass i evaluates p(i) of its
// windows at every bin (thread <-> bin of a 256-bin tile, as scan_kernel) and, in the same pass, accumulates the
// Hermitian sum sum_k p(i)_k a_k a_k^H that is R_(i+1): thread t owns the lower-triangle entry c = t % NE of every
// window and the bins j = t / NE (mod NP) of each tile, NE = M (M + 1) / 2, NP = 256 / NE, and keeps its sums in
// registers across the pass; the NP partial sums of an entry are added in part order after the pass.  Every sum is
// therefore reduced in one fixed order, with no atomics: a window's arithmetic does not depend on W, its slot in the
// CTA, the sub-batch split or the device.  Between passes warp b (window b) adds delta, factors R_i with warp_cholesky
// and forms L^-1 and B.  The last pass writes P64 (and the float spectrum when one is requested); the peaks then go
// through the grid peak rules.  A window fails - every P[k] NaN - when Rh has a non-finite entry or tr Rh <= 0, a
// Cholesky pivot is not > 0 (NaN included), or any p(i)_k is not finite.
#pragma once
#include "music_estimators.cuh"
#include "music_warp_la.cuh"

namespace music {

constexpr int IAA_THREADS = TILE;                 // one bin per thread in the evaluation phase
constexpr int IAA_MAX_ITERATIONS = 64;
constexpr int IAA_DEFAULT_ITERATIONS = 15;

// Windows per CTA: one warp each between passes, and at M > 8 a smaller tile so that the per-window matrices fit
__host__ __device__ constexpr int iaa_windows(int M) { return M > 8 ? 4 : 8; }

// The lower-triangle entries of an M x M Hermitian matrix, and the bin parts of a tile their owners split
__host__ __device__ constexpr int iaa_entries(int M) { return M * (M + 1) / 2; }
__host__ __device__ constexpr int iaa_parts(int M) { return IAA_THREADS / iaa_entries(M); }

// Doubles of dynamic shared memory of iaa_kernel: four M x M complex matrices per window (Rh, B, L^-1, R_i), then a
// region that holds a tile's strengths and rows during a pass and the partial sums of R_(i+1) after it.
__host__ __device__ constexpr size_t iaa_smem_doubles(int M, int T)
{
    return 4 * (size_t)T * 2 * M * M + ((size_t)T * TILE + (size_t)TILE * (2 * M + 1) > (size_t)iaa_parts(M) * iaa_entries(M) * T * 2
                                            ? (size_t)T * TILE + (size_t)TILE * (2 * M + 1)
                                            : (size_t)iaa_parts(M) * iaa_entries(M) * T * 2);
}

// The largest iaa_smem_doubles(M, T) over M = lo .. hi: the dynamic shared memory an instance for those M opts in to
inline size_t iaa_smem_max(int lo, int hi, int T)
{
    size_t m = 0;
    for (int M = lo; M <= hi; ++M) m = iaa_smem_doubles(M, T) > m ? iaa_smem_doubles(M, T) : m;
    return m;
}

// lower-triangle entry c -> (i, j), j <= i, c = i (i + 1) / 2 + j
__device__ __forceinline__ void iaa_entry(int c, int &i, int &j)
{
    i = 0;
    while ((i + 1) * (i + 2) / 2 <= c) ++i;
    j = c - i * (i + 1) / 2;
}

// Window b's preparation for the next pass, by one warp: R_i = (the partial sums in part order) + delta I into A, its
// Cholesky factor, L^-1 into G and B = L^-1 Rh L^-H (through Z = L^-1 Rh in A).  Returns false on a failing pivot.
__device__ bool iaa_prepare(const double *part, int T, int b, int NE, int NP, double delta, const double2 *Rh, double2 *A,
                            double2 *G, double2 *B, int M, int lane)
{
    for (int e = lane; e < NE; e += 32) {
        int i, j;
        iaa_entry(e, i, j);
        double sr = 0.0, si = 0.0;
        for (int q = 0; q < NP; ++q) {
            const double *s = part + 2 * ((size_t)(q * T + b) * NE + e);
            sr += s[0];
            si += s[1];
        }
        if (i == j) A[i * M + i] = make_double2(sr + delta, 0.0);
        else {
            A[i * M + j] = make_double2(sr, si);
            A[j * M + i] = make_double2(sr, -si);
        }
    }
    __syncwarp();
    if (!warp_cholesky(A, M, lane, [](int, double d) { return d > 0.0; })) return false;
    tril_inverse(A, M, G, M, M, lane);  // L^-1, column c by lane c
    __syncwarp();
    for (int e = lane; e < M * M; e += 32) {  // Z = L^-1 Rh (the factor in A is no longer read)
        const int r = e / M, c = e % M;
        double sr = 0.0, si = 0.0;
        for (int q = 0; q <= r; ++q) {
            const double2 g = G[r * M + q], x = Rh[q * M + c];
            sr += g.x * x.x - g.y * x.y;
            si += g.x * x.y + g.y * x.x;
        }
        A[e] = make_double2(sr, si);
    }
    __syncwarp();
    for (int e = lane; e < M * M; e += 32) {  // B = Z L^-H
        const int r = e / M, c = e % M;
        double sr = 0.0, si = 0.0;
        for (int q = 0; q <= c; ++q) {
            const double2 z = A[r * M + q], g = G[c * M + q];
            sr += z.x * g.x + z.y * g.y;
            si += z.y * g.x - z.x * g.y;
        }
        B[e] = make_double2(sr, si);
    }
    __syncwarp();
    return true;
}

// R [W][M][M] (re, im) and the SoA table -> P64 [W][K] = p(I) (and spec [W][K] = (float)P when spec != NULL).
template <int MT, int T>
__global__ void __launch_bounds__(IAA_THREADS) iaa_kernel(const double *__restrict__ soa, const double *__restrict__ R, int Mrt, int K,
                                                          int W, int iters, double loading, double *__restrict__ P64,
                                                          float *__restrict__ spec)
{
    constexpr int MA = MT ? MT : MAXM;
    const int M = MT ? MT : Mrt;
    const int MM2 = 2 * M * M, NE = iaa_entries(M), NP = iaa_parts(M), pitch = 2 * M + 1;
    extern __shared__ __align__(16) double smem[];
    double *sR = smem;             // [T][M][M] complex: Rh
    double *sB = sR + T * MM2;     // [T][M][M] complex: B = L^-1 Rh L^-H
    double *sG = sB + T * MM2;     // [T][M][M] complex: L^-1 (lower triangle)
    double *sA = sG + T * MM2;     // [T][M][M] complex: R_i, its factor, then L^-1 Rh
    double *sP = sA + T * MM2;     // [T][TILE]: p of the tile's bins
    double *sTab = sP + T * TILE;  // [TILE][2M + 1]: the tile's rows (odd pitch)
    double *sPart = sP;            // [NP][T][NE] complex: the partial sums of R_(i+1), after a pass's last tile
    __shared__ int sBad[T];   // Rh or a pivot failed (written between passes, read during them)
    __shared__ int sFail[T];  // a p(i)_k that is not finite (written during a pass, read after it)
    __shared__ double sDelta[T];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int w0 = blockIdx.x * T, nb = min(T, W - w0);

    for (int e = tid; e < nb * MM2; e += IAA_THREADS) sR[e] = R[(size_t)w0 * MM2 + e];
    __syncthreads();
    if (wid < T) {
        bool ok = false;
        double delta = 0.0;
        if (wid < nb) {
            const double *r = sR + wid * MM2;
            bool fin = true;
            for (int e = lane; e < MM2; e += 32) fin = fin && isfinite(r[e]);
            fin = __all_sync(0xffffffffu, fin);
            double tr = 0.0;  // every lane sums the diagonal in the same order
            for (int i = 0; i < M; ++i) tr += r[2 * (i * M + i)];
            ok = fin && tr > 0.0;
            delta = loading * tr / (double)M;
        }
        if (lane == 0) {
            sBad[wid] = !ok;
            sFail[wid] = 0;
            sDelta[wid] = delta;
        }
    }
    // the lower-triangle entry (ei, ej) this thread accumulates, and its part of every tile's bins
    const int c = tid % NE, part = tid / NE;
    const bool accum = part < NP;
    int ei, ej;
    iaa_entry(c, ei, ej);
    __syncthreads();

    const int ntiles = (K + TILE - 1) / TILE;
    for (int pass = 0; pass <= iters; ++pass) {
        const bool last = pass == iters;
        double accr[T], acci[T];
#pragma unroll
        for (int b = 0; b < T; ++b) accr[b] = acci[b] = 0.0;
        for (int tile = 0; tile < ntiles; ++tile) {
            const int k = tile * TILE + tid;
            const double *tb = soa + (size_t)tile * (2 * M + 1) * TILE + tid;
            double ar[MA], ai[MA];
#pragma unroll
            for (int i = 0; i < MA; ++i) {
                if (!MT && i >= M) break;
                ar[i] = tb[(size_t)(2 * i) * TILE];
                ai[i] = tb[(size_t)(2 * i + 1) * TILE];
            }
            const double na = tb[(size_t)(2 * M) * TILE];
            __syncthreads();  // the previous tile's accumulation has read sP and sTab
            if (!last) {
                for (int i = 0; i < M; ++i) {
                    sTab[tid * pitch + 2 * i] = ar[i];
                    sTab[tid * pitch + 2 * i + 1] = ai[i];
                }
            }
#pragma unroll 1
            for (int b = 0; b < T; ++b) {
                double p = 0.0;
                if (b < nb && !sBad[b] && k < K && na != 0.0) {  // rows with nu_k = 0 (and the padding) have p = 0
                    if (pass == 0) {
                        p = bartlett_form<MT>(ar, ai, sR + b * MM2, M) / (na * na);
                    } else {
                        const double *g = sG + b * MM2;
                        double yr[MA], yi[MA];
                        double den = 0.0;
#pragma unroll
                        for (int r = 0; r < MA; ++r) {
                            if (!MT && r >= M) break;
                            double sr = 0.0, si = 0.0;
#pragma unroll
                            for (int q = 0; q <= r; ++q) {
                                const double2 e = *reinterpret_cast<const double2 *>(g + 2 * (r * M + q));
                                sr = fma(e.x, ar[q], fma(-e.y, ai[q], sr));
                                si = fma(e.x, ai[q], fma(e.y, ar[q], si));
                            }
                            yr[r] = sr;
                            yi[r] = si;
                            den = fma(sr, sr, fma(si, si, den));
                        }
                        p = bartlett_form<MT>(yr, yi, sB + b * MM2, M) / (den * den);
                    }
                    if (!isfinite(p)) sFail[b] = 1;
                }
                sP[b * TILE + tid] = p;
                if (last && b < nb && k < K) {
                    P64[(size_t)(w0 + b) * K + k] = p;
                    if (spec) spec[(size_t)(w0 + b) * K + k] = (float)p;
                }
            }
            if (last) continue;
            __syncthreads();
            if (accum) {
                for (int j = part; j < TILE; j += NP) {
                    const double *a = sTab + j * pitch;
                    const double xr = a[2 * ei], xi = a[2 * ei + 1], yr = a[2 * ej], yi = a[2 * ej + 1];
                    const double ur = fma(xr, yr, xi * yi), ui = fma(xi, yr, -(xr * yi));  // a_i conj(a_j)
#pragma unroll
                    for (int b = 0; b < T; ++b) {
                        const double p = sP[b * TILE + j];
                        accr[b] = fma(p, ur, accr[b]);
                        acci[b] = fma(p, ui, acci[b]);
                    }
                }
            }
        }
        if (last) break;
        __syncthreads();  // every thread has left the last tile: the stage region takes the partial sums
        if (accum) {
#pragma unroll
            for (int b = 0; b < T; ++b) {
                double *s = sPart + 2 * ((size_t)(part * T + b) * NE + c);
                s[0] = accr[b];
                s[1] = acci[b];
            }
        }
        __syncthreads();
        if (wid < nb) {
            // a window that failed in this pass is skipped by the remaining passes: its flag moves to sBad, which the
            // evaluation reads (so no pass reads the L^-1 and B a failed window never formed)
            const bool skip = sBad[wid] || sFail[wid];
            if (!skip) {
                const bool ok = iaa_prepare(sPart, T, wid, NE, NP, sDelta[wid], reinterpret_cast<const double2 *>(sR + wid * MM2),
                                            reinterpret_cast<double2 *>(sA + wid * MM2), reinterpret_cast<double2 *>(sG + wid * MM2),
                                            reinterpret_cast<double2 *>(sB + wid * MM2), M, lane);
                if (!ok && lane == 0) sBad[wid] = 1;
            }
            __syncwarp();
            if (skip && lane == 0) sBad[wid] = 1;
        }
        __syncthreads();
    }
    __syncthreads();
    // a failed window: its whole row is NaN (also the bins the last pass wrote before the failure showed)
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (int b = 0; b < nb; ++b) {
        if (!sBad[b] && !sFail[b]) continue;
        for (int k = tid; k < K; k += IAA_THREADS) {
            P64[(size_t)(w0 + b) * K + k] = nan;
            if (spec) spec[(size_t)(w0 + b) * K + k] = (float)nan;
        }
    }
}

}  // namespace music
