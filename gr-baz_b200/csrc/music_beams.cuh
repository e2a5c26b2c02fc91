// music_beams.cuh - beamformed source signals (opt-in, music_b200_set_beamformer and the *_beams entry points).
//
// After the peak stage, each filled slot i of a window (bins[w][i] >= 0) gets a weight vector w_i and a beam
//     y_i(t) = sum_m conj(w_im) x_m(t),   t < N,
// steered at the slot's reported angle (a geometric table) or its table row (a set_table() table):
//   DAS   w_i = a_i / (a_i^H a_i);
//   MVDR  R_L = R + delta I = L L^H,  y_i = L^-1 a_i,  z_i = L^-H y_i,  w_i = z_i / ||y_i||^2;
//   LCMV  G = Y^H Y over the filled slots = C C^H,  W = Z G^-1, so that w_i^H a_j = delta_ij.
// The full definition is in include/music_b200.h and is restated literally by tests/beams_oracle.py.
//
// beam_weights_kernel: one warp per window, R_L and its factor in shared memory as in mvdr_prep_kernel; lanes map to
//   slots for the triangular solves, and to antennas for the LCMV solve against the d x d Gram.
// beam_apply_kernel: a second read of the window stream (the weights depend on the same window's R).  One CTA per
//   (window, BEAM_SPAN snapshots): the span is staged through shared memory with coalesced 16-byte loads marked
//   evict_first, then each lane reads its own snapshot, widens it to fp64 once and forms every slot's beam with the
//   fp64 weights broadcast from shared memory; the float2 stores are streaming (st.global.cs) and coalesced per slot.
//   Why not a bulk-copy ring as in cov4_tma_kernel: a lane reads a whole 32-128 byte snapshot, so an unpadded staging
//   buffer makes 8 lanes of a 16-byte read phase hit the same banks (8-way at M = 16).  The staging pads each snapshot
//   to an odd number of 16-byte units, which a 1-D bulk copy cannot scatter; the coalesced loads can.  (The windows of
//   an odd M are also only 8-byte aligned, below the 16 bytes a bulk copy needs.)
#pragma once
#include "music_kernels.cuh"
#include "music_refine.cuh"
#include "music_warp_la.cuh"

namespace music {

constexpr int BEAM_DAS = 1, BEAM_MVDR = 2, BEAM_LCMV = 3;  // MUSIC_B200_BEAMS_*
constexpr int BEAM_WARPS = 2;                                // windows per weights CTA
constexpr int BEAM_MAXN = MAXM - 1;                          // slots per window (n < M)
constexpr double BEAM_PIVOT_REL = 0x1p-20;                   // LCMV: pivot k must exceed this fraction of G_kk
constexpr int BEAM_SPAN = 128;                               // snapshots per apply CTA, one per thread

// ---- weights ----------------------------------------------------------------------------------------------------------
// R [W][M][M] (re, im); angles / bins [W][n] as the peak stage wrote them; table [K][M] complex64 (read for a set_table()
// table only); geo: the geometry of a geometric table, by value.  wts [W][n][M] (re, im): w_i of every filled slot, 0 for
// unfilled slots and for every slot of a window whose factorisation failed or whose weights are not all finite.
__global__ void __launch_bounds__(BEAM_WARPS * 32) beam_weights_kernel(const double *__restrict__ R, const float *__restrict__ angles,
                                                                      const int32_t *__restrict__ bins, const float2 *__restrict__ table,
                                                                      int M, int n, int W, int rule, double loading, bool geometric,
                                                                      const RefineGeom geo, double *__restrict__ wts)
{
    __shared__ double2 sA[BEAM_WARPS][MAXM * MAXM];            // R_L, overwritten by L
    __shared__ double2 sY[BEAM_WARPS][BEAM_MAXN * MAXM];       // a_i, overwritten by y_i = L^-1 a_i (row i)
    __shared__ double2 sZ[BEAM_WARPS][BEAM_MAXN * MAXM];       // z_i, then w_i (row i)
    __shared__ double2 sG[BEAM_WARPS][BEAM_MAXN * BEAM_MAXN];  // LCMV: G over the filled slots, overwritten by C
    __shared__ double sD[BEAM_WARPS][BEAM_MAXN];               // LCMV: diag(G) before the factorisation
    __shared__ int sS[BEAM_WARPS][BEAM_MAXN];                  // the filled slots, ascending
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int w = blockIdx.x * BEAM_WARPS + wid;
    if (w >= W) return;
    double2 *A = sA[wid], *Y = sY[wid], *Z = sZ[wid], *G = sG[wid];
    double *D = sD[wid];
    int *S = sS[wid];
    const int b = lane < n ? bins[(size_t)w * n + lane] : -1;
    const bool filled = b >= 0;
    const unsigned fmask = __ballot_sync(0xffffffffu, filled);
    const int d = __popc(fmask);
    if (filled) {
        S[__popc(fmask & ((1u << lane) - 1u))] = lane;
        double2 *a = Y + lane * M;
        if (geometric) {
            // refine_eval's steering vector at the reported float angle
            double st, ct;
            sincos((double)angles[(size_t)w * n + lane] * STEER_DEG2RAD, &st, &ct);
            for (int m = 0; m < M; ++m) {
                double phi, psi, sp, cp;
                steer_phase(geo, m, st, ct, &phi, &psi);
                sincos(phi, &sp, &cp);
                a[m] = make_double2(cp, -sp);
            }
        } else {
            const float2 *row = table + (size_t)b * M;
            for (int m = 0; m < M; ++m) {
                const float2 v = row[m];
                a[m] = make_double2((double)v.x, (double)v.y);
            }
        }
    }
    bool ok = true;  // warp-uniform
    if (rule != BEAM_DAS && d > 0) {
        const double2 *Rw = reinterpret_cast<const double2 *>(R) + (size_t)w * M * M;
        for (int e = lane; e < M * M; e += 32) A[e] = Rw[e];
        __syncwarp();
        warp_load_diagonal(A, M, M, loading, lane);
        ok = warp_cholesky(A, M, lane, [](int, double p) { return p > 0.0; });
    }
    __syncwarp();
    if (ok && filled) {
        double2 *y = Y + lane * M, *z = Z + lane * M;
        if (rule == BEAM_DAS) {
            double nrm = 0.0;
            for (int m = 0; m < M; ++m) nrm = fma(y[m].x, y[m].x, fma(y[m].y, y[m].y, nrm));
            for (int m = 0; m < M; ++m) z[m] = make_double2(y[m].x / nrm, y[m].y / nrm);
        } else {
            const auto yk = [&](int k) -> double2 & { return y[k]; };  // y = L^-1 a, in place, then z = L^-H y
            cholesky_solve(A, M, M, yk, yk, [&](int k) -> double2 & { return z[k]; });
            if (rule == BEAM_MVDR) {
                double nrm = 0.0;
                for (int m = 0; m < M; ++m) nrm = fma(y[m].x, y[m].x, fma(y[m].y, y[m].y, nrm));
                for (int m = 0; m < M; ++m) z[m] = make_double2(z[m].x / nrm, z[m].y / nrm);
            }
        }
    }
    __syncwarp();
    if (ok && rule == BEAM_LCMV && d > 0) {
        // G[r][c] = y_{S[r]}^H y_{S[c]} over the filled slots
        for (int e = lane; e < d * d; e += 32) {
            const int r = e / d, c = e - r * d;
            const double2 *yr = Y + S[r] * M, *yc = Y + S[c] * M;
            double gr = 0.0, gi = 0.0;
            for (int m = 0; m < M; ++m) {
                gr += yr[m].x * yc[m].x + yr[m].y * yc[m].y;
                gi += yr[m].x * yc[m].y - yr[m].y * yc[m].x;
            }
            G[e] = make_double2(gr, gi);
            if (r == c) D[r] = gr;
        }
        __syncwarp();
        ok = warp_cholesky(G, d, lane, [D](int k, double p) { return p > BEAM_PIVOT_REL * D[k]; });
        __syncwarp();
        if (ok && lane < M) {
            // lane m: row m of W = Z G^-1, i.e. u = G^-1 conj(Z[S][m]) and w_{S[r], m} = conj(u_r), in place in column m of Z
            const int m = lane;
            const auto zr = [&](int r) -> double2 & { return Z[S[r] * M + m]; };  // C v = conj(z), then C^H u = v
            cholesky_solve(G, d, d, [&](int r) { return make_double2(zr(r).x, -zr(r).y); }, zr, zr);
            for (int r = 0; r < d; ++r) Z[S[r] * M + m].y = -Z[S[r] * M + m].y;
        }
    }
    __syncwarp();
    bool bad = false;
    if (ok)
        for (int e = lane; e < n * M; e += 32)
            if ((fmask >> (e / M)) & 1u) bad = bad || !isfinite(Z[e].x) || !isfinite(Z[e].y);
    const bool any_bad = __any_sync(0xffffffffu, bad);
    ok = ok && !any_bad;
    double2 *out = reinterpret_cast<double2 *>(wts) + (size_t)w * n * M;
    for (int e = lane; e < n * M; e += 32) out[e] = ok && ((fmask >> (e / M)) & 1u) ? Z[e] : make_double2(0.0, 0.0);
}

// ---- beams ------------------------------------------------------------------------------------------------------------
// The stride of one staged snapshot, in floats: 2M, plus one 16-byte unit when M is even and M / 2 is even, so that a
// snapshot spans an odd number of 16-byte units and the 8 lanes of a 16-byte read phase hit distinct banks.  For an odd
// M a lane reads 8-byte pairs at an odd stride of 8-byte units: the 16 lanes of a phase are conflict-free unpadded.
__host__ __device__ constexpr int beam_stride(int M) { return (M % 2 == 0 && (M / 2) % 2 == 0) ? 2 * M + 4 : 2 * M; }

// dynamic shared memory of beam_apply_kernel: the window's weights, then the staged snapshots
__host__ __device__ constexpr size_t beam_apply_smem(int M, int n)
{
    return (size_t)n * M * sizeof(double2) + (size_t)BEAM_SPAN * beam_stride(M) * sizeof(float);
}

__device__ __forceinline__ void st_stream_f2(float2 *p, float2 v)
{
    asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v.x), "f"(v.y) : "memory");
}

// in [W][N][M] complex64; wts [W][n][M] (re, im) from beam_weights_kernel; beams [W][n][N] complex64.  spans = the CTAs
// per window, ceil(N / BEAM_SPAN).  MT = M for the specialised M = 4, 8, 16; MT = 0 reads M at run time.  A slot whose
// weights are all zero (unfilled, or its window failed) gets a zero beam whatever the input holds.
template <int MT>
__global__ void __launch_bounds__(BEAM_SPAN) beam_apply_kernel(const float *__restrict__ in, const double *__restrict__ wts, int M_rt,
                                                               int n, int N, int spans, float *__restrict__ beams)
{
    extern __shared__ __align__(16) unsigned char beam_smem[];
    constexpr int MA = MT ? MT : MAXM;
    const int M = MT ? MT : M_rt;
    const int w = blockIdx.x / spans, t0 = (blockIdx.x - w * spans) * BEAM_SPAN;
    const int cnt = min(BEAM_SPAN, N - t0);
    const int tid = threadIdx.x;
    double2 *sw = reinterpret_cast<double2 *>(beam_smem);
    float *sx = reinterpret_cast<float *>(beam_smem + (size_t)n * M * sizeof(double2));
    const int xs = beam_stride(M);
    const double2 *ww = reinterpret_cast<const double2 *>(wts) + (size_t)w * n * M;
    for (int e = tid; e < n * M; e += BEAM_SPAN) sw[e] = ww[e];
    const uint64_t pol = l2_policy_evict_first();
    if (M % 2 == 0) {
        // a window starts 16-byte aligned when M is even: 16-byte loads, every load of the thread in flight at once
        const int q = M / 2;  // 16-byte units per snapshot
        const float4 *src = reinterpret_cast<const float4 *>(in) + ((size_t)w * N + t0) * q;
        float4 v[MA / 2];
#pragma unroll
        for (int u = 0; u < MA / 2; ++u) {
            const int e = tid + u * BEAM_SPAN;
            if (e < cnt * q) v[u] = ldg_f32x4_hint(src + e, pol);
        }
#pragma unroll
        for (int u = 0; u < MA / 2; ++u) {
            const int e = tid + u * BEAM_SPAN;
            if (e < cnt * q) {
                const int t = e / q, k = e - t * q;
                *reinterpret_cast<float4 *>(sx + t * xs + 4 * k) = v[u];
            }
        }
    } else if (!MT) {
        const float2 *src = reinterpret_cast<const float2 *>(in) + ((size_t)w * N + t0) * M;
        float2 v[MAXM];
#pragma unroll
        for (int u = 0; u < MAXM; ++u) {
            const int e = tid + u * BEAM_SPAN;
            if (e < cnt * M)
                asm volatile("ld.global.nc.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(v[u].x), "=f"(v[u].y) : "l"(src + e), "l"(pol));
        }
#pragma unroll
        for (int u = 0; u < MAXM; ++u) {
            const int e = tid + u * BEAM_SPAN;
            if (e < cnt * M) *reinterpret_cast<float2 *>(sx + 2 * e) = v[u];  // unpadded: stride 2M floats
        }
    }
    __syncthreads();
    if (tid >= cnt) return;
    double xr[MA], xi[MA];
    const float *x = sx + tid * xs;
    if (M % 2 == 0) {
#pragma unroll
        for (int k = 0; k < MA / 2; ++k) {
            if (!MT && 2 * k >= M) break;
            const float4 f = reinterpret_cast<const float4 *>(x)[k];
            xr[2 * k] = f.x; xi[2 * k] = f.y; xr[2 * k + 1] = f.z; xi[2 * k + 1] = f.w;
        }
    } else {
#pragma unroll
        for (int m = 0; m < MA; ++m) {
            if (!MT && m >= M) break;
            const float2 f = reinterpret_cast<const float2 *>(x)[m];
            xr[m] = f.x; xi[m] = f.y;
        }
    }
    float2 *out = reinterpret_cast<float2 *>(beams) + (size_t)w * n * N + t0 + tid;
    for (int i = 0; i < n; ++i) {
        const double2 *wi = sw + i * M;
        double yr = 0.0, yi = 0.0;
        bool live = false;
#pragma unroll
        for (int m = 0; m < MA; ++m) {
            if (!MT && m >= M) break;
            const double2 c = wi[m];  // conj(c) x
            yr = fma(c.x, xr[m], fma(c.y, xi[m], yr));
            yi = fma(c.x, xi[m], fma(-c.y, xr[m], yi));
            live = live || c.x != 0.0 || c.y != 0.0;
        }
        st_stream_f2(out + (size_t)i * N, live ? make_float2((float)yr, (float)yi) : make_float2(0.f, 0.f));
    }
}

}  // namespace music
