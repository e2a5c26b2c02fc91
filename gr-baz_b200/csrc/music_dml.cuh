// music_dml.cuh - deterministic maximum likelihood (DML) angles by alternating projection (opt-in peak mode
// MUSIC_B200_PEAKS_DML).
//
// DML maximises tr(P_A R), the power of the window's covariance R captured by the span of d table rows A, and needs no
// signal-subspace rank: coherent sources (a path and its reflection), whose covariance has rank one, are resolved where
// every subspace method sees one source.  Alternating projection (Ziskind & Wax, 1988) turns the d-dimensional search
// into 1-D table searches S(B): with Q_B an orthonormal basis of the rows already held (B) and P = I - Q_B Q_B^H,
//     f(k) = a_k^H P R P a_k / (||a_k||^2 - ||Q_B^H a_k||^2),
// the power gained by adding row k.  Each search is the Bartlett grid scan (bartlett_form) on R' = P R P,
// plus the denominator.  The full definition (candidate rule, sweeps, least-squares levels, slot order) is in
// include/music_b200.h and is restated by tests/dml_oracle.py.
//
// One CTA of DML_THREADS per window stays resident for all of its searches, so each window stops after its own last
// sweep.  The threads stride over the bins of the fp64 SoA table tiles; warp 0 does the small linear algebra (modified
// Gram-Schmidt twice, the levels) in shared memory, the CTA the M x M products.  Everything is fp64.
#pragma once
#include "music_estimators.cuh"
#include "music_warp_la.cuh"

namespace music {

constexpr int DML_THREADS = 128;
constexpr int DML_WARPS = DML_THREADS / 32;
constexpr int DML_MAX_SWEEPS = 20;
constexpr double DML_DEN_MIN = 9.313225746154785e-10;  // 2^-30: den(k) must exceed this fraction of ||a_k||^2

// Row k of the SoA table, entry i (re, im), and ||a_k||^2
__device__ __forceinline__ const double *dml_row(const double *soa, int k, int M)
{
    return soa + (size_t)(k / TILE) * (2 * M + 1) * TILE + (k % TILE);
}

// Warp 0 of dml_kernel: mgs2 of the table rows bins[0 .. r-1]
__device__ __forceinline__ void dml_mgs2(const double *soa, const int *bins, int r, int M, double2 *Q, double2 *T, int lane)
{
    mgs2([&](int l, int i) {
        const double *a = dml_row(soa, bins[l], M);
        return make_double2(a[(size_t)(2 * i) * TILE], a[(size_t)(2 * i + 1) * TILE]);
    }, r, M, Q, T, lane);
}

// R: per window M * M complex doubles (row-major), the matrix searched; Rl: the matrix the levels are taken from, in the
// same layout (under DML both are the window's covariance; under WSF R is the weighted signal-subspace matrix of
// music_wsf.cuh and Rl the covariance); soa: the table tiles [ceil(K / TILE)][2M + 1][TILE]; counts (may be null): the per-window source
// count d (else d = n).
template <int MT>
__global__ void __launch_bounds__(DML_THREADS) dml_kernel(const double *__restrict__ R, const double *__restrict__ Rl, const double *__restrict__ soa,
                                                          const int32_t *__restrict__ counts, int Mrt, int n, int K, PeakOut out)
{
    constexpr int MA = MT ? MT : MAXM;
    const int M = MT ? MT : Mrt;
    __shared__ double2 sR[MAXM * MAXM];   // R (row-major, stride M)
    __shared__ double2 sP[MAXM * MAXM];   // P = I - Q_B Q_B^H (stride M); U = T^-1 for the levels (stride MAXM)
    __shared__ double2 sX[MAXM * MAXM];   // P R (stride M); the levels' C = Q_A^H R Q_A - s2 I (stride MAXM)
    __shared__ double2 sY[MAXM * MAXM];   // R' = P R P (stride M); the levels' matrix Rl when it is not R
    __shared__ double2 sQ[MAXM * MAXM];   // Q_B or Q_A, vector l at l * MAXM
    __shared__ double2 sT[MAXM * MAXM];   // T of A = Q_A T (stride MAXM)
    __shared__ int slot[MAXM], sB[MAXM];
    __shared__ double rf[DML_WARPS];
    __shared__ int rk[DML_WARPS];
    __shared__ int s_win, s_none;
    __shared__ double s_p[MAXM];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const size_t w = blockIdx.x;
    const int MM = M * M;
    const int d = counts ? counts[w] : n;

    const double2 *Rw = reinterpret_cast<const double2 *>(R) + w * MM;
    bool fin = true;
    for (int e = tid; e < MM; e += DML_THREADS) {
        const double2 v = Rw[e];
        sR[e] = v;
        fin = fin && isfinite(v.x) && isfinite(v.y);
    }
    bool ok = __syncthreads_and(fin) && d > 0;
    double trR = trace_re(sR, M, M);  // every thread sums the diagonal in the same order
    ok = ok && trR > 0.0;

    // S(B) over the r bins in sB: the winner into s_win (-1: no candidate)
    const auto search = [&](int r) {
        if (wid == 0) dml_mgs2(soa, sB, r, M, sQ, nullptr, lane);
        __syncthreads();
        for (int e = tid; e < MM; e += DML_THREADS) {  // P = I - Q Q^H
            const int i = e / M, j = e - i * M;
            double2 s = make_double2(i == j ? 1.0 : 0.0, 0.0);
            for (int l = 0; l < r; ++l) {
                const double2 t = cmul(sQ[l * MAXM + i], make_double2(sQ[l * MAXM + j].x, -sQ[l * MAXM + j].y));
                s.x -= t.x;
                s.y -= t.y;
            }
            sP[e] = s;
        }
        __syncthreads();
        for (int e = tid; e < MM; e += DML_THREADS) {  // X = P R
            const int i = e / M, j = e - i * M;
            double2 s = make_double2(0.0, 0.0);
            for (int q = 0; q < M; ++q) {
                const double2 t = cmul(sP[i * M + q], sR[q * M + j]);
                s.x += t.x;
                s.y += t.y;
            }
            sX[e] = s;
        }
        __syncthreads();
        for (int e = tid; e < MM; e += DML_THREADS) {  // R' = X P
            const int i = e / M, j = e - i * M;
            double2 s = make_double2(0.0, 0.0);
            for (int q = 0; q < M; ++q) {
                const double2 t = cmul(sX[i * M + q], sP[q * M + j]);
                s.x += t.x;
                s.y += t.y;
            }
            sY[e] = s;
        }
        __syncthreads();

        double best = -INFINITY;
        int bk = -1;
        const double *Rp = reinterpret_cast<const double *>(sY);
#pragma unroll 1
        for (int k = tid; k < K; k += DML_THREADS) {  // k ascending per thread: strict > keeps the lower bin
            const double *tb = dml_row(soa, k, M);
            double ar[MA], ai[MA];
#pragma unroll
            for (int i = 0; i < MA; ++i) {
                if (!MT && i >= M) break;
                ar[i] = tb[(size_t)(2 * i) * TILE];
                ai[i] = tb[(size_t)(2 * i + 1) * TILE];
            }
            const double na = tb[(size_t)(2 * M) * TILE];
            double den = na;
#pragma unroll 1
            for (int l = 0; l < r; ++l) {
                const double2 *q = sQ + l * MAXM;
                double cr = 0.0, ci = 0.0;
#pragma unroll
                for (int i = 0; i < MA; ++i) {
                    if (!MT && i >= M) break;
                    const double2 e = q[i];
                    cr = fma(e.x, ar[i], fma(e.y, ai[i], cr));
                    ci = fma(e.x, ai[i], fma(-e.y, ar[i], ci));
                }
                den -= fma(cr, cr, ci * ci);
            }
            const double f = bartlett_form<MT>(ar, ai, Rp, M) / den;
            if (den > DML_DEN_MIN * na && isfinite(f) && f > best) { best = f; bk = k; }
        }
        warp_argmax(best, bk);
        if (lane == 0) { rf[wid] = best; rk[wid] = bk; }
        __syncthreads();
        if (tid == 0) {
            for (int q = 1; q < DML_WARPS; ++q)
                if (peak_better(rf[q], rk[q], best, bk)) { best = rf[q]; bk = rk[q]; }
            s_win = bk;
        }
        __syncthreads();
        return s_win;
    };

    // initialisation: slot i = S(slots 0 .. i-1)
    for (int i = 0; ok && i < d; ++i) {
        if (tid < i) sB[tid] = slot[tid];
        __syncthreads();
        const int k = search(i);
        if (k < 0) ok = false;
        if (tid == 0) slot[i] = k;
        __syncthreads();
    }
    // Gauss-Seidel sweeps: slot i = S(every other slot), until a sweep changes nothing (d = 1 repeats the first search)
    for (int s = 1; ok && d > 1 && s <= DML_MAX_SWEEPS; ++s) {
        bool changed = false;
        for (int i = 0; ok && i < d; ++i) {
            if (tid < d - 1) sB[tid] = slot[tid < i ? tid : tid + 1];
            __syncthreads();
            const int k = search(d - 1);
            if (k < 0) ok = false;
            changed = changed || k != slot[i];
            __syncthreads();
            if (tid == 0) slot[i] = k;
            __syncthreads();
        }
        if (!changed) break;
    }

    // levels: A = Q_A T, s2 = (tr Rl - tr(Q_A^H Rl Q_A)) / (M - d), p = diag(T^-1 (Q_A^H Rl Q_A - s2 I) T^-H)
    if (ok && wid == 0) {
        const double2 *sL = sR;
        if (Rl != R) {
            const double2 *Lw = reinterpret_cast<const double2 *>(Rl) + w * MM;
            for (int e = lane; e < MM; e += 32) sY[e] = Lw[e];
            __syncwarp();
            sL = sY;
            trR = trace_re(sL, M, M);
        }
        dml_mgs2(soa, slot, d, M, sQ, sT, lane);
        // C[a][b] = q_a^H R q_b: lane a < d, then the trace terms
        for (int e = lane; e < d * d; e += 32) {
            const int a = e / d, b = e - a * d;
            double2 s = make_double2(0.0, 0.0);
            for (int i = 0; i < M; ++i) {
                double2 y = make_double2(0.0, 0.0);  // (R q_b)_i
                for (int j = 0; j < M; ++j) {
                    const double2 t = cmul(sL[i * M + j], sQ[b * MAXM + j]);
                    y.x += t.x;
                    y.y += t.y;
                }
                const double2 t = cjmul(sQ[a * MAXM + i], y);
                s.x += t.x;
                s.y += t.y;
            }
            sX[a * MAXM + b] = s;
        }
        __syncwarp();
        const double s2 = (trR - trace_re(sX, MAXM, d)) / (double)(M - d);
        __syncwarp();
        if (lane < d) sX[lane * MAXM + lane].x -= s2;
        triu_inverse(sT, MAXM, sP, MAXM, d, lane);  // U = T^-1 (upper triangular) into sP, column c by lane c
        __syncwarp();
        if (lane < d) s_p[lane] = slot_level(sP, MAXM, sX, MAXM, d, lane);
        __syncwarp();
    }
    if (tid == 0) s_none = !ok;
    __syncthreads();

    // outputs: slots in descending p, exact ties to the lower bin; slots d .. n-1 (every slot without peaks) (0, 0, -1)
    if (tid < n) {
        int rnk = tid, k = -1;
        double p = 0.0;
        if (!s_none && tid < d) {
            p = s_p[tid];
            k = slot[tid];
            rnk = 0;
            for (int j = 0; j < d; ++j)
                if (s_p[j] > p || (s_p[j] == p && slot[j] < k)) ++rnk;
        }
        peak_write(out, w * n + rnk, k, p, K);
    }
}

}  // namespace music
