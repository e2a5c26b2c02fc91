// music_focus.cuh - coherent wideband direction finding on a channel handle (MUSIC_B200_CHANNELS_COHERENT): the
// rotational focusing matrices T_c of Hung and Kaveh (1988) and the focused covariance of the coherent signal-subspace
// method of Wang and Kaveh (1985).
//
// Definition (include/music_b200.h, restated literally by tests/focus_oracle.py): reference channel c_ref = C / 2;
// sector S = {(first + i) mod K : i < count}; fp64 steering vectors a_c(theta_k)[r] = exp(-j 2 pi <p_r, u(theta_k)> / lambda_c);
// B_c = sum_{k in S} a_ref(theta_k) a_c(theta_k)^H + beta |S| I with beta = 1e-3; T_c = U V^H from B_c = U S V^H;
// T_ref = I exactly.  R_foc = (1 / C) sum_c T_c R_c T_c^H in channel order, the c_ref term added as R_ref itself.
//
// Set-up (on a retune): focus_setup_kernel accumulates every B_c on the device (one CTA per channel, the sector in tiles
// of steering vectors in shared memory, one thread per entry: no atomics, a fixed order); the host takes the polar
// factors by a one-sided Jacobi SVD (focus_polar); focus_setup_kernel again sums the focusing errors with the new T_c.
//
// Per call: chan_focus_kernel reads the [C][W] covariances chan_cov_kernel wrote into the handle's channel buffer and
// writes R_foc into the workspace.  A CTA owns 256 / M^2 windows (one thread per matrix entry, so every M keeps the
// threads busy and a sub-batch gives thousands of CTAs) and walks the channels in order, staging T_c and its windows' R_c
// in shared memory: Y = R T^H (M^3 complex MACs per window), then only the upper half of T Y, accumulated in a register
// of the thread that owns the entry for the whole call.  R_foc therefore has the same bits whatever the grid, the
// sub-batch or the call split.
#pragma once
#include <complex>
#include <vector>

#include "music_kernels.cuh"
#include "music_steer.cuh"

namespace music {

constexpr double FOCUS_BETA = 1e-3;       // the regularisation beta |S| I of B_c
constexpr double FOCUS_SINGULAR = 1e-12;  // sigma_min(B_c) <= this * sigma_max(B_c): T_c is not unique, refused
constexpr int FOCUS_THREADS = 256;        // chan_focus_kernel: at most one thread per matrix entry of its windows
constexpr int FOCUS_LD = MAXM + 1;        // padded row length of the staged matrices (rows land on distinct banks)
constexpr int FOCUS_STAGE = 384;          // the most staged entries, windows * M * (M + 1): M = 2, 64 windows

// windows per CTA of chan_focus_kernel: as many M x M matrices as FOCUS_THREADS threads cover, one thread per entry
__host__ __device__ inline int focus_windows(int M) { return FOCUS_THREADS / (M * M); }
__host__ __device__ inline int focus_threads(int M) { return (focus_windows(M) * M * M + 31) / 32 * 32; }
constexpr int FOCUS_TILE = 64;            // sector bins per shared-memory tile of the set-up kernel

// set-up geometry: element positions, and each channel's wavelength
struct FocusGeom {
    double pos[2 * MAXM];
    int M, K, C, ref;
    int first, count;  // the sector
};

// a(theta_k)[r] for lambda, in the literal order of steer_table_kernel, kept in fp64
__device__ __forceinline__ double2 focus_steer(const FocusGeom &g, int k, int r, double lambda)
{
    const double theta = __dmul_rn(__ddiv_rn(__dmul_rn((double)k, 360.0), (double)g.K), STEER_DEG2RAD);
    double s, c;
    sincos(theta, &s, &c);
    const double inner = __fma_rn(g.pos[2 * r + 1], s, __dmul_rn(g.pos[2 * r], c));
    const double phi = -__dmul_rn(STEER_TWO_PI, __ddiv_rn(inner, lambda));
    double sp, cp;
    sincos(phi, &sp, &cp);
    return make_double2(cp, sp);
}

// One CTA per channel c != ref.  T == NULL: B[c] = sum_{k in S} a_ref a_c^H + beta |S| I ([C][M][M] complex).
// Otherwise: e2[c] = sum_{k in S} ||T_c a_c - a_ref||^2, summed per thread in sector order, then over the threads in a
// fixed tree.
__global__ void __launch_bounds__(FOCUS_THREADS) focus_setup_kernel(const FocusGeom g, const double *__restrict__ lambdas,
                                                                   const double2 *__restrict__ T, double2 *__restrict__ B,
                                                                   double *__restrict__ e2)
{
    __shared__ double2 ar[FOCUS_TILE][MAXM], ac[FOCUS_TILE][MAXM];
    __shared__ double2 Ts[MAXM][FOCUS_LD];
    __shared__ double red[FOCUS_THREADS];
    const int c = blockIdx.x, M = g.M, tid = threadIdx.x;
    if (c == g.ref) return;
    const double lam_r = lambdas[g.ref], lam_c = lambdas[c];
    if (T)
        for (int i = tid; i < M * M; i += FOCUS_THREADS) Ts[i / M][i % M] = T[(size_t)c * M * M + i];
    const int ei = tid / M, ek = tid % M;  // B mode: entry (ei, ek) of this thread (M * M <= FOCUS_THREADS)
    double2 b = make_double2(0.0, 0.0);
    double e = 0.0;
    for (int t0 = 0; t0 < g.count; t0 += FOCUS_TILE) {
        const int nt = min(FOCUS_TILE, g.count - t0);
        __syncthreads();
        for (int i = tid; i < nt * M; i += FOCUS_THREADS) {
            const int k = (g.first + t0 + i / M) % g.K, r = i % M;
            ar[i / M][r] = focus_steer(g, k, r, lam_r);
            ac[i / M][r] = focus_steer(g, k, r, lam_c);
        }
        __syncthreads();
        if (!T) {
            if (ei < M)
                for (int j = 0; j < nt; ++j) {  // a_ref[ei] conj(a_c[ek])
                    const double2 x = ar[j][ei], y = ac[j][ek];
                    b.x = fma(x.x, y.x, fma(x.y, y.y, b.x));
                    b.y = fma(x.y, y.x, fma(-x.x, y.y, b.y));
                }
        } else {
            for (int i = tid; i < nt * M; i += FOCUS_THREADS) {
                const int j = i / M, r = i % M;
                double2 d = make_double2(-ar[j][r].x, -ar[j][r].y);
                for (int l = 0; l < M; ++l) {
                    const double2 t = Ts[r][l], a = ac[j][l];
                    d.x = fma(t.x, a.x, fma(-t.y, a.y, d.x));
                    d.y = fma(t.x, a.y, fma(t.y, a.x, d.y));
                }
                e = fma(d.x, d.x, fma(d.y, d.y, e));
            }
        }
    }
    if (!T) {
        if (ei < M) {
            if (ei == ek) b.x += FOCUS_BETA * (double)g.count;
            B[(size_t)c * M * M + ei * M + ek] = b;
        }
        return;
    }
    red[tid] = e;
    __syncthreads();
    for (int s = FOCUS_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) red[tid] += red[tid + s];
        __syncthreads();
    }
    if (tid == 0) e2[c] = red[0];
}

// Rc ([C][W][M][M] complex fp64, one sub-batch) -> Rf ([W][M][M]) = R_foc.  T: [C][M][M] complex.  A CTA owns
// focus_windows(M) windows and has one thread per entry of their M x M matrices (launched with that many threads,
// rounded up to whole warps): that thread stages the entry of R_c and computes the same entry of Y; the threads of the
// Hermitian-half entries then accumulate the upper half of T Y.  R_c and T_c are double-buffered in shared memory, so a
// channel costs two barriers.
__global__ void __launch_bounds__(FOCUS_THREADS) chan_focus_kernel(const double2 *__restrict__ Rc, double2 *__restrict__ Rf, int W,
                                                                  int C, int M, int ref, const double2 *__restrict__ T)
{
    __shared__ double2 Ts[2][MAXM * FOCUS_LD];
    __shared__ double2 Rs[2][FOCUS_STAGE];
    __shared__ double2 Ys[FOCUS_STAGE];
    __shared__ uchar2 pairs[MAXM * (MAXM + 1) / 2];
    const int MM = M * M, E = M * (M + 1) / 2, LD = M + 1, wt = focus_windows(M);
    const int tid = threadIdx.x, w0 = blockIdx.x * wt, nw = min(wt, W - w0);
    const int yw = tid / MM, yi = (tid % MM) / M, yj = tid % M;  // this thread's entry (w, i, j) of R_c and Y
    const int sidx = (yw * M + yi) * LD + yj;
    const bool ythr = tid < nw * MM, zthr = tid < nw * E;        // zthr: this thread owns Hermitian-half entry tid of R_foc
    const int zw = tid / E;
    if (tid == 0) {
        int e = 0;
        for (int i = 0; i < M; ++i)
            for (int k = i; k < M; ++k) pairs[e++] = make_uchar2((unsigned char)i, (unsigned char)k);
    }
    __syncthreads();
    const uchar2 ik = zthr ? pairs[tid % E] : make_uchar2(0, 0);
    double2 acc = make_double2(0.0, 0.0);

    for (int c = 0; c < C; ++c) {
        // buffer b was last read in channel c - 2's stages, which every thread left before channel c - 1's first barrier
        const int b = c & 1;
        if (ythr) Rs[b][sidx] = Rc[((size_t)c * W + w0) * MM + tid];
        if (c != ref && tid < MM) Ts[b][(tid / M) * LD + tid % M] = T[(size_t)c * MM + tid];
        __syncthreads();
        if (c == ref) {  // T_ref = I: R_ref itself
            if (zthr) {
                const double2 r = Rs[b][(zw * M + ik.x) * LD + ik.y];
                acc.x += r.x;
                acc.y += r.y;
            }
            continue;
        }
        if (ythr) {  // Y[w][i][j] = sum_l R[w][i][l] conj(T[j][l])
            double2 y = make_double2(0.0, 0.0);
            for (int l = 0; l < M; ++l) {
                const double2 a = Rs[b][(yw * M + yi) * LD + l], t = Ts[b][yj * LD + l];
                y.x = fma(a.x, t.x, fma(a.y, t.y, y.x));
                y.y = fma(a.y, t.x, fma(-a.x, t.y, y.y));
            }
            Ys[sidx] = y;
        }
        __syncthreads();
        if (zthr) {  // (T Y)[w][i][k], i <= k
            double2 z = make_double2(0.0, 0.0);
            for (int j = 0; j < M; ++j) {
                const double2 t = Ts[b][ik.x * LD + j], y = Ys[(zw * M + j) * LD + ik.y];
                z.x = fma(t.x, y.x, fma(-t.y, y.y, z.x));
                z.y = fma(t.x, y.y, fma(t.y, y.x, z.y));
            }
            acc.x += z.x;
            acc.y += z.y;
        }
    }
    // R_foc = acc / C: upper half as summed, the lower half its mirror, the diagonal real
    if (zthr) {
        const double den = (double)C;
        double2 *Rw = Rf + (size_t)(w0 + zw) * MM;
        const double re = acc.x / den, im = ik.x == ik.y ? 0.0 : acc.y / den;
        Rw[ik.x * M + ik.y] = make_double2(re, im);
        if (ik.x != ik.y) Rw[ik.y * M + ik.x] = make_double2(re, -im);
    }
}

// ---- host side: the polar factor ----

// T = U V^H of the M x M complex matrix B (row-major) from B = U S V^H, by one-sided Jacobi (Hestenes) rotations of the
// columns of B (accumulated in V) until every pair of columns is orthogonal to 1e-15; then U = the columns over their
// norms.  Returns false (T untouched) when sigma_min <= FOCUS_SINGULAR sigma_max, where U V^H is not unique.
inline bool focus_polar(int M, const std::complex<double> *B, std::complex<double> *T)
{
    using cd = std::complex<double>;
    std::vector<cd> A(B, B + (size_t)M * M), V((size_t)M * M, cd(0.0, 0.0));
    for (int i = 0; i < M; ++i) V[(size_t)i * M + i] = 1.0;
    for (int sweep = 0; sweep < 64; ++sweep) {
        bool rotated = false;
        for (int p = 0; p < M - 1; ++p)
            for (int q = p + 1; q < M; ++q) {
                double alpha = 0.0, beta = 0.0;
                cd gamma = 0.0;
                for (int r = 0; r < M; ++r) {
                    const cd ap = A[(size_t)r * M + p], aq = A[(size_t)r * M + q];
                    alpha += std::norm(ap);
                    beta += std::norm(aq);
                    gamma += std::conj(ap) * aq;
                }
                const double g = std::abs(gamma);
                if (!(g > 1e-15 * std::sqrt(alpha * beta))) continue;
                rotated = true;
                const cd ph = std::conj(gamma / g);  // a_q ph makes a_p^H a_q real and positive
                const double zeta = (beta - alpha) / (2.0 * g);
                const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / std::sqrt(1.0 + t * t), s = c * t;
                for (cd *X : {A.data(), V.data()})
                    for (int r = 0; r < M; ++r) {
                        const cd xp = X[(size_t)r * M + p], xq = X[(size_t)r * M + q] * ph;
                        X[(size_t)r * M + p] = c * xp - s * xq;
                        X[(size_t)r * M + q] = s * xp + c * xq;
                    }
            }
        if (!rotated) break;
    }
    std::vector<double> sig(M);
    double smax = 0.0, smin = INFINITY;
    for (int j = 0; j < M; ++j) {
        double s2 = 0.0;
        for (int r = 0; r < M; ++r) s2 += std::norm(A[(size_t)r * M + j]);
        sig[j] = std::sqrt(s2);
        smax = std::max(smax, sig[j]);
        smin = std::min(smin, sig[j]);
    }
    if (!(smin > FOCUS_SINGULAR * smax)) return false;
    for (int i = 0; i < M; ++i)
        for (int k = 0; k < M; ++k) {
            cd v = 0.0;
            for (int j = 0; j < M; ++j) v += A[(size_t)i * M + j] / sig[j] * std::conj(V[(size_t)k * M + j]);
            T[(size_t)i * M + k] = v;
        }
    return true;
}

}  // namespace music
