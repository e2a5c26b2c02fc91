// music_manifold.cuh - gridless root-MUSIC on any planar array by manifold separation (opt-in peak mode
// MUSIC_B200_PEAKS_MANIFOLD).
//
// Each element's response over azimuth is periodic, and by Jacobi-Anger
//     conj(a_i(t)) a_j(t) = exp(-j x_ij cos(t - theta_ij)) = sum_l beta_ij,l e^{j l t},
//     beta_ij,l = (-j)^l J_l(x_ij) e^{-j l theta_ij},   x_ij = 2 pi rho_ij / lambda,
// with (rho_ij, theta_ij) the polar form of p_j - p_i.  The series converges super-exponentially, so the MUSIC
// denominator D(t) = a^H C a, C = G G^H, is to fp64 rounding the trigonometric polynomial sum_{|l| <= L} c_l e^{j l t}
//     c_0 = tr C + 2 sum_{i<j} beta_ij,0 Re C_ij,   c_l = sum_{i<j} beta_ij,l (2 Re C_ij, l even; 2 j Im C_ij, l odd),
// and Q(z) = sum_l c_l z^(l + L) has the directions as roots near the unit circle, arg z = t.  The roots come from
// ROOTS's root finder (roots_solve in music_roots.cuh); the full definition is in
// include/music_b200.h and is restated by tests/manifold_oracle.py.
//
// The order L and the table beta are built on the host with the geometry (manifold_coeffs_host); the kernel reads
// beta from global memory (<= 120 pairs x 65 orders x 16 B = 125 KB, L2-resident and shared by every window).
// One CTA of up to four warps per window, thread r <-> root r (P = 2L <= 128), everything fp64.
#pragma once
#include <cmath>
#include <vector>

#include "music_roots.cuh"

namespace music {

constexpr int MF_MAX_L = 64;               // order cap: an aperture of about 4.4 lambda
constexpr int MF_MAX_P = 2 * MF_MAX_L;     // roots per window
constexpr int MF_MAX_THREADS = MF_MAX_P;   // one thread per root

// ---- host: order and coefficient table ------------------------------------------------------------------------------

// The order L of a geometry of largest element distance rho_max: the smallest L >= 1 with L + 1 >= x and
// 4 tau_{L+1} <= 2^-52, x = 2 pi rho_max / lambda, tau_0 = 1, tau_l = tau_{l-1} (x / 2) / l (|J_l(y)| <= (y/2)^l / l!
// and, once l + 1 >= x, the terms at least halve, so the two-sided tail of every pair is <= 4 tau_{L+1}).  Where tau
// overflows (x > ~1400) L is far above the cap; the running product then continues in logs.
inline uint32_t manifold_order(double x)
{
    const double eps = 2.220446049250313e-16;
    if (!(x <= 1e7)) return 0xffffffffu;  // saturated: far above the cap (the loop below is O(x))
    double tau = x / 2.0;  // tau_1
    uint32_t L = 1;
    double ltau = 0.0;
    bool logd = false;
    for (;;) {
        // tau holds tau_L; tau_{L+1}:
        if (!logd) {
            const double nt = tau * (x / 2.0) / (double)(L + 1);
            if (std::isinf(nt)) {
                logd = true;
                ltau = std::log(tau) + std::log(x / 2.0) - std::log((double)(L + 1));
            } else {
                tau = nt;
            }
        } else {
            ltau += std::log(x / 2.0) - std::log((double)(L + 1));
        }
        const bool small = logd ? (std::log(4.0) + ltau <= std::log(eps)) : (4.0 * tau <= eps);
        if ((double)L + 1.0 >= x && small) return L;
        ++L;
    }
}

// J_0(x) .. J_L(x) for x >= 0 by Miller's backward recurrence, normalised by J_0 + 2 sum_k J_2k = 1: about 1e-16
// absolute at every order (glibc jn is not guaranteed to be at high orders).
inline void bessel_j_all(double x, int L, double *J)
{
    for (int l = 0; l <= L; ++l) J[l] = 0.0;
    if (x < 1e-5) {  // two terms of the power series: relative error below (x/2)^4 / 2
        double term = 1.0;
        for (int l = 0; l <= L; ++l) {
            if (l) term *= (x / 2.0) / l;
            J[l] = term * (1.0 - (x / 2.0) * (x / 2.0) / (l + 1));
        }
        return;
    }
    const int top = std::max(L, (int)std::ceil(x));
    int N = top + 40 + (int)std::sqrt(40.0 * top);
    N += N & 1;  // even start
    std::vector<double> j(N + 2, 0.0);
    j[N + 1] = 0.0;
    j[N] = 1e-300;
    double norm = 0.0;  // J_0 + 2 sum J_2k, as the recurrence runs
    for (int k = N; k >= 1; --k) {
        j[k - 1] = (2.0 * k / x) * j[k] - j[k + 1];
        if (std::fabs(j[k - 1]) > 1e250) {  // rescale what is computed so far
            for (int i = k - 1; i <= N; ++i) j[i] *= 1e-250;
            norm *= 1e-250;
        }
        if (k % 2 == 0) norm += 2.0 * j[k];
    }
    norm += j[0];
    for (int l = 0; l <= L; ++l) J[l] = j[l] / norm;
}

// The order L of positions [M][x, y] (metres) at wavelength lambda and, when beta is not null and L <= MF_MAX_L, the
// table beta [M(M-1)/2][L+1] (complex, pairs (0,1), (0,2), .., (M-2, M-1)).  Returns false when L > MF_MAX_L (L is
// written either way); *aperture (may be null) = rho_max / lambda.
inline bool manifold_coeffs_host(const double *pos, int M, double lambda, uint32_t *L_out, double *beta, double *aperture)
{
    double rho_max = 0.0;
    for (int i = 0; i < M; ++i)
        for (int j = i + 1; j < M; ++j) rho_max = std::max(rho_max, std::hypot(pos[2 * j] - pos[2 * i], pos[2 * j + 1] - pos[2 * i + 1]));
    const double x = STEER_TWO_PI * rho_max / lambda;
    const uint32_t L = manifold_order(x);
    *L_out = L;
    if (aperture) *aperture = rho_max / lambda;
    if (L > (uint32_t)MF_MAX_L) return false;
    if (!beta) return true;
    double J[MF_MAX_L + 1];
    size_t q = 0;
    for (int i = 0; i < M; ++i)
        for (int j = i + 1; j < M; ++j, ++q) {
            const double dx = pos[2 * j] - pos[2 * i], dy = pos[2 * j + 1] - pos[2 * i + 1];
            const double rho = std::hypot(dx, dy), th = std::atan2(dy, dx);
            bessel_j_all(STEER_TWO_PI * rho / lambda, (int)L, J);
            for (uint32_t l = 0; l <= L; ++l) {
                const double c = std::cos(l * th), s = -std::sin(l * th);  // e^{-j l theta}
                double re = J[l] * c, im = J[l] * s;
                switch (l & 3) {  // (-j)^l
                case 1: { const double t = re; re = im; im = -t; break; }
                case 2: re = -re; im = -im; break;
                case 3: { const double t = re; re = -im; im = t; break; }
                default: break;
                }
                double *b = beta + 2 * (q * (L + 1) + l);
                b[0] = re;
                b[1] = im;
            }
        }
    return true;
}

// threads of a window's CTA: one per root, whole warps
inline int manifold_threads(int L) { return (2 * L + 31) / 32 * 32; }

// ---- device: one CTA per window -------------------------------------------------------------------------------------

// Vt: per window M * M complex doubles, eigenvector j contiguous, ascending eigenvalues; counts (may be null): the
// per-window source count d (else d = n).  beta: the table of the current geometry, order L (1 .. MF_MAX_L).  Launched
// with manifold_threads(L) threads per CTA, one CTA per window.
__global__ void __launch_bounds__(MF_MAX_THREADS) manifold_kernel(const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                                  int M, int n, int K, const RefineGeom geo,
                                                                  const double2 *__restrict__ beta, int L, PeakOut out)
{
    __shared__ double2 Cs[MAXM * MAXM];  // C = G G^H, upper triangle
    __shared__ RootsShared<MF_MAX_L> sh;

    const int w = blockIdx.x, r = threadIdx.x, NT = blockDim.x;
    const int d = counts ? counts[w] : n;
    const int p = M - d;
    const double2 *G = reinterpret_cast<const double2 *>(Vt) + (size_t)w * M * M;

    // C_ij = sum_k g_k[i] conj(g_k[j]), i <= j
    for (int e = r; e < M * M; e += NT) {
        const int i = e / M, j = e - i * M;
        if (i > j) continue;
        double2 c = make_double2(0.0, 0.0);
        for (int k = 0; k < p; ++k) {
            const double2 a = G[k * M + i], b = G[k * M + j];
            c.x += a.x * b.x + a.y * b.y;
            c.y += a.y * b.x - a.x * b.y;
        }
        Cs[e] = c;
    }
    __syncthreads();
    // thread l <= L: c_l
    if (r <= L) {
        double2 c = make_double2(0.0, 0.0);
        if (r == 0)
            for (int i = 0; i < M; ++i) c.x += Cs[i * M + i].x;
        int q = 0;
        for (int i = 0; i < M; ++i)
            for (int j = i + 1; j < M; ++j, ++q) {
                const double2 b = beta[(size_t)q * (L + 1) + r], Cij = Cs[i * M + j];
                if (r & 1) {  // b * 2j Im C_ij
                    c.x -= 2.0 * Cij.y * b.y;
                    c.y += 2.0 * Cij.y * b.x;
                } else {      // b * 2 Re C_ij
                    c.x += 2.0 * Cij.x * b.x;
                    c.y += 2.0 * Cij.x * b.y;
                }
            }
        roots_set_coeff(sh, r, c);
    }
    // t* = arg z in [0, 360) degrees
    const RootSlot rs = roots_solve(sh, L, d, [](double2 z) {
        const double t = atan2(z.y, z.x) * REFINE_RAD2DEG;
        return t < 0.0 ? t + 360.0 : t;
    });
    if (rs.slot >= 0) {
        const size_t o = (size_t)w * n + rs.slot;
        if (rs.z.x == 0.0 && rs.z.y == 0.0) {  // a kept root at 0 has no direction
            peak_write(out, o, -1, 0.0, K);
        } else {
            double D, D1, D2;
            refine_eval(geo, G, M, p, rs.tdeg * STEER_DEG2RAD, &D, &D1, &D2);
            ula_store_slot(out, o, rs.tdeg, D, K);
        }
    }
    if (r >= rs.f && r < n) peak_write(out, (size_t)w * n + r, -1, 0.0, K);
}

}  // namespace music
