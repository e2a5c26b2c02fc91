// music_coarray.cuh - the difference co-array of a sparse linear array (music_b200_create_coarray): each window's
// physical covariance R (m x m) mapped to the spatially smoothed covariance R_ss (Mv x Mv) of the virtual uniform
// linear array the lags 0 .. Mv - 1 of the array fill (Pal & Vaidyanathan 2010; Liu & Vaidyanathan 2015).
//
// Definition (include/music_b200.h, restated literally by tests/coarray_oracle.py): for l = 0 .. Mv - 1 the pairs (i, j)
// with p_i - p_j = l in ascending i, c_l of them; z_l = (1 / c_l) sum R_ij over them in table order; T_ab = z_{a-b} for
// a >= b and conj(z_{b-a}) for a < b; R_ss = (1 / Mv) T T^H, each entry a sum over k ascending, computed for a >= b, the
// upper triangle its conjugate mirror, the diagonal real.
//
// Per call: coarray_kernel runs after the covariance, calibration and integration of a sub-batch, reading the physical R
// the handle keeps beside its workspace and writing R_ss into the workspace R, where every later stage reads it.  One
// warp per window: lane l < Mv sums lag l from the lag table (a kernel parameter: at most m (m + 1) / 2 pairs), z goes
// to shared memory, then the lanes share the Mv (Mv + 1) / 2 entries of the lower triangle, each Mv complex products
// long.  At Mv = 16 that is 136 entries, 16 x 136 complex FMAs per window.
#pragma once
#include "music_kernels.cuh"

namespace music {

constexpr int CO_MAX_PAIRS = MAXM * (MAXM + 1) / 2;  // pairs with p_i - p_j >= 0 of an m <= MAXM array
constexpr int CO_WARPS = 4;                          // windows per CTA of coarray_kernel

// The lag table built on the host at create: the pairs of lag l are pi / pj [start[l] .. start[l + 1]).
struct CoarrayLags {
    int mv = 0;
    unsigned char start[MAXM + 1] = {};
    unsigned char pi[CO_MAX_PAIRS] = {}, pj[CO_MAX_PAIRS] = {};
};

// R_phys [W][m][m] complex -> R_ss [W][Mv][Mv] complex
__global__ void __launch_bounds__(CO_WARPS * 32) coarray_kernel(const double2 *__restrict__ R_phys, int m, int W, const CoarrayLags lags,
                                                                double2 *__restrict__ R_ss)
{
    __shared__ double2 zs[CO_WARPS][MAXM];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * CO_WARPS + warp;
    if (w >= W) return;  // (whole warps: only __syncwarp below)
    const int mv = lags.mv;
    const double2 *R = R_phys + (size_t)w * m * m;
    double2 *z = zs[warp];
    if (lane < mv) {
        double sx = 0.0, sy = 0.0;
        const int q0 = lags.start[lane], q1 = lags.start[lane + 1];
        for (int q = q0; q < q1; ++q) {
            const double2 r = R[lags.pi[q] * m + lags.pj[q]];
            sx += r.x;
            sy += r.y;
        }
        const double c = (double)(q1 - q0);
        z[lane] = make_double2(sx / c, sy / c);
    }
    __syncwarp();
    const auto T = [&](int a, int b) {  // T_ab
        const double2 v = z[a >= b ? a - b : b - a];
        return a >= b ? v : make_double2(v.x, -v.y);
    };
    double2 *out = R_ss + (size_t)w * mv * mv;
    const int E = mv * (mv + 1) / 2;
    for (int e = lane; e < E; e += 32) {
        int a = 0;
        while ((a + 1) * (a + 2) / 2 <= e) ++a;
        const int b = e - a * (a + 1) / 2;
        double re = 0.0, im = 0.0;
        for (int k = 0; k < mv; ++k) {
            const double2 x = T(a, k), y = T(b, k);  // x conj(y)
            re += x.x * y.x + x.y * y.y;
            im += x.y * y.x - x.x * y.y;
        }
        re /= (double)mv;
        im = a == b ? 0.0 : im / (double)mv;
        out[a * mv + b] = make_double2(re, im);
        out[b * mv + a] = make_double2(re, -im);
    }
}

}  // namespace music
