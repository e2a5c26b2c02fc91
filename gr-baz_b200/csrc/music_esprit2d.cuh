// music_esprit2d.cuh - 2-D LS-ESPRIT for planar lattice arrays on az-el handles (peak mode MUSIC_B200_PEAKS_ESPRIT).
//
// On a lattice p_m(i, k) = p_0 + i s1 + k s2 (element m = k Mx + i) the steering vectors satisfy two shift invariances,
// one per lattice step: for the doublets P_j (pairs of elements one step s_j apart) B_j = A_j diag(phi_j) with
// phi_j = exp(-j 2 pi (s_j . u) / lambda).  The d signal eigenvectors E_s span the same columns, so with A_j / B_j the
// rows of E_s at the first / second elements of P_j, Psi_j = (A_j^H A_j)^-1 A_j^H B_j = T^-1 diag(phi_j) T with one T
// for both j.  The eigenvectors of Psi_c = Psi_1 + gamma Psi_2 (gamma non-real, |gamma| != 1) are the columns of T^-1,
// and their Rayleigh quotients under Psi_1 and Psi_2 give each source's two phases already paired: no grid, no scan and
// no 2-D peak pick.  The full definition (lattice condition, pairing, angles, levels, bins, slot order) is in
// include/music_b200.h and is restated by tests/esprit2d_oracle.py.
//
// One warp per window; every d x d matrix (d <= ESP2_MAXD) lives in the warp's shared memory, lanes over entries and
// columns as in esprit_kernel.  Everything is fp64.
#pragma once
#include <cmath>

#include "music_azel.cuh"
#include "music_esprit.cuh"
#include "music_warp_la.cuh"

namespace music {

// The lattice condition's result for one geometry (azel_lattice), passed by value like AzelGeom.
struct LatticeGeom {
    int ok;          // 1: the positions form an Mx x My lattice the mode accepts
    int mx, my;      // elements along s1, along s2 (M = mx * my)
    double s1[2];    // (p_1 - p_0)_xy, metres
    double s2[2];    // (p_mx - p_0)_xy, metres
};

constexpr int ESP2_WARPS = 3;     // 3 x 13.5 KB of static shared memory per CTA
constexpr int ESP2_MAXD = 12;     // the largest d_max for M <= 16 (a 4 x 4 lattice)
constexpr double ESP2_PIVOT = 9.094947017729282e-13;  // 2^-40: a Cholesky pivot of A_j^H A_j at most this gives no peaks
constexpr double ESP2_GAMMA_RE = 0.37, ESP2_GAMMA_IM = 0.61;  // gamma of Psi_c = Psi_1 + gamma Psi_2 (DESIGN.md section 5)
constexpr double ESP2_SMIN_REL = 2.220446049250313e-16;       // 2^-52: ztrevc's smin = max(2^-52 |S_kk|, 2^-1022)
constexpr double ESP2_SMIN_ABS = 2.2250738585072014e-308;     // 2^-1022

// d_max = min((Mx - 1) My, Mx (My - 1)): the doublet count of the shorter invariance
__host__ __device__ inline int esp2_dmax(const LatticeGeom &g) { return min((g.mx - 1) * g.my, g.mx * (g.my - 1)); }

// The lattice condition (include/music_b200.h) on positions [M][x, y, z]: the first divisor Mx of M (2 <= Mx <= M / 2)
// with s1 = (p_1 - p_0)_xy and s2 = (p_Mx - p_0)_xy non-zero and independent, every element within
// 1e-6 min(|s1|, |s2|) of p_0 + i s1 + k s2 in xy and of z_0 in z, and |s1|, |s2| <= (lambda / 2)(1 + 1e-12).
inline LatticeGeom azel_lattice(const double *pos, int M, double lambda)
{
    LatticeGeom g = {};
    for (int mx = 2; mx <= M / 2; ++mx) {
        if (M % mx) continue;
        const int my = M / mx;
        const double s1[2] = {pos[3] - pos[0], pos[4] - pos[1]};
        const double s2[2] = {pos[3 * mx] - pos[0], pos[3 * mx + 1] - pos[1]};
        const double a1 = std::hypot(s1[0], s1[1]), a2 = std::hypot(s2[0], s2[1]);
        if (!(a1 > 0.0 && a2 > 0.0)) continue;
        if (!(std::fabs(s1[0] * s2[1] - s1[1] * s2[0]) > 1e-6 * a1 * a2)) continue;
        const double tol = 1e-6 * std::min(a1, a2);
        bool fit = true;
        for (int m = 0; m < M && fit; ++m) {
            const int k = m / mx, i = m - k * mx;
            const double ex = pos[0] + i * s1[0] + k * s2[0], ey = pos[1] + i * s1[1] + k * s2[1];
            fit = std::hypot(pos[3 * m] - ex, pos[3 * m + 1] - ey) <= tol && std::fabs(pos[3 * m + 2] - pos[2]) <= tol;
        }
        if (!fit) continue;
        if (!(a1 <= 0.5 * lambda * (1.0 + 1e-12) && a2 <= 0.5 * lambda * (1.0 + 1e-12))) continue;
        g.ok = 1;
        g.mx = mx;
        g.my = my;
        g.s1[0] = s1[0], g.s1[1] = s1[1], g.s2[0] = s2[0], g.s2[1] = s2[1];
        return g;
    }
    return g;
}

// Psi_j = (A_j^H A_j)^-1 A_j^H B_j into P (row stride d), by the whole warp; Gs (row stride d) is scratch.  Doublet
// (f, f + step) for every first element f = k Mx + i with i < i_end, k < k_end, in ascending f.  False when a Cholesky
// pivot is <= 2^-40 (or NaN) or Psi_j is not finite.
__device__ bool esp2_psi(const double2 *__restrict__ Es, int M, int d, int mx, int i_end, int k_end, int step, double2 *P,
                         double2 *Gs, int lane)
{
    for (int e = lane; e < d * d; e += 32) {
        const int a = e / d, b = e - a * d;
        double2 g = make_double2(0.0, 0.0), c = make_double2(0.0, 0.0);
        for (int k = 0; k < k_end; ++k)
            for (int i = 0; i < i_end; ++i) {
                const int f = k * mx + i;
                const double2 ea = cconj(Es[a * M + f]);
                g = cadd(g, cmul(ea, Es[b * M + f]));
                c = cadd(c, cmul(ea, Es[b * M + f + step]));
            }
        Gs[e] = g;
        P[e] = c;
    }
    __syncwarp();
    const bool ok = warp_cholesky(Gs, d, lane, [](int, double p) { return p > ESP2_PIVOT; });
    __syncwarp();
    bool fin = true;
    if (ok && lane < d) {  // column `lane` of C: L L^H x = c
        const int b = lane;
        for (int k = 0; k < d; ++k) {
            double2 s = P[k * d + b];
            for (int q = 0; q < k; ++q) s = csub(s, cmul(Gs[k * d + q], P[q * d + b]));
            P[k * d + b] = cscale(s, 1.0 / Gs[k * d + k].x);
        }
        for (int k = d - 1; k >= 0; --k) {
            double2 s = P[k * d + b];
            for (int q = k + 1; q < d; ++q) s = csub(s, cmul(cconj(Gs[q * d + k]), P[q * d + b]));
            P[k * d + b] = cscale(s, 1.0 / Gs[k * d + k].x);
            fin = fin && isfinite(P[k * d + b].x) && isfinite(P[k * d + b].y);
        }
    }
    __syncwarp();
    return __all_sync(0xffffffffu, ok && fin);
}

// Vt: per window M * M complex doubles, eigenvector j contiguous, ascending eigenvalues; counts (may be null): the
// per-window source count d (else d = n).  The signal subspace is eigenvectors M - d .. M - 1, the noise subspace (the
// level's D) eigenvectors 0 .. M - d - 1, as in the scan.  Writes azimuths, elevations, levels and bins (no decode).
__global__ void __launch_bounds__(ESP2_WARPS * 32) esprit2d_kernel(const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                                   int M, int n, int W, const AzelGeom geo, const LatticeGeom lat,
                                                                   PeakOut out, float *__restrict__ elev)
{
    constexpr int D2 = ESP2_MAXD * ESP2_MAXD;
    __shared__ double2 sP1[ESP2_WARPS][D2], sP2[ESP2_WARPS][D2], sX[ESP2_WARPS][D2];  // Psi_1, Psi_2 and the eigenvectors
    __shared__ double2 sS[ESP2_WARPS][ESP2_MAXD * ESPRIT_LD], sZ[ESP2_WARPS][ESP2_MAXD * ESPRIT_LD];  // Psi_c -> S, Z
    __shared__ double2 sv[ESP2_WARPS][ESP2_MAXD], sg[ESP2_WARPS][ESP2_MAXD], sev[ESP2_WARPS][ESP2_MAXD];
    const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int w = blockIdx.x * ESP2_WARPS + wi;
    if (w >= W) return;
    const int d = counts ? counts[w] : n;
    const int p = M - d;
    const double2 *G = reinterpret_cast<const double2 *>(Vt) + (size_t)w * M * M;
    const double2 *Es = G + (size_t)p * M;  // Es[a * M + i] = row i of signal eigenvector a
    double2 *P1 = sP1[wi], *P2 = sP2[wi], *X = sX[wi], *S = sS[wi], *Z = sZ[wi];
    const int mx = lat.mx, my = lat.my;

    bool ok = d > 0 && d <= esp2_dmax(lat);
    if (ok) ok = esp2_psi(Es, M, d, mx, mx - 1, my, 1, P1, Z, lane);       // P1: (m(i, k), m(i + 1, k))
    if (ok) ok = esp2_psi(Es, M, d, mx, mx, my - 1, mx, P2, Z, lane);      // P2: (m(i, k), m(i, k + 1))
    if (ok) {
        const double2 gam = make_double2(ESP2_GAMMA_RE, ESP2_GAMMA_IM);
        for (int e = lane; e < d * d; e += 32) {
            const int a = e / d, b = e - a * d;
            S[a * ESPRIT_LD + b] = cadd(P1[e], cmul(gam, P2[e]));
            Z[a * ESPRIT_LD + b] = make_double2(a == b ? 1.0 : 0.0, 0.0);
        }
        __syncwarp();
        ok = esprit_eigvals<true>(S, sv[wi], sg[wi], sev[wi], d, lane, Z);
    }
    __syncwarp();
    // lane k < d: eigenvector k of the triangular S (y_k = 1, ztrevc's back-substitution) into the strict lower
    // triangle of row k of S, then x_k = Z y into row k of X
    if (ok && lane < d) {
        const int k = lane;
        const double2 skk = S[k * ESPRIT_LD + k];
        const double smin = fmax(ESP2_SMIN_REL * sqrt(cabs2(skk)), ESP2_SMIN_ABS);
        for (int j = k - 1; j >= 0; --j) {
            double2 s = S[j * ESPRIT_LD + k];  // y_k = 1
            for (int l = j + 1; l < k; ++l) s = cadd(s, cmul(S[j * ESPRIT_LD + l], S[k * ESPRIT_LD + l]));
            double2 den = csub(S[j * ESPRIT_LD + j], skk);
            if (sqrt(cabs2(den)) < smin) den = make_double2(smin, 0.0);
            S[k * ESPRIT_LD + j] = cscale(cdiv(s, den), -1.0);
        }
        for (int m = 0; m < d; ++m) {
            double2 x = Z[m * ESPRIT_LD + k];
            for (int j = 0; j < k; ++j) x = cadd(x, cmul(Z[m * ESPRIT_LD + j], S[k * ESPRIT_LD + j]));
            X[k * d + m] = x;
        }
    }
    __syncwarp();

    // lane k < d: the Rayleigh quotients phi_1, phi_2 of x_k -> direction, level
    double az = 0.0, el = 0.0, lvl = 0.0;
    bool filled = false;
    if (ok && lane < d) {
        const double2 *x = X + lane * d;
        double xn = 0.0;
        double2 q1 = make_double2(0.0, 0.0), q2 = make_double2(0.0, 0.0);
        for (int a = 0; a < d; ++a) {
            double2 t1 = make_double2(0.0, 0.0), t2 = make_double2(0.0, 0.0);
            for (int b = 0; b < d; ++b) {
                t1 = cadd(t1, cmul(P1[a * d + b], x[b]));
                t2 = cadd(t2, cmul(P2[a * d + b], x[b]));
            }
            xn += cabs2(x[a]);
            q1 = cadd(q1, cmul(cconj(x[a]), t1));
            q2 = cadd(q2, cmul(cconj(x[a]), t2));
        }
        const double2 f1 = cscale(q1, 1.0 / xn), f2 = cscale(q2, 1.0 / xn);
        filled = isfinite(f1.x) && isfinite(f1.y) && isfinite(f2.x) && isfinite(f2.y) && (f1.x != 0.0 || f1.y != 0.0) &&
                 (f2.x != 0.0 || f2.y != 0.0);
        if (filled) {
            // omega_j = -arg(phi_j) lambda / (2 pi) = s_j . u_xy; [s1; s2] u_xy = omega
            const double w1 = -atan2(f1.y, f1.x) * geo.lambda / STEER_TWO_PI, w2 = -atan2(f2.y, f2.x) * geo.lambda / STEER_TWO_PI;
            const double det = lat.s1[0] * lat.s2[1] - lat.s1[1] * lat.s2[0];
            const double ux = (w1 * lat.s2[1] - w2 * lat.s1[1]) / det, uy = (w2 * lat.s1[0] - w1 * lat.s2[0]) / det;
            az = fmod(atan2(uy, ux) * REFINE_RAD2DEG, 360.0);
            if (az < 0.0) az += 360.0;
            el = acos(fmin(hypot(ux, uy), 1.0)) * REFINE_RAD2DEG;
            if (geo.grid.el_hi <= 0.0) el = -el;
            double e[6];
            azel_eval(geo, G, M, p, az * STEER_DEG2RAD, el * STEER_DEG2RAD, e);
            lvl = 1.0 / e[0];
        }
    }
    ok = ok && __all_sync(0xffffffffu, lane >= d || !isnan(lvl));
    filled = filled && ok;
    // slot = rank in descending fp64 level, ties to the lower azimuth, then the lower elevation, then the lower Schur
    // diagonal index
    int r = 0;
    for (int s = 0; s < d; ++s) {
        const bool fs = __shfl_sync(0xffffffffu, filled, s);
        const double ls = __shfl_sync(0xffffffffu, lvl, s), as = __shfl_sync(0xffffffffu, az, s), es = __shfl_sync(0xffffffffu, el, s);
        if (fs && (ls > lvl || (ls == lvl && (as < az || (as == az && (es < el || (es == el && s < lane))))))) ++r;
    }
    const int f = __popc(__ballot_sync(0xffffffffu, filled));
    const AzelGrid &gr = geo.grid;
    if (filled) {
        const size_t o = (size_t)w * n + r;
        float fa = (float)az;
        if (fa >= 360.0f || fa == 0.0f) fa = 0.0f;
        out.angles[o] = fa;
        elev[o] = (float)el;
        if (out.levels) out.levels[o] = (float)lvl;
        int k = (int)floor(az * (double)gr.n_az / 360.0 + 0.5);
        if (k >= gr.n_az) k -= gr.n_az;
        int i = 0;
        if (gr.n_el > 1) {
            i = (int)floor((el - gr.el_lo) * (double)(gr.n_el - 1) / (gr.el_hi - gr.el_lo) + 0.5);
            i = min(max(i, 0), gr.n_el - 1);
        }
        peak_store_bin(out, o, i * gr.n_az + k);
    }
    if (lane >= f && lane < n) {
        const size_t o = (size_t)w * n + lane;
        peak_write(out, o, -1, 0.0, 1);
        elev[o] = 0.f;
    }
}

}  // namespace music
