// music_wsf.cuh - weighted subspace fitting (opt-in peak mode MUSIC_B200_PEAKS_WSF) and the joint Gauss-Newton
// refinement of the DML and WSF angles (MUSIC_B200_REFINE_JOINT).
//
// WSF (Viberg, Ottersten & Kailath 1991) maximises tr(P_A X) with X = sum_i w_i e_i e_i^H over the d signal
// eigenvectors, w_i = (l_i - s2)^2 / l_i.  It has DML's criterion with X in place of R, so wsf_x_kernel forms X and
// dml_kernel (music_dml.cuh) searches it.  Its large-sample variance is the stochastic CRB, and a coherent path's
// surplus eigenvector has l_i ~ s2, so its weight vanishes and no smoothing is needed.
//
// joint_kernel refines all d filled slots of a window together: Gauss-Newton on V(t) = Re tr(P_perp(t) X) over the
// analytic steering of the geometry, from the grid angles, inside the box |t_i - t_b,i| <= 360 / K degrees.  V is
// evaluated as ||P_perp F||_F^2 with a factor X = F F^H (WSF: the columns sqrt(w_i) e_i; DML: the Cholesky factor of R),
// so that it keeps its relative accuracy where V is small and the line search can still tell two iterates apart.
// With A = Q T (modified Gram-Schmidt twice, as the CRB) and G = T^-1 Q^H F = A^+ F:
//   g_i = -2 Re sum_c G_ic ((P_perp F)^H (P_perp D))_ci,   H_ij = 2 Re(B_ij Z_ji),  B = (P_perp D)^H (P_perp D),  Z = G G^H.
// The full definitions are in include/music_b200.h and are restated by tests/wsf_oracle.py.
#pragma once
#include "music_kernels.cuh"
#include "music_refine.cuh"
#include "music_warp_la.cuh"

namespace music {

constexpr int WSF_X_THREADS = 256;
constexpr int JOINT_MAX_STEPS = 50;
constexpr int JOINT_MAX_HALVINGS = 30;
constexpr double JOINT_TOL = 1e-12;          // radians: stop once every entry of a Gauss-Newton step is this small
constexpr double JOINT_T_REL = 0x1p-30;      // |T_ll|^2 (pivot l of A^H A) must exceed this fraction of ||a_l||^2
constexpr double JOINT_H_REL = 0x1p-40;      // pivot k of H must exceed this fraction of H_kk

// The WSF weights of one window from its ascending eigenvalues l[0 .. M-1]: w[i] for i = M-d .. M-1.  Returns false
// when the window has no X: d = 0, l_0 <= 0, a non-finite eigenvalue, or every weight 0 (tr X = 0).
__device__ __forceinline__ bool wsf_weights(const double *__restrict__ l, int M, int d, double *w)
{
    if (d <= 0) return false;
    bool ok = l[0] > 0.0;
    for (int i = 0; i < M; ++i) ok = ok && isfinite(l[i]);
    if (!ok) return false;
    double s = 0.0;
    for (int i = 0; i < M - d; ++i) s += l[i];
    const double s2 = s / (double)(M - d);
    bool any = false;
    for (int i = M - d; i < M; ++i) {
        const double e = l[i] - s2;
        w[i] = l[i] > s2 ? e * e / l[i] : 0.0;
        any = any || w[i] > 0.0;
    }
    return any;
}

// X [W][M][M] (re, im) of W windows from the eigenvalues ev [W][M] and eigenvectors Vt [W][M][M] (vector j contiguous,
// ascending) of the eigensolver; counts (may be null): d per window, else n.  One thread per entry; a window without X
// gets X = 0, which dml_kernel reports as a window with no peaks (tr X <= 0).
__global__ void __launch_bounds__(WSF_X_THREADS) wsf_x_kernel(const double *__restrict__ ev, const double *__restrict__ Vt,
                                                              const int32_t *__restrict__ counts, int M, int n, int W,
                                                              double *__restrict__ X)
{
    const int MM = M * M;
    const long long t = (long long)blockIdx.x * WSF_X_THREADS + threadIdx.x;
    if (t >= (long long)W * MM) return;
    const int w = (int)(t / MM), e = (int)(t - (long long)w * MM), i = e / M, j = e - i * M;
    const int d = counts ? counts[w] : n;
    double wt[MAXM];
    double2 s = make_double2(0.0, 0.0);
    if (wsf_weights(ev + (size_t)w * M, M, d, wt)) {
        const double2 *E = reinterpret_cast<const double2 *>(Vt) + (size_t)w * MM;
        for (int k = M - d; k < M; ++k) {
            const double2 t2 = cmul(E[k * M + i], make_double2(E[k * M + j].x, -E[k * M + j].y));
            s.x += wt[k] * t2.x;
            s.y += wt[k] * t2.y;
        }
    }
    reinterpret_cast<double2 *>(X)[t] = s;
}

// Shared memory of one joint_kernel window (one warp per CTA), in double2 units
__host__ __device__ constexpr int joint_smem_elems(int M, int n)
{
    // R, F, P_perp F (M x M each); A, D, Q, T (n x MAXM each); Q^H F, G (n x M each); T^-1, H (n x n each); then the
    // real vectors (angles, box, step, trial, gradient, norms, pivot scales, levels: 8 x n doubles)
    return 3 * M * M + 4 * n * MAXM + 2 * n * M + 2 * n * n + 4 * n;
}

// Slots o = w * n + i with bins[o] >= 0 of W windows: angles and levels (levels may be null) become JOINT's.  R [W][M][M]
// the covariance the levels are taken from.  WSF: ev, Vt (and counts) give F; DML (ev null): F = chol(R).  A window
// whose F does not exist (WSF without X, a DML R that is not positive definite) or whose A^H A at the grid angles is not
// positive definite keeps what the peak stage wrote.
__global__ void __launch_bounds__(32) joint_kernel(const double *__restrict__ R, const double *__restrict__ ev,
                                                   const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                   const int32_t *__restrict__ bins, int M, int n, int K, const RefineGeom geo,
                                                   float *__restrict__ angles, float *__restrict__ levels)
{
    extern __shared__ double2 joint_smem[];
    const int lane = threadIdx.x, w = blockIdx.x, MM = M * M;
    double2 *sR = joint_smem, *sF = sR + MM, *sPF = sF + MM, *sA = sPF + MM, *sD = sA + n * MAXM, *sQ = sD + n * MAXM,
            *sT = sQ + n * MAXM, *sQF = sT + n * MAXM, *sG = sQF + n * M, *sTi = sG + n * M, *sH = sTi + n * n;
    double *vec = reinterpret_cast<double *>(sH + n * n);
    double *sTh = vec, *sTb = vec + n, *sS = vec + 2 * n, *sTr = vec + 3 * n, *sGr = vec + 4 * n, *sNa = vec + 5 * n,
           *sHd = vec + 6 * n, *sP = vec + 7 * n;

    const int b = lane < n ? bins[(size_t)w * n + lane] : -1;
    const bool filled = b >= 0;
    const unsigned fmask = __ballot_sync(0xffffffffu, filled);
    const int d = __popc(fmask);
    if (d == 0) return;
    const int r = __popc(fmask & ((1u << lane) - 1u));  // a filled lane's column among the filled slots
    const double deg_b = (double)b * 360.0 / (double)K;
    const double delta = (360.0 / (double)K) * STEER_DEG2RAD;
    if (filled) sTh[r] = sTb[r] = deg_b * STEER_DEG2RAD;

    // R, and the factor F (columns stride M) with its column count nc
    const double2 *Rw = reinterpret_cast<const double2 *>(R) + (size_t)w * MM;
    for (int e = lane; e < MM; e += 32) sR[e] = Rw[e];
    int nc = 0;
    bool ok = true;
    if (ev) {
        double wt[MAXM];
        ok = wsf_weights(ev + (size_t)w * M, M, counts ? counts[w] : n, wt);
        const double2 *E = reinterpret_cast<const double2 *>(Vt) + (size_t)w * MM;
        for (int k = M - (counts ? counts[w] : n); ok && k < M; ++k) {
            if (!(wt[k] > 0.0)) continue;
            const double sw = sqrt(wt[k]);
            if (lane < M) sF[nc * M + lane] = make_double2(sw * E[k * M + lane].x, sw * E[k * M + lane].y);
            ++nc;
        }
    } else {
        for (int e = lane; e < MM; e += 32) sF[e] = Rw[e];  // row-major R, factored in place: L[i][j] at i * M + j
        __syncwarp();
        ok = warp_cholesky(sF, M, lane, [](int, double p) { return p > 0.0; });
        __syncwarp();
        if (ok && lane < M)  // column c of L into sPF, then back: F[c][m] = L[m][c] for m >= c, else 0
            for (int c = 0; c < M; ++c) sPF[c * M + lane] = lane >= c ? sF[lane * M + c] : make_double2(0.0, 0.0);
        __syncwarp();
        for (int e = lane; ok && e < MM; e += 32) sF[e] = sPF[e];
        nc = M;
    }
    __syncwarp();
    if (!ok) return;

    // V at the angles sTh (or sTr): A, Q T, P_perp F; with grad also T^-1, P_perp D, G = A^+ F, the gradient sGr and H.
    // Returns whether A^H A passed its pivot test; V in *V (the same value on every lane).
    const auto eval = [&](const double *th, bool grad, double *V) -> bool {
        if (lane < d) {
            double st, ct, na = 0.0;
            sincos(th[lane], &st, &ct);
            for (int m = 0; m < M; ++m) {
                double phi, psi, sp, cp;
                steer_phase(geo, m, st, ct, &phi, &psi);
                sincos(phi, &sp, &cp);
                sA[lane * MAXM + m] = make_double2(cp, -sp);
                sD[lane * MAXM + m] = make_double2(-psi * sp, -psi * cp);  // -j psi a
                na += cp * cp + sp * sp;
            }
            sNa[lane] = na;
        }
        __syncwarp();
        mgs2([&](int l, int i) { return sA[l * MAXM + i]; }, d, M, sQ, sT, lane);
        bool good = true;
        for (int l = 0; l < d; ++l) {
            const double t = sT[l * MAXM + l].x;
            good = good && t * t > JOINT_T_REL * sNa[l];
        }
        if (!good) return false;
        // P_perp F column by column, twice, and Q^H F (the sum of both passes' coefficients) into sQF
        double v2 = 0.0;
        for (int c = 0; c < nc; ++c) {
            double2 v = lane < M ? sF[c * M + lane] : make_double2(0.0, 0.0);
            for (int pass = 0; pass < 2; ++pass)
                for (int l = 0; l < d; ++l) {
                    const double2 q = lane < M ? sQ[l * MAXM + lane] : make_double2(0.0, 0.0);
                    const double2 t = cjmul(q, v);
                    const double2 k = make_double2(warp_sum(t.x), warp_sum(t.y));
                    v.x -= k.x * q.x - k.y * q.y;
                    v.y -= k.x * q.y + k.y * q.x;
                    if (lane == 0) {
                        double2 &f = sQF[l * M + c];
                        f = pass ? make_double2(f.x + k.x, f.y + k.y) : k;
                    }
                }
            if (lane < M) sPF[c * M + lane] = v;
            v2 += warp_sum(v.x * v.x + v.y * v.y);
        }
        *V = v2;
        __syncwarp();
        if (!grad) return true;
        triu_inverse(sT, MAXM, sTi, d, d, lane);  // T^-1 (upper triangular), column c by lane c
        // P_perp D, twice, in place
        for (int c = 0; c < d; ++c) {
            double2 v = lane < M ? sD[c * MAXM + lane] : make_double2(0.0, 0.0);
            for (int pass = 0; pass < 2; ++pass)
                for (int l = 0; l < d; ++l) {
                    const double2 q = lane < M ? sQ[l * MAXM + lane] : make_double2(0.0, 0.0);
                    const double2 t = cjmul(q, v);
                    const double2 k = make_double2(warp_sum(t.x), warp_sum(t.y));
                    v.x -= k.x * q.x - k.y * q.y;
                    v.y -= k.x * q.y + k.y * q.x;
                }
            if (lane < M) sD[c * MAXM + lane] = v;
        }
        __syncwarp();
        // G = T^-1 (Q^H F), row i by lane i
        if (lane < d) {
            const int i = lane;
            for (int c = 0; c < nc; ++c) {
                double2 s = make_double2(0.0, 0.0);
                for (int k = i; k < d; ++k) {
                    const double2 t = cmul(sTi[i * d + k], sQF[k * M + c]);
                    s.x += t.x;
                    s.y += t.y;
                }
                sG[i * M + c] = s;
            }
        }
        __syncwarp();
        // g_i = -2 Re sum_c G_ic (P_perp F)_c^H (P_perp D)_i, lane i
        if (lane < d) {
            const int i = lane;
            double g = 0.0;
            for (int c = 0; c < nc; ++c) {
                double yr = 0.0, yi = 0.0;
                for (int m = 0; m < M; ++m) {
                    const double2 t = cjmul(sPF[c * M + m], sD[i * MAXM + m]);
                    yr += t.x;
                    yi += t.y;
                }
                const double2 gc = sG[i * M + c];
                g += gc.x * yr - gc.y * yi;
            }
            sGr[i] = -2.0 * g;
        }
        // H_ij = 2 Re(B_ij Z_ji), B = (P_perp D)^H (P_perp D), Z = G G^H
        for (int e = lane; e < d * d; e += 32) {
            const int i = e / d, j = e - i * d;
            double br = 0.0, bi = 0.0, zr = 0.0, zi = 0.0;
            for (int m = 0; m < M; ++m) {
                const double2 t = cjmul(sD[i * MAXM + m], sD[j * MAXM + m]);
                br += t.x;
                bi += t.y;
            }
            for (int c = 0; c < nc; ++c) {  // Z_ji = sum_c G_jc conj(G_ic)
                const double2 t = cjmul(sG[i * M + c], sG[j * M + c]);
                zr += t.x;
                zi += t.y;
            }
            const double h = 2.0 * (br * zr - bi * zi);
            sH[e] = make_double2(h, 0.0);
            if (i == j) sHd[i] = h;
        }
        __syncwarp();
        return true;
    };

    double V;
    if (!eval(sTh, true, &V)) return;
    for (int it = 0; it < JOINT_MAX_STEPS; ++it) {
        if (!warp_cholesky(sH, d, lane, [&](int k, double p) { return p > 0.0 && p > JOINT_H_REL * sHd[k]; })) break;
        __syncwarp();
        if (lane == 0) {  // s = -H^-1 g: L y = -g, then L^T s = y
            for (int k = 0; k < d; ++k) {
                double s = -sGr[k];
                for (int q = 0; q < k; ++q) s -= sH[k * d + q].x * sS[q];
                sS[k] = s / sH[k * d + k].x;
            }
            for (int k = d - 1; k >= 0; --k) {
                double s = sS[k];
                for (int q = k + 1; q < d; ++q) s -= sH[q * d + k].x * sS[q];
                sS[k] = s / sH[k * d + k].x;
            }
        }
        __syncwarp();
        double smax = 0.0;
        for (int k = 0; k < d; ++k) smax = fmax(smax, fabs(sS[k]));
        if (!(smax > JOINT_TOL)) break;
        bool accepted = false;
        double Vt = 0.0;
        for (int h = 0; h <= JOINT_MAX_HALVINGS; ++h) {
            if (lane < d) sTr[lane] = fmin(fmax(sTh[lane] + sS[lane], sTb[lane] - delta), sTb[lane] + delta);
            __syncwarp();
            if (eval(sTr, false, &Vt) && Vt < V) { accepted = true; break; }
            if (lane < d) sS[lane] *= 0.5;
            __syncwarp();
        }
        if (!accepted) break;
        if (lane < d) sTh[lane] = sTr[lane];
        __syncwarp();
        eval(sTh, true, &V);
    }

    // levels at the refined angles: A = Q T, C = Q^H R Q, s2 = (tr R - tr C) / (M - d), p = diag(T^-1 (C - s2 I) T^-H)
    double dummy;
    eval(sTh, true, &dummy);  // Q, T and T^-1 at the final angles (A^H A passed there before)
    double2 *sC = sH;
    for (int e = lane; e < d * d; e += 32) {
        const int i = e / d, j = e - i * d;
        double2 s = make_double2(0.0, 0.0);
        for (int k = 0; k < M; ++k) {
            double2 y = make_double2(0.0, 0.0);  // (R q_j)_k
            for (int l = 0; l < M; ++l) {
                const double2 t = cmul(sR[k * M + l], sQ[j * MAXM + l]);
                y.x += t.x;
                y.y += t.y;
            }
            const double2 t = cjmul(sQ[i * MAXM + k], y);
            s.x += t.x;
            s.y += t.y;
        }
        sC[e] = s;
    }
    __syncwarp();
    const double s2 = (trace_re(sR, M, M) - trace_re(sC, d, d)) / (double)(M - d);
    __syncwarp();
    if (lane < d) sC[lane * d + lane].x -= s2;
    __syncwarp();
    if (lane < d) sP[lane] = slot_level(sTi, d, sC, d, d, lane);
    __syncwarp();
    if (filled) {
        const size_t o = (size_t)w * n + lane;
        float ang = (float)deg_b;  // a slot that did not move keeps its grid angle
        if (sTh[r] != sTb[r]) {
            double a = fmod(sTh[r] * REFINE_RAD2DEG, 360.0);
            if (a < 0.0) a += 360.0;
            ang = (float)a;
            if (ang >= 360.0f || ang == 0.0f) ang = 0.0f;
        }
        angles[o] = ang;
        if (levels) levels[o] = (float)sP[r];
    }
}

}  // namespace music
