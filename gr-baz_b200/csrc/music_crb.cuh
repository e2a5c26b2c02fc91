// music_crb.cuh - the stochastic Cramer-Rao bound of every filled peak slot (the *_crb entry points).
//
// After the peak stage, each window's filled slots S = {i : bins[w][i] >= 0} (d = |S|) get the bound on the standard
// deviation of their angle (1-D) or of their (azimuth, elevation) pair, evaluated at the window's own covariance R and
// the reported angles (Stoica, Larsson & Gershman 2001; Stoica & Nehorai 1990):
//   A = [a_i] = Q T (modified Gram-Schmidt applied twice, mgs2), s2 = (tr R - tr(Q^H R Q)) / (M - d),
//   H = T^-1 (Q^H R Q) T^-H,  Gamma = T^-1 T^-H,  P = H - s2 Gamma,  U = P H^-1 P  (H by Cholesky),
//   B = D^H (I - Q Q^H) D over the derivative columns D,  F = (2 N / s2) Re(B o U^T) per parameter pair,  C = F^-1.
// The full definition (failure rules, outputs) is in include/music_b200.h and is restated literally by
// tests/crb_oracle.py.
//
// crb_kernel: one warp per window, everything fp64 in shared memory, as beam_weights_kernel.  Lanes map to antennas for
// the Gram-Schmidt and the projections, to matrix entries for the d x d products and to columns for the triangular
// solves.  The largest problem (az-el, d = 15, 30 parameters) needs about 37 KB of shared memory, so a CTA holds one
// window.
#pragma once
#include "music_kernels.cuh"
#include "music_refine.cuh"
#include "music_azel.cuh"
#include "music_integrate.cuh"
#include "music_warp_la.cuh"

namespace music {

constexpr int CRB_MAXN = MAXM - 1;       // slots per window (n < M)
constexpr int CRB_MAXP = 2 * CRB_MAXN;   // parameters per window (az-el: two per slot)
constexpr double CRB_T_REL = 0x1p-30;    // |T_ii|^2 must exceed this fraction of ||a_i||^2
constexpr double CRB_PIVOT_REL = 0x1p-40;  // pivot k of F must exceed this fraction of F_kk
constexpr double CRB_B_REL = 0x1p-40;      // B_cc must exceed this fraction of the array's derivative scale G

// R [W][M][M] (re, im), the integrated or calibrated covariance the other stages read; angles / elev / bins [W][n] as the
// peak stage wrote them (elev: az-el only); n0 (may be null): the integration count at window 0, for N_eff; Nsnap: the
// snapshots per window.  out [W][n] (1-D) or [W][n][3] (AZEL) floats.
template <bool AZEL>
__global__ void __launch_bounds__(32) crb_kernel(const double *__restrict__ R, const float *__restrict__ angles,
                                                 const float *__restrict__ elev, const int32_t *__restrict__ bins,
                                                 const unsigned long long *__restrict__ n0, int M, int n, int W, int Nsnap,
                                                 double alpha, const RefineGeom geo, const AzelGeom ageo, float *__restrict__ out)
{
    constexpr int PER = AZEL ? 2 : 1;  // parameters per slot
    // pool1: R (stride M), the steering vectors A and Q (stride MAXM) and T (stride MAXM); later F (stride p)
    __shared__ double2 pool1[MAXM * MAXM + 3 * CRB_MAXN * MAXM];
    // pool2: Q^H R Q then P (stride d), T^-1 then U, X = T^-1 C then Y = H^-1 P, H (stride d each); later L_F^-1 (real)
    __shared__ double2 pool2[4 * CRB_MAXN * CRB_MAXN];
    __shared__ double2 sD[CRB_MAXP * MAXM];  // derivative columns, projected onto the complement of span(A) in place
    __shared__ double sNa[CRB_MAXN], sBd[CRB_MAXP], sFd[CRB_MAXP], sCd[CRB_MAXP], sCo[CRB_MAXN];
    const int lane = threadIdx.x, w = blockIdx.x;
    double2 *sR = pool1, *sA = pool1 + MAXM * MAXM, *sQ = sA + CRB_MAXN * MAXM, *sT = sQ + CRB_MAXN * MAXM, *sF = pool1;
    double2 *sC = pool2, *sTi = pool2 + CRB_MAXN * CRB_MAXN, *sX = sTi + CRB_MAXN * CRB_MAXN, *sH = sX + CRB_MAXN * CRB_MAXN;
    double *sLi = reinterpret_cast<double *>(pool2);

    const int b = lane < n ? bins[(size_t)w * n + lane] : -1;
    const bool filled = b >= 0;
    const unsigned fmask = __ballot_sync(0xffffffffu, filled);
    const int d = __popc(fmask), p = PER * d;
    if (d == 0) {
        if (lane < n)
            for (int k = 0; k < (AZEL ? 3 : 1); ++k) out[((size_t)w * n + lane) * (AZEL ? 3 : 1) + k] = 0.f;
        return;
    }
    const int r = __popc(fmask & ((1u << lane) - 1u));  // a filled lane's column among the filled slots
    if (filled) {
        double2 *a = sA + r * MAXM;
        double na = 0.0;
        if constexpr (AZEL) {
            double sp, cp, se, ce;
            sincos((double)angles[(size_t)w * n + lane] * STEER_DEG2RAD, &sp, &cp);
            sincos((double)elev[(size_t)w * n + lane] * STEER_DEG2RAD, &se, &ce);
            for (int m = 0; m < M; ++m) {
                double th, tp, te, tpp, tpe, s, c;
                azel_phase(ageo, m, sp, cp, se, ce, &th, &tp, &te, &tpp, &tpe);
                sincos(th, &s, &c);
                a[m] = make_double2(c, -s);
                sD[(2 * r) * MAXM + m] = make_double2(-tp * s, -tp * c);      // -j theta_az a
                sD[(2 * r + 1) * MAXM + m] = make_double2(-te * s, -te * c);  // -j theta_el a
                na += c * c + s * s;
            }
        } else {
            double st, ct;
            sincos((double)angles[(size_t)w * n + lane] * STEER_DEG2RAD, &st, &ct);
            for (int m = 0; m < M; ++m) {
                double phi, psi, sp, cp;
                steer_phase(geo, m, st, ct, &phi, &psi);
                sincos(phi, &sp, &cp);
                a[m] = make_double2(cp, -sp);
                sD[r * MAXM + m] = make_double2(-psi * sp, -psi * cp);  // -j psi a
                na += cp * cp + sp * sp;
            }
        }
        sNa[r] = na;
    }
    const double2 *Rw = reinterpret_cast<const double2 *>(R) + (size_t)w * M * M;
    for (int e = lane; e < M * M; e += 32) sR[e] = Rw[e];
    __syncwarp();

    // 1. A = Q T
    mgs2([&](int l, int i) { return sA[l * MAXM + i]; }, d, M, sQ, sT, lane);
    bool ok = true;  // warp-uniform
    for (int l = 0; l < d; ++l) {
        const double t = sT[l * MAXM + l].x;
        ok = ok && t * t > CRB_T_REL * sNa[l];
    }

    // 2. C = Q^H R Q, s2 = (tr R - tr C) / (M - d)
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
    triu_inverse(sT, MAXM, sTi, d, d, lane);  // T^-1 (upper triangular), column c by lane c
    __syncwarp();
    const double s2 = (trace_re(sR, M, M) - trace_re(sC, d, d)) / (double)(M - d);
    ok = ok && s2 > 0.0 && isfinite(s2);

    // 3. X = T^-1 C; H = X T^-H; P = H - s2 T^-1 T^-H into sC; U = P H^-1 P
    for (int e = lane; e < d * d; e += 32) {
        const int i = e / d, j = e - i * d;
        double2 s = make_double2(0.0, 0.0);
        for (int k = i; k < d; ++k) {
            const double2 t = cmul(sTi[i * d + k], sC[k * d + j]);
            s.x += t.x;
            s.y += t.y;
        }
        sX[e] = s;
    }
    __syncwarp();
    for (int e = lane; e < d * d; e += 32) {
        const int i = e / d, j = e - i * d;
        double2 h = make_double2(0.0, 0.0), g = make_double2(0.0, 0.0);
        for (int k = 0; k < d; ++k) {
            const double2 t = cmul(sX[i * d + k], make_double2(sTi[j * d + k].x, -sTi[j * d + k].y));
            h.x += t.x;
            h.y += t.y;
        }
        for (int k = i > j ? i : j; k < d; ++k) {
            const double2 t = cmul(sTi[i * d + k], make_double2(sTi[j * d + k].x, -sTi[j * d + k].y));
            g.x += t.x;
            g.y += t.y;
        }
        sH[e] = h;
        sC[e] = make_double2(h.x - s2 * g.x, h.y - s2 * g.y);
    }
    __syncwarp();
    ok = ok && warp_cholesky(sH, d, lane, [](int, double piv) { return piv > 0.0; });
    __syncwarp();
    if (ok && lane < d) {  // column `lane` of Y = H^-1 P: L y = p, then L^H z = y, into sX
        const int c = lane;
        const auto xk = [&](int k) -> double2 & { return sX[k * d + c]; };
        cholesky_solve(sH, d, d, [&](int k) -> const double2 & { return sC[k * d + c]; }, xk, xk);
    }
    __syncwarp();
    for (int e = lane; ok && e < d * d; e += 32) {  // U = P Y into sTi
        const int i = e / d, j = e - i * d;
        double2 s = make_double2(0.0, 0.0);
        for (int k = 0; k < d; ++k) {
            const double2 t = cmul(sC[i * d + k], sX[k * d + j]);
            s.x += t.x;
            s.y += t.y;
        }
        sTi[e] = s;
    }

    // 4. the derivative columns projected onto the orthogonal complement of span(A): twice, as the Gram-Schmidt
    for (int c = 0; ok && c < p; ++c) {
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
    // F (real, in the real parts of pool1, stride p): F_cc' = (2 N / s2) Re(B_cc' U_s(c') s(c)), s(c) = c / PER
    const double N = n0 ? integ_neff(alpha, *n0 + (unsigned long long)w, (double)Nsnap) : (double)Nsnap;
    const double scale = 2.0 * N / s2;
    for (int e = lane; ok && e < p * p; e += 32) {
        const int c = e / p, c2 = e - c * p;
        double br = 0.0, bi = 0.0;
        for (int m = 0; m < M; ++m) {
            const double2 t = cjmul(sD[c * MAXM + m], sD[c2 * MAXM + m]);
            br += t.x;
            bi += t.y;
        }
        const double2 u = sTi[(c2 / PER) * d + c / PER];
        const double f = scale * (br * u.x - bi * u.y);
        sF[e] = make_double2(f, 0.0);
        if (c == c2) {
            sBd[c] = br;
            sFd[c] = f;
        }
    }
    __syncwarp();
    // G = (2 pi / lambda)^2 sum_m |p_m - centroid|^2 bounds B_cc for every direction: B_cc <= 2^-40 G means the parameter
    // is unobservable to first order (its derivative vanishes, or lies in span(A), to rounding).  Every lane forms the
    // same sums in the same order.
    {
        const double *ps = AZEL ? ageo.pos : geo.pos;
        const int dim = AZEL ? 3 : 2;
        double ctr[3] = {0.0, 0.0, 0.0}, G = 0.0;
        for (int m = 0; m < M; ++m)
            for (int k = 0; k < dim; ++k) ctr[k] += ps[dim * m + k];
        for (int k = 0; k < dim; ++k) ctr[k] /= (double)M;
        for (int m = 0; m < M; ++m)
            for (int k = 0; k < dim; ++k) {
                const double v = ps[dim * m + k] - ctr[k];
                G += v * v;
            }
        const double kw = STEER_TWO_PI / (AZEL ? ageo.lambda : geo.lambda);
        G *= kw * kw;
        for (int c = 0; ok && c < p; ++c) ok = sBd[c] > CRB_B_REL * G;
    }
    // 5. C = F^-1 = L^-T L^-1: lane c forms column c of L^-1, then C_cc = ||L^-1 e_c||^2 and the az-el cross term
    ok = ok && warp_cholesky(sF, p, lane, [&](int k, double piv) { return piv > CRB_PIVOT_REL * sFd[k]; });
    __syncwarp();
    if (ok && lane < p) {
        const int c = lane;
        for (int k = 0; k < p; ++k) {
            double s = k == c ? 1.0 : 0.0;
            if (k > c)
                for (int q = c; q < k; ++q) s -= sF[k * p + q].x * sLi[q * p + c];
            sLi[k * p + c] = k < c ? 0.0 : s / sF[k * p + k].x;
        }
    }
    __syncwarp();
    if (ok && lane < p) {
        const int c = lane;
        double cc = 0.0, co = 0.0;
        for (int k = c; k < p; ++k) {
            const double v = sLi[k * p + c];
            cc += v * v;
            if (AZEL && c % 2 == 0) co += v * sLi[k * p + c + 1];
        }
        sCd[c] = cc;
        if (AZEL && c % 2 == 0) sCo[c / 2] = co;
    }
    __syncwarp();

    // 6. outputs: filled slots their bound (NaN when the window failed), unfilled slots 0
    if (lane < n) {
        const float nan = __int_as_float(0x7fc00000);
        if constexpr (AZEL) {
            float *o = out + ((size_t)w * n + lane) * 3;
            if (!filled) {
                o[0] = o[1] = o[2] = 0.f;
            } else if (!ok) {
                o[0] = o[1] = o[2] = nan;
            } else {
                const double caa = sCd[2 * r], cee = sCd[2 * r + 1];
                o[0] = (float)(sqrt(caa) * REFINE_RAD2DEG);
                o[1] = (float)(sqrt(cee) * REFINE_RAD2DEG);
                o[2] = (float)(sCo[r] / sqrt(caa * cee));
            }
        } else {
            out[(size_t)w * n + lane] = !filled ? 0.f : !ok ? nan : (float)(sqrt(sCd[r]) * REFINE_RAD2DEG);
        }
    }
}

}  // namespace music
