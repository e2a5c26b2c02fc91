// music_azel.cuh - MUSIC over an (azimuth, elevation) grid of a 3-D array geometry (music_b200_create_azel).
//
// The covariance, eigensolver and scan kernels do not care what a table row means: they scan any K rows.  An az-el
// handle therefore runs the unfused pipeline unchanged on a table of K = n_az * n_el rows, flat bin b = i * n_az + k
// (elevation-major), and only these stages are its own:
//   azel_table_kernel    the steering table of the grid, fp64, rounded to complex64 (then finish_table as in 1-D);
//   topn_local2d_kernel  the 2-D local-maximum peak rule (the TOP_BINS rule is the 1-D one on the flat index);
//   azel_decode_kernel   flat bins -> (azimuth, elevation); the scan / top-n kernels write b * 360 / K into the angle
//                        slots, this kernel overwrites them;
//   refine_azel_kernel   the 2-D off-grid refinement (projected Newton with a backtracking line search).
// The full definition is in include/music_b200.h and is restated literally by tests/azel_oracle.py.
#pragma once
#include "music_kernels.cuh"
#include "music_steer.cuh"
#include "music_refine.cuh"

namespace music {

struct AzelGrid {
    int n_az, n_el;
    double el_lo, el_hi;  // degrees
};

// The geometry of a table slot, passed by value (as RefineGeom): a later retune of the other slot cannot change what an
// enqueued launch reads.
struct AzelGeom {
    double pos[3 * MAXM];  // [M][x, y, z] in metres
    double lambda;
    AzelGrid grid;
};

// el_i in degrees: el_lo + (i (el_hi - el_lo)) / (n_el - 1), el_lo for n_el = 1.  No multiply feeds an add directly,
// so the compiler cannot contract this into an fma and host and device round alike.
__host__ __device__ inline double azel_el_deg(const AzelGrid &g, int i)
{
    if (g.n_el == 1) return g.el_lo;
    return g.el_lo + ((double)i * (g.el_hi - g.el_lo)) / (double)(g.n_el - 1);
}

// a_m(az_k, el_i) = exp(-j 2 pi <p_m, u> / lambda), u = (cos el cos az, cos el sin az, sin el); one thread per (b, m)
__global__ void azel_table_kernel(const AzelGeom geo, int M, float2 *__restrict__ table)
{
    const int n_az = geo.grid.n_az, K = n_az * geo.grid.n_el;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= K * M) return;
    const int b = idx / M, ant = idx - b * M;
    const int i = b / n_az, k = b - i * n_az;
    const double az = __ddiv_rn(__dmul_rn((double)k, 360.0), (double)n_az);
    const double el = azel_el_deg(geo.grid, i);
    double sa, ca, se, ce;
    sincos(__dmul_rn(az, STEER_DEG2RAD), &sa, &ca);
    sincos(__dmul_rn(el, STEER_DEG2RAD), &se, &ce);
    const double ux = __dmul_rn(ce, ca), uy = __dmul_rn(ce, sa), uz = se;
    const double *p = geo.pos + 3 * ant;
    const double inner = __dadd_rn(__dadd_rn(__dmul_rn(p[0], ux), __dmul_rn(p[1], uy)), __dmul_rn(p[2], uz));
    const double ph = __dmul_rn(STEER_TWO_PI, __ddiv_rn(inner, geo.lambda));
    double s, c;
    sincos(ph, &s, &c);
    table[idx] = make_float2(__double2float_rn(c), __double2float_rn(-s));
}

// ---- 2-D local maxima ----------------------------------------------------------------------------------------------
constexpr int AZEL_LM_THREADS = 256;
constexpr int AZEL_LM_CAP = 2048;  // candidates kept in shared memory per window; more fall back to re-scanning P

// b (strength p > 0) beats each of its up to 8 grid neighbours j: p > P[j], or p == P[j] and b < j.  Azimuth wraps,
// elevation rows do not.
__device__ __forceinline__ bool azel_local_max(const double *__restrict__ P, int b, double p, int n_az, int n_el)
{
    const int i = b / n_az, k = b - i * n_az;
    for (int di = -1; di <= 1; ++di) {
        const int ii = i + di;
        if (ii < 0 || ii >= n_el) continue;
        for (int dk = -1; dk <= 1; ++dk) {
            int kk = k + dk;
            kk = kk < 0 ? kk + n_az : (kk >= n_az ? kk - n_az : kk);
            const int j = ii * n_az + kk;
            if (j == b) continue;
            const double q = P[j];
            if (!(p > q || (p == q && b < j))) return false;
        }
    }
    return true;
}

// Chebyshev grid distance: max(min(|dk|, n_az - |dk|), |di|)
__device__ __forceinline__ int azel_cheb(int a, int b, int n_az)
{
    const int ia = a / n_az, ib = b / n_az;
    int dk = abs((a - ia * n_az) - (b - ib * n_az));
    dk = min(dk, n_az - dk);
    return max(dk, abs(ia - ib));
}

// One CTA per window.  Pass 1 reads the window's P row once (neighbour reads hit L1 / L2) and lists the local maxima in
// shared memory; pass r = 0 .. n-1 takes the strongest listed candidate (ties: lowest b) farther than `excl` from every
// peak taken so far.  A window with more than AZEL_LM_CAP maxima re-tests the whole row in every pass instead.
// counts (may be null, music_sources.cuh): window w fills only its first counts[w] slots.  Writes levels and bins; the
// angles are written by azel_decode_kernel.
__global__ void __launch_bounds__(AZEL_LM_THREADS) topn_local2d_kernel(const double *__restrict__ P64, int n, int n_az, int n_el,
                                                                       int excl, PeakOut out, const int32_t *__restrict__ counts)
{
    __shared__ double cP[AZEL_LM_CAP];
    __shared__ int cb[AZEL_LM_CAP];
    __shared__ int ncand;
    __shared__ double rP[AZEL_LM_THREADS / 32];
    __shared__ int rk[AZEL_LM_THREADS / 32];
    __shared__ int taken[MAXM];
    const int w = blockIdx.x;
    const int K = n_az * n_el;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const double *P = P64 + (size_t)w * K;
    const int nr = counts ? counts[w] : n;
    if (threadIdx.x == 0) ncand = 0;
    __syncthreads();
    if (nr > 0) {
        for (int b = threadIdx.x; b < K; b += AZEL_LM_THREADS) {
            const double p = P[b];
            if (!(p > 0.0) || !azel_local_max(P, b, p, n_az, n_el)) continue;  // also skips NaN
            const int s = atomicAdd(&ncand, 1);
            if (s < AZEL_LM_CAP) { cP[s] = p; cb[s] = b; }
        }
    }
    __syncthreads();
    const int nc = ncand;
    const bool listed = nc <= AZEL_LM_CAP;
    int found = 0;  // peaks taken so far (uniform across the CTA)
    for (int r = 0; r < n; ++r) {
        double bP = 0.0;
        int bk = -1;
        if (r < nr && found == r) {
            const int lim = listed ? nc : K;
            for (int c = threadIdx.x; c < lim; c += AZEL_LM_THREADS) {
                double p;
                int b;
                if (listed) {
                    p = cP[c];
                    b = cb[c];
                } else {
                    b = c;
                    p = P[b];
                    if (!(p > 0.0) || !peak_better(p, b, bP, bk) || !azel_local_max(P, b, p, n_az, n_el)) continue;
                }
                if (!peak_better(p, b, bP, bk)) continue;
                bool ok = true;
                for (int q = 0; q < r; ++q) ok = ok && azel_cheb(b, taken[q], n_az) > excl;
                if (ok) { bP = p; bk = b; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double Po = __shfl_xor_sync(0xffffffffu, bP, o);
            const int ko = __shfl_xor_sync(0xffffffffu, bk, o);
            if (peak_better(Po, ko, bP, bk)) { bP = Po; bk = ko; }
        }
        if (lane == 0) { rP[wid] = bP; rk[wid] = bk; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int q = 1; q < AZEL_LM_THREADS / 32; ++q)
                if (peak_better(rP[q], rk[q], bP, bk)) { bP = rP[q]; bk = rk[q]; }
            const size_t o = (size_t)w * n + r;
            if (out.levels) out.levels[o] = bk >= 0 ? (float)bP : 0.f;
            peak_store_bin(out, o, bk);
            if (r < MAXM) taken[r] = bk;
            rk[0] = bk;
        }
        __syncthreads();
        if (rk[0] >= 0) ++found;
        __syncthreads();  // rk is rewritten in the next pass
    }
}

// angles[o] = (float)(k * 360.0 / n_az) and elev[o] = (float)el_i of the flat bin b = bins[o] = i * n_az + k; (0, 0)
// for an unfilled slot (bin -1)
__global__ void azel_decode_kernel(const int32_t *__restrict__ bins, int slots, const AzelGrid g, float *__restrict__ angles,
                                   float *__restrict__ elev)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= slots) return;
    const int b = bins[o];
    if (b < 0) {
        angles[o] = 0.f;
        elev[o] = 0.f;
        return;
    }
    const int i = b / g.n_az, k = b - i * g.n_az;
    angles[o] = (float)((double)k * 360.0 / (double)g.n_az);
    elev[o] = (float)azel_el_deg(g, i);
}

// ---- 2-D refinement --------------------------------------------------------------------------------------------------
// D(ph, ep) = sum_j |g_j^H a|^2 with its gradient and Hessian, e = {D, D_ph, D_ep, D_phph, D_phep, D_epep}.
// theta_m = 2 pi <p_m, u> / lambda, a_m = exp(-j theta_m); with h = x cos ph + y sin ph, v = y cos ph - x sin ph:
//   theta_ph = 2 pi cos ep v / lambda,      theta_ep = 2 pi (z cos ep - sin ep h) / lambda,
//   theta_phph = -2 pi cos ep h / lambda,   theta_phep = -2 pi sin ep v / lambda,   theta_epep = -theta;
//   conj(g) a_u = -j theta_u c,  conj(g) a_uv = (-theta_u theta_v - j theta_uv) c,  c = conj(g) a;
//   D_u = 2 sum Re(conj(s) s_u),  D_uv = 2 sum (Re(conj(s_u) s_v) + Re(conj(s) s_uv)).
__device__ __noinline__ void azel_eval(const AzelGeom &geo, const double2 *__restrict__ G, int M, int p, double ph, double ep,
                                       double *e)
{
    double sp, cp, se, ce;
    sincos(ph, &sp, &cp);
    sincos(ep, &se, &ce);
    double ar[MAXM], ai[MAXM], th[MAXM], tp[MAXM], te[MAXM], tpp[MAXM], tpe[MAXM];
    for (int m = 0; m < M; ++m) {
        const double x = geo.pos[3 * m], y = geo.pos[3 * m + 1], z = geo.pos[3 * m + 2];
        const double h = x * cp + y * sp, v = y * cp - x * sp;
        th[m] = STEER_TWO_PI * ((ce * h + z * se) / geo.lambda);
        tp[m] = STEER_TWO_PI * ((ce * v) / geo.lambda);
        te[m] = STEER_TWO_PI * ((z * ce - se * h) / geo.lambda);
        tpp[m] = -STEER_TWO_PI * ((ce * h) / geo.lambda);
        tpe[m] = -STEER_TWO_PI * ((se * v) / geo.lambda);
        double s, c;
        sincos(th[m], &s, &c);
        ar[m] = c;
        ai[m] = -s;
    }
    for (int i = 0; i < 6; ++i) e[i] = 0.0;
    for (int j = 0; j < p; ++j) {
        double s0r = 0.0, s0i = 0.0, spr = 0.0, spi = 0.0, ser = 0.0, sei = 0.0;
        double sppr = 0.0, sppi = 0.0, sper = 0.0, spei = 0.0, seer = 0.0, seei = 0.0;
        for (int m = 0; m < M; ++m) {
            const double2 g = G[j * M + m];
            const double cr = g.x * ar[m] + g.y * ai[m], ci = g.x * ai[m] - g.y * ar[m];  // conj(g) a
            s0r += cr;
            s0i += ci;
            spr += tp[m] * ci;
            spi -= tp[m] * cr;
            ser += te[m] * ci;
            sei -= te[m] * cr;
            const double qpp = tp[m] * tp[m], qpe = tp[m] * te[m], qee = te[m] * te[m];
            sppr += -qpp * cr + tpp[m] * ci;
            sppi += -qpp * ci - tpp[m] * cr;
            sper += -qpe * cr + tpe[m] * ci;
            spei += -qpe * ci - tpe[m] * cr;
            seer += -qee * cr - th[m] * ci;  // theta_epep = -theta
            seei += -qee * ci + th[m] * cr;
        }
        e[0] += s0r * s0r + s0i * s0i;
        e[1] += 2.0 * (s0r * spr + s0i * spi);
        e[2] += 2.0 * (s0r * ser + s0i * sei);
        e[3] += 2.0 * (spr * spr + spi * spi + s0r * sppr + s0i * sppi);
        e[4] += 2.0 * (spr * ser + spi * sei + s0r * sper + s0i * spei);
        e[5] += 2.0 * (ser * ser + sei * sei + s0r * seer + s0i * seei);
    }
}

// F = -B, B(ph, ep) = a^H R a, with its gradient and Hessian in e (EST_BARTLETT, music_refine.cuh).  With y = R a,
// y_u = R a_u:  B_u = 2 Re(a_u^H y),  B_uv = 2 (Re(a_u^H y_v) + Re(a_uv^H y)),  a_u = -j theta_u a,
// a_uv = (-theta_u theta_v - j theta_uv) a; theta and its derivatives as in azel_eval.
__device__ __noinline__ void bartlett_azel_eval(const AzelGeom &geo, const double2 *__restrict__ Rw, int M, double ph, double ep,
                                                double *e)
{
    double sp, cp, se, ce;
    sincos(ph, &sp, &cp);
    sincos(ep, &se, &ce);
    double ar[MAXM], ai[MAXM], th[MAXM], tp[MAXM], te[MAXM], tpp[MAXM], tpe[MAXM];
    for (int m = 0; m < M; ++m) {
        const double x = geo.pos[3 * m], y = geo.pos[3 * m + 1], z = geo.pos[3 * m + 2];
        const double h = x * cp + y * sp, v = y * cp - x * sp;
        th[m] = STEER_TWO_PI * ((ce * h + z * se) / geo.lambda);
        tp[m] = STEER_TWO_PI * ((ce * v) / geo.lambda);
        te[m] = STEER_TWO_PI * ((z * ce - se * h) / geo.lambda);
        tpp[m] = -STEER_TWO_PI * ((ce * h) / geo.lambda);
        tpe[m] = -STEER_TWO_PI * ((se * v) / geo.lambda);
        double s, c;
        sincos(th[m], &s, &c);
        ar[m] = c;
        ai[m] = -s;
    }
    double b[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < M; ++i) {
        double yr = 0.0, yi = 0.0, ypr = 0.0, ypi = 0.0, yer = 0.0, yei = 0.0;  // (R a)_i, (R a_ph)_i, (R a_ep)_i
        for (int j = 0; j < M; ++j) {
            const double2 r = Rw[i * M + j];
            const double cr = r.x * ar[j] - r.y * ai[j], ci = r.x * ai[j] + r.y * ar[j];  // R_ij a_j
            yr += cr;
            yi += ci;
            ypr += tp[j] * ci;  // R_ij a_u,j = theta_u (ci - j cr)
            ypi -= tp[j] * cr;
            yer += te[j] * ci;
            yei -= te[j] * cr;
        }
        const double pr = tp[i] * ai[i], pi = -tp[i] * ar[i];  // a_ph,i
        const double er = te[i] * ai[i], ei = -te[i] * ar[i];  // a_ep,i
        const double qpp = tp[i] * tp[i], qpe = tp[i] * te[i], qee = te[i] * te[i];
        const double ppr = -qpp * ar[i] + tpp[i] * ai[i], ppi = -qpp * ai[i] - tpp[i] * ar[i];  // a_phph,i
        const double per = -qpe * ar[i] + tpe[i] * ai[i], pei = -qpe * ai[i] - tpe[i] * ar[i];  // a_phep,i
        const double eer = -qee * ar[i] - th[i] * ai[i], eei = -qee * ai[i] + th[i] * ar[i];   // a_epep,i (theta_epep = -theta)
        b[0] += ar[i] * yr + ai[i] * yi;
        b[1] += 2.0 * (pr * yr + pi * yi);
        b[2] += 2.0 * (er * yr + ei * yi);
        b[3] += 2.0 * (pr * ypr + pi * ypi + ppr * yr + ppi * yi);
        b[4] += 2.0 * (pr * yer + pi * yei + per * yr + pei * yi);
        b[5] += 2.0 * (er * yer + ei * yei + eer * yr + eei * yi);
    }
    for (int q = 0; q < 6; ++q) e[q] = -b[q];
}

template <int EST>
__device__ __forceinline__ void azel_est_eval(const AzelGeom &geo, const double2 *__restrict__ G, int M, int p, double ph, double ep,
                                              double *e)
{
    if constexpr (EST == EST_BARTLETT) bartlett_azel_eval(geo, G, M, ph, ep, e);
    else azel_eval(geo, G, M, p, ph, ep, e);
}

__device__ __forceinline__ double azel_clamp(double v, double lo, double hi) { return v < lo ? lo : (v > hi ? hi : v); }

constexpr double AZEL_T_MIN = 9.313225746154785e-10;  // 2^-30: smallest step fraction of the line search (exclusive)

// Slot o = w * n + i with bins[o] >= 0: projected Newton on D inside the box of one grid step either side of the grid
// point (the elevation range clipped to [el_lo, el_hi]); a result that moved and does not raise D replaces the decoded
// grid angles.  levels[o] (may be null) = 1 / D at the point kept.  counts (may be null): per-window source count.
// EST and Vt as for refine_peaks_kernel (music_refine.cuh); under EST_BARTLETT the level is -F / M^2 = B / M^2.
template <int EST = EST_MUSIC>
__global__ void __launch_bounds__(REFINE_THREADS) refine_azel_kernel(const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                                     const int32_t *__restrict__ bins, int M, int n, int W,
                                                                     const AzelGeom geo, float *__restrict__ angles,
                                                                     float *__restrict__ elev, float *__restrict__ levels)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= W * n) return;
    const int b = bins[o];
    if (b < 0) return;
    const int w = o / n;
    int p = M;
    if constexpr (EST == EST_MUSIC) p = M - (counts ? counts[w] : n);
    const double2 *G = reinterpret_cast<const double2 *>(Vt) + (size_t)w * M * M;
    const AzelGrid &g = geo.grid;
    const int i = b / g.n_az, k = b - i * g.n_az;
    const double ph_b = ((double)k * 360.0 / (double)g.n_az) * STEER_DEG2RAD;
    const double ep_b = azel_el_deg(g, i) * STEER_DEG2RAD;
    const double dph = (360.0 / (double)g.n_az) * STEER_DEG2RAD;
    const double dep = g.n_el > 1 ? ((g.el_hi - g.el_lo) / (double)(g.n_el - 1)) * STEER_DEG2RAD : 0.0;
    const double plo = ph_b - dph, phi = ph_b + dph;
    const double elo = fmax(ep_b - dep, g.el_lo * STEER_DEG2RAD), ehi = fmin(ep_b + dep, g.el_hi * STEER_DEG2RAD);
    double e[6], f[6];
    azel_est_eval<EST>(geo, G, M, p, ph_b, ep_b, e);
    const double Db = e[0];
    double x0 = ph_b, x1 = ep_b;
    for (int it = 0; it < REFINE_MAX_IT; ++it) {
        const double g0 = e[1], g1 = e[2];
        if (g0 == 0.0 && g1 == 0.0) break;
        const double det = e[3] * e[5] - e[4] * e[4];
        double s0, s1;
        if (e[3] > 0.0 && det > 0.0) {
            s0 = -(e[5] * g0 - e[4] * g1) / det;
            s1 = -(e[3] * g1 - e[4] * g0) / det;
        } else {
            const double gn = sqrt(g0 * g0 + g1 * g1);
            s0 = -g0 * dph / gn;
            s1 = -g1 * dph / gn;
        }
        s0 = __dsub_rn(azel_clamp(__dadd_rn(x0, s0), plo, phi), x0);
        s1 = __dsub_rn(azel_clamp(__dadd_rn(x1, s1), elo, ehi), x1);
        double t = 1.0, y0 = x0, y1 = x1;
        bool ok = false;
        while (t > AZEL_T_MIN) {
            y0 = __dadd_rn(x0, __dmul_rn(t, s0));
            y1 = __dadd_rn(x1, __dmul_rn(t, s1));
            azel_est_eval<EST>(geo, G, M, p, y0, y1, f);
            if (f[0] <= e[0]) { ok = true; break; }
            t *= 0.5;
        }
        if (!ok) break;
        const double step = fmax(fabs(__dmul_rn(t, s0)), fabs(__dmul_rn(t, s1)));
        x0 = y0;
        x1 = y1;
        for (int q = 0; q < 6; ++q) e[q] = f[q];
        if (step <= REFINE_TOL) break;
    }
    double D = Db;
    if ((x0 != ph_b || x1 != ep_b) && e[0] <= Db) {
        D = e[0];
        double a = fmod(x0 * REFINE_RAD2DEG, 360.0);
        if (a < 0.0) a += 360.0;
        float az = (float)a;
        if (az >= 360.0f || az == 0.0f) az = 0.0f;
        angles[o] = az;
        elev[o] = (float)(x1 * REFINE_RAD2DEG);
    }
    if constexpr (EST == EST_BARTLETT) {
        if (levels) levels[o] = (float)(-D / ((double)M * (double)M));
    } else {
        if (levels) levels[o] = (float)(1.0 / D);
    }
}

}  // namespace music
