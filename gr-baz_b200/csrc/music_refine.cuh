// music_refine.cuh - off-grid refinement of the reported peaks (opt-in, music_b200_set_refine).
//
// Every angle the scan reports is a grid angle k * 360 / K, so its error is up to half a bin whatever the estimator
// does.  The handle knows the array itself when the table came from music_b200_set_geometry(), so the steering vector
// a(theta) can be evaluated at any angle, and the unfused path already holds the sorted eigenvectors of every window
// (ws.Vt).  This stage moves each filled slot from its grid bin to the minimum of the exact fp64 MUSIC denominator
//     D(theta) = sum_j |g_j^H a(theta)|^2,   g_j = the noise eigenvectors the scan used,
// with a_m(theta) = exp(-j phi_m), phi_m = 2 pi (p_x,m cos theta + p_y,m sin theta) / lambda (the table builder's
// convention, music_steer.cuh) and the analytic derivatives
//     psi_m = dphi_m / dtheta,  phi_m'' = -phi_m,  a' = -j psi a,  a'' = (j phi - psi^2) a,
//     D' = 2 sum Re(conj(s) s'),  D'' = 2 sum (|s'|^2 + Re(conj(s) s'')),  s = G^H a, s' = G^H a', s'' = G^H a''.
// Safeguarded Newton on D' = 0 (rtsafe) inside [theta_b - 360/K, theta_b + 360/K]; the full definition is in
// include/music_b200.h and is restated literally by tests/refine_oracle.py.
//
// One thread per output slot: the stage runs n evaluations' worth of work per window against the scan's K, so it is
// a small fraction of the scan whatever its shape.
#pragma once
#include "music_kernels.cuh"
#include "music_steer.cuh"

namespace music {

// The geometry of the table the scan used, passed by value: a later set_geometry() into the other table slot cannot
// change what an enqueued launch reads.
struct RefineGeom {
    double pos[2 * MAXM];  // [M][x, y] in metres
    double lambda;
};

// One warp per CTA: a call has only W * n slots (8192 at C5), and each thread is a serial fp64 chain, so small CTAs
// spread them over every SM instead of packing them onto half of them.
constexpr int REFINE_THREADS = 32;
constexpr int REFINE_MAX_IT = 50;
constexpr double REFINE_TOL = 1e-12;  // radians: stop once a step is this small
constexpr double REFINE_RAD2DEG = 180.0 / 3.14159265358979323846;

// The phase phi_m and its derivative psi_m of element m at the angle theta with (sin theta, cos theta) = (st, ct); the
// steering entry is a_m = exp(-j phi_m).  Shared by the refinement and the beam weights (music_beams.cuh).
__device__ __forceinline__ void steer_phase(const RefineGeom &geo, int m, double st, double ct, double *phi, double *psi)
{
    const double px = geo.pos[2 * m], py = geo.pos[2 * m + 1];
    *phi = STEER_TWO_PI * (fma(py, st, px * ct) / geo.lambda);
    *psi = STEER_TWO_PI * (fma(py, ct, -(px * st)) / geo.lambda);
}

// D(theta), D'(theta), D''(theta) for the p noise vectors G[j][m] (eigenvector j contiguous) of one window
__device__ __noinline__ void refine_eval(const RefineGeom &geo, const double2 *__restrict__ G, int M, int p, double th,
                                         double *D, double *D1, double *D2)
{
    double st, ct;
    sincos(th, &st, &ct);
    double ar[MAXM], ai[MAXM], ps[MAXM], ph[MAXM];
    for (int m = 0; m < M; ++m) {
        double phi, psi;
        steer_phase(geo, m, st, ct, &phi, &psi);
        double sp, cp;
        sincos(phi, &sp, &cp);
        ar[m] = cp;
        ai[m] = -sp;
        ps[m] = psi;
        ph[m] = phi;
    }
    double d0 = 0.0, d1 = 0.0, d2 = 0.0;
    for (int j = 0; j < p; ++j) {
        double sr = 0.0, si = 0.0, s1r = 0.0, s1i = 0.0, s2r = 0.0, s2i = 0.0;
        for (int m = 0; m < M; ++m) {
            const double2 e = G[j * M + m];
            const double cr = e.x * ar[m] + e.y * ai[m], ci = e.x * ai[m] - e.y * ar[m];  // conj(g) a
            const double q = ps[m] * ps[m];
            sr += cr;
            si += ci;
            s1r += ps[m] * ci;  // conj(g) a' = psi (ci - j cr)
            s1i -= ps[m] * cr;
            s2r += -q * cr - ph[m] * ci;  // conj(g) a'' = (-psi^2 + j phi)(cr + j ci)
            s2i += -q * ci + ph[m] * cr;
        }
        d0 += sr * sr + si * si;
        d1 += 2.0 * (sr * s1r + si * s1i);
        d2 += 2.0 * (s1r * s1r + s1i * s1i + sr * s2r + si * s2i);
    }
    *D = d0;
    *D1 = d1;
    *D2 = d2;
}

// The estimator whose spectrum the refinement follows (music_b200_set_estimator, music_estimators.cuh):
//   EST_MUSIC     D = sum_j |g_j^H a|^2 over the p noise eigenvectors, level 1 / D;
//   EST_MVDR      the same D over p = M vectors g_j = conj(row j of L^-1), i.e. a^H R_L^-1 a, level 1 / D;
//   EST_BARTLETT  D = F = -a^H R a (maximising B = a^H R a is minimising F), level -F / M^2 (||a||^2 = M).

// F = -B, F', F'' with B(theta) = a^H R a for the window's covariance R[i][j] (row i contiguous):
//   B' = 2 Re(a'^H R a),  B'' = 2 (a'^H R a' + Re(a''^H R a)),  a' = -j psi a,  a'' = (j phi - psi^2) a.
__device__ __noinline__ void bartlett_eval(const RefineGeom &geo, const double2 *__restrict__ Rw, int M, double th, double *F,
                                           double *F1, double *F2)
{
    double st, ct;
    sincos(th, &st, &ct);
    double ar[MAXM], ai[MAXM], ps[MAXM], ph[MAXM];
    for (int m = 0; m < M; ++m) {
        double phi, psi;
        steer_phase(geo, m, st, ct, &phi, &psi);
        double sp, cp;
        sincos(phi, &sp, &cp);
        ar[m] = cp;
        ai[m] = -sp;
        ps[m] = psi;
        ph[m] = phi;
    }
    double b0 = 0.0, b1 = 0.0, b2 = 0.0;
    for (int i = 0; i < M; ++i) {
        double yr = 0.0, yi = 0.0, y1r = 0.0, y1i = 0.0;  // (R a)_i, (R a')_i
        for (int j = 0; j < M; ++j) {
            const double2 r = Rw[i * M + j];
            const double cr = r.x * ar[j] - r.y * ai[j], ci = r.x * ai[j] + r.y * ar[j];  // R_ij a_j
            yr += cr;
            yi += ci;
            y1r += ps[j] * ci;  // R_ij a'_j = psi_j (ci - j cr)
            y1i -= ps[j] * cr;
        }
        const double q = ps[i] * ps[i];
        const double d1r = ps[i] * ai[i], d1i = -ps[i] * ar[i];                         // a'_i
        const double d2r = -q * ar[i] - ph[i] * ai[i], d2i = ph[i] * ar[i] - q * ai[i];  // a''_i
        b0 += ar[i] * yr + ai[i] * yi;
        b1 += 2.0 * (d1r * yr + d1i * yi);
        b2 += 2.0 * (d1r * y1r + d1i * y1i + d2r * yr + d2i * yi);
    }
    *F = -b0;
    *F1 = -b1;
    *F2 = -b2;
}

template <int EST>
__device__ __forceinline__ void est_eval(const RefineGeom &geo, const double2 *__restrict__ G, int M, int p, double th, double *D,
                                         double *D1, double *D2)
{
    if constexpr (EST == EST_BARTLETT) bartlett_eval(geo, G, M, th, D, D1, D2);
    else refine_eval(geo, G, M, p, th, D, D1, D2);
}

// Slot o = w * n + i with bins[o] >= 0: angles[o] / levels[o] (levels may be null) become the refined angle and
// 1 / D there; slots with bin -1 are left as the peak rule wrote them.  counts (may be null): per-window source
// count, so that the noise subspace is the M - counts[w] smallest-eigenvalue vectors, as in the scan.
// Vt: per window M * M complex doubles - the sorted eigenvectors (MUSIC), the g_j of mvdr_prep_kernel (MVDR) or R
// (BARTLETT); the non-MUSIC estimators ignore n and counts beyond the bins.  The minimum-blocks hint of the non-MUSIC
// instantiations lets ptxas keep the values live across the evaluation calls in registers (without it the MVDR
// instantiation spills); the MUSIC instantiation keeps its original bounds.
template <int EST = EST_MUSIC>
__global__ void __launch_bounds__(REFINE_THREADS, EST == EST_MUSIC ? 0 : 1) refine_peaks_kernel(const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                           const int32_t *__restrict__ bins, int M, int n, int K, int W,
                                                           const RefineGeom geo, float *__restrict__ angles, float *__restrict__ levels)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= W * n) return;
    const int b = bins[o];
    if (b < 0) return;
    const int w = o / n;
    int p = M;
    if constexpr (EST == EST_MUSIC) p = M - (counts ? counts[w] : n);
    const double2 *G = reinterpret_cast<const double2 *>(Vt) + (size_t)w * M * M;
    const double deg_b = (double)b * 360.0 / (double)K;  // the grid angle the peak rule reported
    const double tb = deg_b * STEER_DEG2RAD, delta = (360.0 / (double)K) * STEER_DEG2RAD;
    double Db, f, df, Dx, fx, dfx;
    est_eval<EST>(geo, G, M, p, tb, &Db, &f, &df);
    double lo = tb - delta, hi = tb + delta;
    double fl, fh;
    est_eval<EST>(geo, G, M, p, lo, &Dx, &fl, &dfx);
    est_eval<EST>(geo, G, M, p, hi, &Dx, &fh, &dfx);
    double x = tb;
    if (fl < 0.0 && fh > 0.0) {
        double dxold = hi - lo, dx = dxold;
        for (int it = 0; it < REFINE_MAX_IT; ++it) {
            if (f == 0.0) break;
            if (((x - hi) * df - f) * ((x - lo) * df - f) > 0.0 || fabs(2.0 * f) > fabs(dxold * df)) {
                dxold = dx;  // Newton would leave the bracket or not halve it: bisect
                dx = 0.5 * (hi - lo);
                x = lo + dx;
            } else {
                dxold = dx;
                dx = f / df;
                x -= dx;
            }
            if (fabs(dx) <= REFINE_TOL) break;
            est_eval<EST>(geo, G, M, p, x, &Dx, &f, &df);
            if (f < 0.0) lo = x;
            else hi = x;
        }
    }
    double D = Db;
    float ang = (float)deg_b;
    if (x != tb) {
        est_eval<EST>(geo, G, M, p, x, &Dx, &fx, &dfx);
        if (Dx <= Db) {  // NaN keeps the grid angle
            D = Dx;
            double a = fmod(x * REFINE_RAD2DEG, 360.0);
            if (a < 0.0) a += 360.0;
            ang = (float)a;
            if (ang >= 360.0f || ang == 0.0f) ang = 0.0f;  // (also turns -0 into +0)
        }
    }
    angles[o] = ang;
    if constexpr (EST == EST_BARTLETT) {
        if (levels) levels[o] = (float)(-D / ((double)M * (double)M));
    } else {
        if (levels) levels[o] = (float)(1.0 / D);
    }
}

}  // namespace music
