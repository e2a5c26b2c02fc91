// music_calib.cuh - receiver calibration (opt-in, music_b200_set_calibration and the music_b200_calib_* entry points).
//
// Each receiver chain multiplies what its element sees by a complex gain g_m (cable, filters, LO phase), after the
// receiver noise: x_raw = diag(g) (A s + n).  The correction is x = diag(c) x_raw, c_m = 1 / g_m, applied to the fp64
// covariance of every window right after the covariance kernel,
//     R_ij <- (c_i R_ij) conj(c_j),
// so that every later stage (eigensolver, source count, scans, every peak mode, refinement, beams) sees the corrected R.
// Beam weights are handed back in raw-input coordinates, w_raw = conj(c) o w, so that the apply pass can read the raw
// input: w_raw^H x_raw = w^H x.
// The gains are estimated from windows of one dominant source at a known direction: the off-diagonal least-squares fit
// R_ij ~ h_i conj(h_j) (i != j) of the mean raw covariance, by Gauss-Seidel sweeps, then g = h / a0.  The full definition
// is in include/music_b200.h and is restated literally by tests/calibration_oracle.py.
//
// calib_apply_kernel:   one thread per (window, entry), coalesced, in place.
// calib_weights_kernel: one thread per (window, slot, element) of the beam weights, in place.
// calib_accum_kernel:   the sum over a sub-batch's windows of the raw R, in a fixed order (deterministic), added to the
//                       handle's [M][M] accumulator by the last CTA to finish.
// calib_solve_kernel:   one warp, lane <-> row: start rule, sweeps, a0, normalisation and residual.
#pragma once
#include "music_kernels.cuh"
#include "music_steer.cuh"
#include "music_refine.cuh"

namespace music {

// c_m = 1 / g_m of every element, by value: a concurrent set_calibration() cannot change what an enqueued launch reads.
struct CalibVec {
    double2 c[MAXM];
};

constexpr int CALIB_THREADS = 256;
constexpr int CALIB_ACC_MAX_CTAS = 1024;   // partial sums per accumulate launch, at most
constexpr int CALIB_ACC_MIN_WPC = 64;      // windows per accumulate CTA, at least
constexpr int CALIB_MAX_SWEEPS = 200;
constexpr double CALIB_TOL = 0x1p-40;      // stop once a sweep moves no entry by more than this times max |h|
constexpr int CALIB_PHASE = 1, CALIB_GAIN_PHASE = 2;  // MUSIC_B200_CALIB_*
// calib_solve_kernel's result: gains [M][2], then residual, sweeps, status (CALIB_OK or the failure)
constexpr int CALIB_OUT = 2 * MAXM + 3;
constexpr int CALIB_OK = 0, CALIB_NOPOWER = 1, CALIB_NONFINITE = 2, CALIB_DEAD = 3;

// c r, and r conj(c), without contraction into fma (so that a host model with the same operation order rounds alike);
// a real c (c.y == 0, the identity included) scales both parts, which keeps every bit, signed zeros too, for c = 1.
__device__ __forceinline__ double2 calib_mul(double2 c, double2 r)
{
    if (c.y == 0.0) return make_double2(__dmul_rn(c.x, r.x), __dmul_rn(c.x, r.y));
    return make_double2(__dsub_rn(__dmul_rn(c.x, r.x), __dmul_rn(c.y, r.y)), __dadd_rn(__dmul_rn(c.x, r.y), __dmul_rn(c.y, r.x)));
}
__device__ __forceinline__ double2 calib_mul_conj(double2 r, double2 c)
{
    if (c.y == 0.0) return make_double2(__dmul_rn(r.x, c.x), __dmul_rn(r.y, c.x));
    return make_double2(__dadd_rn(__dmul_rn(r.x, c.x), __dmul_rn(r.y, c.y)), __dsub_rn(__dmul_rn(r.y, c.x), __dmul_rn(r.x, c.y)));
}

// R [W][M][M] (re, im), in place: R_ij <- (c_i R_ij) conj(c_j)
__global__ void __launch_bounds__(CALIB_THREADS) calib_apply_kernel(double *__restrict__ R, int M, int W, const CalibVec cv)
{
    const size_t e = (size_t)blockIdx.x * CALIB_THREADS + threadIdx.x;
    const int MM = M * M;
    if (e >= (size_t)W * MM) return;
    const int k = (int)(e % (size_t)MM), i = k / M, j = k - i * M;
    double2 *p = reinterpret_cast<double2 *>(R) + e;
    *p = calib_mul_conj(calib_mul(cv.c[i], *p), cv.c[j]);
}

// beam weights wts [W][n][M] (re, im), in place: w_m <- conj(c_m) w_m (zero weights stay zero)
__global__ void __launch_bounds__(CALIB_THREADS) calib_weights_kernel(double *__restrict__ wts, int M, int n, int W, const CalibVec cv)
{
    const size_t e = (size_t)blockIdx.x * CALIB_THREADS + threadIdx.x;
    if (e >= (size_t)W * n * M) return;
    double2 *p = reinterpret_cast<double2 *>(wts) + e;
    *p = calib_mul_conj(*p, cv.c[(int)(e % (size_t)M)]);
}

// windows per CTA of calib_accum_kernel for a sub-batch of W windows (a function of W alone: the sum is deterministic)
__host__ __device__ inline int calib_acc_wpc(int W)
{
    const int w = (W + CALIB_ACC_MAX_CTAS - 1) / CALIB_ACC_MAX_CTAS;
    return w > CALIB_ACC_MIN_WPC ? w : CALIB_ACC_MIN_WPC;
}

// acc [M][M] (re, im) += sum over the W windows of R [W][M][M].  CTA b sums windows [b wpc, (b + 1) wpc): thread t takes
// entry t % MM of the windows g, g + G, ... (g = t / MM, G = CALIB_THREADS / MM groups), so consecutive threads read
// consecutive entries; the groups are summed in order, the CTA's sum goes to part[b], and the last CTA to finish adds
// part[0], part[1], ... to acc in order and re-arms the counter.  part: [gridDim.x][MM]; ctr: one zeroed unsigned.
__global__ void __launch_bounds__(CALIB_THREADS) calib_accum_kernel(const double *__restrict__ R, int M, int W, int wpc,
                                                                    double2 *__restrict__ part, unsigned *__restrict__ ctr,
                                                                    double2 *__restrict__ acc)
{
    __shared__ double2 s[CALIB_THREADS];
    __shared__ bool last;
    const int MM = M * M, G = CALIB_THREADS / MM, t = threadIdx.x;
    const int e = t % MM, g = t / MM;
    const int w0 = blockIdx.x * wpc, w1 = min(W, w0 + wpc);
    const double2 *Rv = reinterpret_cast<const double2 *>(R);
    double2 sum = make_double2(0.0, 0.0);
    if (g < G)
        for (int w = w0 + g; w < w1; w += G) {
            const double2 v = Rv[(size_t)w * MM + e];
            sum.x += v.x;
            sum.y += v.y;
        }
    s[t] = sum;
    __syncthreads();
    if (t < MM) {
        double2 c = s[t];
        for (int q = 1; q < G; ++q) {
            c.x += s[q * MM + t].x;
            c.y += s[q * MM + t].y;
        }
        part[(size_t)blockIdx.x * MM + t] = c;
    }
    __threadfence();
    __syncthreads();
    if (t == 0) last = atomicAdd(ctr, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (t < MM) {
        double2 c = acc[t];
        for (unsigned b = 0; b < gridDim.x; ++b) {
            const double2 v = __ldcg(part + (size_t)b * MM + t);
            c.x += v.x;
            c.y += v.y;
        }
        acc[t] = c;
    }
    if (t == 0) *ctr = 0u;
}

// The known direction of the calibration source and the geometry of the current table, by value.  A 1-D handle has
// z = 0 and el = 0 and takes the refinement's steering vector (steer_phase); an az-el handle the 3-D direction of
// music_azel.cuh, u = (cos el cos az, cos el sin az, sin el).
struct CalibSource {
    double pos[3 * MAXM];  // [M][x, y, z] in metres
    double lambda;
    double az, el;         // radians
    bool azel;
};

// one warp: acc [M][M] / nwin = Rbar; out [CALIB_OUT] (see CALIB_OUT)
__global__ void __launch_bounds__(32) calib_solve_kernel(const double2 *__restrict__ acc, double nwin, int M, const CalibSource src,
                                                         int kind, double *__restrict__ out)
{
    __shared__ double2 S[MAXM * MAXM];
    const int lane = threadIdx.x;
    const bool act = lane < M;
    bool finite = true;
    for (int e = lane; e < M * M; e += 32) {
        const double2 v = acc[e];
        S[e] = make_double2(v.x / nwin, v.y / nwin);
        finite = finite && isfinite(S[e].x) && isfinite(S[e].y);
    }
    __syncwarp();
    const auto fail = [&](int status) {
        if (lane < CALIB_OUT) out[lane] = 0.0;
        __syncwarp();
        if (lane == 0) out[2 * MAXM + 2] = (double)status;
    };
    if (!__all_sync(0xffffffffu, finite)) return fail(CALIB_NONFINITE);
    // start: r = the largest diagonal entry (lowest index on ties), h_r = sqrt(R_rr), h_i = R_ir / sqrt(R_rr)
    int r = 0;
    for (int i = 1; i < M; ++i)
        if (S[i * M + i].x > S[r * M + r].x) r = i;
    const double rr = S[r * M + r].x;
    if (!(rr > 0.0)) return fail(CALIB_NOPOWER);
    const double sr = sqrt(rr);
    double2 h = make_double2(0.0, 0.0);  // lane i: h_i
    if (act) h = lane == r ? make_double2(sr, 0.0) : make_double2(S[lane * M + r].x / sr, S[lane * M + r].y / sr);
    // Gauss-Seidel: h_i <- (sum_{j != i} R_ij h_j) / (sum_{j != i} |h_j|^2), i = 0 .. M-1, with the updated entries
    int sweeps = 0;
    while (sweeps < CALIB_MAX_SWEEPS) {
        ++sweeps;
        double dmax = 0.0;
        for (int i = 0; i < M; ++i) {
            const bool term = act && lane != i;
            const double2 p = term ? cmul(S[i * M + lane], h) : make_double2(0.0, 0.0);
            const double q = term ? fma(h.x, h.x, h.y * h.y) : 0.0;
            const double nr = warp_sum(p.x), ni = warp_sum(p.y), d = warp_sum(q);
            if (lane == i) {
                const double2 hn = make_double2(nr / d, ni / d);
                dmax = fmax(dmax, hypot(hn.x - h.x, hn.y - h.y));
                h = hn;
            }
        }
        double hmax = act ? hypot(h.x, h.y) : 0.0;
        for (int o = 16; o > 0; o >>= 1) {
            dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
            hmax = fmax(hmax, __shfl_xor_sync(0xffffffffu, hmax, o));
        }
        if (!(dmax > CALIB_TOL * hmax)) break;  // (NaN stops too; the checks below reject it)
    }
    const bool bad = act && (!isfinite(h.x) || !isfinite(h.y));
    if (__any_sync(0xffffffffu, bad)) return fail(CALIB_NONFINITE);
    if (__any_sync(0xffffffffu, act && h.x == 0.0 && h.y == 0.0)) return fail(CALIB_DEAD);
    // residual: sum_{i != j} |R_ij - h_i conj(h_j)|^2 / sum_{i != j} |R_ij|^2, lane i summing row i
    double num = 0.0, den = 0.0;
    for (int j = 0; j < M; ++j) {
        const double2 hj = make_double2(__shfl_sync(0xffffffffu, h.x, j), __shfl_sync(0xffffffffu, h.y, j));
        if (act && j != lane) {
            const double2 v = S[lane * M + j];
            const double er = v.x - (h.x * hj.x + h.y * hj.y), ei = v.y - (h.y * hj.x - h.x * hj.y);
            num += er * er + ei * ei;
            den += v.x * v.x + v.y * v.y;
        }
    }
    num = warp_sum(num);
    den = warp_sum(den);
    // a0 of the known direction, g = h / a0, rotated so that g_0 is real and positive, then normalised
    double2 g = make_double2(0.0, 0.0);
    if (act) {
        double phi;
        if (src.azel) {
            double sa, ca, se, ce;
            sincos(src.az, &sa, &ca);
            sincos(src.el, &se, &ce);
            const double *p = src.pos + 3 * lane;
            phi = STEER_TWO_PI * ((p[0] * (ce * ca) + p[1] * (ce * sa) + p[2] * se) / src.lambda);
        } else {
            RefineGeom geo;
            geo.pos[2 * lane] = src.pos[3 * lane];
            geo.pos[2 * lane + 1] = src.pos[3 * lane + 1];
            geo.lambda = src.lambda;
            double st, ct, psi;
            sincos(src.az, &st, &ct);
            steer_phase(geo, lane, st, ct, &phi, &psi);
        }
        double sp, cp;
        sincos(phi, &sp, &cp);
        // h / a0 with a0 = (cp, -sp): h conj(a0) / |a0|^2
        const double na = cp * cp + sp * sp;
        g = make_double2((h.x * cp - h.y * sp) / na, (h.y * cp + h.x * sp) / na);
    }
    const double2 g0 = make_double2(__shfl_sync(0xffffffffu, g.x, 0), __shfl_sync(0xffffffffu, g.y, 0));
    const double a0 = hypot(g0.x, g0.y);
    const double2 rot = make_double2(g0.x / a0, -g0.y / a0);
    g = cmul(g, rot);
    if (kind == CALIB_PHASE) {
        const double a = hypot(g.x, g.y);
        if (act) g = make_double2(g.x / a, g.y / a);
    } else {
        const double s2 = warp_sum(act ? g.x * g.x + g.y * g.y : 0.0);
        const double f = sqrt((double)M / s2);
        g = make_double2(g.x * f, g.y * f);
    }
    const bool gbad = act && (!isfinite(g.x) || !isfinite(g.y));
    if (__any_sync(0xffffffffu, gbad)) return fail(CALIB_NONFINITE);
    if (lane < MAXM) {
        out[2 * lane] = act ? g.x : 0.0;
        out[2 * lane + 1] = act ? g.y : 0.0;
    }
    if (lane == 0) {
        out[2 * MAXM] = sqrt(num / den);
        out[2 * MAXM + 1] = (double)sweeps;
        out[2 * MAXM + 2] = (double)CALIB_OK;
    }
}

}  // namespace music
