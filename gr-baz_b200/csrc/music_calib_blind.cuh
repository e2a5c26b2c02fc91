// music_calib_blind.cuh - receiver self-calibration without a known source (the music_b200_calib_blind_* entry points).
//
// Weiss-Friedlander eigenstructure calibration with the magnitudes read from the diagonal and a multi-start phase
// search; the definition is in include/music_b200.h and is restated literally by tests/calib_blind_oracle.py.  The
// segment covariances R_s are summed by music_calib.cuh's calib_accum_kernel, one launch per segment; the solve runs:
//
// cb_prep_kernel:    one CTA: R_s = sum / windows, the magnitudes from the mean diagonal, the whitened R_s (the input of
//                    the handle's eigensolver) and the non-finite flag.
// cb_proj_kernel:    Pi_s = E_s E_s^H from the eigensolver's sorted eigenvectors, one thread per entry.
// cb_init_kernel:    the start phases (cb_draw) and the solve state.
// cb_scan_kernel:    the hot path, one CTA per (start, segment): P_s(k) = ||E_s^H (phi o a_k)||^2 / M over the table into
//                    shared memory, then the d best local maxima of 1 / P (topn_local_kernel's rule, excl = 0), their
//                    bins and the sum of P at them.
// cb_q_kernel:       one CTA per start: Q = sum_s sum_i D_k^H Pi_s D_k in segment then pick order, thread <-> entry, and
//                    J = sum_s J_s in segment order (J_s: the scan's sum over the picks); Q goes to the handle's eigensolver.
// cb_update_kernel:  one thread per start: phi <- the smallest eigenvector, v_0 made real positive, unit moduli.
// cb_select_kernel:  the start with the smallest J (lowest index on ties, NaN never wins).
// cb_out_kernel:     the gains, angles and stats of the winner.
// In the polish phase the scan, Q and update kernels serve the winner only (the Q slot 0) and return at once after the
// iteration that converged, so the host enqueues fixed counts and synchronises once.
#pragma once
#include "music_kernels.cuh"

namespace music {

constexpr int CB_T1 = 24, CB_T2 = 30;          // iterations of every start; polish iterations of the winner, at most
constexpr double CB_TOL = 0x1p-30;             // polish stops once max_m |phi_new - phi_old| <= this
constexpr int CB_MAX_STARTS = 256;
constexpr int CB_MAX_SEGMENTS = 1024;          // MUSIC_B200_CALIB_MAX_SEGMENTS
constexpr int CB_THREADS = 256;
constexpr int CB_MAX_K = 24576;                // table rows the scan holds in shared memory
constexpr int CB_OUT = 2 * MAXM + 4;           // gains [M][2], misfit, polish iterations, winner, status
constexpr int CB_OK = 0, CB_NONFINITE_INPUT = 1, CB_NONFINITE_FIT = 2;  // status

// the solve's device state: the winner, whether the polish has converged, the polish iterations run, non-finite input
struct CbState {
    int winner, done, used, bad;
};

// the splitmix64 finaliser, and the start phase of (seed, start, element): tests/calib_blind_oracle.py::draw
__host__ __device__ inline unsigned long long cb_mix64(unsigned long long z)
{
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__host__ __device__ inline double cb_draw(unsigned long long seed, int start, int element)
{
    const unsigned long long key = ((unsigned long long)start * 256ull + (unsigned long long)element + 1ull) * 0x9E3779B97F4A7C15ull;
    const unsigned long long z = cb_mix64(seed ^ key);
    return 3.141592653589793 * (2.0 * ((double)(z >> 11) * 0x1p-53) - 1.0);
}

// acc [S][M][M] sums of cnt [S] windows -> Rw [S][M][M] (re, im) whitened, mag [M]; st->bad when anything is not
// finite or some magnitude is not > 0
__global__ void __launch_bounds__(CB_THREADS) cb_prep_kernel(const double2 *__restrict__ acc, const unsigned *__restrict__ cnt,
                                                             int M, int S, double *__restrict__ Rw, double *__restrict__ mag,
                                                             CbState *__restrict__ st)
{
    __shared__ double t[MAXM];
    __shared__ int bad;
    const int MM = M * M;
    if (threadIdx.x == 0) bad = 0;
    __syncthreads();
    if (threadIdx.x < M) {
        const int m = threadIdx.x;
        double sum = 0.0;
        for (int s = 0; s < S; ++s) sum += acc[(size_t)s * MM + m * M + m].x / (double)cnt[s];
        t[m] = sqrt(sum / (double)S);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s2 = 0.0;
        for (int m = 0; m < M; ++m) s2 += t[m] * t[m];
        const double f = sqrt((double)M / s2);
        for (int m = 0; m < M; ++m) {
            const double g = t[m] * f;
            mag[m] = g;
            if (!(g > 0.0) || !isfinite(g)) bad = 1;
            t[m] = 1.0 / g;
        }
    }
    __syncthreads();
    int mybad = 0;
    for (int e = threadIdx.x; e < S * MM; e += CB_THREADS) {
        const int s = e / MM, k = e - s * MM, i = k / M, j = k - i * M;
        const double2 v = acc[e];
        const double n = (double)cnt[s];
        const double re = v.x / n, im = v.y / n;
        if (!isfinite(re) || !isfinite(im)) mybad = 1;
        Rw[2 * (size_t)e] = (t[i] * re) * t[j];
        Rw[2 * (size_t)e + 1] = (t[i] * im) * t[j];
    }
    if (mybad) bad = 1;
    __syncthreads();
    if (threadIdx.x == 0) st->bad = bad;
}

// Pi [S][M][M] = sum_{j < L} e_j e_j^H of the sorted eigenvectors Vt [S][M][M] (vector j, component i)
__global__ void __launch_bounds__(CB_THREADS) cb_proj_kernel(const double *__restrict__ Vt, int M, int L, int S, double2 *__restrict__ Pi)
{
    const size_t e = (size_t)blockIdx.x * CB_THREADS + threadIdx.x;
    const int MM = M * M;
    if (e >= (size_t)S * MM) return;
    const size_t s = e / MM;
    const int k = (int)(e - s * MM), m = k / M, n = k - m * M;
    const double2 *V = reinterpret_cast<const double2 *>(Vt) + s * MM;
    double2 p = make_double2(0.0, 0.0);
    for (int j = 0; j < L; ++j) {
        const double2 a = V[j * M + m], b = V[j * M + n];
        p.x += a.x * b.x + a.y * b.y;
        p.y += a.y * b.x - a.x * b.y;
    }
    Pi[e] = p;
}

// phi [P][M]: start 0 all ones, start p >= 1 the drawn phases; the state cleared
__global__ void cb_init_kernel(double2 *__restrict__ phi, int M, int P, unsigned long long seed, CbState *__restrict__ st)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e == 0) { st->winner = 0; st->done = 0; st->used = 0; }
    if (e >= P * M) return;
    const int p = e / M, m = e - p * M;
    if (p == 0) { phi[e] = make_double2(1.0, 0.0); return; }
    double sn, cs;
    sincos(cb_draw(seed, p, m), &sn, &cs);
    phi[e] = make_double2(cs, sn);
}

// One CTA per (start, segment) pair: blockIdx.x = p * S + s, or in the polish phase s with p the winner.  bins [P][S][d]
// (-1: no further local maximum), jp [P][S] the sum of P_s at the picks in pick order.  Dynamic shared memory: K doubles.
template <int MA>
__global__ void __launch_bounds__(CB_THREADS) cb_scan_kernel(const double *__restrict__ soa, int K, int M, int d, int S,
                                                             const double *__restrict__ Vt, const double2 *__restrict__ phi,
                                                             bool polish, const CbState *__restrict__ st,
                                                             int *__restrict__ bins, double *__restrict__ jp)
{
    extern __shared__ __align__(16) double sP[];
    __shared__ double2 sB[MAXM * MAXM];  // sB[j][i] = phi_i conj(e_j,i): y_j = sum_i sB[j][i] a_i = e_j^H (phi o a)
    __shared__ double rP[CB_THREADS / 32];
    __shared__ int rk[CB_THREADS / 32];
    __shared__ int taken[MAXM];
    if (polish && st->done) return;
    const int p = polish ? st->winner : blockIdx.x / S, s = polish ? blockIdx.x : blockIdx.x % S;
    const int L = M - d, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const double2 *V = reinterpret_cast<const double2 *>(Vt) + (size_t)s * M * M;
    for (int e = tid; e < L * M; e += CB_THREADS) {
        const int j = e / M, i = e - j * M;
        sB[e] = cmul(phi[(size_t)p * M + i], make_double2(V[j * M + i].x, -V[j * M + i].y));
    }
    __syncthreads();
    const double invM = 1.0 / (double)M;
    for (int k = tid; k < K; k += CB_THREADS) {
        const double *tb = soa + (size_t)(k / TILE) * (2 * M + 1) * TILE + (k % TILE);
        double ar[MA], ai[MA];
#pragma unroll
        for (int i = 0; i < MA; ++i) {
            ar[i] = i < M ? tb[(size_t)(2 * i) * TILE] : 0.0;
            ai[i] = i < M ? tb[(size_t)(2 * i + 1) * TILE] : 0.0;
        }
        double acc = 0.0;
        for (int j = 0; j < L; ++j) {
            double yr = 0.0, yi = 0.0;
#pragma unroll
            for (int i = 0; i < MA; ++i) {
                if (i >= M) break;
                const double2 b = sB[j * M + i];
                yr = fma(b.x, ar[i], fma(-b.y, ai[i], yr));
                yi = fma(b.x, ai[i], fma(b.y, ar[i], yi));
            }
            acc = fma(yr, yr, fma(yi, yi, acc));
        }
        sP[k] = acc * invM;
    }
    __syncthreads();
    // the d best circular local maxima of q = 1 / P: q > 0, q[k] > q[k-1], q[k] >= q[k+1]; larger q, then lower k
    double J = 0.0;
    bool dry = false;
    for (int r = 0; r < d; ++r) {
        double bq = 0.0;
        int bk = -1;
        if (!dry)
            for (int k = tid; k < K; k += CB_THREADS) {
                const double q = 1.0 / sP[k];
                if (!(q > 0.0) || !(q > bq)) continue;  // also skips NaN; an equal q at a higher k never wins
                const double ql = 1.0 / sP[k == 0 ? K - 1 : k - 1], qr = 1.0 / sP[k == K - 1 ? 0 : k + 1];
                if (!(q > ql) || !(q >= qr)) continue;
                bool ok = true;
                for (int t = 0; t < r; ++t) ok = ok && taken[t] != k;
                if (ok) { bq = q; bk = k; }
            }
        warp_argmax(bq, bk);
        if (lane == 0) { rP[wid] = bq; rk[wid] = bk; }
        __syncthreads();
        if (tid == 0) {
            double q = rP[0];
            int k = rk[0];
            for (int w = 1; w < CB_THREADS / 32; ++w)
                if (peak_better(rP[w], rk[w], q, k)) { q = rP[w]; k = rk[w]; }
            taken[r] = k;
            bins[((size_t)p * S + s) * d + r] = k;
            if (k >= 0) J += sP[k];
        }
        __syncthreads();
        dry = taken[r] < 0;
    }
    if (tid == 0) jp[(size_t)p * S + s] = J;
}

// One CTA per start (polish: one CTA for the winner, written to slot 0): Q [slot][M][M] (re, im) and J [p]
__global__ void __launch_bounds__(CB_THREADS) cb_q_kernel(const double *__restrict__ soa, int M, int d, int S,
                                                          const double2 *__restrict__ Pi, const int *__restrict__ bins,
                                                          const double *__restrict__ jp, bool polish, const CbState *__restrict__ st,
                                                          double *__restrict__ Q, double *__restrict__ J)
{
    if (polish && st->done) return;
    const int p = polish ? st->winner : blockIdx.x, slot = polish ? 0 : p;
    const int MM = M * M, e = threadIdx.x;
    if (e == 0) {
        double j = 0.0;
        for (int s = 0; s < S; ++s) j += jp[(size_t)p * S + s];
        J[p] = j;
    }
    if (e >= MM) return;
    const int m = e / M, n = e - m * M;
    double2 q = make_double2(0.0, 0.0);
    for (int s = 0; s < S; ++s) {
        const double2 pi = Pi[(size_t)s * MM + e];
        for (int i = 0; i < d; ++i) {
            const int k = bins[((size_t)p * S + s) * d + i];
            if (k < 0) break;
            const double *tb = soa + (size_t)(k / TILE) * (2 * M + 1) * TILE + (k % TILE);
            const double2 am = make_double2(tb[(size_t)(2 * m) * TILE], tb[(size_t)(2 * m + 1) * TILE]);
            const double2 an = make_double2(tb[(size_t)(2 * n) * TILE], tb[(size_t)(2 * n + 1) * TILE]);
            const double2 v = cjmul(am, cmul(pi, an));
            q.x += v.x;
            q.y += v.y;
        }
    }
    Q[2 * ((size_t)slot * MM + e)] = q.x;
    Q[2 * ((size_t)slot * MM + e) + 1] = q.y;
}

// One thread per start (polish: the winner, from slot 0): phi [p] <- the smallest eigenvector of its Q (qV [slot][0]),
// rotated so that element 0 is real and positive, element-wise unit moduli.  Polish: counts the iteration and marks the
// state done once no element moved by more than CB_TOL.
__global__ void cb_update_kernel(const double *__restrict__ qV, int M, int P, bool polish, CbState *__restrict__ st,
                                 double2 *__restrict__ phi)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (polish ? (t != 0 || st->done) : t >= P) return;
    const int p = polish ? st->winner : t, slot = polish ? 0 : t;
    const double2 *v = reinterpret_cast<const double2 *>(qV) + (size_t)slot * M * M;  // vector 0, component i
    const double a0 = hypot(v[0].x, v[0].y);
    const double2 rot = make_double2(v[0].x / a0, -v[0].y / a0);
    double delta = 0.0;
    for (int i = 0; i < M; ++i) {
        const double2 w = cmul(v[i], rot);
        const double a = hypot(w.x, w.y);
        const double2 f = make_double2(w.x / a, w.y / a);
        const double2 o = phi[(size_t)p * M + i];
        delta = fmax(delta, hypot(f.x - o.x, f.y - o.y));
        phi[(size_t)p * M + i] = f;
    }
    if (polish) {
        st->used += 1;
        if (delta <= CB_TOL) st->done = 1;
    }
}

// the start with the smallest J (lowest index on ties; NaN never wins, start 0 when every J is NaN)
__global__ void cb_select_kernel(const double *__restrict__ J, int P, CbState *__restrict__ st)
{
    int b = -1;
    for (int p = 0; p < P; ++p)
        if (!isnan(J[p]) && (b < 0 || J[p] < J[b])) b = p;
    st->winner = b < 0 ? 0 : b;
}

// out [CB_OUT]: the winner's gains (mag o phi, or phi with `phase_only`), misfit J / (S d), polish iterations, winner,
// status (CB_*); angles [S][d]: k 360 / K degrees of the final picks, NaN where none
__global__ void cb_out_kernel(const double2 *__restrict__ phi, const double *__restrict__ mag, const int *__restrict__ bins,
                              const double *__restrict__ J, int M, int S, int d, int K, bool phase_only,
                              const CbState *__restrict__ st, double *__restrict__ out, double *__restrict__ angles)
{
    const int p = st->winner;
    for (int e = threadIdx.x; e < S * d; e += blockDim.x) {
        const int k = bins[(size_t)p * S * d + e];
        angles[e] = k >= 0 ? (double)k * 360.0 / (double)K : __longlong_as_double(0x7ff8000000000000LL);
    }
    __shared__ int fit_bad;
    if (threadIdx.x == 0) fit_bad = 0;
    __syncthreads();
    if (threadIdx.x < M) {
        const int m = threadIdx.x;
        const double2 f = phi[(size_t)p * M + m];
        const double g = phase_only ? 1.0 : mag[m];
        out[2 * m] = g * f.x;
        out[2 * m + 1] = g * f.y;
        // an eigenvector component of exactly zero leaves its phase undefined (NaN): the fit failed
        if (!isfinite(out[2 * m]) || !isfinite(out[2 * m + 1])) fit_bad = 1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        out[2 * MAXM] = J[p] / ((double)S * (double)d);
        out[2 * MAXM + 1] = (double)st->used;
        out[2 * MAXM + 2] = (double)p;
        out[2 * MAXM + 3] = st->bad ? CB_NONFINITE_INPUT : fit_bad || !isfinite(J[p]) ? CB_NONFINITE_FIT : CB_OK;
    }
}

}  // namespace music
