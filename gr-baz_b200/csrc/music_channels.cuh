// music_channels.cuh - frequency-channelised covariance (opt-in, music_b200_create_channels): an FFT filter bank fused
// into the covariance, one M x M Hermitian problem per (window, channel), and the incoherent wideband MUSIC combine.
//
// Definition (include/music_b200.h, restated literally by tests/channels_oracle.py): window w of N snapshots is cut into
// J = N / F consecutive segments of F snapshots; X_j[b] = sum_t h[t] x[jF + t] exp(-2 pi i b t / F) (an M-vector);
// channel c is FFT bin b_c = (first + c) mod F; R_c = sum_j X_j[b_c] X_j[b_c]^H / (J sum_t h[t]^2), all fp64.
//
// chan_cov_kernel: persistent CTAs, each takes whole windows.  A window is streamed once per channel group, in batches of B
// consecutive segments (B the largest divisor of J with B F M <= 2048 samples, so that every barrier interval has work for
// the whole CTA), through a ring of bulk copies (TMA) completed on mbarriers, the idiom of cov4_tma_kernel.  Per batch:
//   1. widen the B x F x M complex64 samples to fp64, times the taper (one rounding; exact for RECT), into B M rows of
//      F + 1 complex values (the odd row length keeps the transposing store off one shared-memory bank);
//   2. log2(F) radix-2 decimation-in-frequency stages in shared memory (natural order in, bit-reversed order out), two
//      stages per pass on four entries in registers, twiddles exp(-2 pi i k / F) from a host-built table;
//   3. every selected channel's rank-one updates X X^H, segment after segment, into fp64 accumulators (Hermitian half,
//      E = M (M + 1) / 2 entries per channel) that live in registers during a batch and in shared memory between
//      batches.  Entry (e, c) belongs to one thread for the whole window (warp = e mod 8, lane = c mod 32), so there are
//      no atomics and the sum over j runs in segment order.
// All F bins are always computed and a channel's accumulator sees the segments in the same order whatever else was
// asked for: R_c does not depend on the channel range, the group split, the grid size or the sub-batch.
// Where the accumulators of all C channels do not fit next to the ring and the FFT buffer, the channels are taken in
// groups of Cg, re-reading the window (from L2 at these sizes) and repeating the FFT: a plain outer loop.
#pragma once
#include "music_kernels.cuh"

namespace music {

constexpr int CHAN_THREADS = 256;
constexpr int CHAN_STAGES = 3;      // segments in flight per CTA
constexpr int CHAN_MIN_F = 8, CHAN_MAX_F = 256;
constexpr size_t CHAN_SMEM_MAX = 232448;  // 227 KiB: the most dynamic shared memory one sm_90 CTA can have
constexpr int CHAN_SEPARATE = 0, CHAN_INCOHERENT = 1;  // = MUSIC_B200_CHANNELS_*
constexpr int CHAN_RECT = 0, CHAN_HANN = 1;            // = MUSIC_B200_TAPER_*

struct ChanShape {
    int M, N, F, logF, J;   // antennas, snapshots per window, FFT length and its log2, segments per window
    int first, C;           // channel c is bin (first + c) mod F
    int B;                  // segments per batch (a divisor of J)
    int Cg, groups;         // channels per group (accumulators resident together), number of groups
    double denom;           // J * sum_t h[t]^2
};

constexpr int CHAN_BATCH_SAMPLES = 2048;  // antenna samples per batch, where a window has that many segments

// the largest divisor of J whose batch holds at most CHAN_BATCH_SAMPLES antenna samples (1 when one segment has more)
inline int chan_batch(int M, int F, int J)
{
    int best = 1;
    for (int b = 1; b <= J && b * F * M <= CHAN_BATCH_SAMPLES; ++b)
        if (J % b == 0) best = b;
    return best;
}

// shared-memory layout of chan_cov_kernel, in bytes from the start of the dynamic segment
struct ChanSmem {
    size_t ring, fft, tw, taper, pairs, acc, total;
};

__host__ __device__ inline ChanSmem chan_smem(int M, int F, int B, int Cg)
{
    ChanSmem s;
    s.ring = 128;                                               // after the mbarriers
    s.fft = s.ring + (size_t)CHAN_STAGES * B * F * M * 8;       // [B][M][F + 1] double2
    s.tw = s.fft + (size_t)B * M * (F + 1) * 16;                // [F / 2] double2
    s.taper = s.tw + (size_t)(F / 2) * 16;                      // [F] double
    s.pairs = s.taper + (size_t)F * 8;                          // [E] (i, k) bytes, padded to 512
    s.acc = s.pairs + 512;                                      // [E][Cg] double2
    s.total = s.acc + (size_t)Cg * (M * (M + 1) / 2) * 16;
    return s;
}

// the most channels whose accumulators fit one CTA (at least 29, at M = 16 and F = 256)
inline int chan_group_size(int M, int F, int B, int C)
{
    const size_t fixed = chan_smem(M, F, B, 0).total, per = (size_t)(M * (M + 1) / 2) * 16;
    return (int)std::min<size_t>((size_t)C, (CHAN_SMEM_MAX - fixed) / per);
}

__global__ void __launch_bounds__(CHAN_THREADS, 3) chan_cov_kernel(const float *__restrict__ in, double *__restrict__ R, int W,
                                                                const ChanShape sh, const double2 *__restrict__ tw_g,
                                                                const double *__restrict__ taper_g)
{
    extern __shared__ __align__(128) unsigned char chan_sm[];
    const int M = sh.M, F = sh.F, logF = sh.logF, B = sh.B, Cg = sh.Cg;
    const int E = M * (M + 1) / 2, FP = F + 1, nb = sh.J / B;
    const ChanSmem L = chan_smem(M, F, B, Cg);
    const float2 *ring = reinterpret_cast<const float2 *>(chan_sm + L.ring);
    double2 *buf = reinterpret_cast<double2 *>(chan_sm + L.fft);
    double2 *tw = reinterpret_cast<double2 *>(chan_sm + L.tw);
    double *taper = reinterpret_cast<double *>(chan_sm + L.taper);
    uchar2 *pairs = reinterpret_cast<uchar2 *>(chan_sm + L.pairs);
    double2 *acc = reinterpret_cast<double2 *>(chan_sm + L.acc);
    const uint32_t bar0 = smem_u32(chan_sm), ring0 = smem_u32(chan_sm + L.ring);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t batch_bytes = (uint32_t)B * F * M * 8;

    const int nwin = (int)blockIdx.x < W ? (W - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    const long long total = (long long)nwin * sh.groups * nb;  // batches this CTA loads

    if (tid == 0) {
        for (int s = 0; s < CHAN_STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    for (int i = tid; i < F / 2; i += CHAN_THREADS) tw[i] = tw_g[i];
    for (int i = tid; i < F; i += CHAN_THREADS) taper[i] = taper_g[i];
    if (tid == 0) {
        int e = 0;
        for (int i = 0; i < M; ++i)
            for (int k = i; k < M; ++k) pairs[e++] = make_uchar2((unsigned char)i, (unsigned char)k);
    }
    __syncthreads();

    // The stream is read once when the channels fit one group; with more groups only the last pass is marked
    // evict_first, so that the passes before it leave the window in L2.
    const uint64_t pol_stream = l2_policy_evict_first();
    const unsigned char *src0 = reinterpret_cast<const unsigned char *>(in);
    int wi_i = 0, g_i = 0, jb_i = 0, slot_i = 0;  // thread 0: the next batch to load (window, group, batch) and its slot
    auto issue = [&]() {
        const size_t w = (size_t)blockIdx.x + (size_t)wi_i * gridDim.x;
        const unsigned char *src = src0 + ((w * (size_t)sh.N + (size_t)jb_i * B * F) * M) * 8;
        mbar_expect_tx(bar0 + 8 * slot_i, batch_bytes);
        if (g_i == sh.groups - 1) bulk_g2s_hint(ring0 + slot_i * batch_bytes, src, batch_bytes, bar0 + 8 * slot_i, pol_stream);
        else bulk_g2s(ring0 + slot_i * batch_bytes, src, batch_bytes, bar0 + 8 * slot_i);
        if (++slot_i == CHAN_STAGES) slot_i = 0;
        if (++jb_i == nb) {
            jb_i = 0;
            if (++g_i == sh.groups) { g_i = 0; ++wi_i; }
        }
    };
    if (tid == 0)
        for (long long q = 0; q < total && q < CHAN_STAGES; ++q) issue();

    // thread (u0, r) of the widening step: antenna r, snapshots u0, u0 + tpr, ... of the batch
    const int tpr = CHAN_THREADS / M, r_ld = tid % M, u0_ld = tid / M;
    const int half_f = F >> 1, rows = B * M;

    int wi = 0, g = 0, jb = 0, slot = 0;
    uint32_t parity = 0;
    for (long long q = 0; q < total; ++q) {
        while (!mbar_try_wait(bar0 + 8 * slot, parity)) {}
        const float2 *seg = ring + (size_t)slot * B * F * M;
        if (u0_ld < tpr) {
            for (int u = u0_ld; u < B * F; u += tpr) {
                const float2 x = seg[u * M + r_ld];
                const int t = u & (F - 1);
                const double h = taper[t];
                buf[((u >> logF) * M + r_ld) * FP + t] = make_double2((double)x.x * h, (double)x.y * h);
            }
        }
        __syncthreads();  // the slot has been read: it may be refilled
        if (tid == 0 && q + CHAN_STAGES < total) issue();
        if (++slot == CHAN_STAGES) { slot = 0; parity ^= 1; }

        // Two radix-2 stages at a time on four entries held in registers (the arithmetic of the two stages, unchanged):
        // half the passes over shared memory and half the barriers; an odd log2(F) leaves one single stage.
        int s = 0;
        for (; s + 1 < logF; s += 2) {
            const int lh = logF - 1 - s, half = 1 << lh, quarter = half >> 1;  // stage s spans `half`, stage s + 1 `quarter`
            for (int b = tid; b < rows * (F >> 2); b += CHAN_THREADS) {
                const int row = b >> (logF - 2), p = b & ((F >> 2) - 1);
                const int k = p & (quarter - 1);
                const int i0 = row * FP + ((p >> (lh - 1)) << (lh + 1)) + k;
                const double2 wa = tw[k << s], wb = tw[(k + quarter) << s], wc = tw[k << (s + 1)];
                const double2 x0 = buf[i0], x1 = buf[i0 + quarter], x2 = buf[i0 + half], x3 = buf[i0 + half + quarter];
                // stage s: (x0, x2) with wa, (x1, x3) with wb
                const double d0r = x0.x - x2.x, d0i = x0.y - x2.y, d1r = x1.x - x3.x, d1i = x1.y - x3.y;
                const double2 y0 = make_double2(x0.x + x2.x, x0.y + x2.y), y1 = make_double2(x1.x + x3.x, x1.y + x3.y);
                const double2 y2 = make_double2(fma(d0r, wa.x, -(d0i * wa.y)), fma(d0r, wa.y, d0i * wa.x));
                const double2 y3 = make_double2(fma(d1r, wb.x, -(d1i * wb.y)), fma(d1r, wb.y, d1i * wb.x));
                // stage s + 1: (y0, y1) and (y2, y3), both with wc
                const double e0r = y0.x - y1.x, e0i = y0.y - y1.y, e1r = y2.x - y3.x, e1i = y2.y - y3.y;
                buf[i0] = make_double2(y0.x + y1.x, y0.y + y1.y);
                buf[i0 + quarter] = make_double2(fma(e0r, wc.x, -(e0i * wc.y)), fma(e0r, wc.y, e0i * wc.x));
                buf[i0 + half] = make_double2(y2.x + y3.x, y2.y + y3.y);
                buf[i0 + half + quarter] = make_double2(fma(e1r, wc.x, -(e1i * wc.y)), fma(e1r, wc.y, e1i * wc.x));
            }
            __syncthreads();
        }
        if (s < logF) {  // the last stage of an odd log2(F): neighbours, twiddle 1
            for (int b = tid; b < rows * half_f; b += CHAN_THREADS) {
                const int row = b >> (logF - 1), p = b & (half_f - 1);
                const int lo = row * FP + (p << 1);
                const double2 w = tw[0];
                const double2 a = buf[lo], c = buf[lo + 1];
                const double dr = a.x - c.x, di = a.y - c.y;
                buf[lo] = make_double2(a.x + c.x, a.y + c.y);
                buf[lo + 1] = make_double2(fma(dr, w.x, -(di * w.y)), fma(dr, w.y, di * w.x));
            }
            __syncthreads();
        }

        const int c_base = g * Cg, cg = min(Cg, sh.C - c_base);
        for (int e = warp; e < E; e += CHAN_THREADS / 32) {
            const uchar2 ik = pairs[e];
            for (int cl = lane; cl < cg; cl += 32) {
                const int bin = (sh.first + c_base + cl) & (F - 1);
                const int pos = (int)(__brev((unsigned)bin) >> (32 - logF));  // where the transform left bin `bin`
                const double2 *xi = buf + (int)ik.x * FP + pos, *xk = buf + (int)ik.y * FP + pos;
                double2 v = jb == 0 ? make_double2(0.0, 0.0) : acc[e * Cg + cl];
                for (int sg = 0; sg < B; ++sg) {
                    const double2 a = xi[sg * M * FP], c = xk[sg * M * FP];
                    v.x = fma(a.x, c.x, fma(a.y, c.y, v.x));
                    v.y = fma(a.y, c.x, fma(-a.x, c.y, v.y));
                }
                if (jb == nb - 1) {
                    // R[c][w][i][k] = x_i conj(x_k) summed, and its mirror; the diagonal is real
                    const size_t w = (size_t)blockIdx.x + (size_t)wi * gridDim.x;
                    double *Rw = R + (((size_t)(c_base + cl) * W + w) * M * M) * 2;
                    const double re = v.x / sh.denom, im = v.y / sh.denom;
                    Rw[2 * (ik.x * M + ik.y)] = re;
                    Rw[2 * (ik.x * M + ik.y) + 1] = ik.x == ik.y ? 0.0 : im;
                    if (ik.x != ik.y) {
                        Rw[2 * (ik.y * M + ik.x)] = re;
                        Rw[2 * (ik.y * M + ik.x) + 1] = -im;
                    }
                } else {
                    acc[e * Cg + cl] = v;
                }
            }
        }
        __syncthreads();  // the FFT buffer is free for the next batch
        if (++jb == nb) {
            jb = 0;
            if (++g == sh.groups) { g = 0; ++wi; }
        }
    }
}

// Incoherent wideband MUSIC (Wax, Shan and Kailath 1984): P64 holds the C channels' MUSIC strengths [C][W][K] of one
// sub-batch.  D = sum_c 1 / P_c in channel order (one thread per (w, k): no atomics, reproducible), P = 1 / D into channel
// 0's block, which the peak rules then read, and into the float spectrum row when asked.
__global__ void __launch_bounds__(256) chan_combine_kernel(double *__restrict__ P64, int C, size_t WK, float *__restrict__ spectrum)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= WK) return;
    double D = 0.0;
    for (int c = 0; c < C; ++c) D += 1.0 / P64[(size_t)c * WK + i];
    const double P = 1.0 / D;
    P64[i] = P;
    if (spectrum) spectrum[i] = (float)P;
}

// ---- host side of the filter bank: correctly rounded twiddles and the taper ----

// (cos, sin)(2 pi k / F) for 0 <= k < F, F a power of two: reduced to the first octant, where the long double
// evaluation rounds to the correctly rounded fp64 value, and exact at the multiples of pi / 2
inline void chan_cos_sin(int k, int F, double &c, double &s)
{
    const long double two_pi = 6.283185307179586476925286766559005768L;
    const int q = F / 4;
    if (F >= 4 && k >= q) {  // rotate by a quarter turn: cos(t + pi/2) = -sin t, sin(t + pi/2) = cos t
        double c1, s1;
        chan_cos_sin(k - q, F, c1, s1);
        c = -s1;
        s = c1;
        if (c == 0.0) c = 0.0;  // no negative zero
        return;
    }
    if (k == 0) { c = 1.0; s = 0.0; return; }
    if (8 * k == F) { c = s = (double)sqrtl(0.5L); return; }
    if (8 * k < F) {
        const long double t = two_pi * k / F;
        c = (double)cosl(t);
        s = (double)sinl(t);
    } else {  // second octant: reflect about pi / 4
        const long double t = two_pi * (q - k) / F;
        c = (double)sinl(t);
        s = (double)cosl(t);
    }
}

// tw[k] = exp(-2 pi i k / F), k < F / 2;  taper[t] = 1 (RECT) or 1/2 - 1/2 cos(2 pi t / F) (periodic HANN);
// returns sum_t taper[t]^2 summed in ascending t
inline double chan_tables_host(int F, int taper_kind, double2 *tw, double *taper)
{
    for (int k = 0; k < F / 2; ++k) {
        double c, s;
        chan_cos_sin(k, F, c, s);
        tw[k] = make_double2(c, -s);
    }
    double sum = 0.0;
    for (int t = 0; t < F; ++t) {
        double c, s;
        chan_cos_sin(t, F, c, s);
        taper[t] = taper_kind == CHAN_HANN ? 0.5 - 0.5 * c : 1.0;
        sum += taper[t] * taper[t];
    }
    return sum;
}

}  // namespace music
