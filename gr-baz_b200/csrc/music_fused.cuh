// music_fused.cuh - FUSED persistent kernel for the headline shape class (M = 4 antennas, n = 1
// source, peak outputs only): covariance + eigenvectors + pseudospectrum scan + peak pick in
// ONE launch, persistent CTAs of 8 warps, two per SM (one of this launch, one of the next), warp-specialised.  R and the
// eigenvectors never leave shared memory.
//
//   warps 0..3   covariance (FP64 pipe): per-warp TMA ring exactly as cov4_tma_kernel; a finished
//                window's R is written to a 32-slot shared-memory queue and marked ready (per-slot flag).
//   warp  4      eigenvectors, four lanes per queued window (8 windows per round): principal eigenvector by
//                repeated squaring + Householder basis of its complement (music_eig4p.cuh; 7.5 k cycles per
//                round under the covariance warps' FP64 load); windows that do not converge (noise only, NaN) go through the full Jacobi solver
//                (herm_eig4_coop in music_kernels.cuh, ~26 k cycles), which MUSIC_B200_EIG=jacobi selects for all.
//   warps 5..7   pseudospectrum scan + peak pick, 8 windows per pass (two sweeps of the table):
//                  1. SCREEN on the tensor cores: c_k = e_s^H a_k for all bins k and the 4 windows as a
//                     [bins x 8] x [8 x 8] product in 3xTF32 (mma.sync m16n8k8, hi/lo split of both
//                     operands, fp32 accumulate), d~_k = ||a_k||^2 - |c_k|^2 in fp32.  The FP64 pipe -
//                     which the covariance warps need - is not touched.
//                  2. the screen's error is bounded by FZ_B * ||a_k||^2 (derivation below), so only
//                     bins whose lower bound d~_k - B||a_k||^2 does not exceed the smallest upper bound
//                     U = min_k (d~_k + B||a_k||^2) can hold the fp64 minimum: a first sweep finds U, a second
//                     one lists the survivors, which are re-evaluated EXACTLY in fp64 (same complement/direct formula as
//                     the unfused kernels) and the peak is picked among them with the reference's rule
//                     (strength desc, bin asc, strict '>', /root/reference/lib/baz_music_doa.cc:129-141).
//                     Typically 2-60 bins per window; if more than FZ_CMAX bins of a window survive (flat
//                     spectra, e.g. an all-zero window) every bin of that window is evaluated in fp64 instead.
//                The result is therefore bit-identical to an all-fp64 scan.
//   DRAIN        A tensor-core pass has a latency of ~35 k cycles whatever it holds, and that latency (plus the
//                eigensolver's) used to be the tail of the launch: 58 k cycles per CTA with HBM idle.  Once the
//                window tickets have run out and `mma_fin_max` covariance warps are done, no new pass is started:
//                every warp that has nothing left to do - covariance warps as they finish, the scan warps after
//                their last pass, the eigenvector warp at the end - becomes a drain worker and takes (group of 4
//                windows - fewer only for the CTA's very last ones -, 1/FZ_NCH of the bins, interleaved in steps of 32)
//                units of an all-fp64 scan (drain_bin = scan_bin's arithmetic from the unfused scan_peak1_kernel; the
//                FP64 pipe is free by then), merged per group by the warp that finishes the group's last unit.  Same
//                formula, same tie rule: bit-identical to the tensor-core path, at ~4 k cycles of the whole SM per
//                window instead of a 35 k-cycle pass.  With the spectrum port connected every window goes this way.
//   LAUNCH       programmatic dependent launch: the grid takes one half of every SM (grid <= SM count) and signals
//                griddepcontrol.launch_dependents at its start, so the next launch's CTAs move into the other halves at once
//                and stream their input while this launch finishes its last windows - no SM's input stream stands still
//                between calls.  Results still land in stream order (OUTPUT ORDER at fused_emit); per-launch ticket counters.
//
// Screen error bound.  a is stored in fp32 exactly (the block's table IS complex64) and split at run
// time by truncation: a_hi = a & ~0x1fff (|a - a_hi| < 2^-10|a|), a_lo = (a - a_hi) & ~0x1fff (the
// subtraction is exact), residual < 2^-20|a|.  e is rounded to fp32 (2^-24) and split with cvt.rna
// (residual <= 2^-22|e|).  The three products hi*hi, hi*lo, lo*hi are exact in fp32 (11-bit x 11-bit
// significands); the dropped lo*lo term is <= 2^-21|a||e|.  Allowing every one of the <= 24 fp32
// accumulations a full 2^-23 (truncating adder), |c~ - c| <= (2^-18.4 + 2^-19.2) sum|a_i||e_i| <= 2^-17.8||a||,
// hence ||c~|^2 - |c|^2| <= 2^-16.8||a||^2, plus 2^-22 for the fp32 squares and the subtraction from
// fl32(||a||^2).  FZ_B = 2^-15 leaves > 3x margin over this (already pessimistic) bound; a CPU emulation of the
// screen with truncating fp32 accumulation measures <= 5e-7 ||a||^2, 60x below FZ_B (tests/test_screen_bound.py).
// The bound assumes fp32 never overflows or goes subnormal: a table with a non-zero row whose fl32(||a||^2) lies outside
// [2^-100, 2^100] (screen_bounds_table in music_b200.cu) runs every window on the fp64 drain instead (tests/test_gpu_tables.py).
//
// INSTRUCTION FOOTPRINT.  Sixteen warps in four roles (two CTAs) share one SM's instruction caches (L0 ~6 KB per sub-partition,
// L1.5 32 KB per SM; beyond that instructions come from the L2, which this kernel keeps saturated with the input stream).
// The first version of this file inlined everything (211 KB of SASS): code that runs once per pass / per drain unit then
// cost ~50 cycles per INSTRUCTION (a 500-instruction lane merge: 26 k cycles) while loop bodies ran at ~6.  Hence:
// everything rare or once-per-unit is out of line and shared (fused_exact_d, fused_recip, the Jacobi fallback), the two
// table sweeps of a pass are one loop body, merges are rolled loops, and the clock64 trace exists only in the TRACE
// instantiation of the kernel.
//
// Reference lines covered: /root/reference/lib/baz_music_doa.cc:74-155 (everything work() does per window; with the
// optional spectrum port connected, :120-121, every window takes the fp64 drain workers, which also write (float)P[k]).
#pragma once
#include "music_kernels.cuh"
#include "music_eig4p.cuh"
#include "music_planar.cuh"

namespace music {

// Half an SM per CTA (two CTAs per SM): a launch's grid takes one of the two slots of every SM, so the next launch on the
// stream is placed in the other slot at once and streams its input while this one finishes its last windows.
constexpr int FZ_COV_WARPS = 4;
constexpr int FZ_SCAN_WARPS = 3;
constexpr int FZ_THREADS = 32 * (FZ_COV_WARPS + 1 + FZ_SCAN_WARPS);  // 256
constexpr int FZ_SCAN_THREADS = 32 * FZ_SCAN_WARPS;                  // 96
constexpr int FZ_MPW = 4;        // MMA tiles (16 rows) per scan warp and table tile: more work per ring iteration
                                 // amortises the fixed load -> split -> MMA -> reduce latency chain of a warp
constexpr int FZ_BINS = 16 * FZ_SCAN_WARPS * FZ_MPW;  // table rows per ring tile
constexpr int FZ_Q = 32;        // window queue slots per CTA
constexpr int FZ_WPT = 8;       // windows per scan pass = 2 column groups of 4 windows x {re, im} (8 MMA columns each)
constexpr int FZ_STAGES = 4;    // 4 KiB TMA stages per covariance warp
constexpr int FZ_TS = 3;        // steering-table tile stages (cp.async ring shared by the scan warps)
constexpr int FZ_FRAG_BYTES = 512;  // one 16 x 8 fp32 A tile in fragment order (16 B per lane)
constexpr int FZ_TILE_BYTES = (FZ_BINS / 16) * FZ_FRAG_BYTES + FZ_BINS * 4;  // fragment tiles + fp32 ||a||^2
constexpr int FZ_CMAX = 192;    // exact candidates kept per window before falling back to a full fp64 scan
constexpr float FZ_B = 3.0517578125e-05f;  // 2^-15, see "Screen error bound"

constexpr int FZ_TRACE = 40;    // int64 trace words per CTA (MUSIC_B200_TRACE=1)
constexpr int FZ_TRACE_CTAS = 1024;    // trace rows per launch
constexpr int FZ_TRACE_LAUNCHES = 32;  // launches kept in the trace ring: launch l writes rows [(l % 32) * 1024, ..)
constexpr int FZ_DG = 4;         // windows per drain group (= scan_bin's windows per thread)
constexpr int FZ_NCH = 16;       // interleaved bin chunks per drain group: (group, chunk) is the unit a drain worker (one warp) takes
constexpr int FZ_NGS = 4;        // drain groups in flight
constexpr unsigned FZ_IDLE_NS = 100;  // sleep of a drain worker that found no unit
constexpr int FZ_STG = 64;       // finished windows staged per CTA until the previous launch's outputs are written (fused_emit)
constexpr int FZ_IPT = 4;        // exact candidates per scan thread and pass (kept in registers)

struct FusedCtl {               // shared-memory control block
    unsigned cov_seq;           // queue sequence numbers handed to finished covariances (atomic)
    unsigned lock;              // spin lock: claim, scan_done, drain group slots
    volatile unsigned eig_done; // windows whose eigenvectors are in the queue
    volatile unsigned scan_done;// every window below this is finished (its queue slot is free)
    volatile unsigned cov_finished;  // covariance warps that ran out of windows
    volatile unsigned batch_start, batch_cnt;
    volatile unsigned claim;    // windows below this were handed to a tensor-core pass or to a drain group
    volatile unsigned tout;     // the global ticket counter has run out
    volatile unsigned mma_off;  // no further tensor-core passes: the drain workers take what is left
    volatile int dg_open;       // drain group currently handing out chunks (-1: none)
    unsigned drained_windows;   // statistics (trace)
    unsigned drain_groups;
    unsigned stg_lock;          // spin lock of the output stage
    volatile unsigned stg_n;    // windows in the output stage
    volatile unsigned ordered;  // the previous launch's outputs are written: results go straight to global memory
};
struct StagedPeak {             // a finished window waiting in the output stage
    unsigned o;
    int kk;
    double P;
};
struct DrainGroup {
    volatile unsigned gs;       // first queue sequence number of the group
    volatile int gc;            // windows in the group (1..FZ_DG)
    unsigned next_chunk, done;  // chunks handed out / finished
    volatile int busy;
    int pad[3];
};

constexpr size_t fz_align(size_t x, size_t a) { return (x + a - 1) / a * a; }
// uint64 cov barriers [FZ_COV_WARPS][FZ_STAGES] at offset 0
constexpr size_t FZ_OFF_TBAR = fz_align(8 * FZ_COV_WARPS * FZ_STAGES, 64);  // uint64 tfull[FZ_TS], tempty[FZ_TS]
constexpr size_t FZ_OFF_WRING = fz_align(FZ_OFF_TBAR + 16 * FZ_TS, 64);     // int wring[FZ_COV_WARPS][8]: window ids claimed by each covariance warp
constexpr size_t FZ_OFF_CTL = FZ_OFF_WRING + 32 * FZ_COV_WARPS;             // FusedCtl (64 B)
constexpr size_t FZ_OFF_WIN = FZ_OFF_CTL + 64;                              // int qwin[FZ_Q]
constexpr size_t FZ_OFF_RMIN = FZ_OFF_WIN + 4 * FZ_Q;                       // float redmin[FZ_SCAN_WARPS][FZ_WPT]
constexpr size_t FZ_OFF_CCNT = FZ_OFF_RMIN + 4 * FZ_SCAN_WARPS * FZ_WPT;    // int cand_cnt[FZ_WPT]
constexpr size_t FZ_OFF_CBIN = FZ_OFF_CCNT + 4 * FZ_WPT;                    // int cand_bin[FZ_WPT][FZ_CMAX]
constexpr size_t FZ_OFF_RED = fz_align(FZ_OFF_CBIN + 4 * FZ_WPT * FZ_CMAX, 16);  // double redP[FZ_SCAN_WARPS]; int redk[FZ_SCAN_WARPS]  (fallback scan)
constexpr size_t FZ_OFF_BEST = fz_align(FZ_OFF_RED + 12 * FZ_SCAN_WARPS, 16);    // u64 bestP[FZ_WPT]; int bestk[FZ_WPT]; int admitted[FZ_WPT]
constexpr size_t FZ_OFF_QRDY = FZ_OFF_BEST + 16 * FZ_WPT;   // unsigned qready[FZ_Q]: sequence number + 1 of the R held by the slot
constexpr size_t FZ_OFF_QDONE = FZ_OFF_QRDY + 4 * FZ_Q;    // unsigned qdone[FZ_Q]: the slot's window is finished
constexpr size_t FZ_OFF_DGRP = FZ_OFF_QDONE + 4 * FZ_Q;    // DrainGroup grp[FZ_NGS]
constexpr size_t FZ_OFF_DRES = FZ_OFF_DGRP + 32 * FZ_NGS;  // double resP[FZ_NGS][FZ_NCH][FZ_DG]; int resk[...]
constexpr size_t FZ_OFF_STG = fz_align(FZ_OFF_DRES + 12 * FZ_NGS * FZ_NCH * FZ_DG, 16);  // StagedPeak stg[FZ_STG]
constexpr size_t FZ_OFF_RQ = fz_align(FZ_OFF_STG + sizeof(StagedPeak) * FZ_STG, 256);   // double Rq[FZ_Q][32]
constexpr size_t FZ_OFF_VQ = FZ_OFF_RQ + (size_t)FZ_Q * 256;  // double Vq[FZ_Q][32]
constexpr size_t FZ_OFF_TBL = FZ_OFF_VQ + (size_t)FZ_Q * 256; // FZ_TS table tiles
constexpr size_t FZ_OFF_RING = fz_align(FZ_OFF_TBL + (size_t)FZ_TS * FZ_TILE_BYTES, 128);
constexpr size_t FZ_SMEM = FZ_OFF_RING + (size_t)FZ_COV_WARPS * FZ_STAGES * COV_CHUNK;
static_assert(sizeof(FusedCtl) <= 64 && sizeof(DrainGroup) == 32 && sizeof(StagedPeak) == 16, "control block layout");
// two CTAs per SM: 228 KiB of shared memory per SM, 1 KiB of it reserved per CTA
static_assert(FZ_SMEM <= (228 - 2 * 1) * 1024 / 2, "fused kernel shared memory: two CTAs must fit on one SM");
constexpr int FZ_CPT = (FZ_TILE_BYTES / 16 + FZ_SCAN_THREADS - 1) / FZ_SCAN_THREADS;  // 16-byte copies per thread and tile
static_assert(FZ_TILE_BYTES % 16 == 0, "table tile copy plan");

__device__ __forceinline__ void bar_sync_scan() { asm volatile("bar.sync 1, %0;" ::"n"(FZ_SCAN_THREADS) : "memory"); }

__host__ __device__ inline int fused_tiles(int K) { return (K + FZ_BINS - 1) / FZ_BINS; }
// Decimated table (tiles 0 .. FZ_NDEC-1): every fused_stride(K)-th row, at most FZ_NDEC * FZ_BINS of them.  The
// first sweep only needs an upper bound of the minimum; a subsample gives one at a fraction of the cost, and
// the finer it is the fewer bins survive into the exact evaluation.
constexpr int FZ_NDEC = 2;
__host__ __device__ inline int fused_stride(int K) { return (K + FZ_NDEC * FZ_BINS - 1) / (FZ_NDEC * FZ_BINS); }
__host__ __device__ inline size_t fused_table_bytes(int K) { return (size_t)(FZ_NDEC + fused_tiles(K)) * FZ_TILE_BYTES; }

__device__ __forceinline__ uint32_t to_tf32(float x)
{
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// Steering table in the tensor-core screen's layout.  Per FZ_BINS-row tile: FZ_BINS / 16 MMA A-fragment tiles
// (16 rows x 8 columns; the complex64 row [Re a0, Im a0, .., Re a3, Im a3] IS the A row), stored in
// fragment order - lane l holds {a0..a3} (fp32, split into tf32 hi/lo at run time) with a0 = A[g][t], a1 = A[g+8][t],
// a2 = A[g][t+4], a3 = A[g+8][t+4], g = l/4, t = l%4 - followed by fl32(||a||^2) per row
// (+inf for padding rows, which therefore never win).  Tiles 0..FZ_NDEC-1 hold every fused_stride(K)-th row
// (the subsample of the first sweep), the following tiles the whole table.  na_max = max ||a||^2 over the K real rows.
__global__ void prep_table_tc_kernel(const float *__restrict__ tab, unsigned char *__restrict__ tbl, float *__restrict__ na_max,
                                     int K)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // one thread per (16-row tile, lane)
    const int tile16 = idx >> 5, lane = idx & 31;           // tile16 < FZ_BINS/16: decimated tile, then the full table
    const int per = FZ_BINS / 16;
    const int ntile16 = (FZ_NDEC + fused_tiles(K)) * per;
    if (tile16 >= ntile16) return;
    const int g = lane >> 2, t = lane & 3;
    const bool dec = tile16 < FZ_NDEC * per;
    const int stride = dec ? fused_stride(K) : 1;
    const int row0 = dec ? tile16 * 16 : (tile16 - FZ_NDEC * per) * 16;  // first (sub)sampled row of this 16-row tile
    unsigned char *tile = tbl + (size_t)(tile16 / per) * FZ_TILE_BYTES;
    float *frag = reinterpret_cast<float *>(tile) + (size_t)(tile16 % per) * (FZ_FRAG_BYTES / 4) + lane * 4;
    const int rows[4] = {g, g + 8, g, g + 8};
    const int cols[4] = {t, t, t + 4, t + 4};
    for (int i = 0; i < 4; ++i) {
        const int bin = (row0 + rows[i]) * stride;
        frag[i] = bin < K ? tab[(size_t)bin * 8 + cols[i]] : 0.f;
    }
    if (lane < 16) {  // ||a||^2 of row `lane` of this 16-row tile, same fma order as prep_table_kernel
        const int bin = (row0 + lane) * stride;
        double na = 0.0;
        for (int i = 0; i < 4; ++i) {
            double re = 0.0, im = 0.0;
            if (bin < K) { re = tab[(size_t)bin * 8 + 2 * i]; im = tab[(size_t)bin * 8 + 2 * i + 1]; }
            na = fma(re, re, fma(im, im, na));
        }
        float *na32 = reinterpret_cast<float *>(tile + per * FZ_FRAG_BYTES) + (tile16 % per) * 16 + lane;
        if (bin < K) {
            const float f = (float)na;
            *na32 = f;
            atomicMax(reinterpret_cast<int *>(na_max), __float_as_int(f));  // non-negative floats order like ints
        } else {
            *na32 = __int_as_float(0x7f800000);
        }
    }
}

// Exact fp64 denominator d_k = ||G^H a_k||^2 of bin k for the window whose eigenvectors sit at shared address `ev`:
// the same formula (and the same ||a||^2 fma order) as the unfused kernels.  ONE out-of-line copy serves the exact phase
// of the tensor-core passes, the flat-spectrum fallback and the cold path of the drain workers.
__device__ __noinline__ double fused_exact_d(const float *__restrict__ tab_c64, const int k, const uint32_t ev, const uint64_t pol_keep)
{
    const float4 *row = reinterpret_cast<const float4 *>(tab_c64 + (size_t)k * 8);
    const float4 x0 = ldg_f32x4_hint(row, pol_keep), x1 = ldg_f32x4_hint(row + 1, pol_keep);
    double ar[4], ai[4];
    ar[0] = x0.x; ai[0] = x0.y; ar[1] = x0.z; ai[1] = x0.w;
    ar[2] = x1.x; ai[2] = x1.y; ar[3] = x1.z; ai[3] = x1.w;
    double na = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) na = fma(ar[i], ar[i], fma(ai[i], ai[i], na));
    double d = complement_denominator<4>(ar, ai, na, ev + 16 * 3 * 4);
    if (d < COMPLEMENT_GUARD * na) d = direct_denominator<4>(ar, ai, ev);
    return d;
}
__device__ __noinline__ double fused_recip(const double d) { return 1.0 / d; }
// the reference's replacement rule "1/d > 1/best" (strict '>' on the strengths, :132) for a d already known to be < best
__device__ __noinline__ bool fused_recip_greater(const double d, const double best)
{
    return d < best * 0.99999999999999911182 /* 1 - 2^-50 */ || 1.0 / d > 1.0 / best;
}
__device__ __forceinline__ double fused_exact_P(const float *__restrict__ tab_c64, const int k, const uint32_t ev, const uint64_t pol_keep)
{
    return fused_recip(fused_exact_d(tab_c64, k, ev, pol_keep));
}
__device__ __noinline__ void fused_jacobi4(const double *Rw, double *vw, const bool active, const int j) { herm_eig4_coop(Rw, vw, active, j); }

// One steering-table row against FZ_DG windows: scan_bin's hot path (music_kernels.cuh) with the rare exact evaluation
// out of line.  Same arithmetic, same decisions: bit-identical results.
// SPEC = true (the spectrum port is connected, /root/reference/lib/baz_music_doa.cc:120-121): every (bin, window) strength
// is needed, so each d is made exact (direct form inside the cancellation guard), P = 1 / d goes to spec_row[b][k] as float
// and the peak is kept on the strengths themselves (strict '>', :132); bestP = the running maxima.
template <bool SPEC>
__device__ __forceinline__ void drain_bin(const double (&ar)[4], const double (&ai)[4], const double na, const int k,
                                          const uint32_t (&ev)[4], PeakState<4> &ps, const float *__restrict__ tab_c64,
                                          const uint64_t pol_keep, double (&bestP)[4], float *const (&spec_row)[4], const int gc)
{
    constexpr int sig = 16 * 3 * 4;  // byte offset of the signal vector (largest eigenvalue)
    double cr[4], ci[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        double e0x;
        asm volatile("ld.shared.f64 %0, [%1];" : "=d"(e0x) : "r"(ev[b] + sig));
        cr[b] = e0x * ar[0];
        ci[b] = e0x * ai[0];
    }
#pragma unroll
    for (int i = 1; i < 4; ++i) {
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const double2 e = lds_f64x2(ev[b] + sig + 16 * i);
            cr[b] = fma(e.y, ai[i], cr[b]);
            ci[b] = fma(-e.y, ar[i], ci[b]);
            cr[b] = fma(e.x, ar[i], cr[b]);
            ci[b] = fma(e.x, ai[i], ci[b]);
        }
    }
    const int hg = __double2hiint(COMPLEMENT_GUARD * na);
    if (SPEC) {
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            double d = fma(-cr[b], cr[b], fma(-ci[b], ci[b], na));
            if (!(__double2hiint(d) > hg)) d = fused_exact_d(tab_c64, k, ev[b], pol_keep);  // inside the guard, negative or NaN
            const double P = fused_recip(d);
            if (b < gc) spec_row[b][k] = (float)P;
            if (P > bestP[b]) { bestP[b] = P; ps.bestd[b] = d; ps.bestk[b] = k; }
        }
        return;
    }
    unsigned cold = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        const double d = fma(-cr[b], cr[b], fma(-ci[b], ci[b], na));
        const int hds = __double2hiint(d);
        const unsigned hd = (unsigned)hds;
        const bool guard = hds <= hg;
        if ((hd - ps.hbm1[b]) <= 1u || guard) cold |= 1u << b;
        if (hd < ps.hbm1[b] && !guard) { ps.bestd[b] = d; ps.bestk[b] = k; ps.hbm1[b] = max(hd, 1u) - 1u; }
    }
    if (cold) {
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            if (cold & (1u << b)) {
                const double d = fused_exact_d(tab_c64, k, ev[b], pol_keep);
                if (d < ps.bestd[b] && fused_recip_greater(d, ps.bestd[b])) {
                    ps.bestd[b] = d;
                    ps.bestk[b] = k;
                    ps.hbm1[b] = max((unsigned)__double2hiint(d), 1u) - 1u;
                }
            }
        }
    }
}

// ---- shared-memory spin lock ----
// WARP-UNIFORM CONTROL FLOW.  Every wait in this kernel is a loop that ALL lanes of the warp run, with lane 0 doing the
// atomic / the polling read and the outcome broadcast by __shfl_sync.  The first version let lane 0 spin alone inside
// `if (lane == 0) { for (;;) { lock ... __nanosleep } }`: after such a block the warp stayed split (lane 0 | lanes 1-31,
// measured with __activemask() in the TRACE build: every drain unit ran twice, every warp collective took its
// divergent slow path - 26 k cycles for a 60-shuffle merge).
__device__ __forceinline__ void fz_lock(unsigned *lock, const int lane)  // all lanes call; lane 0 holds the lock afterwards
{
    for (;;) {
        unsigned got = 0u;
        if (lane == 0) got = atomicCAS(lock, 0u, 1u) == 0u ? 1u : 0u;
        if (__shfl_sync(0xffffffffu, got, 0)) break;
    }
    __threadfence_block();
}
__device__ __forceinline__ void fz_unlock(unsigned *lock, const int lane)  // all lanes call
{
    __threadfence_block();
    if (lane == 0) atomicExch(lock, 0u);
    __syncwarp();
}
__device__ __forceinline__ void fz_lock(FusedCtl *ctl, const int lane) { fz_lock(&ctl->lock, lane); }
__device__ __forceinline__ void fz_unlock(FusedCtl *ctl, const int lane) { fz_unlock(&ctl->lock, lane); }

// OUTPUT ORDER.  Results must land after those of the previous launch on the stream, which under programmatic dependent
// launch runs alongside this one (often in the other half of the same SM) for most of this launch.  Waiting for it
// (griddepcontrol.wait) before the first store would stall the scan, fill the queue and stop the covariance warps, so
// finished windows are staged in shared memory instead.  The first writer that finds the stage full - or warp 0 at CTA exit -
// waits for the previous launch once, flushes the stage and marks the CTA `ordered`; from then on results are stored directly.
// fused_stage_flush: the whole calling warp, holding stg_lock (or alone in the CTA).
__device__ __noinline__ void fused_stage_flush(unsigned char *smem, const PeakOut out, const int K)
{
    FusedCtl *ctl = reinterpret_cast<FusedCtl *>(smem + FZ_OFF_CTL);
    const StagedPeak *stg = reinterpret_cast<const StagedPeak *>(smem + FZ_OFF_STG);
    asm volatile("griddepcontrol.wait;" ::: "memory");  // the previous launch has finished and its writes are visible
    const unsigned n = ctl->stg_n;
    for (unsigned i = threadIdx.x & 31; i < n; i += 32) peak_write(out, stg[i].o, stg[i].kk, stg[i].P, K);
    __syncwarp();
    if ((threadIdx.x & 31) == 0) { ctl->stg_n = 0u; ctl->ordered = 1u; }
    __syncwarp();
}
// The peak (kk, P) of window o, for every lane with `valid`; all lanes of one warp call.
__device__ __forceinline__ void fused_emit(unsigned char *smem, const PeakOut out, const bool valid, const unsigned o, const int kk,
                                        const double P, const int K)
{
    FusedCtl *ctl = reinterpret_cast<FusedCtl *>(smem + FZ_OFF_CTL);
    StagedPeak *stg = reinterpret_cast<StagedPeak *>(smem + FZ_OFF_STG);
    const int lane = threadIdx.x & 31;
    unsigned ord = 0u;
    if (lane == 0) ord = ctl->ordered;
    if (!__shfl_sync(0xffffffffu, ord, 0)) {
        fz_lock(&ctl->stg_lock, lane);
        const unsigned mask = __ballot_sync(0xffffffffu, valid);
        unsigned n = 0u;
        if (lane == 0) { n = ctl->stg_n; ord = ctl->ordered; }
        n = __shfl_sync(0xffffffffu, n, 0);
        ord = __shfl_sync(0xffffffffu, ord, 0);
        if (!ord) {
            if (n + __popc(mask) > (unsigned)FZ_STG) {
                fused_stage_flush(smem, out, K);
                ord = 1u;
            } else {
                if (valid) stg[n + __popc(mask & ((1u << lane) - 1u))] = StagedPeak{o, kk, P};
                if (lane == 0) ctl->stg_n = n + __popc(mask);
            }
        }
        fz_unlock(&ctl->stg_lock, lane);
        if (!ord) return;
    }
    if (valid) peak_write(out, o, kk, P, K);
}

// windows [start, start + cnt) are finished: mark their queue slots and advance scan_done over every finished slot
// (tensor-core passes and drain groups complete out of order).  All lanes of one warp call.
__device__ __forceinline__ void fused_retire(unsigned char *smem, const unsigned start, const unsigned cnt, const int lane)
{
    FusedCtl *ctl = reinterpret_cast<FusedCtl *>(smem + FZ_OFF_CTL);
    volatile unsigned *qdone = reinterpret_cast<volatile unsigned *>(smem + FZ_OFF_QDONE);
    __threadfence_block();
    fz_lock(ctl, lane);
    if (lane == 0) {
        for (unsigned w = 0; w < cnt; ++w) qdone[(start + w) % FZ_Q] = 1u;
        unsigned sd = ctl->scan_done;
        while (sd != ctl->claim && qdone[sd % FZ_Q]) { qdone[sd % FZ_Q] = 0u; ++sd; }
        ctl->scan_done = sd;
    }
    fz_unlock(ctl, lane);
}

// Drain worker (a whole warp; see the file header): takes (group, bin chunk) units of an all-fp64 scan until every
// window of this CTA has been handed out.  The table is the complex64 one the block was given (32 bytes per bin; it is
// also what the exact phase of the tensor-core passes reads, so it is L2-resident), widened here, ||a||^2 in the fma
// order of the table preparation.  A group is FZ_DG windows (one table row serves four windows) - fewer only for the
// CTA's very last windows; its FZ_NCH units interleave the table in steps of 32 bins (unit c: bins (i * FZ_NCH + c) * 32
// + lane, i = 0, 1, ..), the next row is requested before the current one is evaluated.  Returns the number of units
// this warp processed.
template <bool TRACE, bool SPEC>
__device__ __noinline__ int fused_drain_worker(unsigned char *smem, const float *__restrict__ tab_c64, const int K,
                                               float *__restrict__ spec /* [W][K] or null */, const PeakOut out, long long *__restrict__ dbg_in, const long long t_start)
{
    long long *const dbg_cta = TRACE ? dbg_in : nullptr;
    FusedCtl *ctl = reinterpret_cast<FusedCtl *>(smem + FZ_OFF_CTL);
    DrainGroup *grp = reinterpret_cast<DrainGroup *>(smem + FZ_OFF_DGRP);
    double *resP = reinterpret_cast<double *>(smem + FZ_OFF_DRES);
    int *resk = reinterpret_cast<int *>(smem + FZ_OFF_DRES + 8 * FZ_NGS * FZ_NCH * FZ_DG);
    const int *qwin = reinterpret_cast<const int *>(smem + FZ_OFF_WIN);
    const uint32_t Vq0 = smem_u32(smem + FZ_OFF_VQ);
    const int lane = threadIdx.x & 31;
    int units = 0;
    long long ph[4] = {0, 0, 0, 0};  // trace: table sweep | merge + publish | whole unit | waiting for a unit
    int ndiv0 = 0, ndiv1 = 0;
    const uint64_t pol_keep = l2_policy_evict_last();
    // the spectrum rows are stored as they are computed, not staged: they wait for the previous launch here (peaks: fused_emit)
    if (SPEC) asm volatile("griddepcontrol.wait;" ::: "memory");
    for (;;) {
        int slot = -1, chunk = 0, gc = 0;
        unsigned gs = 0;
        const long long tw0 = dbg_cta ? clock64() : 0;
        for (;;) {  // (all lanes loop; lane 0 decides inside the lock, the outcome is broadcast)
            int all_done = 0;
            fz_lock(ctl, lane);
            if (lane == 0) {
                const int cur = ctl->dg_open;
                if (cur >= 0 && grp[cur].next_chunk < (unsigned)FZ_NCH) {
                    slot = cur; chunk = (int)grp[cur].next_chunk++; gs = grp[cur].gs; gc = grp[cur].gc;
                } else if (ctl->mma_off) {
                    const unsigned start = ctl->claim, avail = ctl->eig_done - start;
                    // every window of this CTA has its eigenvectors: what is left may go out as a partial group
                    const bool last = ctl->cov_finished == (unsigned)FZ_COV_WARPS &&
                                      ctl->eig_done == *reinterpret_cast<volatile unsigned *>(&ctl->cov_seq);
                    if (avail >= (unsigned)FZ_DG || (avail > 0 && last)) {
                        int f = -1;
                        for (int i = 0; i < FZ_NGS; ++i)
                            if (!grp[i].busy) { f = i; break; }
                        if (f >= 0) {
                            gc = (int)min(avail, (unsigned)FZ_DG);
                            grp[f].gs = start; grp[f].gc = gc; grp[f].next_chunk = 1u; grp[f].done = 0u; grp[f].busy = 1;
                            ctl->claim = start + gc;
                            ctl->dg_open = f;
                            ctl->drained_windows += gc;
                            ctl->drain_groups += 1;
                            slot = f; chunk = 0; gs = start;
                        }
                    } else if (avail == 0) {
                        all_done = last ? 1 : 0;
                    }
                }
            }
            fz_unlock(ctl, lane);
            slot = __shfl_sync(0xffffffffu, slot, 0);
            all_done = __shfl_sync(0xffffffffu, all_done, 0);
            if (slot >= 0) break;
            if (all_done) { slot = -2; break; }
            __nanosleep(FZ_IDLE_NS);
        }
        if (dbg_cta && lane == 0) ph[3] += clock64() - tw0;
        if (slot < 0) {
            if (dbg_cta && lane == 0) {
                atomicAdd(reinterpret_cast<unsigned long long *>(dbg_cta + 22), (unsigned long long)ph[2]);
                atomicAdd(reinterpret_cast<unsigned long long *>(dbg_cta + 25), (unsigned long long)ph[0]);
                atomicAdd(reinterpret_cast<unsigned long long *>(dbg_cta + 26), (unsigned long long)ph[1]);
                atomicAdd(reinterpret_cast<unsigned long long *>(dbg_cta + 28), (unsigned long long)ph[3]);
                atomicAdd(reinterpret_cast<unsigned long long *>(dbg_cta + 29), (unsigned long long)units);
                atomicAdd(reinterpret_cast<unsigned long long *>(dbg_cta + 24), (unsigned long long)ndiv0);
                atomicAdd(reinterpret_cast<unsigned long long *>(dbg_cta + 27), (unsigned long long)ndiv1);
            }
            return units;
        }
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        gc = __shfl_sync(0xffffffffu, gc, 0);
        gs = __shfl_sync(0xffffffffu, gs, 0);
        ++units;
        const long long tu0 = dbg_cta ? clock64() : 0;
        uint32_t ev[FZ_DG];
#pragma unroll
        for (int b = 0; b < FZ_DG; ++b) ev[b] = Vq0 + 256u * ((gs + (unsigned)min(b, gc - 1)) % FZ_Q);
        PeakState<FZ_DG> ps;
        ps.reset();
        double ar[4], ai[4], na = 0.0, nr[4], ni[4], nna = 0.0;
        auto load_row = [&](const int k, double (&r)[4], double (&im)[4], double &n) {  // k < K
            const float4 *row = reinterpret_cast<const float4 *>(tab_c64 + (size_t)k * 8);
            const float4 x0 = ldg_f32x4_hint(row, pol_keep), x1 = ldg_f32x4_hint(row + 1, pol_keep);
            r[0] = x0.x; im[0] = x0.y; r[1] = x0.z; im[1] = x0.w;
            r[2] = x1.x; im[2] = x1.y; r[3] = x1.z; im[3] = x1.w;
            double a = 0.0;
#pragma unroll
            for (int i = 0; i < 4; ++i) a = fma(r[i], r[i], fma(im[i], im[i], a));
            n = a;
        };
        int k = chunk * 32 + lane;
        if (TRACE && dbg_cta && __activemask() != 0xffffffffu) ++ndiv0;  // (trace: is the warp converged at the sweep?)
        if (k < K) load_row(k, ar, ai, na);
        double bestP[FZ_DG] = {0.0, 0.0, 0.0, 0.0};
        float *spec_row[FZ_DG];
#pragma unroll
        for (int b = 0; b < FZ_DG; ++b) spec_row[b] = SPEC ? spec + (size_t)qwin[(gs + (unsigned)min(b, gc - 1)) % FZ_Q] * K : nullptr;
        if (SPEC) {  // (compile time: the default instantiation carries neither the strengths nor the row pointers)
#pragma unroll 1
            while (k < K) {
                const int kn = k + FZ_NCH * 32;
                if (kn < K) load_row(kn, nr, ni, nna);
                drain_bin<true>(ar, ai, na, k, ev, ps, tab_c64, pol_keep, bestP, spec_row, gc);
#pragma unroll
                for (int i = 0; i < 4; ++i) { ar[i] = nr[i]; ai[i] = ni[i]; }
                na = nna;
                k = kn;
            }
        } else {
#pragma unroll 1
            while (k < K) {
                const int kn = k + FZ_NCH * 32;
                if (kn < K) load_row(kn, nr, ni, nna);
                drain_bin<false>(ar, ai, na, k, ev, ps, tab_c64, pol_keep, bestP, spec_row, gc);
#pragma unroll
                for (int i = 0; i < 4; ++i) { ar[i] = nr[i]; ai[i] = ni[i]; }
                na = nna;
                k = kn;
            }
        }
        __syncwarp();
        if (TRACE && dbg_cta && __activemask() != 0xffffffffu) ++ndiv1;  // (... and at the merge?)
        long long tp2 = 0;
        if (dbg_cta) { asm volatile("" ::"d"(ps.bestd[0]), "d"(ps.bestd[3]), "r"(ps.bestk[1]) : "memory"); tp2 = clock64(); }
        // per-window merge over the lanes, order (P desc, bin asc); a lane without a bin holds d = +inf -> P = 0, bin -1.
        // Three warp reductions per window (redux.sync) instead of a 5-round shuffle butterfly: non-negative doubles
        // order like their bit patterns, so max(high word), then max(low word) among the lanes that hold it, then
        // min(bin) among the lanes that hold both.
        double P[FZ_DG];
        int kk[FZ_DG];
#pragma unroll
        for (int b = 0; b < FZ_DG; ++b) {
            const double Pl = fused_recip(ps.bestd[b]);
            const unsigned hi = (unsigned)__double2hiint(Pl), lo = (unsigned)__double2loint(Pl);
            const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
            const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? lo : 0u);
            const unsigned mk = __reduce_min_sync(0xffffffffu, (hi == mh && lo == ml && ps.bestk[b] >= 0) ? (unsigned)ps.bestk[b] : 0x7fffffffu);
            P[b] = __hiloint2double((int)mh, (int)ml);
            kk[b] = mk == 0x7fffffffu ? -1 : (int)mk;
        }
        int last = 0;
        if (lane == 0) {
#pragma unroll
            for (int b = 0; b < FZ_DG; ++b) {
                resP[(slot * FZ_NCH + chunk) * FZ_DG + b] = P[b];
                resk[(slot * FZ_NCH + chunk) * FZ_DG + b] = kk[b];
            }
            __threadfence_block();
            last = atomicAdd(&grp[slot].done, 1u) == (unsigned)FZ_NCH - 1 ? 1 : 0;
            __threadfence_block();
            if (dbg_cta) {  // phases of this unit, accumulated in registers and written once when the worker returns
                const long long tp4 = clock64();
                ph[0] += tp2 - tu0; ph[1] += tp4 - tp2; ph[2] += tp4 - tu0;
            }
        }
        last = __shfl_sync(0xffffffffu, last, 0);
        __syncwarp();  // (memory ordering for the lanes that read the other units' results below)
        if (last) {
            // this warp finished the group's last unit: merge the chunks (lane b <-> window b; any order gives the same
            // result, (P desc, bin asc) is a total order)
            double Pm = 0.0;
            int km = -1;
            unsigned o = 0u;
            if (lane < gc) {
                Pm = resP[(slot * FZ_NCH) * FZ_DG + lane];
                km = resk[(slot * FZ_NCH) * FZ_DG + lane];
#pragma unroll 1
                for (int c = 1; c < FZ_NCH; ++c) {
                    const double Pc = resP[(slot * FZ_NCH + c) * FZ_DG + lane];
                    const int kc = resk[(slot * FZ_NCH + c) * FZ_DG + lane];
                    if (peak_better(Pc, kc, Pm, km)) { Pm = Pc; km = kc; }
                }
                o = (unsigned)qwin[(gs + lane) % FZ_Q];
            }
            fused_emit(smem, out, lane < gc, o, km, Pm, K);
            __syncwarp();
            fused_retire(smem, gs, (unsigned)gc, lane);
            if (lane == 0) {
                grp[slot].busy = 0;  // (results were read above; a new group may reuse the slot)
                if (dbg_cta) dbg_cta[23] = clock64() - t_start;  // (the last group to finish writes last)
            }
            __syncwarp();
        }
    }
}

// PLANAR = true: the window is read from four per-antenna streams (music_planar.cuh) - window w = snapshots
// [first_snapshot + w * hop, ... + N) of each stream - by four 1 KiB bulk copies per stage instead of one 4 KiB copy;
// the stage then holds [antenna][128 snapshots] and a lane gathers its snapshot with four LDS.64.  Requires 16-byte
// aligned streams and even first_snapshot, hop and N (bulk copies move multiples of 16 bytes).
// TRACE = true: the instantiation tools/fused_trace.py runs (MUSIC_B200_TRACE=1): per-CTA clock64 trace in dbg_in.
template <bool PLANAR, bool TRACE>
__global__ void __launch_bounds__(FZ_THREADS, 2)
music4_fused_kernel(const float *__restrict__ in, const PlanarStreams S, unsigned long long first_snapshot, unsigned hop,
                    const unsigned char *__restrict__ tbl /* fused_table_bytes(K) */,
                    const float *__restrict__ tab_c64 /* [K][4] complex64 */, const float *__restrict__ na_max_p, int W, int N,
                    int K, PeakOut out, unsigned *__restrict__ work_ctr /* [0]: window tickets, [1]: finished CTAs; both zero between launches */,
                    long long *__restrict__ dbg_in /* TRACE: [grid][FZ_TRACE] clock64 trace */,
                    const int eig_mode /* 0: principal eigenvector by squaring (Jacobi fallback), otherwise: Jacobi, four lanes per window */,
                    const GatherFlags gather_flags /* epoch flags of the fused bins all-gather (out.npeer > 0) */,
                    const int mma_fin_max /* no tensor-core pass starts once the window tickets have run out and this many covariance warps are done (0: once the tickets have run out); < 0: never any */,
                    float *__restrict__ spec /* optional spectrum port [W][K] (float): every window then goes through the fp64 drain workers, which write it */)
{
    long long *const dbg = TRACE ? dbg_in : nullptr;
    // programmatic dependent launch: the next launch on this stream may be placed at once, in the other half of each SM;
    // see OUTPUT ORDER (fused_emit) for the other half
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const long long t_start = clock64();
    unsigned long long g_start = 0;
    if (dbg) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g_start));
    extern __shared__ __align__(128) unsigned char fz_smem[];
    FusedCtl *ctl = reinterpret_cast<FusedCtl *>(fz_smem + FZ_OFF_CTL);
    int *qwin = reinterpret_cast<int *>(fz_smem + FZ_OFF_WIN);
    volatile unsigned *qready = reinterpret_cast<volatile unsigned *>(fz_smem + FZ_OFF_QRDY);
    double *Rq = reinterpret_cast<double *>(fz_smem + FZ_OFF_RQ);
    double *Vq = reinterpret_cast<double *>(fz_smem + FZ_OFF_VQ);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x < FZ_Q) {
        reinterpret_cast<unsigned *>(fz_smem + FZ_OFF_QRDY)[threadIdx.x] = 0u;
        reinterpret_cast<unsigned *>(fz_smem + FZ_OFF_QDONE)[threadIdx.x] = 0u;
    }
    if (threadIdx.x < FZ_NGS * 8) reinterpret_cast<unsigned *>(fz_smem + FZ_OFF_DGRP)[threadIdx.x] = 0u;
    if (threadIdx.x == 0) {
        if (dbg) { dbg[blockIdx.x * FZ_TRACE + 22] = 0; for (int i = 24; i < 30; ++i) dbg[blockIdx.x * FZ_TRACE + i] = 0; }  // (accumulated by the drain workers)
        ctl->cov_seq = 0; ctl->lock = 0; ctl->eig_done = 0; ctl->scan_done = 0; ctl->cov_finished = 0;
        ctl->batch_start = 0; ctl->batch_cnt = 0; ctl->claim = 0; ctl->tout = 0; ctl->mma_off = (mma_fin_max < 0 || spec != nullptr) ? 1u : 0u;
        ctl->dg_open = -1; ctl->drained_windows = 0; ctl->drain_groups = 0;
        ctl->stg_lock = 0; ctl->stg_n = 0; ctl->ordered = 0;
        const uint32_t tb0 = smem_u32(fz_smem + FZ_OFF_TBAR);
        for (int s = 0; s < FZ_TS; ++s) {
            mbar_init(tb0 + 8 * s, FZ_SCAN_THREADS);            // tfull: one cp.async-completion arrival per scan thread
            mbar_init(tb0 + 8 * (FZ_TS + s), FZ_SCAN_WARPS);    // tempty: one arrival per scan warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp < FZ_COV_WARPS) {
        // ================= covariance warps =================
        uint64_t *bars = reinterpret_cast<uint64_t *>(fz_smem) + warp * FZ_STAGES;
        unsigned char *ring = fz_smem + FZ_OFF_RING + (size_t)warp * FZ_STAGES * COV_CHUNK;
        const uint32_t bar0 = smem_u32(bars), ring0 = smem_u32(ring);
        // Windows are claimed one at a time from a global ticket counter (dynamic balance: 10 000 windows over
        // 528 warps would otherwise leave 18 or 19 per warp, i.e. a 5 % longer critical path).  The producer
        // (lane 0) claims the next window when it requests the last chunk of the current one and hands the id
        // to the consumer side through a small per-warp ring; -1 ends the stream.
        volatile int *wring = reinterpret_cast<volatile int *>(fz_smem + FZ_OFF_WRING) + warp * 8;
        unsigned *ctr = work_ctr;
        const size_t win_bytes = (size_t)N * 32;
        const int cpw = (int)((win_bytes + COV_CHUNK - 1) / COV_CHUNK);
        const unsigned char *src0 = reinterpret_cast<const unsigned char *>(in);
        if (lane == 0) {
            for (int s = 0; s < FZ_STAGES; ++s) mbar_init(bar0 + 8 * s, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
        __syncwarp();
        // producer state (lane 0): next chunk to request = chunk iq of window iw (-1: stream exhausted)
        int iq = 0, iw = -1, islot = 0, wr = 0;
        // the stream is read once: evict_first, so that it does not push the steering tables out of L2 (overlapping
        // planar windows, hop < N, are re-read from L2 by the next windows and keep the default policy)
        const bool stream_once = !PLANAR || hop >= (unsigned)N;
        const uint64_t pol_stream = l2_policy_evict_first();
        auto claim = [&]() {
            const unsigned tkt = atomicAdd(ctr, 1u);
            iw = tkt < (unsigned)W ? (int)tkt : -1;
            if (iw < 0) ctl->tout = 1u;
            wring[wr & 7] = iw;
            ++wr;
        };
        auto issue = [&]() {
            if (iw < 0) return;
            const size_t off = (size_t)iq * COV_CHUNK;
            const uint32_t bytes = (uint32_t)min((size_t)COV_CHUNK, win_bytes - off);
            mbar_expect_tx(bar0 + 8 * islot, bytes);
            if (PLANAR) {
                const unsigned long long s0 = first_snapshot + (unsigned long long)iw * hop + (unsigned long long)iq * (COV_CHUNK / 32);
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (stream_once) bulk_g2s_hint(ring0 + islot * COV_CHUNK + r * (COV_CHUNK / 4), S.p[r] + s0, bytes / 4, bar0 + 8 * islot, pol_stream);
                    else bulk_g2s(ring0 + islot * COV_CHUNK + r * (COV_CHUNK / 4), S.p[r] + s0, bytes / 4, bar0 + 8 * islot);
                }
            } else {
                bulk_g2s_hint(ring0 + islot * COV_CHUNK, src0 + (size_t)iw * win_bytes + off, bytes, bar0 + 8 * islot, pol_stream);
            }
            if (++islot == FZ_STAGES) islot = 0;
            if (++iq == cpw) { iq = 0; claim(); }
        };
        if (lane == 0) {
            claim();
            for (int s = 0; s < FZ_STAGES; ++s) issue();
        }
        __syncwarp();
        double acc[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = 0.0;
        int slot = 0;
        uint32_t parity = 0;
        for (int rd = 0;; ++rd) {
            const int wcur = wring[rd & 7];  // written by lane 0 at least one chunk request ago
            if (wcur < 0) break;
            for (int q = 0; q < cpw; ++q) {
                while (!mbar_try_wait(bar0 + 8 * slot, parity)) {}
                if (dbg && warp == 0 && lane == 0 && rd == 0 && q == 0) {  // first input bytes of this CTA have arrived
                    unsigned long long g;
                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
                    dbg[blockIdx.x * FZ_TRACE + 32] = (long long)g;
                }
                const size_t off = (size_t)q * COV_CHUNK;
                const int nsnap = (int)(min((size_t)COV_CHUNK, win_bytes - off) >> 5);
                const float4 *buf = reinterpret_cast<const float4 *>(ring + (size_t)slot * COV_CHUNK);
                const float2 *pbuf = reinterpret_cast<const float2 *>(buf);  // PLANAR: [antenna][COV_CHUNK / 32 snapshots]
                auto snap = [&](int s, float4 &a, float4 &b) {
                    if (PLANAR) {
                        const float2 x0 = pbuf[s], x1 = pbuf[COV_CHUNK / 32 + s], x2 = pbuf[2 * (COV_CHUNK / 32) + s], x3 = pbuf[3 * (COV_CHUNK / 32) + s];
                        a = make_float4(x0.x, x0.y, x1.x, x1.y);
                        b = make_float4(x2.x, x2.y, x3.x, x3.y);
                    } else {
                        a = buf[2 * s];
                        b = buf[2 * s + 1];
                    }
                };
                if (nsnap == COV_CHUNK / 32) {
                    float4 xa[4], xb[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) snap(lane + 32 * u, xa[u], xb[u]);
#pragma unroll
                    for (int u = 0; u < 4; ++u) cov4_accumulate(acc, xa[u], xb[u]);
                } else {
                    for (int s = lane; s < nsnap; s += 32) {
                        float4 a, b;
                        snap(s, a, b);
                        cov4_accumulate(acc, a, b);
                    }
                }
                __syncwarp();  // every lane is done reading the slot -> it may be refilled
                if (lane == 0) issue();
                if (++slot == FZ_STAGES) { slot = 0; parity ^= 1; }
            }
            __syncwarp();  // makes lane 0's ring writes (claims during this window) visible to the next read
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = warp_sum(acc[i]);
            unsigned seq = 0u;
            if (lane == 0) seq = atomicAdd(&ctl->cov_seq, 1u);
            seq = __shfl_sync(0xffffffffu, seq, 0);
            for (;;) {  // queue slot free?
                unsigned sd = 0u;
                if (lane == 0) sd = ctl->scan_done;
                if (seq - __shfl_sync(0xffffffffu, sd, 0) < (unsigned)FZ_Q) break;
                __nanosleep(100);
            }
            if (lane == 0) {
                const double dn = (double)N;
                double *Rw = Rq + (size_t)(seq % FZ_Q) * 32;
                Rw[0] = acc[0] / dn;   Rw[1] = 0.0;
                Rw[10] = acc[1] / dn;  Rw[11] = 0.0;
                Rw[20] = acc[2] / dn;  Rw[21] = 0.0;
                Rw[30] = acc[3] / dn;  Rw[31] = 0.0;
                int e = 4;
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = a + 1; b < 4; ++b) {
                        const double re = acc[e] / dn, im = acc[e + 1] / dn;
                        Rw[2 * (a * 4 + b)] = re;  Rw[2 * (a * 4 + b) + 1] = im;
                        Rw[2 * (b * 4 + a)] = re;  Rw[2 * (b * 4 + a) + 1] = -im;
                        e += 2;
                    }
                qwin[seq % FZ_Q] = wcur;
                __threadfence_block();
                qready[seq % FZ_Q] = seq + 1u;  // per-slot ready flag: no ordering between the covariance warps
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[i] = 0.0;
        }
        if (lane == 0) {
            __threadfence_block();
            const unsigned fin = atomicAdd((unsigned *)&ctl->cov_finished, 1u);
            if (dbg && fin == (unsigned)FZ_COV_WARPS - 1) {  // last covariance warp: this SM's input stream ends here
                dbg[blockIdx.x * FZ_TRACE + 0] = clock64() - t_start;
                unsigned long long g;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
                dbg[blockIdx.x * FZ_TRACE + 33] = (long long)g;
            }
            if (dbg && fin == 0) dbg[blockIdx.x * FZ_TRACE + 1] = clock64() - t_start;                           // first one
        }
        __syncwarp();
        if (spec) fused_drain_worker<TRACE, true>(fz_smem, tab_c64, K, spec, out, dbg ? dbg + blockIdx.x * FZ_TRACE : nullptr, t_start);
        else fused_drain_worker<TRACE, false>(fz_smem, tab_c64, K, nullptr, out, dbg ? dbg + blockIdx.x * FZ_TRACE : nullptr, t_start);
    } else if (warp == FZ_COV_WARPS) {
        // ================= eigensolver warp =================
        long long eig_busy = 0, eig_rounds = 0, eig_jacobi = 0;
        for (;;) {
            const unsigned done = ctl->eig_done;
            // ready windows in queue order: slot (done + i) holds sequence number done + i iff its flag says so
            const bool rdy = lane < 8 && qready[(done + lane) % FZ_Q] == done + lane + 1u;
            const unsigned mask = __ballot_sync(0xffffffffu, rdy);
            const unsigned avail = (unsigned)__ffs(~mask) - 1u;  // leading run of ready slots (0..8)
            if (avail == 0) {
                if (ctl->cov_finished == (unsigned)FZ_COV_WARPS && done == *reinterpret_cast<volatile unsigned *>(&ctl->cov_seq)) break;
                __nanosleep(100);
                continue;
            }
            __threadfence_block();
            const long long t0 = clock64();
            const unsigned cnt = min(avail, 8u);
            {
                const unsigned grp = (unsigned)lane >> 2;
                const unsigned slot = (done + min(grp, cnt - 1)) % FZ_Q;
                bool jac = grp < cnt;  // windows the Jacobi solver must take
                if (eig_mode == 0) {  // (every lane must make the call: it shuffles and synchronises over the whole warp)
                    const bool solved = eig4_principal_coop(Rq + (size_t)slot * 32, Vq + (size_t)slot * 32, jac, lane & 3);
                    jac = jac && !solved;
                }
                if (__any_sync(0xffffffffu, jac)) {
                    fused_jacobi4(Rq + (size_t)slot * 32, Vq + (size_t)slot * 32, jac, lane & 3);
                    ++eig_jacobi;
                }
            }
            __syncwarp();
            __threadfence_block();
            if (lane == 0) ctl->eig_done = done + cnt;
            __syncwarp();
            eig_busy += clock64() - t0;
            ++eig_rounds;
        }
        if (dbg && lane == 0) {
            dbg[blockIdx.x * FZ_TRACE + 8] = clock64() - t_start;
            dbg[blockIdx.x * FZ_TRACE + 9] = eig_busy;
            dbg[blockIdx.x * FZ_TRACE + 10] = eig_rounds;
            dbg[blockIdx.x * FZ_TRACE + 19] = eig_jacobi;
        }
        if (spec) fused_drain_worker<TRACE, true>(fz_smem, tab_c64, K, spec, out, dbg ? dbg + blockIdx.x * FZ_TRACE : nullptr, t_start);
        else fused_drain_worker<TRACE, false>(fz_smem, tab_c64, K, nullptr, out, dbg ? dbg + blockIdx.x * FZ_TRACE : nullptr, t_start);
    } else {
        // ================= scan warps =================
        const int st = threadIdx.x - 32 * (FZ_COV_WARPS + 1);  // 0 .. FZ_SCAN_THREADS - 1
        const int swarp = st >> 5;
        const int g = lane >> 2, t = lane & 3;                 // MMA fragment coordinates; t = this thread's window
        float *redmin = reinterpret_cast<float *>(fz_smem + FZ_OFF_RMIN);
        int *cand_cnt = reinterpret_cast<int *>(fz_smem + FZ_OFF_CCNT);
        int *cand_bin = reinterpret_cast<int *>(fz_smem + FZ_OFF_CBIN);
        double *redP = reinterpret_cast<double *>(fz_smem + FZ_OFF_RED);
        int *redk = reinterpret_cast<int *>(fz_smem + FZ_OFF_RED + 8 * FZ_SCAN_WARPS);
        const uint32_t Vq0 = smem_u32(Vq);
        const int ntile_full = fused_tiles(K);
        const uint32_t tb0 = smem_u32(fz_smem + FZ_OFF_TBAR), tbuf0 = smem_u32(fz_smem + FZ_OFF_TBL);
        const float na_max = __ldg(na_max_p);
        const uint64_t pol_keep = l2_policy_evict_last();
        unsigned T = 0;  // table tiles consumed so far (identical in every scan thread)
        long long scan_busy = 0, scan_passes = 0, scan_exact = 0, scan_fallbacks = 0, scan_ncand = 0;
        long long tr_issue = 0, tr_full = 0, tr_comp = 0;

        for (;;) {
            if (swarp == 0) {  // (the whole first scan warp, in uniform control flow; lane 0 decides)
                // A pass streams the whole table from L2 once and costs ~27 k cycles whatever it holds, so it takes exactly
                // FZ_WPT windows, and none is started once the launch is running out (see DRAIN in the file header).
                unsigned start = 0, cnt = 0;
                for (;;) {
                    unsigned stop = 0u;
                    fz_lock(ctl, lane);
                    if (lane == 0) {
                        start = ctl->claim;
                        const unsigned avail = ctl->eig_done - start;
                        const int fin = (int)ctl->cov_finished;
                        const bool closing = (ctl->tout && fin >= mma_fin_max) || fin == FZ_COV_WARPS;  // the launch is running out
                        if (ctl->mma_off) {
                            stop = 1u;
                        } else if (closing) {
                            ctl->mma_off = 1u;
                            stop = 1u;
                        } else if (avail >= (unsigned)FZ_WPT) {
                            cnt = FZ_WPT;
                            ctl->claim = start + cnt;
                        }
                    }
                    fz_unlock(ctl, lane);
                    cnt = __shfl_sync(0xffffffffu, cnt, 0);
                    stop = __shfl_sync(0xffffffffu, stop, 0);
                    if (cnt || stop) break;
                    __nanosleep(200);
                }
                if (lane == 0) {
                    if (dbg && cnt == 0) dbg[blockIdx.x * FZ_TRACE + 16] = clock64() - t_start;  // when the tensor-core passes ended
                    ctl->batch_start = start;
                    ctl->batch_cnt = cnt;
                    __threadfence_block();
                }
                __syncwarp();
            }
            if (st < FZ_WPT) cand_cnt[st] = 0;
            bar_sync_scan();
            const unsigned start = ctl->batch_start, cnt = ctl->batch_cnt;
            if (cnt == 0) break;
            const long long t0 = clock64();

            // B fragments per column group gi (windows 4*gi .. 4*gi+3): column n = lane/4 = 2*(window%4) + {0: Re
            // row, 1: Im row} of e^H, rows k = t and t + 4 of
            //   Re column: [ er0, ei0, er1, ei1, er2, ei2, er3, ei3 ]     Im column: [ -ei0, er0, -ei1, er1, ... ]
            // (c = sum_i conj(e_i) a_i with a row = [Re a0, Im a0, ...]); windows beyond cnt duplicate the last one.
            uint32_t bh0[2], bh1[2], bl0[2], bl1[2];
#pragma unroll
            for (int gi = 0; gi < 2; ++gi) {
                const int wn = min(4 * gi + (g >> 1), (int)cnt - 1), im = g & 1;
                const double *e = Vq + 32 * ((start + wn) % FZ_Q) + 2 * 3 * 4;  // signal vector (largest eigenvalue)
                auto col = [&](int k) -> float {  // element k of this thread's column
                    const int i = k >> 1, part = k & 1;  // antenna; 0 -> multiplies Re a_i, 1 -> multiplies Im a_i
                    const double er = e[2 * i], ei = e[2 * i + 1];
                    return (float)(im == 0 ? (part == 0 ? er : ei) : (part == 0 ? -ei : er));
                };
                const float v0 = col(t), v1 = col(t + 4);
                bh0[gi] = to_tf32(v0); bl0[gi] = to_tf32(v0 - __uint_as_float(bh0[gi]));
                bh1[gi] = to_tf32(v1); bl1[gi] = to_tf32(v1 - __uint_as_float(bh1[gi]));
            }
            // The table streams through the FZ_TS-deep ring; every thread handles two rows (g, g + 8) of every MMA tile its
            // warp owns and both column groups (its windows are 4*gi + t).
            // T counts tiles since kernel start: slot = T % FZ_TS, tfull parity = (T / FZ_TS) & 1; a tile is
            // released by one arrival per scan warp on tempty.
            // Table tiles arrive by cp.async (LDGSTS, 16 B per request through the LSU): the SM's TMA queue is FIFO
            // and permanently holds ~100 KB of HBM-bound covariance requests, behind which an L2-resident
            // table tile would wait for thousands of cycles.  Every scan thread copies its 2-3 chunks of tile
            // T + D and its completion arrives on tfull[slot]; a slot is reused once all warps released it.
            constexpr int D = FZ_TS - 1;  // prefetch distance in tiles
            auto issue_tile = [&](const int ia, const unsigned Ta) {
                const int sa = (int)(Ta % FZ_TS);
                if (Ta >= FZ_TS) while (!mbar_try_wait(tb0 + 8 * (FZ_TS + sa), (uint32_t)((Ta / FZ_TS - 1) & 1))) {}
                const unsigned char *src = tbl + (size_t)ia * FZ_TILE_BYTES;
                const uint32_t dst = tbuf0 + sa * FZ_TILE_BYTES;
#pragma unroll
                for (int c = 0; c < FZ_CPT; ++c) {
                    const int chunk = st + c * FZ_SCAN_THREADS;  // 16-byte chunk of the tile
                    if (chunk < FZ_TILE_BYTES / 16)
                        asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst + 16 * chunk), "l"(src + 16 * chunk), "l"(pol_keep) : "memory");
                }
                asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(tb0 + 8 * sa) : "memory");
            };
            // ---- the two sweeps of a pass share ONE loop body (instruction footprint, see the file header) ----
            //   phase 0 (the decimated tiles only): an upper bound U >= min_k d_k per window, U = min over the subsample
            //           of d~ + B||a||^2 (any bin's upper bound bounds the minimum from above);
            //   phase 1 (the whole table): the candidates, lower bound d~ - B||a||^2 <= U (1 + 2^-10); the relative slack
            //           makes every rejected bin's exact d larger than the best one's by > 2^-11 relative, so its
            //           reciprocal is strictly smaller (no tie can be lost to the rounding of 1/d).  Columns that
            //           duplicate a window (beyond cnt) do not report.
            const float INF = __int_as_float(0x7f800000);
            float umin[2] = {INF, INF}, thr[2] = {-INF, -INF};
#pragma unroll 1
            for (int phase = 0; phase < 2; ++phase) {
                const int tile0 = phase ? FZ_NDEC : 0, ntile = phase ? ntile_full : FZ_NDEC;
                for (int a = 0; a < D && a < ntile; ++a) issue_tile(tile0 + a, T + a);
#pragma unroll 1
                for (int it = 0; it < ntile; ++it, ++T) {
                    const int slot = (int)(T % FZ_TS);
                    const long long tk0 = dbg ? clock64() : 0;
                    if (it + D < ntile) issue_tile(tile0 + it + D, T + D);
                    const long long tk1 = dbg ? clock64() : 0;
                    while (!mbar_try_wait(tb0 + 8 * slot, (uint32_t)((T / FZ_TS) & 1))) {}
                    const long long tk2 = dbg ? clock64() : 0;
                    const uint32_t tile = tbuf0 + slot * FZ_TILE_BYTES;
                    // all MMA tiles of this warp: loads and the truncating tf32 split (ALU pipe) first
                    uint32_t ah[FZ_MPW][4], al[FZ_MPW][4];
                    float na0[FZ_MPW], na1[FZ_MPW];
#pragma unroll
                    for (int m = 0; m < FZ_MPW; ++m) {
                        const int mt = m * FZ_SCAN_WARPS + swarp;  // MMA tile within the FZ_BINS-row tile (round-robin over warps)
                        uint32_t av[4];
                        asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(av[0]), "=r"(av[1]), "=r"(av[2]), "=r"(av[3]) : "r"(tile + mt * FZ_FRAG_BYTES + lane * 16));
                        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(na0[m]) : "r"(tile + (FZ_BINS / 16) * FZ_FRAG_BYTES + 4 * (mt * 16 + g)));
                        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(na1[m]) : "r"(tile + (FZ_BINS / 16) * FZ_FRAG_BYTES + 4 * (mt * 16 + g + 8)));
#pragma unroll
                        for (int i = 0; i < 4; ++i) {  // a = hi + lo + r, |r| < 2^-20|a|
                            ah[m][i] = av[i] & 0xffffe000u;
                            al[m][i] = __float_as_uint(__uint_as_float(av[i]) - __uint_as_float(ah[m][i])) & 0xffffe000u;
                        }
                    }
                    __syncwarp();
                    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tb0 + 8 * (FZ_TS + slot)) : "memory");
                    // 3 MMAs (a_lo e_hi, a_hi e_lo, a_hi e_hi; small terms first) for each of the 2 FZ_MPW (tile, column
                    // group) accumulators, issued round-robin so that dependent MMAs are 8 instructions (~64
                    // cycles at one HMMA.1688 per 8 cycles) apart - more than the ~20-cycle MMA latency.
                    float c[FZ_MPW][2][4];
#pragma unroll
                    for (int m = 0; m < FZ_MPW; ++m)
#pragma unroll
                        for (int gi = 0; gi < 2; ++gi)
                            asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                                : "=f"(c[m][gi][0]), "=f"(c[m][gi][1]), "=f"(c[m][gi][2]), "=f"(c[m][gi][3])
                                : "r"(al[m][0]), "r"(al[m][1]), "r"(al[m][2]), "r"(al[m][3]), "r"(bh0[gi]), "r"(bh1[gi]), "f"(0.f));
#pragma unroll
                    for (int m = 0; m < FZ_MPW; ++m)
#pragma unroll
                        for (int gi = 0; gi < 2; ++gi)
                            asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                                : "+f"(c[m][gi][0]), "+f"(c[m][gi][1]), "+f"(c[m][gi][2]), "+f"(c[m][gi][3])
                                : "r"(ah[m][0]), "r"(ah[m][1]), "r"(ah[m][2]), "r"(ah[m][3]), "r"(bl0[gi]), "r"(bl1[gi]));
#pragma unroll
                    for (int m = 0; m < FZ_MPW; ++m)
#pragma unroll
                        for (int gi = 0; gi < 2; ++gi)
                            asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                                : "+f"(c[m][gi][0]), "+f"(c[m][gi][1]), "+f"(c[m][gi][2]), "+f"(c[m][gi][3])
                                : "r"(ah[m][0]), "r"(ah[m][1]), "r"(ah[m][2]), "r"(ah[m][3]), "r"(bh0[gi]), "r"(bh1[gi]));
                    // (c0, c1) = (Re, Im) of e^H a for row g, window 4*gi + t; (c2, c3) the same for row g + 8
                    if (phase == 0) {
#pragma unroll
                        for (int m = 0; m < FZ_MPW; ++m)
#pragma unroll
                            for (int gi = 0; gi < 2; ++gi) {
                                const float d0 = na0[m] - fmaf(c[m][gi][0], c[m][gi][0], c[m][gi][1] * c[m][gi][1]);
                                const float d1 = na1[m] - fmaf(c[m][gi][2], c[m][gi][2], c[m][gi][3] * c[m][gi][3]);
                                umin[gi] = fminf(umin[gi], fminf(fmaf(FZ_B, na0[m], d0), fmaf(FZ_B, na1[m], d1)));
                            }
                    } else {
#pragma unroll
                        for (int m = 0; m < FZ_MPW; ++m) {
                            const int row = it * FZ_BINS + (m * FZ_SCAN_WARPS + swarp) * 16 + g;
#pragma unroll
                            for (int gi = 0; gi < 2; ++gi) {
                                const float d0 = na0[m] - fmaf(c[m][gi][0], c[m][gi][0], c[m][gi][1] * c[m][gi][1]);
                                const float d1 = na1[m] - fmaf(c[m][gi][2], c[m][gi][2], c[m][gi][3] * c[m][gi][3]);
                                if (fmaf(-FZ_B, na0[m], d0) <= thr[gi]) {
                                    const int sc = atomicAdd(&cand_cnt[4 * gi + t], 1);
                                    if (sc < FZ_CMAX) cand_bin[(4 * gi + t) * FZ_CMAX + sc] = row;
                                }
                                if (fmaf(-FZ_B, na1[m], d1) <= thr[gi]) {
                                    const int sc = atomicAdd(&cand_cnt[4 * gi + t], 1);
                                    if (sc < FZ_CMAX) cand_bin[(4 * gi + t) * FZ_CMAX + sc] = row + 8;
                                }
                            }
                        }
                    }
                    if (dbg) { const long long tk3 = clock64(); tr_issue += tk1 - tk0; tr_full += tk2 - tk1; tr_comp += tk3 - tk2; }
                }
                if (phase == 0) {
#pragma unroll
                    for (int gi = 0; gi < 2; ++gi) {
                        float u = umin[gi];
                        u = fminf(u, __shfl_xor_sync(0xffffffffu, u, 4));
                        u = fminf(u, __shfl_xor_sync(0xffffffffu, u, 8));
                        u = fminf(u, __shfl_xor_sync(0xffffffffu, u, 16));
                        if (lane < 4) redmin[swarp * FZ_WPT + 4 * gi + lane] = u;
                    }
                    bar_sync_scan();
#pragma unroll
                    for (int gi = 0; gi < 2; ++gi) {
                        const int w = 4 * gi + t;
                        float u = redmin[w];
#pragma unroll
                        for (int q = 1; q < FZ_SCAN_WARPS; ++q) u = fminf(u, redmin[q * FZ_WPT + w]);
                        thr[gi] = (unsigned)w < cnt ? fmaf(fabsf(u), 0.0009765625f, u) : -INF;
                    }
                }
            }
            bar_sync_scan();

            // ---- exact fp64 evaluation: the candidates of all windows flattened over the scan threads ----
            // (strength desc, bin asc) is resolved with two shared-memory atomics per candidate: max over the
            // fp64 bit pattern of P (positive doubles order like their bits), then min over the bins that hold it.
            const long long te0 = dbg ? clock64() : 0;
            unsigned long long *bestP = reinterpret_cast<unsigned long long *>(fz_smem + FZ_OFF_BEST);
            int *bestk = reinterpret_cast<int *>(fz_smem + FZ_OFF_BEST + 8 * FZ_WPT);
            int *admitted = reinterpret_cast<int *>(fz_smem + FZ_OFF_BEST + 12 * FZ_WPT);
            constexpr int IPT = FZ_IPT;
            int pre[FZ_WPT + 1];
            pre[0] = 0;
#pragma unroll
            for (int w = 0; w < FZ_WPT; ++w) {
                const int nc = ((unsigned)w < cnt) ? cand_cnt[w] : 0;
                const bool ok = nc <= FZ_CMAX && pre[w] + nc <= IPT * FZ_SCAN_THREADS;
                pre[w + 1] = pre[w] + (ok ? nc : 0);
                if (st == w) { bestP[w] = 0ull; bestk[w] = 0x7fffffff; admitted[w] = ok ? 1 : 0; }
            }
            bar_sync_scan();
            double myP[IPT];
            int myk[IPT], myw[IPT];
#pragma unroll
            for (int r = 0; r < IPT; ++r) {
                const int i = st + r * FZ_SCAN_THREADS;
                myk[r] = -1; myw[r] = 0; myP[r] = 0.0;
                if (i < pre[FZ_WPT]) {
                    int w = 0;
#pragma unroll
                    for (int q = 1; q < FZ_WPT; ++q) w += (i >= pre[q]) ? 1 : 0;
                    const int k = cand_bin[w * FZ_CMAX + (i - pre[w])];
                    const double P = fused_exact_P(tab_c64, k, Vq0 + 256 * ((start + w) % FZ_Q), pol_keep);
                    if (P > 0.0) {  // NaN and non-positive strengths are never inserted (reference :132)
                        myP[r] = P; myk[r] = k; myw[r] = w;
                        atomicMax(&bestP[w], (unsigned long long)__double_as_longlong(P));
                    }
                }
            }
            bar_sync_scan();
#pragma unroll
            for (int r = 0; r < IPT; ++r)
                if (myk[r] >= 0 && (unsigned long long)__double_as_longlong(myP[r]) == bestP[myw[r]]) atomicMin(&bestk[myw[r]], myk[r]);
            bar_sync_scan();
            if (swarp == 0) {  // (cnt <= FZ_WPT: every window of the pass belongs to a lane of the first scan warp)
                const bool v = (unsigned)st < cnt && admitted[st];
                const int kk = v ? (bestk[st] == 0x7fffffff ? -1 : bestk[st]) : -1;
                const double P = v ? __longlong_as_double((long long)bestP[st]) : 0.0;
                fused_emit(fz_smem, out, v, v ? (unsigned)qwin[(start + st) % FZ_Q] : 0u, kk, P, K);
            }
            if (dbg && st == 0) scan_ncand += pre[FZ_WPT];
            // ---- fallback: too many candidates (flat spectrum) -> every bin in fp64 ----
            for (unsigned w = 0; w < cnt; ++w) {
                if (admitted[w]) continue;  // uniform over the scan group
                const uint32_t ev = Vq0 + 256 * ((start + w) % FZ_Q);
                double P = 0.0;
                int kk = -1;
                for (int k = st; k < K; k += FZ_SCAN_THREADS) {
                    const double p = fused_exact_P(tab_c64, k, ev, pol_keep);
                    if (p > P) { P = p; kk = k; }  // k ascending per thread: strict '>' keeps the lower bin
                }
                warp_argmax(P, kk);
                if (lane == 0) { redP[swarp] = P; redk[swarp] = kk; }
                bar_sync_scan();
                if (st == 0) {
                    for (int q = 1; q < FZ_SCAN_WARPS; ++q)
                        if (peak_better(redP[q], redk[q], P, kk)) { P = redP[q]; kk = redk[q]; }
                    ++scan_fallbacks;
                }
                if (swarp == 0) fused_emit(fz_smem, out, st == 0, (unsigned)qwin[(start + w) % FZ_Q], kk, P, K);
                bar_sync_scan();
            }
            if (dbg) scan_exact += clock64() - te0;
            bar_sync_scan();  // scratch and the queue slots may be reused from here on
            if (swarp == 0) fused_retire(fz_smem, start, cnt, lane);
            scan_busy += clock64() - t0;
            ++scan_passes;
        }
        if (dbg && st == 0) {
            dbg[blockIdx.x * FZ_TRACE + 11] = clock64() - t_start;
            dbg[blockIdx.x * FZ_TRACE + 12] = scan_busy;
            dbg[blockIdx.x * FZ_TRACE + 13] = scan_passes;
            dbg[blockIdx.x * FZ_TRACE + 14] = scan_exact;
            dbg[blockIdx.x * FZ_TRACE + 15] = scan_fallbacks;
            dbg[blockIdx.x * FZ_TRACE + 7] = scan_ncand;
            dbg[blockIdx.x * FZ_TRACE + 4] = tr_issue;  // (overwrite covariance warps 4..6 slots)
            dbg[blockIdx.x * FZ_TRACE + 5] = tr_full;
            dbg[blockIdx.x * FZ_TRACE + 6] = tr_comp;
            unsigned long long g_end;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g_end));
            dbg[blockIdx.x * FZ_TRACE + 3] = (long long)(g_end - g_start);   // ns, this CTA's lifetime (overwrites covariance warp 3's slot)
            dbg[blockIdx.x * FZ_TRACE + 2] = (long long)g_start;             // ns, absolute start (overwrites covariance warp 2's slot)
        }
        if (spec) fused_drain_worker<TRACE, true>(fz_smem, tab_c64, K, spec, out, dbg ? dbg + blockIdx.x * FZ_TRACE : nullptr, t_start);
        else fused_drain_worker<TRACE, false>(fz_smem, tab_c64, K, nullptr, out, dbg ? dbg + blockIdx.x * FZ_TRACE : nullptr, t_start);
    }
    // The last CTA to finish re-arms the ticket counter for the next launch (launches of one handle are
    // serialised by the host, and by now every covariance warp has drawn a ticket >= W).
    __syncthreads();
    if (warp == 0 && !ctl->ordered) fused_stage_flush(fz_smem, out, K);  // (uniform: no warp is left to change `ordered`)
    if (threadIdx.x == 0) {
        if (dbg) {
            dbg[blockIdx.x * FZ_TRACE + 17] = ctl->drained_windows;
            dbg[blockIdx.x * FZ_TRACE + 20] = ctl->drain_groups;
            dbg[blockIdx.x * FZ_TRACE + 18] = clock64() - t_start;  // every window of this CTA is finished
            unsigned long long g;
            unsigned smid;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g));
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            dbg[blockIdx.x * FZ_TRACE + 31] = (long long)g;  // ns, absolute: CTA exit
            dbg[blockIdx.x * FZ_TRACE + 30] = (long long)smid;
        }
        if (out.npeer > 0) __threadfence_system(); else __threadfence();
        if (atomicAdd(&work_ctr[1], 1u) == gridDim.x - 1) {
            work_ctr[0] = 0;
            work_ctr[1] = 0;
            __threadfence();
            // every CTA's peak bins (fenced at system scope above) are on their way to the peers: raise this GPU's
            // epoch flag in every peer's flag array - the consumer side of the fused all-gather waits on these
            if (out.npeer > 0 && gather_flags.epoch) {
                __threadfence_system();
                for (int p = 0; p < out.npeer; ++p)
                    asm volatile("red.release.sys.global.max.u32 [%0], %1;" ::"l"(gather_flags.peer[p] + out.rank), "r"(gather_flags.epoch) : "memory");  // (max: launches may retire out of order)
            }
        }
    }
}

}  // namespace music
