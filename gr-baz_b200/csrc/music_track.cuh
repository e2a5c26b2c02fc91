// music_track.cuh - angle tracking across windows (opt-in, music_b200_set_tracking; the *_tracks entry points).
//
// After the peak stage (and the beams and the CRB) every window's filled slots are measurements of a bank of at most 32
// constant-velocity Kalman filters, one per track: predict, gate by the Mahalanobis distance, assign by global nearest
// neighbour, update in Joseph form, confirm M of N, delete after consecutive misses, start tracks on the measurements
// left over.  The full definition is in include/music_b200.h and is restated literally by tests/track_oracle.py.
//
// The recurrence is serial in window order, so the work is to keep each window's dependent chain short rather than to
// move bytes.  track_kernel<D> (D = 1: angle; D = 2: azimuth and elevation) runs one warp per handle per sub-batch:
//   - lane r owns carry row r (state, covariance and counters in registers); prediction, distances, the gating masks
//     and the updates are lane-local, the measurements of a window are shared through shared memory;
//   - the inputs (angles, elevations, bins, CRB) of TRK_CHUNK windows are copied into a shared-memory buffer by
//     asynchronous copies issued one chunk ahead, so no window waits on a global load; each window's outputs are
//     written by the lanes as whole rows;
//   - the assignment: a row whose only gated measurement has no other gated row is an isolated pair and is matched at
//     once (the common case needs no solver).  The rows and measurements left form the ambiguous clusters, solved
//     together by a Hungarian (Jonker-Volgenant shortest augmenting path) solve on a shared-memory cost view with one
//     lane per column of the larger side.  With cost d2 - gate <= 0 on gated pairs and 0 elsewhere a minimum-cost
//     assignment of the smaller side equals the minimum over partial matchings of gated pairs (a non-gated pair taken
//     by the solve is no match), so no dummy rows are needed.
// The carry (the rows and next_id) lives in the handle's device buffers, read at the start of each sub-batch and
// written at its end; the handle orders consecutive sub-batches, on whichever streams they run, with one event.
#pragma once
#include <cuda_pipeline.h>
#include "music_kernels.cuh"

namespace music {

constexpr int TRK_ROWS = 32;          // carry rows (max_tracks <= 32): lane r owns row r
constexpr int TRK_MAXN = MAXM - 1;    // slots per window (n < M)
constexpr int TRK_CHUNK = 32;         // windows per shared-memory input buffer
constexpr int TRK_ROW_INTS = 5;       // id, status, age, hits, misses
constexpr int TRK_INT_MAX = 0x7fffffff;
constexpr double TRK_INF = __builtin_huge_val();

enum : int { TRK_EMPTY = 0, TRK_TENTATIVE = 1, TRK_CONFIRMED = 2 };  // MUSIC_B200_TRACK_EMPTY, _TENTATIVE, _CONFIRMED

struct TrackParams {
    bool crb;                          // measurement covariance from the CRB (MUSIC_B200_TRACK_CRB), else floor^2 I
    double q, rate0, floor, crb_scale, gate;
    int confirm_hits, confirm_window, max_misses, T;
};

// doubles of one carry row's state: x [2D] then P [2D][2D] row-major
__host__ __device__ constexpr int track_state_len(int D) { return 2 * D + 4 * D * D; }

__device__ __forceinline__ double trk_wrap360(double v) { return v - 360.0 * floor(v / 360.0); }
__device__ __forceinline__ double trk_wrap180(double v) { return v - 360.0 * floor((v + 180.0) / 360.0); }

// The cost view of the ambiguous clusters: the smaller side are the solve's rows, the larger its columns.
struct TrkCost {
    const double *d2;          // [TRK_ROWS][16] distances of (row, slot)
    const uint32_t *gated;     // [TRK_ROWS] gating masks over the slots
    const int *rows, *slots;   // the ambiguous rows and slots, ascending
    bool swap;                 // the solve's rows are slots (fewer ambiguous slots than rows)
    double gate;
    __device__ void pair(int hr, int hc, int &t, int &i) const
    {
        t = swap ? rows[hc] : rows[hr];
        i = swap ? slots[hr] : slots[hc];
    }
    __device__ double operator()(int hr, int hc) const
    {
        int t, i;
        pair(hr, hc, t, i);
        return (gated[t] >> i) & 1u ? d2[t * 16 + i] - gate : 0.0;
    }
};

// Minimum-cost assignment of nr rows to nc >= nr columns (nc <= 32), warp-wide: the shortest augmenting path form of the
// Hungarian method (Jonker & Volgenant 1987), lane j holding column j + 1 (column 0 is the virtual start), its potential,
// its running minimum and its path link.  sU [33]: row potentials.  Returns in `p` the 1-based row given column lane + 1
// (0: none).  Ties go to the lowest column, so the result is the same on every run.
__device__ int trk_hungarian(const TrkCost &cost, int nr, int nc, double *sU, int lane)
{
    constexpr unsigned full = 0xffffffffu;
    int p = 0, way = 0;
    double v = 0.0;
    if (lane <= nr) sU[lane] = 0.0;
    if (lane == 0) sU[32] = 0.0;
    __syncwarp();
    for (int i = 1; i <= nr; ++i) {
        int j0 = 0;
        double minv = TRK_INF;
        bool used = false;
        while (true) {
            const int pj0 = __shfl_sync(full, p, j0 > 0 ? j0 - 1 : 0);
            const int i0 = j0 == 0 ? i : pj0;
            if (lane == j0 - 1) used = true;
            const double ui0 = sU[i0];
            double cand = TRK_INF;
            if (lane < nc && !used) {
                const double cur = cost(i0 - 1, lane) - ui0 - v;
                if (cur < minv) { minv = cur; way = j0; }
                cand = minv;
            }
            int cj = lane;
            for (int off = 16; off; off >>= 1) {
                const double ov = __shfl_xor_sync(full, cand, off);
                const int oj = __shfl_xor_sync(full, cj, off);
                if (ov < cand || (ov == cand && oj < cj)) { cand = ov; cj = oj; }
            }
            const double delta = cand;
            __syncwarp();  // every lane has read sU[i0]
            if (lane < nc) {
                if (used) { sU[p] += delta; v -= delta; }
                else minv -= delta;
            }
            if (lane == 0) sU[i] += delta;  // the virtual column holds row i (no used column holds it)
            __syncwarp();
            j0 = cj + 1;
            if (__shfl_sync(full, p, cj) == 0) break;
        }
        while (j0 != 0) {  // augment along the links
            const int w = __shfl_sync(full, way, j0 - 1);
            const int pw = __shfl_sync(full, p, w > 0 ? w - 1 : 0);
            if (lane == j0 - 1) p = w == 0 ? i : pw;
            j0 = w;
        }
    }
    return p;
}

// angles / bins [W][n] (the azimuths on an az-el handle), elev [W][n] (D = 2), crb [W][n] (D = 1) or [W][n][3] (D = 2),
// read under CRB variance only.  Carry: rows [T][5], state [T][track_state_len(D)], next [1]; `fresh`: start from empty
// rows and next_id 0 instead.  Outputs slot_track [W][n]; track_ids [W][T] and track_state [W][T][3 D] (both or neither).
template <int D>
__global__ void __launch_bounds__(32) track_kernel(const float *__restrict__ angles, const float *__restrict__ elev,
                                                   const int32_t *__restrict__ bins, const float *__restrict__ crb, int n, int W,
                                                   const TrackParams tp, bool fresh, int32_t *__restrict__ carry_rows,
                                                   double *__restrict__ carry_state, unsigned *__restrict__ carry_next,
                                                   int32_t *__restrict__ slot_track, int32_t *__restrict__ track_ids,
                                                   float *__restrict__ track_state)
{
    constexpr unsigned full = 0xffffffffu;
    constexpr int NS = 2 * D, SL = track_state_len(D), CW = D == 2 ? 3 : 1, OUT = 3 * D;
    __shared__ float sAng[2][TRK_CHUNK * TRK_MAXN], sEl[2][D == 2 ? TRK_CHUNK * TRK_MAXN : 1];
    __shared__ float sCrb[2][TRK_CHUNK * TRK_MAXN * CW];
    __shared__ int32_t sBin[2][TRK_CHUNK * TRK_MAXN];
    __shared__ double sZ[16][2], sR[16][3];       // the window's measurements
    __shared__ double sD2[TRK_ROWS * 16];         // distances (row, slot)
    __shared__ uint32_t sGated[TRK_ROWS];
    __shared__ int sRows[TRK_ROWS], sSlots[16], sMatch[TRK_ROWS], sSlotTrack[16];
    __shared__ double sU[33];
    const int lane = threadIdx.x, T = tp.T;
    const bool crbv = tp.crb;

    // this lane's row of the carry
    int id = -1, status = TRK_EMPTY, age = 0, hits = 0, misses = 0;
    double x[NS], P[NS][NS];
    for (int a = 0; a < NS; ++a) {
        x[a] = 0.0;
        for (int b = 0; b < NS; ++b) P[a][b] = 0.0;
    }
    unsigned next_id = 0;
    if (!fresh) {
        if (lane < T) {
            const int32_t *rw = carry_rows + lane * TRK_ROW_INTS;
            id = rw[0]; status = rw[1]; age = rw[2]; hits = rw[3]; misses = rw[4];
            const double *st = carry_state + lane * SL;
            for (int a = 0; a < NS; ++a) x[a] = st[a];
            for (int a = 0; a < NS; ++a)
                for (int b = 0; b < NS; ++b) P[a][b] = st[NS + a * NS + b];
        }
        next_id = *carry_next;
    }

    const auto stage = [&](int buf, int w0) {
        const int e = min(TRK_CHUNK, W - w0) * n;
        for (int k = lane; k < e; k += 32) {
            __pipeline_memcpy_async(&sAng[buf][k], angles + (size_t)w0 * n + k, sizeof(float));
            __pipeline_memcpy_async(&sBin[buf][k], bins + (size_t)w0 * n + k, sizeof(int32_t));
            if constexpr (D == 2) __pipeline_memcpy_async(&sEl[buf][k], elev + (size_t)w0 * n + k, sizeof(float));
        }
        if (crbv)
            for (int k = lane; k < e * CW; k += 32)
                __pipeline_memcpy_async(&sCrb[buf][k], crb + (size_t)w0 * n * CW + k, sizeof(float));
        __pipeline_commit();
    };

    const double c2 = tp.crb_scale * tp.crb_scale, f2 = tp.floor * tp.floor, gate = tp.gate;
    const double q3 = tp.q * (1.0 / 3.0), q2 = tp.q * 0.5, rs2 = tp.rate0 * tp.rate0;
    const uint32_t nmask = (1u << n) - 1u;
    stage(0, 0);
    for (int w0 = 0, c = 0; w0 < W; w0 += TRK_CHUNK, ++c) {
        const int buf = c & 1;
        if (w0 + TRK_CHUNK < W) {
            stage(buf ^ 1, w0 + TRK_CHUNK);
            __pipeline_wait_prior(1);
        } else {
            __pipeline_wait_prior(0);
        }
        __syncwarp();
        const int cw = min(TRK_CHUNK, W - w0);
        for (int wi = 0; wi < cw; ++wi) {
            const size_t w = (size_t)w0 + wi;
            const bool live = status != TRK_EMPTY;
            // 1. predict
            if (live) {
                for (int u = 0; u < D; ++u)
                    for (int v = 0; v < D; ++v) {
                        double &a = P[2 * u][2 * v], &b = P[2 * u][2 * v + 1], &cc = P[2 * u + 1][2 * v], &d = P[2 * u + 1][2 * v + 1];
                        const double bd = b + d, cd = cc + d;
                        a = (a + cc) + bd;
                        b = bd;
                        cc = cd;
                        if (u == v) { a += q3; b += q2; cc += q2; d += tp.q; }
                    }
                for (int u = 0; u < D; ++u) x[2 * u] = x[2 * u] + x[2 * u + 1];
                x[0] = trk_wrap360(x[0]);
                age = age < TRK_INT_MAX ? age + 1 : age;
            }
            // 2. measurements: lane i holds slot i
            bool valid = false;
            if (lane < n) {
                const int k = wi * n + lane;
                valid = sBin[buf][k] >= 0;
                const double z0 = (double)sAng[buf][k];
                double z1 = 0.0;
                if constexpr (D == 2) z1 = (double)sEl[buf][k];
                double r00 = f2, r01 = 0.0, r11 = f2;
                if (crbv) {
                    if constexpr (D == 1) {
                        const double s = (double)sCrb[buf][k];
                        valid = valid && isfinite(s);
                        r00 = c2 * (s * s) + f2;
                    } else {
                        const double sa = (double)sCrb[buf][3 * k], se = (double)sCrb[buf][3 * k + 1], rho = (double)sCrb[buf][3 * k + 2];
                        valid = valid && isfinite(sa) && isfinite(se) && isfinite(rho);
                        r00 = c2 * (sa * sa) + f2;
                        r01 = c2 * ((rho * sa) * se);
                        r11 = c2 * (se * se) + f2;
                    }
                }
                sZ[lane][0] = z0; sZ[lane][1] = z1;
                sR[lane][0] = r00; sR[lane][1] = r01; sR[lane][2] = r11;
                sSlotTrack[lane] = -1;
            }
            const uint32_t mmask = __ballot_sync(full, valid) & nmask;
            __syncwarp();
            // 3. distances and the gating mask of this lane's row
            uint32_t g = 0;
            if (live)
                for (uint32_t mm = mmask; mm; mm &= mm - 1) {
                    const int i = __ffs(mm) - 1;
                    double d2;
                    if constexpr (D == 1) {
                        const double nu = trk_wrap180(sZ[i][0] - x[0]), S = P[0][0] + sR[i][0];
                        d2 = (nu * nu) / S;
                    } else {
                        const double nu0 = trk_wrap180(sZ[i][0] - x[0]), nu1 = sZ[i][1] - x[2];
                        const double S00 = P[0][0] + sR[i][0], S01 = P[0][2] + sR[i][1], S11 = P[2][2] + sR[i][2];
                        const double det = S00 * S11 - S01 * S01;
                        d2 = ((S11 * nu0) * nu0 - ((2.0 * S01) * nu0) * nu1 + (S00 * nu1) * nu1) / det;
                    }
                    sD2[lane * 16 + i] = d2;
                    if (d2 <= gate) g |= 1u << i;
                }
            sGated[lane] = g;
            // lane i < n: the rows that gate slot i
            uint32_t col = 0;
            for (int i = 0; i < n; ++i) {
                const uint32_t b = __ballot_sync(full, (g >> i) & 1u);
                if (lane == i) col = b;
            }
            // 4. assignment: isolated pairs at once, the ambiguous clusters by one solve
            const int gi = g ? __ffs(g) - 1 : 0;
            const uint32_t col_gi = __shfl_sync(full, col, gi);
            const int gr = col ? __ffs(col) - 1 : 0;
            const uint32_t g_gr = __shfl_sync(full, g, gr);
            int match = -1;
            bool amb_row = false, amb_slot = false;
            if (g) {
                if (__popc(g) == 1 && __popc(col_gi) == 1) match = gi;
                else amb_row = true;
            }
            if (col) amb_slot = __popc(col) > 1 || __popc(g_gr) > 1;
            const uint32_t rows_amb = __ballot_sync(full, amb_row), slots_amb = __ballot_sync(full, amb_slot);
            sMatch[lane] = match;
            if (rows_amb) {
                if (amb_row) sRows[__popc(rows_amb & ((1u << lane) - 1u))] = lane;
                if (amb_slot) sSlots[__popc(slots_amb & ((1u << lane) - 1u))] = lane;
                __syncwarp();
                const int a = __popc(rows_amb), s = __popc(slots_amb);
                TrkCost cost{sD2, sGated, sRows, sSlots, s < a, gate};
                const int nr = min(a, s), nc = max(a, s);
                const int pr = trk_hungarian(cost, nr, nc, sU, lane);
                if (lane < nc && pr > 0) {
                    int t, i;
                    cost.pair(pr - 1, lane, t, i);
                    if ((sGated[t] >> i) & 1u) sMatch[t] = i;
                }
                __syncwarp();
                match = sMatch[lane];
            }
            const uint32_t matched = __reduce_or_sync(full, match >= 0 ? 1u << match : 0u);
            // 5. update
            if (match >= 0) {
                const int i = match;
                double K[NS][D], Rm[D][D];
                double nu[D];
                if constexpr (D == 1) {
                    Rm[0][0] = sR[i][0];
                    nu[0] = trk_wrap180(sZ[i][0] - x[0]);
                    const double S = P[0][0] + Rm[0][0];
                    for (int j = 0; j < NS; ++j) K[j][0] = P[j][0] / S;
                } else {
                    Rm[0][0] = sR[i][0]; Rm[0][D - 1] = sR[i][1]; Rm[D - 1][0] = sR[i][1]; Rm[D - 1][D - 1] = sR[i][2];
                    nu[0] = trk_wrap180(sZ[i][0] - x[0]);
                    nu[D - 1] = sZ[i][1] - x[2 * (D - 1)];
                    const double S00 = P[0][0] + Rm[0][0], S01 = P[0][2 * (D - 1)] + Rm[0][D - 1], S11 = P[2 * (D - 1)][2 * (D - 1)] + Rm[D - 1][D - 1];
                    const double det = S00 * S11 - S01 * S01;
                    for (int j = 0; j < NS; ++j) {
                        K[j][0] = (P[j][0] * S11 - P[j][2 * (D - 1)] * S01) / det;
                        K[j][D - 1] = (P[j][2 * (D - 1)] * S00 - P[j][0] * S01) / det;
                    }
                }
                for (int j = 0; j < NS; ++j) {
                    double kn = 0.0;
                    for (int u = 0; u < D; ++u) kn += K[j][u] * nu[u];
                    x[j] = x[j] + kn;
                }
                x[0] = trk_wrap360(x[0]);
                // Joseph form: P <- A P A^T + K R K^T with A = I - K H, the lower triangle mirrored
                double A[NS][NS], M[NS][NS], KR[NS][D];
                for (int j = 0; j < NS; ++j)
                    for (int cc = 0; cc < NS; ++cc) A[j][cc] = (j == cc ? 1.0 : 0.0) - ((cc & 1) == 0 ? K[j][cc / 2] : 0.0);
                for (int j = 0; j < NS; ++j)
                    for (int b = 0; b < NS; ++b) {
                        double s = 0.0;
                        for (int a = 0; a < NS; ++a) s += A[j][a] * P[a][b];
                        M[j][b] = s;
                    }
                for (int j = 0; j < NS; ++j)
                    for (int v = 0; v < D; ++v) {
                        double s = 0.0;
                        for (int u = 0; u < D; ++u) s += K[j][u] * Rm[u][v];
                        KR[j][v] = s;
                    }
                for (int j = 0; j < NS; ++j)
                    for (int l = j; l < NS; ++l) {
                        double s = 0.0, t = 0.0;
                        for (int b = 0; b < NS; ++b) s += M[j][b] * A[l][b];
                        for (int v = 0; v < D; ++v) t += KR[j][v] * K[l][v];
                        P[j][l] = s + t;
                    }
                for (int j = 0; j < NS; ++j)
                    for (int l = 0; l < j; ++l) P[j][l] = P[l][j];
                hits = hits < TRK_INT_MAX ? hits + 1 : hits;
                misses = 0;
                sSlotTrack[i] = id;
            } else if (live) {
                misses = misses < TRK_INT_MAX ? misses + 1 : misses;
            }
            // 6. status
            bool drop = false;
            if (status == TRK_TENTATIVE) {
                if (hits >= tp.confirm_hits) status = TRK_CONFIRMED;
                else drop = (long long)hits + ((long long)tp.confirm_window - age) < tp.confirm_hits;
            } else if (status == TRK_CONFIRMED) {
                drop = misses >= tp.max_misses;
            }
            if (drop) {
                id = -1; status = TRK_EMPTY; age = hits = misses = 0;
                for (int a = 0; a < NS; ++a) {
                    x[a] = 0.0;
                    for (int b = 0; b < NS; ++b) P[a][b] = 0.0;
                }
            }
            // 7. initiation: each unmatched measurement in slot order takes the lowest empty row
            uint32_t empty = __ballot_sync(full, status == TRK_EMPTY && lane < T);
            for (uint32_t um = mmask & ~matched; um; um &= um - 1) {
                if (!empty) break;
                const int i = __ffs(um) - 1, r = __ffs(empty) - 1;
                empty &= empty - 1;
                if (lane == r) {
                    id = (int)next_id;
                    status = tp.confirm_hits == 1 ? TRK_CONFIRMED : TRK_TENTATIVE;
                    age = hits = 1;
                    misses = 0;
                    x[0] = sZ[i][0];
                    P[0][0] = sR[i][0];
                    P[1][1] = rs2;
                    if constexpr (D == 2) {
                        x[2] = sZ[i][1];
                        P[0][2] = P[2][0] = sR[i][1];
                        P[2][2] = sR[i][2];
                        P[3][3] = rs2;
                    }
                    sSlotTrack[i] = id;
                }
                next_id = (next_id + 1u) & 0x7fffffffu;
            }
            __syncwarp();
            // 8. outputs
            if (lane < n) slot_track[w * n + lane] = sSlotTrack[lane];
            if (track_ids && lane < T) {
                const bool conf = status == TRK_CONFIRMED;
                track_ids[w * T + lane] = conf ? id : -1;
                float *o = track_state + (w * T + lane) * OUT;
                if constexpr (D == 1) {
                    o[0] = conf ? (float)x[0] : 0.f;
                    o[1] = conf ? (float)x[1] : 0.f;
                    o[2] = conf ? (float)sqrt(P[0][0]) : 0.f;
                } else {
                    for (int k = 0; k < 4; ++k) o[k] = conf ? (float)x[k] : 0.f;
                    o[4] = conf ? (float)sqrt(P[0][0]) : 0.f;
                    o[5] = conf ? (float)sqrt(P[2][2]) : 0.f;
                }
            }
            __syncwarp();  // the next window rewrites the shared measurements
        }
        __syncwarp();  // this buffer is refilled two chunks on
    }
    if (lane < T) {
        int32_t *rw = carry_rows + lane * TRK_ROW_INTS;
        rw[0] = id; rw[1] = status; rw[2] = age; rw[3] = hits; rw[4] = misses;
        double *st = carry_state + lane * SL;
        for (int a = 0; a < NS; ++a) st[a] = x[a];
        for (int a = 0; a < NS; ++a)
            for (int b = 0; b < NS; ++b) st[NS + a * NS + b] = P[a][b];
    }
    if (lane == 0) *carry_next = next_id;
}

}  // namespace music
