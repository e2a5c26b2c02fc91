// music_sources.cuh - per-window estimate of the number of sources (opt-in, music_b200_set_source_rule).
//
// The block is created with a fixed number of sources n.  When fewer emitters are on the air the spare slots report
// the flank of the strongest peak or a noise bump; when more are present the noise subspace holds signal and every
// peak is biased.  The information-theoretic criteria of Wax and Kailath (IEEE Trans. ASSP 33(2), 1985) estimate the
// model order from the eigenvalues alone, which the unfused path already holds for every window (ws.ev, ascending).
//
// Definition (restated literally by tests/source_count_oracle.py::estimate_source_count): with the ascending fp64
// eigenvalues l_0 <= ... <= l_{M-1} and N snapshots, for d = 0 .. nmax and p = M - d, summing i = 0 .. p-1 in
// ascending order
//     S = sum l_i,  G = sum log l_i,  L(d) = N (p log(S / p) - G),
//     MDL(d) = L(d) + 1/2 d (2M - d) log N,     AIC(d) = 2 L(d) + 2 d (2M - d);
// the count is the smallest d with the minimum criterion (NaN never wins), and 0 when l_0 <= 0 or any eigenvalue is
// not finite.  One thread per window; the sums are prefix sums, so every p reuses the previous one's in the same order.
#pragma once
#include "music_kernels.cuh"

namespace music {

constexpr int SOURCES_FIXED = 0, SOURCES_MDL = 1, SOURCES_AIC = 2;  // = MUSIC_B200_SOURCES_*

// counts[w] (workspace) and, when given, counts_out[w] (the caller's) for the W windows of ev ([W][M], ascending)
__global__ void __launch_bounds__(128) source_count_kernel(const double *__restrict__ ev, int M, int nmax, int N, int rule, int W,
                                                           int32_t *__restrict__ counts, int32_t *__restrict__ counts_out)
{
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    const double *lam = ev + (size_t)w * M;
    bool ok = lam[0] > 0.0;
    for (int i = 0; i < M; ++i) ok = ok && isfinite(lam[i]);
    int best = 0;
    if (ok) {
        // explicit roundings: no contraction into FMAs, so that each criterion is the literal expression above
        const double Nd = (double)N, logN = log(Nd);
        double S = 0.0, G = 0.0, bestc = 0.0;
        bool have = false;
        for (int p = 1; p <= M; ++p) {  // p ascending = d descending: "<=" keeps the smallest d among equal minima
            S = __dadd_rn(S, lam[p - 1]);
            G = __dadd_rn(G, log(lam[p - 1]));
            const int d = M - p;
            if (d > nmax) continue;
            const double L = __dmul_rn(Nd, __dsub_rn(__dmul_rn((double)p, log(S / (double)p)), G));
            const double pen = (double)(d * (2 * M - d));
            const double c = rule == SOURCES_MDL ? __dadd_rn(L, __dmul_rn(0.5 * pen, logN)) : __dadd_rn(2.0 * L, 2.0 * pen);
            if (have ? (c <= bestc) : !isnan(c)) {
                best = d;
                bestc = c;
                have = true;
            }
        }
    }
    counts[w] = best;
    if (counts_out) counts_out[w] = best;
}

// a FIXED handle asked for counts: every window has the handle's n
__global__ void fill_counts_kernel(int32_t *__restrict__ counts, int n, int W)
{
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w < W) counts[w] = n;
}

}  // namespace music
