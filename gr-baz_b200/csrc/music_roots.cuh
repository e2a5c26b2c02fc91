// music_roots.cuh - root-MUSIC for uniform linear arrays (opt-in peak mode MUSIC_B200_PEAKS_ROOTS).
//
// On a ULA p_m = p_0 + m s the steering vector is a_m = e^{-j 2 pi p_0.u / lambda} z0^m with
// z0 = exp(-j 2 pi (s.u) / lambda), so the MUSIC denominator is a Laurent polynomial in z0:
//     D = a^H G G^H a = sum_l c_l z0^l,   c_l = sum_{j - i = l} (G G^H)_ij,   l = -(M-1) .. M-1,
// and Q(z) = sum_l c_l z^(l + M - 1) (degree 2M - 2) has the directions as roots near the unit circle.  Each window's
// roots come from an Aberth-Ehrlich iteration; the full definition (selection, angles, levels, bins) is in
// include/music_b200.h and is restated by tests/root_music_oracle.py.
//
// One warp per window, lane r <-> root r (2M - 2 <= 30).  Everything is fp64.
#pragma once
#include "music_kernels.cuh"
#include "music_refine.cuh"
#include "music_steer.cuh"

namespace music {

// The ULA parameters of a geometric table (set_geometry), passed by value like RefineGeom.
struct UlaGeom {
    double p0[2];  // first element, metres
    double s[2];   // element step (p_{M-1} - p_0) / (M - 1), metres
    int ula;       // 1: the positions form a ULA with |s| <= lambda / 2 (the root mode's condition)
};

constexpr int ROOTS_WARPS = 4;
constexpr int ROOTS_MAX_IT = 100;
constexpr double ROOTS_EPS = 2.220446049250313e-16;  // 2^-52
constexpr double ROOTS_STOP = 4.0 * ROOTS_EPS;        // a lane stops once its correction is <= 4 ulps of |z|,
constexpr double ROOTS_BACK = 8.0;                    // or once |Q(z)| <= ROOTS_BACK P eps sum_k |b_k| |z|^k
constexpr double ROOTS_MERGE = 1e-6;                  // two roots this close (relative) are one double root

__device__ __forceinline__ double2 cdiv(double2 a, double2 b)
{
    const double r = 1.0 / (b.x * b.x + b.y * b.y);
    return make_double2((a.x * b.x + a.y * b.y) * r, (a.y * b.x - a.x * b.y) * r);
}
__device__ __forceinline__ double2 shfl2(double2 v, int src)
{
    return make_double2(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src));
}

// The direction of z0 = z on the ULA (shared by the gridless ULA modes, ROOTS and ESPRIT): cos(t - alpha) =
// -arg(z) lambda / (2 pi |s|); the lower of alpha +- psi in [0, 360) degrees
__device__ __forceinline__ double ula_direction(double2 z, const RefineGeom &geo, const UlaGeom &ula)
{
    const double sabs = hypot(ula.s[0], ula.s[1]);
    double cpsi = -atan2(z.y, z.x) * geo.lambda / (STEER_TWO_PI * sabs);
    cpsi = fmin(1.0, fmax(-1.0, cpsi));
    const double psi = acos(cpsi), alpha = atan2(ula.s[1], ula.s[0]);
    double a1 = fmod((alpha + psi) * REFINE_RAD2DEG, 360.0), a2 = fmod((alpha - psi) * REFINE_RAD2DEG, 360.0);
    if (a1 < 0.0) a1 += 360.0;
    if (a2 < 0.0) a2 += 360.0;
    return fmin(a1, a2);
}

// A filled slot of a gridless ULA mode: the angle t* (float cast, 360 -> 0), level 1 / D(t*) and the nearest grid bin
__device__ __forceinline__ void ula_store_slot(const PeakOut &out, size_t o, double tdeg, double D, int K)
{
    float ang = (float)tdeg;
    if (ang >= 360.0f || ang == 0.0f) ang = 0.0f;
    out.angles[o] = ang;
    if (out.levels) out.levels[o] = (float)(1.0 / D);
    int b = (int)floor(tdeg * (double)K / 360.0 + 0.5);
    if (b >= K) b -= K;
    peak_store_bin(out, o, b);
}

// Vt: per window M * M complex doubles, eigenvector j contiguous, ascending eigenvalues; counts (may be null): the
// per-window source count d (else d = n); the noise subspace is eigenvectors 0 .. M - d - 1, as in the scan.
__global__ void __launch_bounds__(ROOTS_WARPS * 32) roots_kernel(const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                                int M, int n, int K, int W, const RefineGeom geo, const UlaGeom ula,
                                                                PeakOut out)
{
    const int w = blockIdx.x * ROOTS_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (w >= W) return;
    const int d = counts ? counts[w] : n;
    const int p = M - d;
    const double2 *G = reinterpret_cast<const double2 *>(Vt) + (size_t)w * M * M;

    // lane l < M: c_l = sum_j sum_i g_j[i] conj(g_j[i + l]); c_{-l} = conj(c_l)
    double2 c = make_double2(0.0, 0.0);
    if (lane < M) {
        for (int j = 0; j < p; ++j)
            for (int i = 0; i + lane < M; ++i) {
                const double2 a = G[j * M + i], b = G[j * M + i + lane];
                c.x += a.x * b.x + a.y * b.y;
                c.y += a.y * b.x - a.x * b.y;
            }
    }
    const bool finite = __all_sync(0xffffffffu, lane >= M || (isfinite(c.x) && isfinite(c.y)));
    // t: outermost coefficient pairs c_{+-(M-1)}, c_{+-(M-2)}, .. that are exactly zero (each a root at 0 and at infinity)
    const unsigned nz = __ballot_sync(0xffffffffu, lane < M && (c.x != 0.0 || c.y != 0.0));
    const int t = nz ? M - 1 - (31 - __clz(nz)) : M - 1;
    const int P = 2 * (M - 1 - t);  // degree of the reduced polynomial sum_k b_k z^k, b_k = c_{k - (M - 1 - t)}
    const int H = M - 1 - t;

    double2 z = make_double2(0.0, 0.0);
    bool ok = finite && d > 0 && P > 0;
    if (ok) {
        // starting points on the circles of the Newton polygon (Bini): the upper convex hull of (k, log2 |b_k|), with
        // |b_k| = |c_{|k - H|}|, every lane building the same hull; the roots of hull segment [i, j) start on the circle
        // of radius (|b_i| / |b_j|)^(1 / (j - i)), so that roots decades away from the unit circle start near it
        const double lgc = (lane < M && (c.x != 0.0 || c.y != 0.0)) ? log2(hypot(c.x, c.y)) : -INFINITY;
        int hull[32], nh = 1;
        hull[0] = 0;
        for (int k = 1; k <= P; ++k) {
            const double lk = __shfl_sync(0xffffffffu, lgc, k >= H ? k - H : H - k);
            if (lk == -INFINITY) continue;
            while (nh >= 2) {
                const int i = hull[nh - 2], j = hull[nh - 1];
                const double li = __shfl_sync(0xffffffffu, lgc, i >= H ? i - H : H - i);
                const double lj = __shfl_sync(0xffffffffu, lgc, j >= H ? j - H : H - j);
                if ((lj - li) * (k - i) <= (lk - li) * (j - i)) --nh;  // j on or below the chord i -> k
                else break;
            }
            hull[nh++] = k;
        }
        int si = 0;
        while (si + 2 < nh && hull[si + 1] <= lane) ++si;
        const int i0 = hull[si], j0 = hull[si + 1];
        const double li = __shfl_sync(0xffffffffu, lgc, i0 >= H ? i0 - H : H - i0);
        const double lj = __shfl_sync(0xffffffffu, lgc, j0 >= H ? j0 - H : H - j0);
        const double u = exp2((li - lj) / (j0 - i0));
        double sn, cs;
        sincospi(2.0 * (lane - i0) / (j0 - i0) + 2.0 * i0 / P + 0.5 / P, &sn, &cs);
        z = make_double2(u * cs, u * sn);
        bool done = lane >= P, conv = false;
        for (int it = 0; it < ROOTS_MAX_IT; ++it) {
            // Horner for Q and Q' (coefficients broadcast from the lanes that built them); outside the unit circle for
            // R(w) = w^P Q(1 / w) and R' at w = 1 / z instead, so that no power of z overflows.  acc = sum_k |b_k| |w|^k
            const bool outside = z.x * z.x + z.y * z.y > 1.0;
            const double2 w = outside ? cdiv(make_double2(1.0, 0.0), z) : z;
            const double aw = hypot(w.x, w.y);
            double2 q = shfl2(c, H), dq = make_double2(0.0, 0.0);  // b_0 = conj(c_H), b_P = c_H: equal modulus
            if (outside) q.y = -q.y;
            double acc = hypot(q.x, q.y);
            for (int k = 1; k <= P; ++k) {
                const int l = (outside ? k : P - k) - H;
                double2 b = shfl2(c, l >= 0 ? l : -l);
                if (l < 0) b.y = -b.y;
                dq = cmul(dq, w);
                dq.x += q.x; dq.y += q.y;
                q = cmul(q, w);
                q.x += b.x; q.y += b.y;
                acc = acc * aw + hypot(b.x, b.y);
            }
            // a lane whose residual is at rounding level holds an exact root of a polynomial within that rounding
            if (hypot(q.x, q.y) <= ROOTS_BACK * P * ROOTS_EPS * acc) done = true;
            // Aberth term sum_{s != r} 1 / (z_r - z_s)
            double2 S = make_double2(0.0, 0.0);
            for (int s = 0; s < P; ++s) {
                const double2 zs = shfl2(z, s);
                if (s != lane) {
                    const double dx = z.x - zs.x, dy = z.y - zs.y, r = 1.0 / (dx * dx + dy * dy);
                    S.x += dx * r;
                    S.y -= dy * r;
                }
            }
            // Aberth correction N / (1 - N S) with N = Q / Q', as one division: Q / (Q' - Q S); outside, N = z R / (P R -
            // w R'), so z R / (P R - w R' - z R S)
            double2 wc;
            if (outside) {
                const double2 num = cmul(z, q), nS = cmul(num, S), wd = cmul(w, dq);
                wc = cdiv(num, make_double2(P * q.x - wd.x - nS.x, P * q.y - wd.y - nS.y));
            } else {
                const double2 qS = cmul(q, S);
                wc = cdiv(q, make_double2(dq.x - qS.x, dq.y - qS.y));
            }
            if (!done) {  // a converged lane stays put
                z.x -= wc.x;
                z.y -= wc.y;
                done = wc.x * wc.x + wc.y * wc.y <= ROOTS_STOP * ROOTS_STOP * (z.x * z.x + z.y * z.y);
            }
            if (__all_sync(0xffffffffu, done)) {
                conv = true;
                break;
            }
        }
        // a window whose iteration has not converged in ROOTS_MAX_IT steps reports no peaks
        ok = conv && __all_sync(0xffffffffu, lane >= P || (isfinite(z.x) && isfinite(z.y)));
    }

    // a double root on the unit circle (the two approximants are each other's nearest root, closer than
    // ROOTS_MERGE |z|) counts once: both move to the midpoint, the lower lane keeps it with modulus 1
    double key = hypot(z.x, z.y);
    bool dup = false;
    if (ok) {
        int nn = -1;
        double best = 0.0;
        for (int s = 0; s < P; ++s) {
            const double2 zs = shfl2(z, s);
            const double dd = hypot(z.x - zs.x, z.y - zs.y);
            if (s != lane && (nn < 0 || dd < best)) { nn = s; best = dd; }
        }
        const int src = nn < 0 ? 0 : nn;
        const int back = __shfl_sync(0xffffffffu, nn, src);
        const double2 zn = shfl2(z, src);
        const double keyn = __shfl_sync(0xffffffffu, key, src);
        if (lane < P && back == lane && best <= ROOTS_MERGE * fmax(key, keyn)) {
            z = make_double2(0.5 * (z.x + zn.x), 0.5 * (z.y + zn.y));
            key = 1.0;
            dup = lane > nn;
        }
    }

    const double tdeg = ula_direction(z, geo, ula);

    // keep the M - 1 - t inside roots (ascending modulus, a double root's second copy after every other root of equal
    // modulus, then lane); fill slots in descending modulus, ties to the lower angle
    int r1 = 0, r2 = 0;
    for (int s = 0; s < P; ++s) {
        const double ks = __shfl_sync(0xffffffffu, key, s);
        const bool ds = __shfl_sync(0xffffffffu, dup, s);
        if (ks < key || (ks == key && (ds < dup || (ds == dup && s < lane)))) ++r1;
    }
    const bool kept = ok && lane < P && r1 < H;
    for (int s = 0; s < P; ++s) {
        const bool ks_kept = __shfl_sync(0xffffffffu, kept, s);
        const double ks = __shfl_sync(0xffffffffu, key, s);
        const double ts = __shfl_sync(0xffffffffu, tdeg, s);
        if (ks_kept && (ks > key || (ks == key && (ts < tdeg || (ts == tdeg && s < lane))))) ++r2;
    }
    const int f = ok ? min(d, H) : 0;  // filled slots
    if (kept && r2 < f) {
        const size_t o = (size_t)w * n + r2;
        double D, D1, D2;
        refine_eval(geo, G, M, p, tdeg * STEER_DEG2RAD, &D, &D1, &D2);
        ula_store_slot(out, o, tdeg, D, K);
    }
    if (lane >= f && lane < n) peak_write(out, (size_t)w * n + lane, -1, 0.0, K);
}

}  // namespace music
