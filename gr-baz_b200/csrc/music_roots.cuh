// music_roots.cuh - root-MUSIC for uniform linear arrays (opt-in peak mode MUSIC_B200_PEAKS_ROOTS).
//
// On a ULA p_m = p_0 + m s the steering vector is a_m = e^{-j 2 pi p_0.u / lambda} z0^m with
// z0 = exp(-j 2 pi (s.u) / lambda), so the MUSIC denominator is a Laurent polynomial in z0:
//     D = a^H G G^H a = sum_l c_l z0^l,   c_l = sum_{j - i = l} (G G^H)_ij,   l = -(M-1) .. M-1,
// and Q(z) = sum_l c_l z^(l + M - 1) (degree 2M - 2) has the directions as roots near the unit circle.  Each window's
// roots come from an Aberth-Ehrlich iteration; the full definition (selection, angles, levels, bins) is in
// include/music_b200.h and is restated by tests/root_music_oracle.py.
//
// The root finder (roots_solve) is shared with the manifold mode (music_manifold.cuh), which differs only in how it
// forms the coefficients and turns a root into an angle.  One CTA of one warp per window, thread r <-> root r
// (2M - 2 <= 30).  Everything is fp64.
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

// ---- the root finder of ROOTS and MANIFOLD ----------------------------------------------------------------------------
//
// Q(z) = sum_{l = -L .. L} c_l z^(l + L), c_{-l} = conj(c_l), solved by one CTA per window, thread r <-> root r, with
// the approximants in shared memory.  MAXL bounds L (P = 2L <= 2 MAXL roots), so each kernel sizes the state for its own
// largest polynomial.

// One window's root-finder state
template <int MAXL> struct RootsShared {
    double2 cf[MAXL + 1];   // c_0 .. c_L
    double lg[MAXL + 1];    // log2 |c_l| (-inf for 0)
    double ac[MAXL + 1];    // |c_l|
    int hull[2 * MAXL + 1], nh;
    double2 zs[2 * MAXL];   // the current approximants
    double keys[2 * MAXL], tds[2 * MAXL];
    int nns[2 * MAXL];
    unsigned char dups[2 * MAXL], kepts[2 * MAXL];
};

// thread l <= L hands over c_l
template <int MAXL> __device__ __forceinline__ void roots_set_coeff(RootsShared<MAXL> &sh, int l, double2 c)
{
    sh.cf[l] = c;
    sh.ac[l] = hypot(c.x, c.y);
    sh.lg[l] = (c.x != 0.0 || c.y != 0.0) ? log2(hypot(c.x, c.y)) : -INFINITY;
}

// A thread's root after roots_solve: its direction and the slot it fills (-1: none); the window fills slots 0 .. f - 1
struct RootSlot {
    double2 z;
    double tdeg;
    int slot, f;
};

// Called by every thread of the CTA (at least max(P, n) of them) once threads 0 .. L have called roots_set_coeff; d is
// the window's source count and dir(z) the direction of a root in degrees, which breaks slot ties.
template <int MAXL, class Dir> __device__ __forceinline__ RootSlot roots_solve(RootsShared<MAXL> &sh, int L, int d, Dir dir)
{
    __syncthreads();
    const int r = threadIdx.x;
    // t: outermost pairs c_{+-L}, c_{+-(L-1)}, .. that are exactly zero (each a root at 0 and at infinity)
    bool finite = true;
    int t = L;
    for (int l = 0; l <= L; ++l) {
        const double2 c = sh.cf[l];
        finite = finite && isfinite(c.x) && isfinite(c.y);
        if (c.x != 0.0 || c.y != 0.0) t = L - l;
    }
    const int H = L - t, P = 2 * H;  // Q reduced to sum_k b_k z^k, k = 0 .. P, b_k = c_{k - H}
    bool ok = finite && d > 0 && P > 0;  // uniform over the CTA
    double2 z = make_double2(0.0, 0.0);
    if (ok) {
        // starting points on the circles of the Newton polygon (Bini): the upper convex hull of (k, log2 |b_k|), with
        // |b_k| = |c_{|k - H|}|, built by one thread; the roots of hull segment [i, j) start on the circle of radius
        // (|b_i| / |b_j|)^(1 / (j - i)), so that roots decades away from the unit circle start near it
        if (r == 0) {
            int nh = 1;
            sh.hull[0] = 0;
            for (int k = 1; k <= P; ++k) {
                const double lk = sh.lg[k >= H ? k - H : H - k];
                if (lk == -INFINITY) continue;
                while (nh >= 2) {
                    const int i = sh.hull[nh - 2], j = sh.hull[nh - 1];
                    const double li = sh.lg[i >= H ? i - H : H - i], lj = sh.lg[j >= H ? j - H : H - j];
                    if ((lj - li) * (k - i) <= (lk - li) * (j - i)) --nh;  // j on or below the chord i -> k
                    else break;
                }
                sh.hull[nh++] = k;
            }
            sh.nh = nh;
        }
        __syncthreads();
        const int nh = sh.nh;
        int si = 0;
        while (si + 2 < nh && sh.hull[si + 1] <= r) ++si;
        const int i0 = sh.hull[si], j0 = sh.hull[si + 1];
        const double li = sh.lg[i0 >= H ? i0 - H : H - i0], lj = sh.lg[j0 >= H ? j0 - H : H - j0];
        const double u = exp2((li - lj) / (j0 - i0));
        double sn, cs;
        sincospi(2.0 * (r - i0) / (j0 - i0) + 2.0 * i0 / P + 0.5 / P, &sn, &cs);
        z = make_double2(u * cs, u * sn);
        if (r < P) sh.zs[r] = z;
        __syncthreads();
        bool done = r >= P, conv = false;
        for (int it = 0; it < ROOTS_MAX_IT; ++it) {
            double2 wc = make_double2(0.0, 0.0);
            if (!done) {  // a converged root stays put, so only the others evaluate
                // Horner for Q and Q'; outside the unit circle for R(w) = w^P Q(1 / w) and R' at w = 1 / z instead, so
                // that no power of z overflows.  acc = sum_k |b_k| |w|^k
                const bool outside = z.x * z.x + z.y * z.y > 1.0;
                const double2 w1 = outside ? cdiv(make_double2(1.0, 0.0), z) : z;
                const double aw = hypot(w1.x, w1.y);
                double2 q = sh.cf[H], dq = make_double2(0.0, 0.0);  // b_0 = conj(c_H), b_P = c_H: equal modulus
                if (outside) q.y = -q.y;
                double acc = sh.ac[H];
                for (int k = 1; k <= P; ++k) {
                    const int l = (outside ? k : P - k) - H;
                    double2 b = sh.cf[l >= 0 ? l : -l];
                    if (l < 0) b.y = -b.y;
                    dq = cmul(dq, w1);
                    dq.x += q.x; dq.y += q.y;
                    q = cmul(q, w1);
                    q.x += b.x; q.y += b.y;
                    acc = acc * aw + sh.ac[l >= 0 ? l : -l];
                }
                // a root whose residual is at rounding level is an exact root of a polynomial within that rounding
                if (hypot(q.x, q.y) <= ROOTS_BACK * P * ROOTS_EPS * acc) done = true;
                // Aberth term sum_{s != r} 1 / (z_r - z_s)
                double2 S = make_double2(0.0, 0.0);
                for (int s = 0; s < P; ++s) {
                    const double2 zz = sh.zs[s];
                    if (s != r) {
                        const double dx = z.x - zz.x, dy = z.y - zz.y, rr = 1.0 / (dx * dx + dy * dy);
                        S.x += dx * rr;
                        S.y -= dy * rr;
                    }
                }
                // Aberth correction N / (1 - N S) with N = Q / Q', as one division: Q / (Q' - Q S); outside, N = z R /
                // (P R - w R'), so z R / (P R - w R' - z R S)
                if (outside) {
                    const double2 num = cmul(z, q), nS = cmul(num, S), wd = cmul(w1, dq);
                    wc = cdiv(num, make_double2(P * q.x - wd.x - nS.x, P * q.y - wd.y - nS.y));
                } else {
                    const double2 qS = cmul(q, S);
                    wc = cdiv(q, make_double2(dq.x - qS.x, dq.y - qS.y));
                }
            }
            __syncthreads();  // every thread has read this step's approximants
            if (!done) {
                z.x -= wc.x;
                z.y -= wc.y;
                done = wc.x * wc.x + wc.y * wc.y <= ROOTS_STOP * ROOTS_STOP * (z.x * z.x + z.y * z.y);
                sh.zs[r] = z;
            }
            if (__syncthreads_and(done)) {
                conv = true;
                break;
            }
        }
        // a window whose iteration has not converged in ROOTS_MAX_IT steps reports no peaks
        ok = __syncthreads_and(conv && (r >= P || (isfinite(z.x) && isfinite(z.y))));
    }

    // a double root on the unit circle (the two approximants are each other's nearest root, closer than
    // ROOTS_MERGE |z|) counts once: both move to the midpoint, the lower index keeps it with modulus 1
    double key = hypot(z.x, z.y);
    bool dup = false;
    if (ok) {
        int nn = -1;
        double best = 0.0;
        if (r < P) {
            for (int s = 0; s < P; ++s) {
                const double2 zz = sh.zs[s];
                const double dd = hypot(z.x - zz.x, z.y - zz.y);
                if (s != r && (nn < 0 || dd < best)) { nn = s; best = dd; }
            }
            sh.nns[r] = nn;
            sh.keys[r] = key;
        }
        __syncthreads();
        if (r < P && nn >= 0 && sh.nns[nn] == r && best <= ROOTS_MERGE * fmax(key, sh.keys[nn])) {
            const double2 zn = sh.zs[nn];
            z = make_double2(0.5 * (z.x + zn.x), 0.5 * (z.y + zn.y));
            key = 1.0;
            dup = r > nn;
        }
        __syncthreads();  // zs and keys are read above before they are rewritten below
    }
    const double tdeg = dir(z);
    if (r < P) {
        sh.keys[r] = key;
        sh.dups[r] = dup;
        sh.tds[r] = tdeg;
    }
    __syncthreads();

    // keep the H inside roots (ascending modulus, a double root's second copy after every other root of equal modulus,
    // then index); fill slots in descending modulus, ties to the lower angle
    int r1 = 0, r2 = 0;
    for (int s = 0; s < P; ++s) {
        const double ks = sh.keys[s];
        const bool ds = sh.dups[s];
        if (ks < key || (ks == key && (ds < dup || (ds == dup && s < r)))) ++r1;
    }
    const bool kept = ok && r < P && r1 < H;
    if (r < P) sh.kepts[r] = kept;
    __syncthreads();
    for (int s = 0; s < P; ++s) {
        const double ks = sh.keys[s], ts = sh.tds[s];
        if (sh.kepts[s] && (ks > key || (ks == key && (ts < tdeg || (ts == tdeg && s < r))))) ++r2;
    }
    const int f = ok ? min(d, H) : 0;  // filled slots
    return {z, tdeg, kept && r2 < f ? r2 : -1, f};
}

// ---- ROOTS: one warp per window -------------------------------------------------------------------------------------

constexpr int ROOTS_THREADS = 32;  // P = 2M - 2 <= 30 roots, n < M slots

// Vt: per window M * M complex doubles, eigenvector j contiguous, ascending eigenvalues; counts (may be null): the
// per-window source count d (else d = n); the noise subspace is eigenvectors 0 .. M - d - 1, as in the scan.  Launched
// with ROOTS_THREADS threads per CTA, one CTA per window.
__global__ void __launch_bounds__(ROOTS_THREADS) roots_kernel(const double *__restrict__ Vt, const int32_t *__restrict__ counts,
                                                              int M, int n, int K, const RefineGeom geo, const UlaGeom ula,
                                                              PeakOut out)
{
    __shared__ RootsShared<MAXM - 1> sh;
    const int w = blockIdx.x, r = threadIdx.x;
    const int d = counts ? counts[w] : n;
    const int p = M - d;
    const double2 *G = reinterpret_cast<const double2 *>(Vt) + (size_t)w * M * M;

    // thread l < M: c_l = sum_j sum_i g_j[i] conj(g_j[i + l]); c_{-l} = conj(c_l)
    if (r < M) {
        double2 c = make_double2(0.0, 0.0);
        for (int j = 0; j < p; ++j)
            for (int i = 0; i + r < M; ++i) {
                const double2 a = G[j * M + i], b = G[j * M + i + r];
                c.x += a.x * b.x + a.y * b.y;
                c.y += a.y * b.x - a.x * b.y;
            }
        roots_set_coeff(sh, r, c);
    }
    const RootSlot rs = roots_solve(sh, M - 1, d, [&](double2 z) { return ula_direction(z, geo, ula); });
    if (rs.slot >= 0) {
        double D, D1, D2;
        refine_eval(geo, G, M, p, rs.tdeg * STEER_DEG2RAD, &D, &D1, &D2);
        ula_store_slot(out, (size_t)w * n + rs.slot, rs.tdeg, D, K);
    }
    if (r >= rs.f && r < n) peak_write(out, (size_t)w * n + r, -1, 0.0, K);
}

}  // namespace music
