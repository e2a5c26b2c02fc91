// music_warp_la.cuh - the fp64 dense linear algebra of the one-warp solvers, on small complex matrices in shared
// memory: mvdr_prep_kernel (music_estimators.cuh), iaa_kernel (music_iaa.cuh), beam_weights_kernel (music_beams.cuh),
// dml_kernel (music_dml.cuh), joint_kernel (music_wsf.cuh), crb_kernel (music_crb.cuh) and esprit2d_kernel.
//
// Matrices are row-major double2 with an explicit row stride ld (warp_cholesky: its order M; mgs2: MAXM).  A routine
// marked "warp" is called by all 32 lanes of one warp with the same arguments; a routine marked "per lane" does one
// lane's share and may be called by any subset of the lanes.  Each routine keeps one loop order, one accumulation order
// and one way of writing every product, which the CPU restatements (tools/emulate_solves_warp.py, tests/*_oracle.py)
// follow, so it must not be reordered or re-expressed.  Every caller compiles to the machine code of the loop it
// replaced, up to register names and the order of independent instructions.  That is not automatic: moving a loop into
// a routine can change which product of a * b + c * d nvcc fuses into an FMA elsewhere in the kernel, and so the
// rounding.  This is why C = Q^H R Q (dml_kernel, joint_kernel, crb_kernel) and the twice-applied projection onto the
// complement of span(Q) (joint_kernel, crb_kernel) stay written out in their kernels; compare each kernel's SASS with
// the parent's before moving another loop here.
#pragma once
#include "music_kernels.cuh"

namespace music {

// Warp: in-place right-looking Cholesky A = L L^H of the M x M Hermitian matrix A (row stride M, lower triangle read);
// L overwrites the lower triangle with a real diagonal.  Lanes map to rows for the column scaling and to entries of the
// trailing block for the update.  The caller syncs A before the call; every column ends with a __syncwarp, so L is
// visible to every lane on return.  pivot_ok(k, d) tests pivot k before its square root; every lane reads the same
// value, so the warp leaves the loop together.  Returns false on the first pivot that fails (the factor is then
// incomplete, and what was written of it is synced).
template <class PivotOk>
__device__ __forceinline__ bool warp_cholesky(double2 *A, int M, int lane, PivotOk pivot_ok)
{
    bool ok = true;
    for (int k = 0; k < M; ++k) {
        const double d = A[k * M + k].x;
        if (!pivot_ok(k, d)) { ok = false; break; }
        const double l = sqrt(d);
        __syncwarp();
        if (lane == k) A[k * M + k] = make_double2(l, 0.0);
        if (lane > k && lane < M) {
            const double2 v = A[lane * M + k];
            A[lane * M + k] = make_double2(v.x / l, v.y / l);
        }
        __syncwarp();
        const int r = M - 1 - k;  // trailing block: A[i][j] -= L[i][k] conj(L[j][k]) for k < j <= i
        for (int e = lane; e < r * r; e += 32) {
            const int i = k + 1 + e / r, j = k + 1 + e % r;
            if (j > i) continue;
            const double2 a = A[i * M + k], b = A[j * M + k];
            double2 &t = A[i * M + j];
            t.x -= a.x * b.x + a.y * b.y;
            t.y -= a.y * b.x - a.x * b.y;
        }
        __syncwarp();
    }
    return ok;
}

// Warp: Q[0 .. r-1] (row stride MAXM) = modified Gram-Schmidt, applied twice, of the vectors a_0 .. a_(r-1) in that
// order, a_l[i] = row(l, i); T (row stride MAXM, may be null) receives the upper triangle of A = Q T.  Lane i holds
// component i (row() is read by lanes i < M only).  The caller syncs whatever row() reads; every vector ends with a
// __syncwarp, so Q and T are visible to every lane on return.  No failure test: a vector in the span of the earlier
// ones gets T_ll = 0 and a non-finite q_l, and the callers test T's diagonal.
template <class Row>
__device__ __forceinline__ void mgs2(Row row, int r, int M, double2 *Q, double2 *T, int lane)
{
    for (int l = 0; l < r; ++l) {
        double2 v = make_double2(0.0, 0.0);
        if (lane < M) v = row(l, lane);
        for (int j = 0; j < l; ++j) {
            if (T && lane == 0) T[j * MAXM + l] = make_double2(0.0, 0.0);
        }
        for (int pass = 0; pass < 2; ++pass) {
            for (int j = 0; j < l; ++j) {
                const double2 q = lane < M ? Q[j * MAXM + lane] : make_double2(0.0, 0.0);
                const double2 p = cjmul(q, v);
                const double2 c = make_double2(warp_sum(p.x), warp_sum(p.y));
                v.x -= c.x * q.x - c.y * q.y;
                v.y -= c.x * q.y + c.y * q.x;
                if (T && lane == 0) { T[j * MAXM + l].x += c.x; T[j * MAXM + l].y += c.y; }
            }
        }
        const double nrm = sqrt(warp_sum(v.x * v.x + v.y * v.y));
        if (lane < M) Q[l * MAXM + lane] = make_double2(v.x / nrm, v.y / nrm);
        if (T && lane == 0) T[l * MAXM + l] = make_double2(nrm, 0.0);
        __syncwarp();
    }
}

// Per lane: the real part of the trace of the n x n matrix A (row stride ld), summed in index order, so that every lane
// that calls it gets the same value.  The caller syncs A before the call.
__device__ __forceinline__ double trace_re(const double2 *A, int ld, int n)
{
    double t = 0.0;
    for (int i = 0; i < n; ++i) t += A[i * ld + i].x;
    return t;
}

// Warp: diagonal loading of the M x M matrix A (row stride ld): delta = loading * tr(A) / M added to the diagonal, lane i
// adding to A_ii.  The caller syncs A before the call; the routine syncs before the write and after it, so the loaded A is
// visible to every lane on return.  No failure rule: a non-finite trace loads a non-finite diagonal, which the
// factorisation that follows rejects.
__device__ __forceinline__ void warp_load_diagonal(double2 *A, int ld, int M, double loading, int lane)
{
    const double delta = loading * trace_re(A, ld, M) / (double)M;
    __syncwarp();
    if (lane < M) A[lane * ld + lane].x += delta;
    __syncwarp();
}

// Per lane, lane c < n: column c of the inverse Li (row stride ldi) of the n x n lower-triangular L (row stride ldl, real
// diagonal) by forward substitution, x_c = 1 / L_cc, x_i = -(sum_{c <= q < i} L_iq x_q) / L_ii, and zeros above the
// diagonal.  Lanes c >= n do nothing.  The caller syncs L before the call and Li after it (the routine does not sync).
// No pivot test: the caller has checked L's diagonal (a Cholesky factor that passed its pivot rule).
__device__ __forceinline__ void tril_inverse(const double2 *L, int ldl, double2 *Li, int ldi, int n, int lane)
{
    if (lane < n) {
        const int c = lane;
        for (int i = 0; i < c; ++i) Li[i * ldi + c] = make_double2(0.0, 0.0);
        Li[c * ldi + c] = make_double2(1.0 / L[c * ldl + c].x, 0.0);
        for (int i = c + 1; i < n; ++i) {
            double sr = 0.0, si = 0.0;
            for (int q = c; q < i; ++q) {
                const double2 l = L[i * ldl + q], x = Li[q * ldi + c];
                sr += l.x * x.x - l.y * x.y;
                si += l.x * x.y + l.y * x.x;
            }
            const double li = L[i * ldl + i].x;
            Li[i * ldi + c] = make_double2(-sr / li, -si / li);
        }
    }
}

// Per lane, lane c < n: column c of the inverse Ti (row stride ldi) of the n x n upper-triangular T (row stride ldt, real
// diagonal) by back substitution, rows n-1 down to 0, and zeros below the diagonal.  Lanes c >= n do nothing.  The caller
// syncs T before the call and Ti after it (the routine does not sync).  No pivot test: the caller has checked T's
// diagonal (the |T_ll|^2 rule of the Gram-Schmidt that made it).
__device__ __forceinline__ void triu_inverse(const double2 *T, int ldt, double2 *Ti, int ldi, int n, int lane)
{
    if (lane < n) {
        const int c = lane;
        for (int i = n - 1; i >= 0; --i) {
            double2 s = make_double2(0.0, 0.0);
            if (i <= c) {
                s.x = i == c ? 1.0 : 0.0;
                for (int q = i + 1; q <= c; ++q) {
                    const double2 t = cmul(T[i * ldt + q], Ti[q * ldi + c]);
                    s.x -= t.x;
                    s.y -= t.y;
                }
                const double tii = T[i * ldt + i].x;
                s = make_double2(s.x / tii, s.y / tii);
            }
            Ti[i * ldi + c] = s;
        }
    }
}

// Per lane: one right-hand side through the n x n Cholesky factor L (row stride ld, lower triangle, real diagonal):
// L y = b, then L^H z = y.  The vectors are reached through accessors so that each caller keeps its own layout: b(k)
// returns b_k by value, y(k) and z(k) return references to y_k and z_k (y may be b's storage, z may be y's).  The lane
// that owns a right-hand side owns its y and z, so the routine does not sync; the caller syncs L before the call and z
// after it when other lanes read z.  No pivot test: L passed the pivot rule of its factorisation.
template <class Rhs, class Fwd, class Sol>
__device__ __forceinline__ void cholesky_solve(const double2 *L, int ld, int n, Rhs b, Fwd y, Sol z)
{
    for (int k = 0; k < n; ++k) {  // L y = b
        double sr = b(k).x, si = b(k).y;
        for (int q = 0; q < k; ++q) {
            const double2 l = L[k * ld + q], v = y(q);
            sr -= l.x * v.x - l.y * v.y;
            si -= l.x * v.y + l.y * v.x;
        }
        const double lk = L[k * ld + k].x;
        y(k) = make_double2(sr / lk, si / lk);
    }
    for (int k = n - 1; k >= 0; --k) {  // L^H z = y
        double sr = y(k).x, si = y(k).y;
        for (int q = k + 1; q < n; ++q) {
            const double2 l = L[q * ld + k], v = z(q);  // conj(L[q][k]) z_q
            sr -= l.x * v.x + l.y * v.y;
            si -= l.x * v.y - l.y * v.x;
        }
        const double lk = L[k * ld + k].x;
        z(k) = make_double2(sr / lk, si / lk);
    }
}

// Per lane, slot l < d: the least-squares level p_l = (Ti C Ti^H)_ll = sum_{a, b >= l} Ti_la C_ab conj(Ti_lb) of the
// d x d matrix C (row stride ldc) and the upper-triangular Ti (row stride ldt), the inner sum over b first.  The caller
// syncs C and Ti before the call (the routine does not sync).  No failure rule.
__device__ __forceinline__ double slot_level(const double2 *Ti, int ldt, const double2 *C, int ldc, int d, int l)
{
    double p = 0.0;
    for (int a = l; a < d; ++a) {
        double2 y = make_double2(0.0, 0.0);
        for (int b = l; b < d; ++b) {
            const double2 t = cmul(C[a * ldc + b], make_double2(Ti[l * ldt + b].x, -Ti[l * ldt + b].y));
            y.x += t.x;
            y.y += t.y;
        }
        p += cmul(Ti[l * ldt + a], y).x;
    }
    return p;
}

}  // namespace music
