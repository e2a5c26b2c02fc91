/*
 * music_b200.h - C ABI of the H100-native (sm_90a) MUSIC direction-of-arrival hot path.
 *
 * This is the drop-in boundary for gr-baz's `baz_music_doa` block: everything that
 * /root/reference/lib/baz_music_doa.cc does per window inside work() (lines 72-161) runs
 * behind these entry points as hand-written CUDA; the GNU Radio block (lib/baz_music_doa.cc
 * in this repo), the Python helper and the bench harness are the only callers.
 *
 * Plain C types only: pointers and sizes, no C++/torch types, no exceptions.  Every function
 * returns 0 on success or a negative MUSIC_B200_E* code; the message is available from
 * music_b200_last_error().  There is NO CPU fallback: create() fails if the device is not a
 * compute-capability 9.0 (sm_90, H100) GPU.
 *
 * Data layouts (identical to the reference's GNU Radio item layouts):
 *   input window : nsamples complex64 (re, im floats), antennas sample-interleaved,
 *                  x(r, c) = in[c*m + r]            (reference lib/baz_music_doa.cc:37, :82-84)
 *   array response table : [resolution][m] complex64  (reference lib/baz_music_doa.h:32-33,
 *                  marshalled by swig/baz_swig.i:564)
 *   angles / levels : n floats per window             (reference lib/baz_music_doa.cc:38, :146-155)
 *   spectrum        : resolution floats per window    (reference lib/baz_music_doa.cc:38, :120-121)
 *   bins            : n int32 per window - the integer peak-bin index k behind each angle
 *                     (angle = (float)(k*360.0/resolution), :134); -1 where the reference
 *                     would leave its (0, 0) initial pair in place (:95).
 */
#ifndef MUSIC_B200_H
#define MUSIC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MUSIC_B200_OK 0
#define MUSIC_B200_EINVAL (-1)   /* bad argument (same conditions as the reference's ctor asserts) */
#define MUSIC_B200_ECUDA (-2)    /* CUDA runtime error */
#define MUSIC_B200_ENODEVICE (-3) /* no sm_90 device / device index out of range */
#define MUSIC_B200_ENOMEM (-4)

#define MUSIC_B200_MAX_M 16 /* antennas supported by this build */

typedef struct music_b200 music_b200;

/* ABI version of this header (bumped on any signature change). */
int music_b200_version(void);  /* 2: multi-device handles, fused bins all-gather */

/*
 * Replaces baz_make_music_doa() + the constructor
 * (/root/reference/lib/baz_music_doa.cc:29-53, lib/baz_music_doa.h:36-43).
 * Argument checks are the reference's asserts (:45-50) made real, plus 1 <= n < m
 * (m == n underflows eigvec.cols(0, m-n-1) at :93) and m <= MUSIC_B200_MAX_M.
 * table_c64: [resolution][m] interleaved (re, im) floats, copied (the block owns its table,
 * :42).  device: CUDA device ordinal.
 */
int music_b200_create(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples,
                      uint32_t resolution, const float *table_c64, int device);

/*
 * The same block spread over `ndev` GPUs of one node (SURVEY.md section 8e: windows are independent, so they shard
 * round-robin, window w -> devices[w mod ndev], and every device keeps a full copy of the array response).  The handle
 * behaves like one from music_b200_create():
 *   process_host()     deals the call's windows round-robin at WINDOW granularity to the devices (strided 2-D copies,
 *                      one PCIe link per device, no interleaving pass on the host) and returns the outputs in stream
 *                      order - one work() call of one flowgraph block uses every GPU and every PCIe link;
 *   set_table() / set_geometry() / set_peak_mode()  apply to every device;
 *   process_device()   goes to the device the input pointer lives on;  process_device_sharded() (below) runs all of them;
 *   planar, reducer, stage-timing entries are served by devices[0].
 * lib/baz_music_doa.cc picks the devices from the environment variable BAZ_MUSIC_DOA_DEVICES ("0,1,2,3" or "all").
 */
int music_b200_create_multi(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution,
                            const float *table_c64, const int *devices, int ndev);
int music_b200_device_count(const music_b200 *h);

/*
 * Device-resident, sharded form of work() on a multi-device handle: device g (= devices[g] of create_multi) holds in
 * d_in_c64[g] the windows w = i * G + g of a stream of nwindows_total windows (i = local index, compacted) and receives
 * their angles / levels in d_angles[g] / d_levels[g] ([ceil((nwindows_total - g) / G)][n], levels may be NULL).
 * d_bins_all (may be NULL): G device arrays, d_bins_all[p] on device p, each int32 [nwindows_total][n] in STREAM order.
 * The all-gather of the peak bins is fused into the scan epilogue: the kernel of shard g stores bin w into
 * d_bins_all[p][w] for every p over NVLink (peer-mapped memory; no NCCL, no separate collective kernel), so when the
 * G streams have finished every device holds all peaks.  streams (may be NULL): one cudaStream_t per device.
 */
int music_b200_process_device_sharded(music_b200 *h, const float *const *d_in_c64, uint32_t nwindows_total, float *const *d_angles,
                                      float *const *d_levels, int32_t *const *d_bins_all, void *const *streams);

/*
 * The same fused all-gather when every GPU belongs to its own PROCESS (one rank per GPU, e.g. under torchrun): each rank
 *   1. gather_create(h, total_windows, handles)  allocates its stream-ordered gather buffer (int32 [total_windows][n]) and
 *      epoch flags and returns their two 64-byte CUDA IPC handles;
 *   2. exchanges the handles with the other ranks by any means (bench.py: one all_gather of 128 bytes at start-up);
 *   3. gather_attach(h, nranks, rank, all_handles)  maps the peers' buffers.
 * From then on every process_device() call of this handle treats its nwindows windows as the shard w = i * nranks + rank
 * and its scan epilogue stores the peak bins into every rank's gather buffer; the last CTA raises this rank's epoch flag
 * at every peer.  gather_wait(h, stream) enqueues a one-warp kernel that returns when all ranks' flags have reached this
 * rank's call count, i.e. when gather_buffer(h) holds every rank's bins of the latest call (all ranks must make the same
 * sequence of calls, as with any collective).  ncclAllGather stays the reference implementation the tests compare with.
 */
int music_b200_gather_create(music_b200 *h, uint32_t total_windows, unsigned char *ipc_handles /* [2][64] */);
int music_b200_gather_attach(music_b200 *h, int nranks, int rank, const unsigned char *all_handles /* [nranks][2][64] */);
int music_b200_gather_wait(music_b200 *h, void *stream);
const int32_t *music_b200_gather_buffer(const music_b200 *h);
int music_b200_gather_read(music_b200 *h, int32_t *host_out, uint32_t count); /* synchronous copy of the first `count` entries */

/*
 * Replaces baz_music_doa::set_array_response() (/root/reference/lib/baz_music_doa.cc:60-70).
 * Thread-safe against a concurrent process_*() call, like the reference's d_mutex (:67, :101):
 * a call in flight finishes with the old table, later calls see the new one.
 */
int music_b200_set_table(music_b200 *h, const float *table_c64);

/*
 * Peak rule.  MUSIC_B200_PEAKS_TOP_BINS (default) is the reference's: the n largest bins, ties to the
 * lower bin (/root/reference/lib/baz_music_doa.cc:129-141) - for n >= 2 usually neighbouring bins of one
 * peak.  MUSIC_B200_PEAKS_LOCAL_MAXIMA is an opt-in extension with no reference counterpart: the n
 * largest circular local maxima (P[k] > P[k-1] and P[k] >= P[k+1], P[k] > 0), each more than
 * exclusion_bins away from every stronger peak taken; outputs in descending strength, unfilled slots
 * (0, 0, bin -1).  Applies to later process_*() calls.
 *
 * MUSIC_B200_PEAKS_ROOTS (extension, root-MUSIC): angles from the roots of the noise-subspace polynomial instead of a
 * search over the table, for a uniform linear array.  Covariance, eigensolver, source rules and spectrum are unchanged.
 *   ULA        the geometry set_geometry() recorded with the current table, p_0 .. p_{M-1}, s = (p_{M-1} - p_0) / (M - 1):
 *              |s| > 0, max_m ||p_m - (p_0 + m s)|| <= 1e-6 |s| and |s| <= (lambda / 2)(1 + 1e-12) (either element order,
 *              any origin and axis direction; a wider spacing maps a root to several directions).
 *   polynomial G = the M - d noise eigenvectors the scan would use (d = n, or the MDL / AIC count), C = G G^H,
 *              c_l = sum_{j - i = l} C_ij (l = -(M-1) .. M-1, c_{-l} = conj(c_l)), Q(z) = sum_l c_l z^(l + M - 1), so that
 *              D(t) = sum_l c_l z0^l with z0 = exp(-j 2 pi (s . u(t)) / lambda), all fp64.  Each outermost pair
 *              c_{+-l} that is exactly zero contributes a root at 0 and one at infinity.
 *   roots      Aberth-Ehrlich iteration in fp64: starting points on the circles of the Newton polygon of |b_k| (Bini),
 *              evaluation in 1 / z outside the unit circle (no power of z overflows), a root done once its correction is
 *              within 4 ulps of |z| or |Q(z)| <= 8 (2M - 2) 2^-52 sum_k |b_k| |z|^k; a window whose roots are not all done
 *              after 100 steps reports no peaks.  Two roots that
 *              are each other's nearest and closer than 1e-6 max(|z_a|, |z_b|) are one double root on the unit circle
 *              (D >= 0 there, so a root on the circle has even multiplicity): both become their midpoint, with modulus
 *              taken as 1, and the copy of the higher index sorts after every other root of modulus 1.
 *   selection  sort the 2M - 2 roots by ascending modulus and keep the first M - 1 (one of each pair z, 1 / conj(z));
 *              slots 0 .. d-1 take the d kept roots of largest modulus, in descending modulus, exact ties to the lower
 *              angle.  A kept root at 0 has no direction: its slot stays unfilled.
 *   angle      cpsi = clamp(-arg(z) lambda / (2 pi |s|), -1, 1), psi = acos(cpsi), alpha = atan2(s_y, s_x); the slot
 *              reports t* = the smaller of alpha + psi and alpha - psi wrapped into [0, 360) degrees (the mirror the grid's
 *              lower-bin tie rule picks: on an x-axis ULA [0, 180]); float cast and 360 -> 0 as in refinement.
 *   outputs    level = (float)(1 / D(t*)), D the direct fp64 form of the refinement; bin = floor(t* K / 360 + 0.5) mod K.
 *              Slots d .. n-1, windows with d = 0 and windows whose C or roots are not finite report (0, 0, bin -1).
 *              Spectrum, P64, R, eigenvalues and counts are unchanged; the MUSIC grid spectrum is computed only when the
 *              spectrum or P64 is requested (then by the unfused scan), otherwise no table scan runs at all.
 * Caveats: near end-fire (psi -> 0 or 180 degrees) acos amplifies the root error; as |s| / lambda shrinks every root
 * crowds towards z = 1 (a placeholder geometry such as 1 m elements at 1 Hz is meaningless here).
 * ROOTS needs exclusion_bins = 0, estimator MUSIC and refinement OFF (set_peak_mode(ROOTS) under MVDR / Bartlett or
 * NEWTON, and set_estimator(MVDR / BARTLETT) or set_refine(NEWTON) under ROOTS, return EINVAL), and a current table from
 * set_geometry() of a ULA: set_peak_mode(ROOTS) returns EINVAL otherwise, and so does a process_*() call whose current
 * table came from set_table() or from set_geometry() of another geometry (no fall-back to grid peaks).  Az-el handles
 * return EINVAL.  It runs the unfused kernels: covariance, eigensolver (+ source count), [scan], then one root kernel
 * per sub-batch, timed in the top-n slot of the stage timing.
 *
 * MUSIC_B200_PEAKS_ESPRIT (extension, LS-ESPRIT): angles from the shift invariance of the signal subspace, for the same
 * uniform linear arrays as ROOTS (the ULA condition, p_0, s and the angle rule above).
 *   subspace   E_s = the d eigenvectors of largest eigenvalue (M x d, orthonormal; d = n, or the MDL / AIC count),
 *              E1 = rows 0 .. M-2 of E_s, E2 = rows 1 .. M-1.
 *   matrix     Psi = (E1^H E1)^-1 E1^H E2 (d x d, fp64).  Windows where E1^H E1 is not positive definite or Psi is not
 *              finite report no peaks.  (E1^H E1 = I - r^H r with r = the last row of E_s, so the condition is
 *              |r|^2 < 1, and the inverse is I + r^H r / (1 - |r|^2).)
 *   eigenvalues  phi_1 .. phi_d of Psi in fp64: Householder reduction to Hessenberg form, then single-shift complex QR
 *              with Wilkinson shifts (exceptional shifts h + 0.75 |h_sub| (0.6 + 0.8 j) at the 10th and 20th step
 *              without a deflation, after LAPACK zlahqr), deflating a subdiagonal h_{l,l-1} once |h_{l,l-1}| <= 2^-52 (|h_{l-1,l-1}| +
 *              |h_{l,l}|); a window that needs more than 30 QR steps between two deflations reports no peaks.  On a ULA
 *              each phi is z0 = exp(-j 2 pi (s . u) / lambda) of one source, the z of ROOTS.
 *   outputs    each eigenvalue phi gives t* by ROOTS's angle rule (z = phi), level = (float)(1 / D(t*)) with D the direct
 *              fp64 form over the M - d noise eigenvectors, bin = floor(t* K / 360 + 0.5) mod K.  An eigenvalue exactly
 *              0 has no direction: its slot stays unfilled.  All d directions fill slots 0 .. d-1 in descending fp64
 *              level 1 / D, exact ties to the lower t*, then to the lower eigenvalue index (the diagonal position at
 *              which the QR deflated it).  Slots d .. n-1, windows with d = 0 and windows with a NaN level report (0, 0, bin -1).
 *              Spectrum, P64, R, eigenvalues and counts are unchanged, and the grid scan runs only for the spectrum
 *              or P64, as under ROOTS.
 * ESPRIT has ROOTS's restrictions, checked the same way in either order: exclusion_bins = 0, estimator MUSIC,
 * refinement OFF, a current table from set_geometry() of a ULA (a process_*() call on any other table returns EINVAL,
 * with no fall-back to grid peaks).  On an az-el handle the mode is 2-D ESPRIT (defined with the az-el entries below).  It
 * runs the unfused kernels: covariance, eigensolver (+ source count), [scan], then one ESPRIT kernel per sub-batch, timed
 * in the top-n slot of the stage timing.
 *
 * MUSIC_B200_PEAKS_DML (extension, deterministic maximum likelihood by alternating projection): the d table rows whose
 * span captures the most power of R, tr(P_A R).  It needs no signal-subspace rank, so it resolves coherent sources (a
 * path and its reflection, one emitter seen twice) that every subspace method merges, on any 1-D table.
 *   inputs     R = the window's fp64 covariance (the R output); a_k = table row k widened to fp64, ||a_k||^2 in fp64;
 *              d = n, or the MDL / AIC count.  d = 0, any non-finite entry of R, or tr R <= 0 (no power to place)
 *              gives a window with no peaks.
 *   search     S(B), B a set of slot bins: Q_B = modified Gram-Schmidt, applied twice, of the rows a_b (b in B) in slot
 *              order; P = I - Q_B Q_B^H; num(k) = a_k^H P R P a_k (a_k^H R a_k for B empty); den(k) = ||a_k||^2 -
 *              ||Q_B^H a_k||^2.  Bin k is a candidate iff den(k) > 2^-30 ||a_k||^2 and f(k) = num(k) / den(k) is
 *              finite (so a row in span(B), such as a line array's mirror row or a row already in B, and a zero row are
 *              never candidates).  S(B) = the candidate of largest f, exact ties to the lower bin; no candidate: the
 *              window reports no peaks.
 *   init       slot i = S({slots 0 .. i-1}), i = 0 .. d-1.
 *   sweeps     s = 1 .. 20: for i = 0 .. d-1, slot i = S({every other slot}) with the updated slots (Gauss-Seidel);
 *              stop after the first sweep that changed no slot, else keep the bins of sweep 20.  tr(P_A R) never
 *              decreases; with d = 1 a sweep repeats the first search and is skipped.
 *   levels     A = [a_slot0 .. a_slot(d-1)] = Q_A T (MGS twice as above), s2 = (tr R - tr(Q_A^H R Q_A)) / (M - d),
 *              p = diag(T^-1 (Q_A^H R Q_A - s2 I) T^-H): least-squares source powers in R's units (as MVDR's and
 *              Bartlett's levels; unlike MUSIC's 1 / D).  A level can be <= 0 at low SNR; its slot is still filled.
 *   outputs    slots 0 .. d-1 in descending fp64 p, exact ties to the lower bin; angle = (float)(bin * 360 / K) as
 *              under TOP_BINS, level = (float)p, bin through the peak-bin all-gather of sharded calls.  Slots d .. n-1
 *              report (0, 0, bin -1).  Spectrum, P64, R, eigenvalues and counts are unchanged.
 * Coherent sources lower the rank MDL / AIC count: use FIXED for them.  DML needs exclusion_bins = 0, estimator MUSIC
 * and refinement OFF or JOINT (NEWTON refines the MUSIC objective), checked in either order, and no az-el handle; any table from
 * set_table() or set_geometry() is accepted.  It runs the unfused kernels: covariance, the eigensolver only for MDL /
 * AIC, the eigenvalues, the spectrum or P64, the MUSIC scan only for the spectrum or P64, then one DML kernel per
 * sub-batch (one CTA per window for all its searches), timed in the top-n slot of the stage timing.
 *
 * MUSIC_B200_PEAKS_WSF (extension, weighted subspace fitting, also called MODE; Viberg, Ottersten & Kailath 1991): DML's
 * search on a weighted signal-subspace matrix X in place of R.  Its large-sample variance is the stochastic CRB of the
 * _crb entries, on any 1-D geometry, and coherent sources need no smoothing.
 *   inputs     l_0 <= .. <= l_{M-1} and e_0 .. e_{M-1}: the eigenvalues and eigenvectors of the window's R (the R output,
 *              after calibration and integration); d = n, or the MDL / AIC count.
 *   matrix     s2 = (l_0 + .. + l_{M-d-1}) / (M - d); for i = M-d .. M-1, w_i = (l_i - s2)^2 / l_i if l_i > s2, else 0;
 *              X = sum_i w_i e_i e_i^H (M x M, fp64).  X does not depend on eigenvector phase or on a rotation inside a
 *              degenerate eigenspace.  d = 0, l_0 <= 0, a non-finite eigenvalue, or every w_i = 0 (tr X = 0) gives a
 *              window with no peaks.  Under FIXED n with coherent sources the surplus signal eigenvalue is close to s2, so
 *              its weight is close to 0.
 *   search     DML's (init, up to 20 Gauss-Seidel sweeps, candidate and tie rules) word for word, with X for R.
 *   levels     DML's least-squares powers, taken from R (not X) at the chosen rows.
 *   outputs    as DML: slot order, angles, bins, the peak-bin all-gather and unfilled slots.
 * WSF has DML's restrictions, checked the same way in either order: exclusion_bins = 0, estimator MUSIC, refinement
 * OFF or JOINT, no az-el handle and no SEPARATE / INCOHERENT channel handle; any 1-D table from set_table() or
 * set_geometry().  It runs the unfused kernels: covariance, the eigensolver (always) and the count, one kernel per
 * sub-batch that forms X (timed in the eigensolver slot of the stage timing), [scan], then the DML kernel on X.
 *
 * MUSIC_B200_PEAKS_MANIFOLD (extension, root-MUSIC by manifold separation): gridless angles over the whole 360 degrees
 * on any planar array, from the roots of one polynomial per window (Belloni, Richter & Koivunen 2007; Rubsamen &
 * Gershman 2009).  Covariance, eigensolver, source rules and spectrum are unchanged.
 *   geometry   the positions p_m = (x_m, y_m) and wavelength set_geometry() recorded with the current table (on a
 *              COHERENT channel handle the reference channel's geometry and lambda_ref).
 *   order      rho_max = max_{i<j} ||p_j - p_i|| (fp64 hypot), x = 2 pi rho_max / lambda; L = the smallest integer >= 1
 *              with L + 1 >= x and 4 tau_{L+1} <= 2^-52, tau_0 = 1, tau_l = tau_{l-1} (x / 2) / l (a running fp64
 *              product).  Since |J_l(y)| <= (y/2)^l / l!, the truncation moves D by at most M^2 2^-52.  L must be <= 64
 *              (an aperture of about 4.4 lambda); on lambda / 2 UCAs M = 3, 4, 5, 8, 12, 16 give L = 21, 24, 26, 32, 39, 46.
 *   table      built in fp64 with the geometry, for each pair i < j in the order (0,1), (0,2), .., (M-2, M-1):
 *              (rho_ij, theta_ij) the polar form of p_j - p_i, beta_ij,l = (-j)^l J_l(2 pi rho_ij / lambda) e^{-j l theta_ij},
 *              l = 0 .. L (J_l by Miller's backward recurrence normalised by J_0 + 2 sum J_2k = 1);
 *              music_b200_manifold_coeffs_host() returns it.
 *   polynomial G = the M - d noise eigenvectors the scan would use (d = n, or the MDL / AIC count), C = G G^H in fp64;
 *              c_0 = tr C + 2 sum_{i<j} beta_ij,0 Re C_ij, c_l = sum_{i<j} beta_ij,l (2 Re C_ij for even l, 2 j Im C_ij for
 *              odd l), l = 1 .. L, c_{-l} = conj(c_l).  Then sum_{|l|<=L} c_l e^{j l t} = D(t) = a(t)^H C a(t) with
 *              a_m(t) = exp(-j 2 pi (x_m cos t + y_m sin t) / lambda), the refinement's steering.  Q(z) = sum_l c_l z^(l+L),
 *              degree P = 2L, and on |z| = 1 Q(z) = z^L D(arg z).  Each outermost pair c_{+-l} that is exactly zero
 *              contributes a root at 0 and one at infinity.
 *   roots      ROOTS's rules word for word: Aberth-Ehrlich from the Newton-polygon circles, evaluation in 1 / z outside
 *              the unit circle, the two stop tests (with P for 2M - 2), 100 steps and then no peaks, and the double-root
 *              merge.
 *   selection  ROOTS's: sort the P roots by ascending modulus and keep the first P / 2; slots 0 .. d-1 take the d kept
 *              roots of largest modulus, in descending modulus, exact ties to the lower angle; a kept root at 0 leaves
 *              its slot unfilled.
 *   angle      t* = atan2(Im z, Re z) in degrees, + 360 if negative; float cast and 360 -> 0 as in refinement.  The map
 *              is one-to-one: there is no mirror rule.
 *   outputs    level = (float)(1 / D(t*)), D the direct fp64 form of the refinement; bin = floor(t* K / 360 + 0.5) mod K.
 *              Slots d .. n-1, windows with d = 0, windows whose C or roots are not finite and windows with P = 0 (every
 *              element at one point) report (0, 0, bin -1).  Spectrum, P64, R, eigenvalues and counts are unchanged, and
 *              the grid scan runs only for the spectrum or P64, as under ROOTS.
 * Caveats: on a collinear array D is symmetric about the array line, so every source has a mirror root of equal modulus
 * and the slots fill with mirror pairs (ROOTS and ESPRIT are the modes for line arrays; MANIFOLD accepts them).  Elements
 * more than lambda / 2 apart carry the grid spectrum's ambiguities.
 * MANIFOLD has ROOTS's restrictions, checked the same way in either order: exclusion_bins = 0, estimator MUSIC,
 * refinement OFF, no az-el handle and no SEPARATE / INCOHERENT channel handle; a current table from set_geometry() (a
 * process_*() call on a set_table() table returns EINVAL, with no fall-back) whose order is <= 64 (EINVAL otherwise,
 * with the aperture in wavelengths in the message).  COHERENT channel handles, multi-device handles, every 1-D entry
 * point, calibration and MDL / AIC work as under ROOTS.  It runs the unfused kernels: covariance, eigensolver (+ source
 * count), [scan], then one manifold kernel per sub-batch (one CTA per window), timed in the top-n slot of the stage
 * timing.
 */
#define MUSIC_B200_PEAKS_TOP_BINS 0
#define MUSIC_B200_PEAKS_LOCAL_MAXIMA 1
#define MUSIC_B200_PEAKS_ROOTS 2
#define MUSIC_B200_PEAKS_ESPRIT 3
#define MUSIC_B200_PEAKS_DML 4
#define MUSIC_B200_PEAKS_MANIFOLD 5
#define MUSIC_B200_PEAKS_WSF 6
int music_b200_set_peak_mode(music_b200 *h, int mode, uint32_t exclusion_bins);

/*
 * Test hook of MUSIC_B200_PEAKS_MANIFOLD (no device needed): the order L of positions [m][x, y] (metres) at `wavelength`
 * and, when beta is not NULL, the coefficient table beta[m(m-1)/2][L+1][re, im] the peak mode uses (caller-allocated for
 * that L: call once with beta NULL to learn it).  Returns EINVAL for L > 64, after writing L, and for invalid arguments.
 */
int music_b200_manifold_coeffs_host(const double *positions_xy, uint32_t m, double wavelength, uint32_t *L, double *beta);

/*
 * Source-count rule (extension, no reference counterpart).  MUSIC_B200_SOURCES_FIXED (default) uses the n of
 * create() for every window.  With MUSIC_B200_SOURCES_MDL or _AIC, n becomes the MAXIMUM number of sources: for each
 * window the engine estimates d in [0, n] from the window's ascending eigenvalues l_0 <= ... <= l_{m-1} and the
 * N = nsamples / m snapshots (Wax & Kailath, 1985).  For d = 0 .. n, p = m - d, sums over i = 0 .. p-1:
 *     L(d) = N (p log(sum l_i / p) - sum log l_i)
 *     MDL(d) = L(d) + d (2m - d) log(N) / 2          AIC(d) = 2 L(d) + 2 d (2m - d)
 * d is the smallest minimiser (NaN never wins), and 0 when l_0 <= 0 or any eigenvalue is not finite.  The noise
 * subspace is then the m - d smallest-eigenvalue eigenvectors, the peak rule fills the first d slots and slots
 * d .. n-1 stay unfilled (angle 0, level 0, bin -1).  With d = 0 the spectrum is 1 / ||a||^2 and no peak is reported.
 * MDL and AIC run the unfused kernels (the fused m = 4 / m = 8 kernels do not compute every eigenvalue).
 * Returns EINVAL for an unknown rule, or for MDL / AIC when N <= m (R is rank-deficient, the criteria meaningless).
 * Applies to later process_*() calls and to every device of a multi-device handle.
 */
#define MUSIC_B200_SOURCES_FIXED 0
#define MUSIC_B200_SOURCES_MDL 1
#define MUSIC_B200_SOURCES_AIC 2
int music_b200_set_source_rule(music_b200 *h, int rule);

/*
 * Off-grid peak refinement (extension, no reference counterpart).  MUSIC_B200_REFINE_OFF (default) reports grid
 * angles k * 360 / K.  With MUSIC_B200_REFINE_NEWTON every filled slot (w, i) with grid bin b >= 0 is moved to the
 * minimum of the exact MUSIC denominator of the array geometry near b:
 *   G      the noise eigenvectors the scan used (the m - n smallest, or m - d under MDL / AIC);
 *   a(t)   the unrounded fp64 steering vector of the current geometry (music_b200_set_geometry), t in radians:
 *          a_m(t) = exp(-j phi_m),  phi_m = 2 pi (p_x,m cos t + p_y,m sin t) / lambda;
 *   D(t)   = sum_j |g_j^H a(t)|^2 (always the direct noise-subspace form), with the analytic derivatives
 *          psi_m = dphi_m/dt = 2 pi (-p_x,m sin t + p_y,m cos t) / lambda,  phi_m'' = -phi_m,
 *          a' = -j psi a,  a'' = (j phi - psi^2) a,  s = G^H a, s' = G^H a', s'' = G^H a'':
 *          D' = 2 sum Re(conj(s) s'),  D'' = 2 sum (|s'|^2 + Re(conj(s) s''));
 *   bracket [lo, hi] = [t_b - delta, t_b + delta], t_b = b * 360 / K degrees, delta = 360 / K degrees.
 *          If D'(lo) < 0 < D'(hi), safeguarded
 *          Newton on D' = 0 starts at t_b: a step that would leave the bracket or not halve it is a bisection step
 *          (rtsafe); it stops at D' = 0 exactly, when a step is at most 1e-12 rad, or after 50 iterations.  The result
 *          t* is accepted iff t* != t_b and D(t*) <= D(t_b) (same fp64 formula); otherwise the slot keeps t_b.
 * Outputs: angles[w][i] = (float) of t* in degrees wrapped into [0, 360) (a value that rounds to 360.0f becomes 0.0f;
 * a kept slot keeps its grid angle); levels[w][i] = (float)(1 / D(t*)).  bins, spectrum, P64, R, eigenvalues and
 * counts are the grid results, unchanged; unfilled slots stay (0, 0, bin -1).
 * Caveats: with refinement on a level is the analytic fp64 spectrum, not the value from the float32-rounded table.  P
 * is conditioned about 4000x (DESIGN.md section 3), so even where t* = t_b the level can differ from the unrefined
 * level by about 1e-4 relative.  With TOP_BINS and n >= 2, neighbouring bins of one peak can refine to the same angle:
 * use MUSIC_B200_PEAKS_LOCAL_MAXIMA for n >= 2.
 * Refinement runs the unfused kernels (the fused m = 4 / m = 8 kernels keep only the principal eigenvector) plus one
 * fp64 kernel per sub-batch, timed in the top-n slot of the stage timing.
 * Returns EINVAL for an unknown mode, and for NEWTON when the current table came from music_b200_set_table() (it has
 * no geometry).  A process_*() call with refinement on whose current table came from set_table() (set_table() after
 * set_refine()) fails with EINVAL; there is no silent fall-back to grid angles.
 * Applies to later process_*() calls and to every device of a multi-device handle.
 */
/*
 * MUSIC_B200_REFINE_JOINT (extension): a joint Gauss-Newton refinement of all d filled slots of a DML or WSF window on
 * the analytic steering a(t), a'(t) = -j psi a(t) of NEWTON above.
 *   factor     X = F F^H: under WSF the columns sqrt(w_i) e_i with w_i > 0 in ascending i; under DML F = L of the
 *              Cholesky factorisation R = L L^H (X = R).  A DML window whose R is not positive definite (a pivot <= 0)
 *              keeps what the peak stage wrote, and so does a WSF window without X.
 *   criterion  t = the slot angles in radians (filled slots in slot order), A(t) = [a(t_i)], D = [a'(t_i)],
 *              A+ = (A^H A)^-1 A^H, P_perp = I - A A+, V(t) = Re tr(P_perp X) = ||P_perp F||_F^2 (evaluated in this form,
 *              which stays accurate where V is small).  A^H A counts as positive definite when every pivot l of its
 *              factorisation exceeds 2^-30 ||a_l||^2.
 *   step       g_i = -2 Re(A+ X P_perp D)_ii, H = 2 Re((D^H P_perp D) o (A+ X A+^H)^T) (the structure of the CRB's
 *              Fisher matrix), s = -H^-1 g.  H counts as positive definite when every pivot k of its Cholesky
 *              factorisation is > 0 and > 2^-40 H_kk.
 *   iteration  start at t_b,i = (b_i * 360 / K) degrees in radians, box |t_i - t_b,i| <= (360 / K) degrees.  A window
 *              whose A^H A at the start is not positive definite keeps what the peak stage wrote.  Each step: stop if H
 *              is not positive definite or max |s_i| <= 1e-12; else try t + s projected onto the box, accepted iff
 *              A^H A is positive definite there and V strictly decreases, else halve s (up to 30 times); stop when no
 *              try is accepted, or after 50 steps.
 *   outputs    angles[w][i] = (float) of t*_i in degrees wrapped into [0, 360), 360 -> 0 as under NEWTON (a slot whose
 *              t*_i = t_b,i keeps its grid angle); levels = (float) of DML's least-squares powers from R at the analytic
 *              A(t*).  Bins, spectrum, P64, R, eigenvalues and counts keep their grid values, as under NEWTON, and so
 *              does the slot order.
 * JOINT is accepted only with DML or WSF (JOINT under any other peak mode, and any peak mode other than DML and WSF under
 * JOINT, returns EINVAL; NEWTON under DML and WSF stays EINVAL), on 1-D single- and multi-device handles (channel and
 * az-el handles return EINVAL), on a table from set_geometry(): a process_*() call on a set_table() table returns EINVAL,
 * with no fall-back.  One warp per window runs after the peak stage and before beams, CRB and tracking, timed in the
 * top-n slot of the stage timing; the beams, the CRB and the tracker read the refined angles.
 * Not built: az-el WSF and JOINT, JOINT for the grid modes (NEWTON serves them), stochastic ML proper, a fused path.
 */
#define MUSIC_B200_REFINE_OFF 0
#define MUSIC_B200_REFINE_NEWTON 1
#define MUSIC_B200_REFINE_JOINT 2
int music_b200_set_refine(music_b200 *h, int mode);

/*
 * Spectrum estimator (extension, no reference counterpart).  R is the window's covariance, a = a_k table row k widened
 * to fp64, M = m.
 *   MUSIC_B200_ESTIMATOR_MUSIC (default)  P[k] = 1 / ||G^H a||^2, unchanged.
 *   MUSIC_B200_ESTIMATOR_BARTLETT         P[k] = (a^H R a) / (a^H a)^2: the output power of the unit-gain beam
 *                                         w = a / ||a||^2 (delay-and-sum beamscan).  No eigendecomposition, no n.
 *   MUSIC_B200_ESTIMATOR_MVDR             delta = loading * tr(R) / M,  R_L = R + delta I,  P[k] = 1 / (a^H R_L^-1 a):
 *                                         the output power of the distortionless (Capon) beam.  Evaluated as
 *                                         ||L^-1 a||^2 with the Cholesky factor R_L = L L^H.  If the factorisation meets
 *                                         a pivot that is not > 0 (NaN included), every P[k] of that window is NaN: the
 *                                         window reports no peak, (0, 0, bin -1), and its spectrum row is NaN (as a NaN
 *                                         window under MUSIC).
 * For one source, R = p a0 a0^H + s2 I with ||a0||^2 = M, both give P(theta0) = p + (s2 + delta) / M (delta = 0 for
 * Bartlett): their levels are power estimates.
 * Unchanged: the peak rules, the float casts, levels = (float)P at the peak, the spectrum / P64 outputs and the bins,
 * now of the chosen estimator's P; n (1 <= n < m) is the number of peak slots.  Under MDL / AIC the eigensolver runs
 * only to count: the peak rule fills d slots of the estimator's spectrum, which does not depend on d.
 * Refinement (MUSIC_B200_REFINE_NEWTON, geometric tables only) works for all three, with the 1-D bracket and accept
 * rule and the az-el projected Newton steps of music_b200_set_refine, on:
 *   MVDR      D(t) = a(t)^H R_L^-1 a(t) (minimised), level = (float)(1 / D(t*));
 *   BARTLETT  F(t) = -B(t), B(t) = a(t)^H R a(t) (B maximised): the 1-D bracket condition is B'(lo) > 0 > B'(hi), a step
 *             is accepted iff B(t*) >= B(t_b), level = (float)(B(t*) / M^2) (||a(t)||^2 = M for the analytic a).
 * BARTLETT and MVDR run the unfused kernels: covariance, [eigensolver + source count only under MDL / AIC or when
 * process_device_ex asks for the eigenvalues], [MVDR: Cholesky preparation, timed in the eigensolver slot], the
 * quadratic-form scan, then the peak rule / decode / refinement as for MUSIC.
 * Returns EINVAL for an unknown estimator, loading not finite or < 0, loading != 0 for MUSIC or BARTLETT, and MVDR with
 * loading == 0 when N <= m (R is singular).  Setting MUSIC (loading 0) again restores the default behaviour exactly.
 * Applies to later process_*() calls (host, device, _ex, _counts, planar, sharded, az-el) and to every device of a
 * multi-device handle.
 *
 * MUSIC_B200_ESTIMATOR_IAA, the iterative adaptive approach (Yardibi, Li, Stoica, Xue & Baggeroer 2010): a
 * nonparametric weighted-least-squares power spectrum on the grid.  It needs no source count and works from R alone, so
 * it also runs when R is singular (N <= m), and it resolves coherent sources (a path and its reflection).  Its level at
 * a peak is that source's power in R's units.  Definition, with Rh the window's fp64 covariance every other estimator
 * reads (the R output, after calibration and integration; per channel R_c on a SEPARATE channel handle, the focused R
 * on a COHERENT one), a_k table row k widened to fp64, nu_k = ||a_k||^2, I the iteration count
 * (music_b200_set_iaa_iterations) and delta = loading * tr(Rh) / M:
 *   p0_k = a_k^H Rh a_k / nu_k^2                  (the Bartlett P, so I = 0 would be Bartlett);
 *   rows with nu_k = 0 have p_k = 0 at every step and add nothing;
 *   for i = 1 .. I:  R_i = sum_k p(i-1)_k a_k a_k^H + delta I (fp64),  R_i = L L^H (Cholesky),  S_i = R_i^-1,
 *                    p(i)_k = (a_k^H S_i Rh S_i a_k) / (a_k^H S_i a_k)^2,  the denominator evaluated as ||L^-1 a_k||^2
 *                    (a sum of squares that cannot cancel, as MVDR);
 *   P = p(I).
 * Every P[k] of a window is NaN - the window reports no peak, (0, 0, bin -1), and its spectrum row is NaN, as under
 * MVDR - when Rh has a non-finite entry or tr Rh <= 0, when a Cholesky pivot is not > 0 (NaN included), or when any
 * p(i)_k is not finite.  The spectrum and P64 are P; TOP_BINS, LOCAL_MAXIMA and the az-el 2-D rules pick the peaks from
 * P unchanged, level = (float)P at the peak; bins, counts (MDL / AIC count from the eigenvalues, as under MVDR) and R
 * are unchanged.
 * Accepted on every 1-D entry point (host, device, _ex, _counts, planar, sharded and gather, multi-device, _beams,
 * _crb, _tracks), on az-el handles (host, device, _crb, _tracks) and on SEPARATE and COHERENT channel handles, with any
 * finite loading >= 0: loading 0 is accepted for any N, N <= m included.  EINVAL with the ROOTS, ESPRIT, MANIFOLD, DML
 * or WSF peak modes (they need the MUSIC estimator), with NEWTON or JOINT refinement and with the INCOHERENT combine.
 * Runs unfused: covariance, [eigensolver + source count under MDL / AIC or when the eigenvalues are asked for], then one
 * iaa_kernel launch per sub-batch (and per channel), timed in the scan slot, then the grid peak rule.  Its cost is
 * about 3 K M^2 fp64 FMA per window per iteration (K = table rows; 9x the 1-D cost on a 360 x 91 az-el grid).
 * Weakness: IAA does not replace MUSIC for closely spaced *uncorrelated* sources with plenty of snapshots.  Two
 * uncorrelated sources 6 degrees apart on an 8-element lambda / 2 ULA at 10 dB and N = 64 are resolved by MUSIC in every
 * window and by IAA in none: IAA's resolution there is that of a (sharpened) beam, MUSIC's that of the noise subspace.
 * Not built: off-grid refinement of IAA peaks, SPICE, a fused path.
 */
#define MUSIC_B200_ESTIMATOR_MUSIC 0
#define MUSIC_B200_ESTIMATOR_MVDR 1
#define MUSIC_B200_ESTIMATOR_BARTLETT 2
/* IAA is 4, not the next free code 3: releases before IAA answered set_estimator(3) with EINVAL (unknown estimator),
 * and that answer is kept, so code 3 stays unassigned. */
#define MUSIC_B200_ESTIMATOR_IAA 4
int music_b200_set_estimator(music_b200 *h, int estimator, double loading);

/*
 * The IAA iteration count I (MUSIC_B200_ESTIMATOR_IAA): 1 .. 64, default 15; EINVAL outside.  Applies to later calls
 * and to every device of a multi-device handle; read only under the IAA estimator.
 */
#define MUSIC_B200_IAA_DEFAULT_ITERATIONS 15
#define MUSIC_B200_IAA_MAX_ITERATIONS 64
int music_b200_set_iaa_iterations(music_b200 *h, int iterations);

/*
 * Beamformed source signals (extension, no reference counterpart): receive each reported source, a beam steered at
 * every filled peak slot of a window, from the same window's covariance.
 * music_b200_set_beamformer() takes MUSIC_B200_BEAMS_OFF (default), _DAS, _MVDR or _LCMV and a diagonal loading.  The
 * setting is read only by music_b200_process_device_beams() and music_b200_process_host_beams(); every other entry point
 * ignores it.  It applies to every device of a multi-device handle.  EINVAL: an unknown rule; loading not finite or < 0;
 * loading != 0 with OFF or DAS; MVDR or LCMV with loading == 0 when N <= m (R is singular); an az-el handle.
 * For window w the filled slots are S = {i : bins[w][i] >= 0} as the call's peak stage reported them, under every peak
 * mode, source rule, estimator and refinement setting (the slots need not form a prefix).  M = m, x(r, c) = in[c m + r].
 *   steering   a_i (fp64): if the current table came from set_geometry(), a_m = exp(-j phi_m),
 *              phi_m = 2 pi (p_x,m cos t + p_y,m sin t) / lambda, t = the reported float angle (double)angles[w][i] in
 *              radians (the refinement's convention, so refined, ROOTS and ESPRIT angles steer off the grid); if it came
 *              from set_table(), table row bins[w][i] widened to fp64.
 *   DAS        w_i = a_i / (a_i^H a_i).  It reads no R.
 *   MVDR       R_L = R + delta I, delta = loading * tr(R) / M; R_L = L L^H with the MVDR estimator's Cholesky (a pivot
 *              that is not > 0 fails); y_i = L^-1 a_i, z_i = L^-H y_i, w_i = z_i / ||y_i||^2.
 *   LCMV       unit gain on its own source, a null on every other filled slot: Y = [y_i], Z = [z_i] over i in S (slot
 *              order), G = Y^H Y (d x d), G = C C^H where every pivot g_k (before its square root) must satisfy
 *              g_k > 2^-20 G_kk (G_kk = the diagonal entry before elimination); W = Z G^-1, column i is w_i, and
 *              w_i^H a_j = delta_ij.  With d = 1, LCMV equals MVDR.
 *   failure    every weight and beam of the window is 0 when the Cholesky of R_L fails (MVDR, LCMV), when LCMV's pivot
 *              test fails (e.g. the two mirror slots of an x-axis ULA under LOCAL_MAXIMA: their steering vectors are
 *              nearly identical), or when any weight is not finite.  Unfilled slots always get zero weights and beams.
 *   outputs    weights[w][i][m] = w_i as fp64 (re, im) pairs; beams[w][i][t] = (float)(sum_m conj(w_im) x_m(t)) for
 *              t < N, accumulated in fp64, re and im each rounded once; layout [W][n][N] complex64, one contiguous time
 *              series per slot.
 * Caveat: with coherent sources (what the DML peak mode resolves) an MVDR or LCMV beam built from R suffers signal
 * cancellation; that is physics, not a defect.  Use DAS there.
 * The beams entry points take the outputs of music_b200_process_device_counts() / _host_counts() plus weights and beams;
 * either of the two may be NULL, not both (EINVAL).  With the rule OFF they return EINVAL.  beams must be 8-byte
 * aligned and weights 16-byte aligned.  The host entry deals windows over a multi-device handle as process_host does;
 * the device entry goes to the device the input lives on.  A beams call always runs the unfused kernels (the fused
 * kernels keep no R): its angles, levels, spectrum, bins and counts are byte-identical to process_device_ex() with d_R
 * on the same windows.  Per sub-batch it adds beam_weights_kernel and (with beams) beam_apply_kernel after the peak
 * stage, timed in the top-n slot of the stage timing.  The apply kernel reads the input a second time: n N complex64
 * out, m N in per window.
 */
#define MUSIC_B200_BEAMS_OFF 0
#define MUSIC_B200_BEAMS_DAS 1
#define MUSIC_B200_BEAMS_MVDR 2
#define MUSIC_B200_BEAMS_LCMV 3
int music_b200_set_beamformer(music_b200 *h, int rule, double loading);
int music_b200_process_device_beams(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles, float *d_levels,
                                    float *d_spectrum, int32_t *d_bins, int32_t *d_counts, double *d_weights, float *d_beams,
                                    void *stream);
int music_b200_process_host_beams(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels,
                                  float *spectrum, int32_t *bins, int32_t *counts, double *weights, float *beams);

/*
 * Receiver calibration (extension, no reference counterpart): estimate each element's complex gain from a known source
 * and correct it on the device in every mode.
 *   model      each receiver chain multiplies what its element sees by a gain g_m (cable length, filter group delay, the
 *              LO phase of each channel, which changes at every retune), after the receiver noise:
 *              x_raw(t) = G (A s(t) + n(t)), G = diag(g).  The correction is x = C x_raw, C = diag(c), c_m = 1 / g_m,
 *              which makes the noise white again.  (Correcting the table instead, a -> g o a, would leave the noise
 *              coloured by |g_m|^2: the correction goes on the data side, as a transform of R.)
 *   apply      music_b200_set_calibration(h, gains) sets gains [m][2] doubles (re, im); NULL clears it.  Every entry must
 *              be finite, every |g_m| > 0 and 1 / g_m finite, otherwise EINVAL and the old setting stays.  While a
 *              calibration is set, every process call transforms each window's fp64 covariance right after the covariance
 *              kernel: R_ij <- (c_i R_ij) conj(c_j), with c_m = 1 / g_m = conj(g_m) / |g_m|^2 computed on the host in fp64.
 *              Everything downstream sees the corrected R: eigensolver, source count, MVDR preparation, scans, every peak
 *              mode, refinement, ROOTS, ESPRIT, DML, az-el decode and refinement, and beam weights; process_device_ex's
 *              d_R returns the corrected R.  Beam weights are returned in raw-input coordinates, w_raw = conj(c) o w, and
 *              the beams are formed from the raw input: beams = w_raw^H x_raw = w^H x, and LCMV's w_i^H a_j = delta_ij
 *              still holds in corrected coordinates.  The setting persists across set_table(), set_geometry() and
 *              set_geometry_azel() (it belongs to the receivers, not to the table), applies to every device of a
 *              multi-device handle and is read by every process entry (host, device, _ex, _counts, planar, sharded, az-el,
 *              beams).  A calibrated call runs the unfused kernels (the fused M = 4 / M = 8 kernels keep R in registers),
 *              plus calib_apply_kernel per sub-batch, timed in the covariance slot of the stage timing, and with beams
 *              calib_weights_kernel after the weights, timed in the top-n slot.
 *              music_b200_get_calibration returns the gains in use, all (1, 0) when none is set.
 *   estimate   from windows of one dominant source at a known direction (az, el) in degrees; el must be 0 on a 1-D handle.
 *              a0 = the unrounded fp64 steering vector of the current geometry (the refinement's convention on a 1-D
 *              handle, the 3-D direction u(az, el) on an az-el handle); a table from set_table() gives EINVAL.
 *              Rbar = (1 / W) sum_w R_w, the fp64 covariance of each raw window (before any calibration that is set),
 *              accumulated over one or more accumulate calls.  h minimises the off-diagonal misfit
 *              sum_{i != j} |Rbar_ij - h_i conj(h_j)|^2: noise and its colouring live on the diagonal only, so unlike the
 *              principal eigenvector of Rbar the minimiser recovers g o a0 exactly on a population covariance at any
 *              noise level.
 *                start   r = argmax_i Rbar_ii (lowest index on ties), h_r = sqrt(Rbar_rr), h_i = Rbar_ir / sqrt(Rbar_rr);
 *                sweeps  Gauss-Seidel: for i = 0 .. M-1 in turn, h_i <- (sum_{j != i} Rbar_ij h_j) / (sum_{j != i} |h_j|^2),
 *                        with the updated entries; stop after the first sweep whose largest change |h_i,new - h_i,old| is
 *                        <= 2^-40 max_i |h_i|, or after 200 sweeps.
 *              g_m = h_m / a0_m, rotated by a common phase so that g_0 is real and positive, then
 *                MUSIC_B200_CALIB_GAIN_PHASE  scaled to sum |g_m|^2 = M; needs m >= 3 (with two elements the split of the
 *                                             magnitudes between the chains cannot be identified);
 *                MUSIC_B200_CALIB_PHASE       g_m <- g_m / |g_m|; any m >= 2, including a two-channel receiver.
 *              stats: the residual rho = sqrt(sum_{i != j} |Rbar_ij - h_i conj(h_j)|^2 / sum_{i != j} |Rbar_ij|^2) (small
 *              when one source dominates) and the number of sweeps.
 *              EINVAL, and nothing written, when no windows were accumulated, Rbar_rr <= 0, anything is not finite, or
 *              some h_m = 0 (a dead channel).
 *   calls      accumulation and solving run on the device.  calib_accumulate_device needs d_in 16-byte aligned, is enqueued
 *              on `stream` and does not synchronise; calib_accumulate_host copies in chunks and returns when done.  solve
 *              synchronises, leaves the accumulator unchanged (more windows can be added and solved again) and does not
 *              apply the gains: the caller inspects rho, then calls set_calibration.  reset empties the accumulator.  On
 *              a multi-device handle the accumulator and solve are served by devices[0], and accumulate_device needs
 *              its input there.  The accumulated sum is deterministic for a given sequence of calls; its rounding may
 *              depend on how the windows are split across calls.
 */
#define MUSIC_B200_CALIB_PHASE 1
#define MUSIC_B200_CALIB_GAIN_PHASE 2
int music_b200_set_calibration(music_b200 *h, const double *gains /* [m][2] or NULL */);
int music_b200_get_calibration(music_b200 *h, double *gains /* [m][2] */);
int music_b200_calib_reset(music_b200 *h);
int music_b200_calib_accumulate_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, void *stream);
int music_b200_calib_accumulate_host(music_b200 *h, const float *in_c64, uint32_t nwindows);
int music_b200_calib_solve(music_b200 *h, double az_deg, double el_deg, int kind, double *gains /* host [m][2] */,
                           double *stats /* host [2]: residual, sweeps; may be NULL */);

/*
 * Receiver self-calibration without a known source (extension, no reference counterpart): the element gains from windows
 * of unknown emitters, so that the array can be recalibrated after every retune without a beacon at a surveyed bearing.
 * Weiss-Friedlander eigenstructure calibration (1990) with the magnitudes read from the diagonal and a multi-start phase
 * search.  Model as above: x_raw = G (A s + n), G = diag(g).  tests/calib_blind_oracle.py restates it literally.
 *   segments   music_b200_calib_blind_accumulate_*(h, in, nwindows, segment): nwindows must be a multiple of segment
 *              (>= 1); every `segment` consecutive windows form one segment, R_s = the mean fp64 covariance of its raw
 *              windows (before any calibration that is set).  The sources may move between segments but are assumed
 *              still within one: a single emitter moving past the array, or different emitters in different segments.
 *              More distinct, well spread directions identify the gains better.  A segment never straddles calls; at
 *              most MUSIC_B200_CALIB_MAX_SEGMENTS segments are held (EINVAL, nothing added, beyond).  R_s is
 *              deterministic and does not depend on how the windows are split across calls.
 *   magnitudes mag_m = sqrt(sum_s Re R_s,mm / S), scaled to sum mag_m^2 = M (exact on a population covariance with a
 *              geometric table, |a_m| = 1); R_s <- T R_s T with T = diag(1 / mag), which whitens the noise.
 *   projectors E_s = the M - d smallest-eigenvalue eigenvectors of the whitened R_s from the handle's eigensolver,
 *              Pi_s = E_s E_s^H, computed once.
 *   starts     start 0 is phi = 1; start p >= 1 takes phi_m = exp(j theta), theta = pi (2 u - 1), u = (z >> 11) 2^-53,
 *              z = mix64(seed xor ((p * 256 + m + 1) * 0x9E3779B97F4A7C15 mod 2^64)), mix64 the splitmix64 finaliser
 *              (z ^= z >> 30, z *= 0xBF58476D1CE4E5B9, z ^= z >> 27, z *= 0x94D049BB133111EB, z ^= z >> 31).
 *   iteration  for each segment: P_s(k) = ||E_s^H (phi o a_k)||^2 / M over the rows a_k of the handle's table, and the d
 *              best circular local maxima of q = 1 / P_s by the LOCAL_MAXIMA rule (q > 0, q[k] > q[k-1], q[k] >= q[k+1];
 *              larger q first, lowest k on ties), bins k_s,1..d in pick order (fewer when fewer exist);
 *              Q = sum_s sum_i D_k^H Pi_s D_k (D_k = diag(a_k)) in segment then pick order, and J = sum_s J_s in segment
 *              order with J_s = sum_i P_s(k_s,i) in pick order.
 *              Then phi <- v / |v| element-wise, v the eigenvector of the smallest eigenvalue of Q (handle's eigensolver)
 *              rotated so that v_0 is real and positive.  (At a population Q the true phases are its null vector; the
 *              eigenvector form stays well conditioned there, where W-F's linear constraint Q^-1 e_0 does not.)
 *   schedule   every start runs 24 iterations; the winner is the start with the smallest J of its 24th iteration (lowest
 *              index on ties; NaN never wins).  It is polished for up to 30 iterations, stopping after the first one whose
 *              max_m |phi_new - phi_old| <= 2^-30.  The counts are fixed, so the result is deterministic.
 *   outputs    gains [m][2]: mag o phi (MUSIC_B200_CALIB_GAIN_PHASE) or phi (MUSIC_B200_CALIB_PHASE); g_0 is real and
 *              positive.  angles [S][d] (may be NULL): k 360 / K degrees of the last iteration's picks, NaN where a
 *              segment had fewer than d local maxima.  stats [4] (may be NULL): the misfit J / (S d) of the last
 *              iteration (in [0, 1], small when calibrated), the polish iterations run, the winning start, S.
 *   limits     the grid is discrete: a fit can settle where the phase error looks to every segment like a shift of its
 *              directions by one bin, with a small non-zero misfit and phase errors of the order of the grid step.  24
 *              iterations per start avoid it in the exact-covariance cases of tests/test_calib_blind_oracle.py (UCA-4 and
 *              UCA-8, d = 1 and 2, 8 and 16 segments spread over the circle, seeds 0 - 9) but one, UCA-8 with d = 1 and 8
 *              segments at seed 5, which neither more starts nor more iterations reach.  More segments and spread
 *              directions avoid it.  On exact covariances the misfit tells it apart (about 1e-4 against 1e-30); on
 *              measured windows the estimation noise sets the misfit of a good fit too.
 *   refusals   EINVAL, nothing written, for: an az-el or channel handle (not built); a set_table() table; collinear element
 *              positions (a phase ramp along the line cannot be told from a shift of every direction); m < 3; d outside
 *              1 .. m - 2; no segments; starts outside 1 .. 256; a table of more than 24576 rows (the scan holds a
 *              segment's spectrum in shared memory); non-finite segment covariances or an element without power.
 *   calls      calib_blind_accumulate_device needs d_in 16-byte aligned, is enqueued on `stream` and does not synchronise;
 *              _host copies in chunks and returns when done.  solve enqueues a fixed number of kernels on one stream,
 *              synchronises once, leaves the segments unchanged and does not apply the gains: the caller inspects the
 *              misfit, then calls set_calibration.  reset empties the segments.  On a multi-device handle devices[0]
 *              serves them all, and accumulate_device needs its input there.
 */
#define MUSIC_B200_CALIB_MAX_SEGMENTS 1024
int music_b200_calib_blind_reset(music_b200 *h);
int music_b200_calib_blind_accumulate_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, uint32_t segment, void *stream);
int music_b200_calib_blind_accumulate_host(music_b200 *h, const float *in_c64, uint32_t nwindows, uint32_t segment);
int music_b200_calib_blind_solve(music_b200 *h, uint32_t d, int kind, uint32_t starts, uint64_t seed, double *gains /* host [m][2] */,
                                 double *angles /* host [S][d] or NULL */, double *stats /* host [4] or NULL */);

/*
 * Covariance integration across windows (extension, no reference counterpart): an exponentially weighted covariance
 * carried from window to window and from call to call, so that a weak source is detected and located from the recent
 * past while every window keeps its own output rate and latency.
 *   setting    music_b200_set_integration(h, alpha): the forgetting factor, finite with 0 <= alpha < 1, otherwise EINVAL
 *              and the old setting stays.  alpha = 0 (the default) is off: every output, the launch count and the fused /
 *              unfused path choice are those of a handle that never had integration.  music_b200_reset_integration(h)
 *              restarts the recurrence at the next window.
 *   inputs     R_j: the window's fp64 covariance as process_device_ex's d_R returns it with integration off (after the
 *              calibration when one is set); j = 0, 1, 2, ... the handle's windows in stream order since the last reset,
 *              through the windows of one call and on into the next call.
 *   recurrence S_{-1} = 0, c_{-1} = q_{-1} = 0;  S_j = alpha S_{j-1} + R_j,  c_j = alpha c_{j-1} + 1,
 *              q_j = alpha^2 q_{j-1} + 1;  the integrated covariance is Rbar_j = S_j / c_j (the first window after a reset
 *              is its own R, bit for bit).
 *   reads      every stage that reads R reads Rbar_j instead: eigensolver, source count, MVDR preparation, every scan,
 *              every peak mode (TOP_BINS, LOCAL_MAXIMA, ROOTS, ESPRIT, 2-D ESPRIT, DML, MANIFOLD), refinement, the az-el
 *              decode and the beam weights; beams are still formed from the window's own raw samples with those
 *              weights; d_R returns Rbar_j.  Rbar_j keeps R_j's exact Hermitian form (mirrored lower triangle, real
 *              diagonal): both parts of every entry follow the same operations.
 *   numerics   the sums are evaluated as a parallel scan over each sub-batch's windows, so their order is not the
 *              recurrence's.  Against the exact recurrence on the same R_j, per entry and part (eps = 2^-53):
 *              |Rbar_gpu - Rbar| <= eps |Rbar| + 1.01 eps (L(W_b) Abar_j + carry_j / c_j), where Abar_j =
 *              sum_k alpha^(j-k) |R_k| / c_j, L(W_b) = 2 ceil(W_b / 32) + 2 ceil(W_b / 8192) + 130 is the rounding depth of
 *              a sub-batch of W_b windows, and carry_j (in units of eps) the carried error of the sub-batches before:
 *              E_b = alpha^(W_b) E_(b-1) + L(W_b) c_end Abar_end at the end of sub-batch b, and carry_j = alpha^(windows
 *              since) E_(b-1) inside sub-batch b (tests/covariance_oracle.py).  c_j and N_eff,j are accurate to a few ulp
 *              at every alpha, including alpha within 2^-52 of 1.  The split of the windows into calls changes Rbar
 *              within that bound only.
 *   counts     MDL / AIC use N_eff,j = N c_j^2 / q_j (fp64, per window) in place of N: N at the first window after a
 *              reset, tending to N (1 + alpha) / (1 - alpha).  The "N <= m" refusals stay on N.
 *   resets     reset_integration(), every set_integration() (the same alpha included), every table setter (set_table,
 *              set_geometry, set_geometry_azel: old covariances describe another manifold) and set_calibration() (the
 *              carry is in corrected coordinates).  Not reset by the peak mode, estimator, source rule, refinement and
 *              beamformer setters.  calib_accumulate_* keep reading raw, unintegrated covariances.  A call with
 *              nwindows = 0, or refused with EINVAL before it enqueues anything, leaves the carry untouched.
 *   ordering   call k + 1 integrates after call k on the same handle, whichever streams they use (an event orders them);
 *              the host entries' chunks, staged on two streams, and the sub-batches of a call integrate in window order.
 *   handles    single-device 1-D handles (process_host, _device, _ex, _counts, both planar entries, both beams entries)
 *              and az-el handles (process_azel_*).  Not built, and refused with EINVAL by set_integration() and
 *              reset_integration(): multi-device handles (their windows are dealt round-robin over the devices) and with
 *              them the sharded entry, handles with a bins all-gather (gather_create() is refused while alpha > 0), and
 *              channel handles (per-channel integration).
 *   kernels    while alpha > 0 every call runs the unfused kernels (the fused M = 4 / M = 8 kernels keep R in registers)
 *              plus integ_tiles_kernel, integ_carry_kernel and integ_apply_kernel per sub-batch, timed in the covariance
 *              slot of the stage timing; MDL / AIC run source_count_neff_kernel.  The carry (S and the window count) lives
 *              in device buffers of the handle.
 */
int music_b200_set_integration(music_b200 *h, double alpha);
int music_b200_reset_integration(music_b200 *h);

/*
 * How precise every direction is (extension, no reference counterpart): the stochastic Cramer-Rao bound of each filled
 * peak slot, evaluated on the device at the window's own covariance and its reported angles (Stoica, Larsson &
 * Gershman, IEEE SP Letters 8(5), 2001; Stoica & Nehorai, IEEE Trans. ASSP 38(10), 1990).  It is the bound for
 * Gaussian sources in white noise at the estimated parameters: the measurement variance a tracker, a triangulation or
 * a display needs, the same whatever peak mode or estimator produced the angles.  It is NOT the variance of the
 * estimator that produced the angle.  For window w:
 *   R          the covariance every other stage reads (what process_device_ex's d_R returns: after the calibration and
 *              the integration).  M = m.
 *   N          nsamples / m, or while integration is on N_eff,j = N c_j^2 / q_j, the value MDL / AIC use.
 *   S          the filled slots {i : bins[w][i] >= 0} in slot order (they need not form a prefix), d = |S|.
 *   steering   for each i in S the reported float angle, widened to fp64, in radians (az-el: the (azimuth, elevation)
 *              pair): a_i with the refinement's convention (1-D: a_m = exp(-j phi_m); az-el: a_m = exp(-j theta_m)), and
 *              the derivative columns, 1-D d_i = da/dt = -j psi o a_i; az-el da/daz = -j theta_az o a_i and
 *              da/del = -j theta_el o a_i (the refinement's psi, theta_az and theta_el).
 *   algorithm  in fp64:
 *              1. A = [a_i] = Q T by modified Gram-Schmidt applied twice (as the DML levels).  The window fails if any
 *                 |T_ii|^2 <= 2^-30 ||a_i||^2.
 *              2. s2 = (tr R - tr(Q^H R Q)) / (M - d), DML's noise level.  The window fails if s2 <= 0 or not finite.
 *              3. H = T^-1 (Q^H R Q) T^-H (= A^+ R A^+H), Gamma = T^-1 T^-H (= (A^H A)^-1), P = H - s2 Gamma (the
 *                 concentrated stochastic-ML source covariance), U = P H^-1 P with H by Cholesky; a pivot that is not
 *                 > 0 fails the window.  P is never inverted: coherent sources (a rank-deficient P) are fine.
 *              4. B = D^H (I - Q Q^H) D over the derivative columns (the columns are projected twice, as step 1).  The
 *                 Fisher matrix over the parameters in slot order: 1-D F_ij = (2 N / s2) Re(B_ij U_ji); az-el with the
 *                 parameters (az_0, el_0, az_1, el_1, ...) F_(i,u),(j,v) = (2 N / s2) Re((d_iu^H P_perp d_jv) U_ji).
 *                 With p_m the element positions and pbar their centroid, G = (2 pi / lambda)^2 sum_m |p_m - pbar|^2 bounds
 *                 B_cc for every direction; the window fails if any B_cc <= 2^-40 G (the parameter is unobservable to
 *                 first order: its derivative vanishes, or lies in span(A), to rounding).
 *              5. C = F^-1 by Cholesky: a pivot <= 2^-40 F_kk (before its square root), or NaN, fails the window.
 *   outputs    1-D std[w][i] = (float)(sqrt(C_ii) 180 / pi), degrees.  Az-el crb[w][i] = {std_az, std_el, rho}: both
 *              standard deviations in degrees and rho = C_(az,el) / sqrt(C_(az,az) C_(el,el)), the dimensionless
 *              correlation (from C in radians).  Unfilled slots get 0; in a failed window every filled slot gets NaN.
 *   caveats    the bound is that of a model with d sources at the reported angles; nothing here tests whether the data
 *              contain them.  n >= 2 under TOP_BINS puts the slots on neighbouring bins of one peak: such windows get
 *              finite values, the bound of two sources one bin apart, which mean nothing for one source (use LOCAL_MAXIMA
 *              or a gridless mode with n >= 2).  The two mirror slots of a line array fail the window (step 1).  A ULA at
 *              end-fire (0 or 180 degrees, where psi vanishes to rounding), a planar array at el = 0 (da/del = 0) and the
 *              azimuth at el = +-90 degrees (da/daz = 0) fail it (step 4).
 * The 1-D entries take the outputs of the beams entries plus d_std [W][n] floats (required); d_weights and d_beams may
 * both be NULL, and otherwise need a beamformer set (as process_*_beams), so that one call returns angles, beams and
 * their bounds (two calls would advance the integration twice).  The az-el entries take the outputs of
 * process_azel_device / _host plus d_crb [W][n][3] floats (required).  Every output is 4-byte aligned (weights and beams
 * as for the beams entries).  The host entry deals windows over a multi-device handle as process_host does; the device
 * entry goes to the device the input lives on.  A CRB call runs the unfused kernels: its angles, levels, spectrum, bins,
 * counts, weights and beams are byte-identical to process_device_ex() with d_R (process_device_beams with weights or
 * beams) on the same windows.  Per sub-batch it adds crb_kernel after the peak stage (and the refinement and the beam
 * weights), timed in the top-n slot of the stage timing.
 * EINVAL, with no fall-back: a current table from set_table() (it has no geometry); channel handles; a 1-D entry on an
 * az-el handle or the reverse; NULL d_std / d_crb; a misaligned output; weights or beams without a beamformer.
 * Not built: the CRB of set_table() manifolds (they would need the table's derivative), of channel handles and of the
 * planar, sharded and gather entries.
 */
int music_b200_process_device_crb(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles, float *d_levels,
                                  float *d_spectrum, int32_t *d_bins, int32_t *d_counts, double *d_weights, float *d_beams,
                                  float *d_std, void *stream);
int music_b200_process_host_crb(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels,
                                float *spectrum, int32_t *bins, int32_t *counts, double *weights, float *beams, float *std_out);
int music_b200_process_azel_device_crb(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_azimuth,
                                       float *d_elevation, float *d_levels, float *d_spectrum, int32_t *d_bins,
                                       int32_t *d_counts, float *d_crb, void *stream);
int music_b200_process_azel_host_crb(music_b200 *h, const float *in_c64, uint32_t nwindows, float *azimuth, float *elevation,
                                     float *levels, float *spectrum, int32_t *bins, int32_t *counts, float *crb);

/*
 * Angle tracking (extension, no reference counterpart): the per-window directions become tracks, each with an identity,
 * an angle, a rate and an uncertainty, carried across windows and calls on the device.  Slot i of window w and slot i
 * of window w + 1 need not be the same emitter (slots are filled in order of strength); a track id is.  One
 * constant-velocity Kalman filter per track (Bar-Shalom, Li & Kirubarajan 2001), global-nearest-neighbour assignment
 * of each window's measurements to the tracks inside a chi-square gate, M-of-N confirmation and deletion after
 * consecutive misses (Blackman & Popoli 1999).  Time is counted in windows, so rates are in degrees per window; the
 * windows are numbered in stream order since the last reset, within a call and on into the next call, as for the
 * integration.  Everything is fp64 in the order written; float outputs are single casts.
 *   setting    variance MUSIC_B200_TRACK_OFF (default), _FIXED: the measurement covariance R_i = floor_deg^2 I (needs
 *              floor_deg > 0), or _CRB: R_i = crb_scale^2 C_crb + floor_deg^2 I (needs crb_scale > 0), where C_crb is the
 *              slot's CRB (process_*_crb) in degrees^2: sigma^2 in 1-D, [[sa^2, rho sa se], [rho sa se, se^2]] in az-el
 *              (evaluated as c2 = crb_scale crb_scale, f2 = floor_deg floor_deg, 1-D R = c2 (s s) + f2; az-el R_00 =
 *              c2 (sa sa) + f2, R_01 = R_10 = c2 ((rho sa) se), R_11 = c2 (se se) + f2; FIXED: R = f2 I).  EINVAL, with the
 *              old setting kept, unless q >= 0, rate_std0 >= 0, floor_deg >= 0 and gate > 0 are all finite,
 *              1 <= confirm_hits <= confirm_window <= 64, max_misses >= 1 and 1 <= max_tracks <= 32.
 *   carry      T = max_tracks rows and a counter next_id (0 after a reset).  A row is empty or a track: id, status
 *              (TENTATIVE or CONFIRMED), state x, covariance P, age, hits and misses (consecutive).  1-D x = (theta,
 *              omega); az-el x = (az, omega_az, el, omega_el), two independent axes with the same model.  H picks the
 *              angle components (theta; az and el).
 *   window w, in this order:
 *              1. predict every live row, per axis: F = [[1, 1], [0, 1]], Q = q [[1/3, 1/2], [1/2, 1]] (the white-noise
 *                 acceleration model with a step of 1; Q = (q / 3, q / 2, q / 2, q)), x <- F x, P <- F P F^T + Q (for each
 *                 2 x 2 block [[a, b], [c, d]] of P: [[(a + c) + (b + d), b + d], [c + d, d]], then + Q on the diagonal
 *                 blocks).  theta (az) is wrapped into [0, 360) by v - 360 floor(v / 360).  age += 1 (age, hits and
 *                 misses saturate at 2^31 - 1).
 *              2. measurements: the slots i in ascending order with bins[w][i] >= 0 (under CRB also with every CRB entry
 *                 of the slot finite: a failed CRB window contributes none), z_i = (double)angles[w][i] (az-el: the
 *                 (azimuth, elevation) pair), R_i as above.
 *              3. for every live row t and measurement i: nu = z_i - H x_t with the angle (azimuth) component wrapped into
 *                 [-180, 180) by v - 360 floor((v + 180) / 360); S = H P H^T + R_i; 1-D d2 = (nu nu) / S; az-el with det
 *                 = S00 S11 - S01 S01, d2 = ((S11 nu0) nu0 - ((2 S01) nu0) nu1 + (S00 nu1) nu1) / det.  The pair is gated
 *                 in iff d2 <= gate (a NaN d2 never is).
 *              4. global nearest neighbour: a matching of gated pairs, each row and each measurement used at most once,
 *                 that minimises sum (d2 - gate) over the matched pairs (the linear assignment on the (rows +
 *                 measurements)-square matrix of the gated d2 augmented with dummy costs gate / 2).  On exact ties any
 *                 minimiser may be taken, the same on every run.
 *              5. update every matched row: 1-D K = P H^T / S; az-el K_j0 = (P_j0 S11 - P_j2 S01) / det, K_j1 = (P_j2 S00 -
 *                 P_j0 S01) / det; x <- x + K nu, wrapped; P <- (I - K H) P (I - K H)^T + K R K^T (Joseph form), the lower
 *                 triangle mirrored from the upper; hits += 1, misses = 0.  Every unmatched live row: misses += 1.
 *              6. status: a TENTATIVE row is confirmed once hits >= confirm_hits, else deleted once it can no longer get
 *                 there, hits + (confirm_window - age) < confirm_hits; a CONFIRMED row is deleted once misses >=
 *                 max_misses.
 *              7. initiation: each unmatched measurement, in ascending slot order, takes the lowest empty row if there is
 *                 one: id = next_id++ (mod 2^31), TENTATIVE (CONFIRMED at once when confirm_hits = 1), x = (z, 0) per
 *                 axis, P with R_i in its angle block and rate_std0^2 on each rate diagonal, age = hits = 1, misses = 0.
 *              8. outputs: slot_track[w][i] = the id of the track slot i's measurement updated or started (tentative or
 *                 confirmed), -1 otherwise (no measurement, or no free row).  track_ids[w][r] = the id of row r if it holds
 *                 a CONFIRMED track after step 7, else -1.  track_state[w][r] for those rows, 0 for the others: 1-D
 *                 {theta, omega, sqrt(P_00)}, az-el {az, omega_az, el, omega_el, sqrt(P_00), sqrt(P_22)}.
 *   entries    the _tracks entries take the outputs of the CRB entries (d_std / d_crb may be NULL: under CRB variance the
 *              bound then goes to a workspace) plus d_slot_track [W][n] (required), and d_track_ids [W][T] with
 *              d_track_state [W][T][3] (az-el [W][T][6]), both or neither; every output 4-byte aligned.  One call
 *              returns everything a window produces, because two calls would advance the integration and the track
 *              carry twice.  Every other output is byte-identical to the matching CRB call (process_device_beams with
 *              weights or beams, process_device_ex with d_R otherwise) on the same windows.  Only the _tracks entries
 *              read the setting: every other entry ignores it and leaves the carry untouched, so windows sent through
 *              other entries are a gap in the tracker's time.  Per sub-batch a tracks call adds one track_kernel launch
 *              (one CTA) after the peak stage, the beams and the CRB, timed in the top-n slot of the stage timing.
 *              get_tracks() waits for the last tracking call and returns the carry: rows [T][5] = {id, status, age, hits,
 *              misses} (an empty row is {-1, MUSIC_B200_TRACK_EMPTY, 0, 0, 0}), state [T][2D + (2D)^2] = x then P
 *              row-major (zeros for an empty row; D = 1, or 2 on an az-el handle), and next_id; any of the three may be
 *              NULL.
 *   resets     reset_tracks(), every set_tracking() (the same parameters included) and every table setter (set_table,
 *              set_geometry, set_geometry_azel).  Not reset by the peak mode, estimator, source rule, refinement,
 *              beamformer, integration or calibration setters.  A call with nwindows = 0, or refused before it enqueues
 *              anything, leaves the carry untouched.  Call k + 1 tracks after call k whatever streams they use; the host
 *              entries' chunks and the sub-batches of a call track in window order.
 *   EINVAL     with no fall-back: a _tracks call while the variance is OFF; CRB variance with a current table from
 *              set_table() (FIXED takes any table); set_tracking() / reset_tracks() on multi-device handles, handles with a
 *              bins all-gather (gather_create() is refused while tracking is on) and channel handles; a 1-D entry on an
 *              az-el handle or the reverse; NULL d_slot_track; only one of d_track_ids / d_track_state; a misaligned
 *              output; weights or beams without a beamformer.
 *   caveats    TOP_BINS with n >= 2 reports neighbouring bins of one peak, which gives two tracks per source: use
 *              LOCAL_MAXIMA or a gridless mode.  The two mirror slots of a line array under the grid modes become two
 *              tracks.  Under integration consecutive measurements are correlated, so the filter's sigma is optimistic.
 *              The CRB is a lower bound: crb_scale and floor_deg absorb the estimator's excess variance and the grid's
 *              quantisation (without refinement a grid angle carries about (360 / K) / sqrt(12) degrees).
 */
#define MUSIC_B200_TRACK_OFF 0
#define MUSIC_B200_TRACK_FIXED 1
#define MUSIC_B200_TRACK_CRB 2
#define MUSIC_B200_TRACK_EMPTY 0      /* get_tracks() row status */
#define MUSIC_B200_TRACK_TENTATIVE 1
#define MUSIC_B200_TRACK_CONFIRMED 2
#define MUSIC_B200_TRACK_MAX_ROWS 32
int music_b200_set_tracking(music_b200 *h, int variance, double q, double rate_std0, double floor_deg, double crb_scale,
                            double gate, uint32_t confirm_hits, uint32_t confirm_window, uint32_t max_misses,
                            uint32_t max_tracks);
int music_b200_reset_tracks(music_b200 *h);
int music_b200_get_tracks(music_b200 *h, int32_t *rows, double *state, uint32_t *next_id);
int music_b200_process_device_tracks(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles,
                                     float *d_levels, float *d_spectrum, int32_t *d_bins, int32_t *d_counts,
                                     double *d_weights, float *d_beams, float *d_std, int32_t *d_slot_track,
                                     int32_t *d_track_ids, float *d_track_state, void *stream);
int music_b200_process_host_tracks(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels,
                                   float *spectrum, int32_t *bins, int32_t *counts, double *weights, float *beams,
                                   float *std_out, int32_t *slot_track, int32_t *track_ids, float *track_state);
int music_b200_process_azel_device_tracks(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_azimuth,
                                          float *d_elevation, float *d_levels, float *d_spectrum, int32_t *d_bins,
                                          int32_t *d_counts, float *d_crb, int32_t *d_slot_track, int32_t *d_track_ids,
                                          float *d_track_state, void *stream);
int music_b200_process_azel_host_tracks(music_b200 *h, const float *in_c64, uint32_t nwindows, float *azimuth,
                                        float *elevation, float *levels, float *spectrum, int32_t *bins, int32_t *counts,
                                        float *crb, int32_t *slot_track, int32_t *track_ids, float *track_state);

/*
 * Downstream reducers (extension, no reference counterpart): what a GUI-rate consumer such as the DOA
 * compass (/root/reference/python/doa_compass_control.py:102-108) or a plot sink
 * (/root/reference/python/plot_sink.py:38) needs from millions of windows per second.
 *   reduce_angles: for every angle slot i < n the CIRCULAR mean over nwindows of angles[w][i] (degrees in
 *     [0, 360)), the mean resultant length (1: all windows agree, 0: spread uniformly) and the total
 *     weight.  A window counts iff levels == NULL or levels[w][i] > 0 (unfilled slots carry level 0);
 *     weighted != 0 weights each window by its level.  resultant / weight_sum may be NULL.
 *   reduce_spectrum: mean over nwindows of spectrum[w][k], k < resolution.
 * _device: buffers in device memory, enqueued on `stream`; _host: host buffers (upload, reduce, download).
 */
int music_b200_reduce_angles_device(music_b200 *h, const float *d_angles, const float *d_levels, uint32_t nwindows, int weighted,
                                    float *d_mean_deg, float *d_resultant, float *d_weight_sum, void *stream);
int music_b200_reduce_spectrum_device(music_b200 *h, const float *d_spectrum, uint32_t nwindows, float *d_mean, void *stream);
int music_b200_reduce_angles_host(music_b200 *h, const float *angles, const float *levels, uint32_t nwindows, int weighted,
                                  float *mean_deg, float *resultant, float *weight_sum);
int music_b200_reduce_spectrum_host(music_b200 *h, const float *spectrum, uint32_t nwindows, float *mean);

/*
 * Planar input: one c64 stream per antenna instead of interleaved items.  Window w is
 *     x_w(r, c) = streams[r][w * hop + c],   r < m, c < N = nsamples / m,
 * i.e. what the flowgraph in front of the reference block builds on the CPU by interleaving the
 * antenna streams (/root/reference/lib/baz_interleaver.cc:152-229), cutting vectors and, for
 * sliding windows, re-copying the overlap (/root/reference/lib/baz_overlap.cc:107-129) before
 * baz_music_doa::work() reshapes it back (/root/reference/lib/baz_music_doa.cc:82-84).
 * hop == N: back-to-back windows; hop < N: windows overlap by N - hop snapshots; hop > N: gaps.
 * Each stream must hold (nwindows - 1) * hop + N samples.  Outputs as in process_host/_device.
 * Results equal those of process_*() on the interleaved windows up to fp64 rounding of R (the planar kernels sum the
 * snapshots in a different order for m > 4): P(theta) agrees to ~1e-12 relative, peak bins are equal except where two
 * bins' strengths tie to within that rounding (in practice the 90/270 degree pair of an x-axis ULA).
 *   _host  : streams[r] are host pointers (copied to the device in chunks, planar, no interleave)
 *   _device: d_streams is a HOST array of m device pointers (8-byte aligned), work is enqueued on `stream`
 */
int music_b200_process_planar_host(music_b200 *h, const float *const *streams, uint32_t hop, uint32_t nwindows,
                                   float *angles, float *levels, float *spectrum, int32_t *bins);
int music_b200_process_planar_device(music_b200 *h, const float *const *d_streams, uint32_t hop, uint32_t nwindows,
                                     float *d_angles, float *d_levels, float *d_spectrum, int32_t *d_bins, void *stream);

/*
 * Retune without marshalling a table: builds the array response ON THE DEVICE from the element
 * positions and the wavelength, i.e. replaces calculate_antenna_array_response() + the SWIG
 * complex128 -> complex64 conversion + set_array_response()
 * (/root/reference/python/music_doa_helper.py:29-46, :100-103; swig/baz_swig.i:564) by one call.
 * positions_xy: [m][2] doubles in metres, already multiplied by array_spacing
 * (music_doa_helper.py:56); wavelength = 299792458 / frequency (:55, :101).
 * The resulting table is bit-identical to the one the Python helper computes on this host:
 * entries whose float32 rounding could depend on the last bits of sin/cos are re-evaluated
 * with the host libm; *guarded (may be NULL) receives how many (typically ~3e-5 of 2*m*K).
 * Same locking and double buffering as music_b200_set_table().
 */
int music_b200_set_geometry(music_b200 *h, const double *positions_xy, double wavelength, uint32_t *guarded);

/*
 * Test hook (no device needed): the host-libm evaluation of one table entry that
 * music_b200_set_geometry() uses for the guarded entries; re_im = {Re, Im} as float32.
 */
void music_b200_steer_entry_host(const double *positions_xy, double wavelength, uint32_t resolution, uint32_t step,
                                 uint32_t antenna, float *re_im);

/*
 * (azimuth, elevation) MUSIC over a 3-D array geometry (extension, no reference counterpart).
 * An az-el handle has n_az azimuth steps, n_el elevation steps, an elevation range [el_lo, el_hi] in degrees
 * (-90 <= el_lo <= el_hi <= 90), element positions p_m = (x, y, z) in metres and a wavelength lambda.
 *   grid       az_k = k * 360 / n_az degrees (k < n_az);  el_i = el_lo + (i * (el_hi - el_lo)) / (n_el - 1), el_0 = el_lo
 *              for n_el = 1; both evaluated in fp64 in exactly this order.
 *   direction  u(az, el) = (cos el cos az, cos el sin az, sin el), el measured from the xy-plane (at el = 0 this is the
 *              reference helper's unit_vect).
 *   steering   a_m(az, el) = exp(-j 2 pi <p_m, u> / lambda) (the helper's sign convention).
 *   table      table[i][k][m] = a_m(az_k, el_i) in fp64 rounded to complex64, flat bin b = i * n_az + k, so the handle
 *              scans K = n_az * n_el rows, elevation-major.  Each component is within one float32 ulp of the fp64 value
 *              (there is no host helper to be bit-identical to); music_b200_get_table() returns the table in use.
 *   per window R, eigenvectors, noise subspace and P[b] = 1 / ||G^H a_b||^2 exactly as for a 1-D handle with K = n_az * n_el;
 *              the source rules (FIXED / MDL / AIC) apply unchanged.
 *   outputs    bins = b;  azimuth = (float)(k * 360.0 / n_az) (the 1-D angle expression);  elevation = (float)el_i;
 *              level = (float)P[b];  unfilled slots (0, 0, 0, bin -1);  spectrum [W][n_el][n_az] float32.
 *   peak rules MUSIC_B200_PEAKS_TOP_BINS (default): the reference's rule on the flat index (the n largest bins, strict
 *              '>', lowest b on ties).  MUSIC_B200_PEAKS_LOCAL_MAXIMA: b is a candidate iff P[b] > 0 and, for each of its
 *              up to 8 grid neighbours j (azimuth circular, elevation rows do not wrap), P[b] > P[j] or (P[b] == P[j] and
 *              b < j); peaks are taken in descending strength, ties to the lowest b, skipping a candidate whose Chebyshev
 *              grid distance max(min(|dk|, n_az - |dk|), |di|) to a peak already taken is <= exclusion_bins.  The tie
 *              clause gives a constant row (the zenith row of a planar array) exactly one maximum.
 *   refinement MUSIC_B200_REFINE_NEWTON (geometric tables only, as in 1-D) minimises the exact fp64
 *              D(az, el) = sum_j |g_j^H a(az, el)|^2 (G the noise eigenvectors the scan used) inside the box
 *              [az_b -+ d_az] x [max(el_b - d_el, el_lo), min(el_b + d_el, el_hi)], d_az = 360 / n_az, d_el = one
 *              elevation step (0 for n_el = 1), angles in radians, gradient g and Hessian H analytic
 *              (theta_m = 2 pi <p_m, u> / lambda; d2 theta_m / d el2 = -theta_m).  At most 50 iterations of:
 *                1. s = -H^-1 g if H11 > 0 and det H > 0, else s = -g d_az / ||g||; stop if g = 0;
 *                2. s = clamp(x + s) - x, the clamp componentwise into the box;
 *                3. halve t from 1 while t > 2^-30 until D(x + t s) <= D(x); stop if there is no such t;
 *                4. x = x + t s; stop once max |t s| <= 1e-12 rad.
 *              x* is kept iff x* != x_b and D(x*) <= D(x_b): azimuth = (float) of x*_az in degrees wrapped into
 *              [0, 360) as in 1-D, elevation = (float) of x*_el in degrees; otherwise the slot keeps its grid angles.
 *              level = (float)(1 / D) at the point kept (as in 1-D, the analytic level even where the grid point is
 *              kept).  Bins, spectrum and counts stay the grid results.
 * Caveat: for a planar array (all z equal) +el and -el have bit-identical table rows, so on a grid with el_lo < 0 the
 * tie rules resolve every such pair to the negative elevation (the lower b).  Use el_lo >= 0 for planar arrays.
 * An az-el handle is single-device and always runs the unfused kernels (plus the decode and, with refinement, the 2-D
 * refinement kernel, both timed in the top-n slot of the stage timing).  set_table() accepts a [n_el][n_az][m] table (a
 * measured or calibrated manifold; refinement then returns EINVAL, as in 1-D); set_peak_mode(), set_source_rule(),
 * set_refine(), the stage timing, get_table(), the reducers and launch_count() work as on a 1-D handle.  The 1-D
 * process_* entries, set_geometry(), the planar entries and the gather / sharded entries return EINVAL on an az-el
 * handle; set_geometry_azel() and the _azel entries return EINVAL on a 1-D handle.
 *
 * create_azel: positions_xyz [m][3] doubles (finite), wavelength finite and > 0, 1 <= n < m <= MUSIC_B200_MAX_M,
 * nsamples a positive multiple of m, n_az, n_el >= 1 with n_az * n_el <= MUSIC_B200_AZEL_MAX_BINS, el_lo < el_hi when
 * n_el >= 2.  The argument checks come first (EINVAL); ENODEVICE without an sm_90 device.
 * set_geometry_azel: retune, with the locking and double buffering of music_b200_set_table().
 * process_azel_host / _device: as process_host_counts / process_device_counts, plus the elevations (n floats per
 * window, required like the azimuths); levels, spectrum, bins and counts may be NULL.
 *
 * MUSIC_B200_PEAKS_ESPRIT on an az-el handle (extension, 2-D LS-ESPRIT): gridless (azimuth, elevation) pairs from the two
 * shift invariances of a planar lattice (uniform rectangular or any other 2-D lattice) array.  Covariance, eigensolver,
 * source rules and spectrum are unchanged.  (On a 1-D handle the mode keeps the ULA meaning above.)
 *   lattice    evaluated on the positions p_m = (x, y, z) at create_azel / set_geometry_azel and kept with the table: for
 *              each divisor Mx of M with 2 <= Mx <= M / 2, ascending, My = M / Mx, s1 = (p_1 - p_0)_xy,
 *              s2 = (p_Mx - p_0)_xy.  The geometry is the lattice (Mx, My, s1, s2) when |s1|, |s2| > 0,
 *              |s1 x s2| > 1e-6 |s1| |s2|, every element m = k Mx + i lies within 1e-6 min(|s1|, |s2|) of
 *              p_0 + i s1 + k s2 in xy with |z_m - z_0| within the same bound, and |s1|, |s2| <= (lambda / 2)(1 + 1e-12).
 *              At most one Mx passes.  Row-major element order; column-major passes with s1 and s2 swapped; rotated,
 *              non-orthogonal (e.g. triangular) lattices, any p_0 and z_0 pass.  music_b200_azel_lattice_host() tests it.
 *   doublets   P1 = {(m(i, k), m(i + 1, k)) : i < Mx - 1}, P2 = {(m(i, k), m(i, k + 1)) : k < My - 1}, both in ascending
 *              first index; d_max = min((Mx - 1) My, Mx (My - 1)).
 *   subspace   E_s = the d eigenvectors of largest eigenvalue (d = n, or the MDL / AIC count); A_j = the rows of E_s at
 *              the first indices of P_j, B_j = the rows at the second indices.
 *   matrices   G_j = A_j^H A_j, C_j = A_j^H B_j, Psi_j = G_j^-1 C_j in fp64 by Cholesky of G_j (lower, row by row).  G_j =
 *              I - (excluded rows)^H (excluded rows) has its eigenvalues in [0, 1]: a pivot <= 2^-40 before its square
 *              root (or NaN) means no peaks for the window, as do d = 0, d > d_max and a non-finite Psi_j.
 *   pairing    Psi_c = Psi_1 + gamma Psi_2, gamma = 0.37 + 0.61 j.  Complex Schur form Psi_c = Z S Z^H by ESPRIT's
 *              Householder + shifted QR (above) with the whole rows and columns updated and Z accumulated (zlahqr's
 *              wantt / wantz); a window needing more than 30 QR steps between deflations reports no peaks.  Eigenvector
 *              k of S: y_k = 1, y_j = 0 for j > k, y_j = -(sum_{l=j+1..k} S_jl y_l) / (S_jj - S_kk) for j = k-1 .. 0,
 *              a divisor of modulus < smin = max(2^-52 |S_kk|, 2^-1022) replaced by smin (LAPACK ztrevc); x_k = Z y_k.
 *              phi_jk = x_k^H Psi_j x_k / x_k^H x_k, the two phases of one source, already paired.  They depend only on
 *              span(E_s).
 *   direction  omega_j = -arg(phi_j) lambda / (2 pi) = s_j . u_xy; [s1; s2] u_xy = omega solved in fp64, rho = |u_xy|;
 *              az = atan2(u_y, u_x) in degrees wrapped into [0, 360), el = acos(min(rho, 1)) in degrees (>= 0: a planar
 *              array cannot tell +el from -el), negated when the handle's el_hi <= 0.  A phi exactly 0 or not finite
 *              leaves its slot unfilled.
 *   outputs    azimuth, elevation = float casts (360 -> 0 as in refinement); level = (float)(1 / D(az, el)), D the direct
 *              fp64 form of the refinement over the M - d noise eigenvectors at the unrounded angles; bin = i n_az + k,
 *              k = floor(az n_az / 360 + 0.5) mod n_az, i = clamp(floor((el - el_lo)(n_el - 1) / (el_hi - el_lo) + 0.5),
 *              0, n_el - 1) (i = 0 for n_el = 1).  Slots 0 .. d-1 in descending fp64 level, exact ties to the lower
 *              azimuth, then the lower elevation, then the lower Schur diagonal index.  Slots d .. n-1, windows without
 *              peaks and windows with a NaN level report (0, 0, 0, bin -1).  Spectrum and counts are unchanged; the grid
 *              scan runs only when the spectrum is requested; the bin decode does not run.
 * Restrictions, checked in either order like 1-D ESPRIT: exclusion_bins = 0, estimator MUSIC, refinement OFF; a current
 * table from set_geometry_azel() of a lattice (a process_*() call on a set_table() table or on another geometry returns
 * EINVAL, with no fall-back to grid peaks); n <= d_max (the MDL / AIC count never exceeds n, so it never exceeds d_max
 * either).  ROOTS, MANIFOLD and DML stay refused on az-el handles.  A call runs covariance (+ calibration), eigensolver
 * (+ source count), [scan], then one ESPRIT kernel per sub-batch, timed in the top-n slot of the stage timing.
 */
#define MUSIC_B200_AZEL_MAX_BINS (1u << 20)
int music_b200_create_azel(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t n_az, uint32_t n_el,
                           double el_lo_deg, double el_hi_deg, const double *positions_xyz /* [m][3] */, double wavelength,
                           int device);
int music_b200_set_geometry_azel(music_b200 *h, const double *positions_xyz /* [m][3] */, double wavelength);
int music_b200_process_azel_host(music_b200 *h, const float *in_c64, uint32_t nwindows, float *azimuth, float *elevation,
                                 float *levels, float *spectrum, int32_t *bins, int32_t *counts);
int music_b200_process_azel_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_azimuth, float *d_elevation,
                                   float *d_levels, float *d_spectrum, int32_t *d_bins, int32_t *d_counts, void *stream);

/*
 * Test hook of the az-el ESPRIT mode's lattice condition (no device needed): for positions [m][x, y, z] (metres) at
 * `wavelength`, the lattice shape Mx, My and the steps s = {s1_x, s1_y, s2_x, s2_y}.  Returns EINVAL for a geometry that
 * is not a lattice, and for invalid arguments.
 */
int music_b200_azel_lattice_host(const double *positions_xyz, uint32_t m, double wavelength, int *mx, int *my, double s[4]);

/*
 * Frequency-channelised direction finding (extension, no reference counterpart): an FFT filter bank fused into the
 * covariance, one direction-finding problem per frequency channel, and the incoherent wideband MUSIC spectrum.  Every
 * other mode starts from one covariance over the whole sampled bandwidth; a channel handle separates emitters at
 * different frequencies and matches each channel against a table built for that channel's own wavelength.
 * A channel handle has, besides m, n, nsamples (N = nsamples / m snapshots) and resolution (K): an FFT length F = nfft
 * (a power of two, 8 <= F <= 256, F | N), a channel range (chan_first < F, 1 <= chan_count = C <= F), a taper and a
 * combine rule.
 *   segments   window w is cut into J = N / F consecutive, non-overlapping segments of F snapshots.
 *   filter bank  X_j[b] = sum_{t<F} h[t] x[jF + t] exp(-2 pi i b t / F) (an m-vector), h = 1 (MUSIC_B200_TAPER_RECT) or the
 *              periodic Hann h[t] = 1/2 - 1/2 cos(2 pi t / F) (MUSIC_B200_TAPER_HANN).
 *   channels   channel c in [0, C) is FFT bin b_c = (chan_first + c) mod F, so a range may wrap through the negative
 *              frequencies, at frequency offset f_c = fs * (s(b_c) / F), s(b) = b for b < F / 2 and b - F otherwise
 *              (evaluated in fp64 in exactly this order; music_b200_channel_frequencies returns f_c).
 *   covariance R_c = sum_j X_j[b_c] X_j[b_c]^H / (J sum_t h[t]^2), fp64 throughout (the inputs widen exactly).  White
 *              noise of power s2 gives R_c ~ s2 I in every channel; for RECT (1 / F) sum_b R_b is the plain handle's R.
 *              R_c does not depend on which other channels the handle has.
 *   tables     set_geometry_channels(positions_xy, f_centre, fs) builds one table per channel with the device builder of
 *              music_b200_set_geometry(): a_c(theta)[r] = exp(-j 2 pi <p_r, u(theta)> / lambda_c),
 *              lambda_c = 299792458.0 / (f_centre + f_c), bit-identical to set_geometry(positions_xy, lambda_c) on a plain
 *              handle.  f_centre must exceed fs / 2.  music_b200_set_table() on a channel handle installs ONE measured
 *              table for all channels: that is the narrowband assumption, and the caller's choice.  create_channels()
 *              installs no table: a process call before either returns EINVAL.  music_b200_get_table_channel() returns
 *              channel c's table; music_b200_get_table() returns EINVAL on a channel handle.
 *   SEPARATE   every (window, channel) is an ordinary problem on (R_c, table_c): estimator MUSIC / MVDR / BARTLETT, peak
 *              mode TOP_BINS / LOCAL_MAXIMA, source rule FIXED / MDL / AIC with their definitions above, except that MDL,
 *              AIC and the N <= m conditions use J, the number of segments (the independent looks), in place of N.  Under
 *              MDL a count of 0 is how an empty channel shows.
 *              Outputs are channel-major: angles / levels / bins [C][W][n], counts [C][W], spectrum [C][W][K]; channel
 *              c's block is what a plain handle would have written for (R_c, table_c).
 *   INCOHERENT (Wax, Shan and Kailath 1984) one problem per window: P(theta_k) = 1 / sum_c (1 / P_c(theta_k)), P_c channel
 *              c's MUSIC strength with its own table, i.e. 1 / sum_c ||G_c^H a_c(theta_k)||^2, summed in channel order;
 *              then the peak mode on P.  MUSIC estimator and FIXED rule only.  angles / levels / bins [W][n],
 *              spectrum [W][K], counts must be NULL.
 *   COHERENT   (the coherent signal-subspace method, Wang and Kaveh 1985, with the rotational focusing matrices of Hung and
 *              Kaveh 1988) one ordinary problem per window on a focused covariance:
 *     reference  channel c_ref = C / 2 (integer division) at lambda_ref = lambda_{c_ref}; its table is the reference table.
 *     sector     grid bins S = {(first + i) mod K : i < count}, the whole grid (0, K) unless music_b200_set_focusing()
 *                chose another; the sector persists across set_geometry_channels() retunes.
 *     steering   fp64 vectors from the geometry (not the float tables): a_c(theta)[r] = exp(-j 2 pi <p_r, u(theta)> / lambda_c).
 *     focusing   B_c = sum_{k in S} a_ref(theta_k) a_c(theta_k)^H + beta |S| I, beta = 1e-3; T_c = U V^H from the SVD
 *                B_c = U S V^H, the unitary minimiser of sum_k ||a_ref - T a_c||^2; T_{c_ref} = I exactly (not computed).
 *                beta keeps T_c unique on sectors narrower than the array's degrees of freedom.  When
 *                sigma_min(B_c) <= 1e-12 sigma_max(B_c) for some c, set_geometry_channels() / set_focusing() return EINVAL
 *                and name the channel; the handle keeps its previous matrices.  The matrices are built on every
 *                set_geometry_channels() and set_focusing(), in the idle table slot beside its channel tables, which then
 *                becomes current (set_focusing() copies the current tables into it), after a device synchronise as in
 *                every table setter.
 *     error      e_c = ||T_c A_c - A_ref||_F / ||A_ref||_F over the columns a(theta_k), k in S (music_b200_get_focusing).
 *     covariance R_foc = (1 / C) sum_c T_c R_c T_c^H in fp64, summed in channel order, the c_ref term R_ref itself (added
 *                without multiplication); upper triangle as summed, lower triangle its mirror, diagonal real.
 *     problem    (R_foc, reference table) with J * C looks in place of N (MDL, AIC and the N <= m conditions): estimator
 *                MUSIC / MVDR / BARTLETT, peak mode TOP_BINS / LOCAL_MAXIMA / ROOTS / ESPRIT / DML (ROOTS and ESPRIT need
 *                a ULA with spacing <= lambda_ref / 2), source rule FIXED / MDL / AIC, refinement OFF / NEWTON on the
 *                reference geometry.  With C = 1 every output equals SEPARATE's.
 *     outputs    angles / levels / bins [W][n], spectrum [W][K], counts [W], R [W][m][m] holding R_foc.
 *     caveat     the focusing error moves signal power into the noise eigenvalues, so MDL and AIC over-count at high
 *                SNR (in a two-path UCA-8 case at 20 dB per element, MDL gave 4 for 2).
 *              music_b200_set_table() is refused on a COHERENT handle (one shared table gives no focusing).
 *   R          (SEPARATE, INCOHERENT, may be NULL) [C][W][m][m] complex fp64.
 * Not built, and refused with EINVAL rather than ignored: under SEPARATE and INCOHERENT the ROOTS, ESPRIT and DML peak modes and refinement; on every channel handle beams
 * (set_beamformer), calibration (set_calibration and the calib entries), the planar, sharded, gather and az-el entries and
 * set_geometry() on a channel handle; create_multi() makes no channel handle.  The plain process entries on a channel
 * handle and the channel entries on a plain handle return EINVAL.  Segments do not overlap.
 * A call runs, per sub-batch: chan_cov_kernel (the filter bank and all C covariances, one read of the input per channel
 * group; timed in the covariance slot of the stage timing), then the eigensolver, source count and MVDR preparation of the
 * plain unfused path once over all C * W (window, channel) pairs, then one scan and one peak-rule launch per channel on
 * that channel's table, and under INCOHERENT one combine kernel and one peak-rule launch.  Under COHERENT a sub-batch runs
 * chan_cov_kernel, chan_focus_kernel (timed in the covariance slot) and the plain unfused stages once over its W focused
 * covariances, whatever C is.  set_estimator, set_peak_mode,
 * set_source_rule, stage timing, the reducers and launch_count work as on any handle.
 * The device entry is enqueued on `stream` and does not synchronise; d_in must be 16-byte aligned.  The host entry copies
 * in chunks and returns when done.
 */
#define MUSIC_B200_TAPER_RECT 0
#define MUSIC_B200_TAPER_HANN 1
#define MUSIC_B200_CHANNELS_SEPARATE 0
#define MUSIC_B200_CHANNELS_INCOHERENT 1
#define MUSIC_B200_CHANNELS_COHERENT 2
int music_b200_create_channels(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution, uint32_t nfft,
                               uint32_t chan_first, uint32_t chan_count, int taper, int combine, int device);
int music_b200_set_geometry_channels(music_b200 *h, const double *positions_xy /* [m][2] */, double centre_frequency_hz,
                                     double sample_rate_hz);
int music_b200_channel_frequencies(music_b200 *h, double *offsets_hz /* [C] */);
int music_b200_get_table_channel(music_b200 *h, uint32_t channel, float *table_c64);
/* COHERENT handles only (EINVAL otherwise).  set_focusing: the sector (1 <= bin_count <= K, first_bin < K), rebuilding the
 * matrices when a geometry exists.  get_focusing: T [C][m][m] complex fp64 and e_c [C] (either may be NULL); EINVAL
 * before set_geometry_channels(). */
int music_b200_set_focusing(music_b200 *h, uint32_t first_bin, uint32_t bin_count);
int music_b200_get_focusing(music_b200 *h, double *T, double *err);
int music_b200_process_channels_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles, float *d_levels,
                                       float *d_spectrum, int32_t *d_bins, int32_t *d_counts, double *d_R, void *stream);
int music_b200_process_channels_host(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels,
                                     float *spectrum, int32_t *bins, int32_t *counts, double *R);

/*
 * Sparse linear arrays through the difference co-array (music_coarray.cuh; Moffet 1968, Pillai, Bar-Ness & Haber 1985,
 * Pal & Vaidyanathan 2010, Vaidyanathan & Pal 2011, Liu & Vaidyanathan 2015): up to Mv - 1 uncorrelated sources from
 * m < Mv antennas.  Restated literally by tests/coarray_oracle.py.
 *   inputs     m physical elements (2 <= m <= MUSIC_B200_MAX_M) at integer positions p_0 = 0 < p_1 < ... < p_{m-1} in
 *              units of the step s = (s_x, s_y) metres (finite, 0 < |s| <= (lambda / 2)(1 + 1e-12)), the wavelength lambda
 *              (finite, > 0) and the virtual size Mv.  Each input snapshot holds the m physical channels, nsamples a
 *              positive multiple of m, N = nsamples / m snapshots per window.
 *   extent     U = the largest value with every lag 0 .. U - 1 some p_i - p_j.  2 <= Mv <= min(U, 16); mv = 0 chooses
 *              min(U, 16) (music_b200_coarray_size() reads it back).  E.g. the nested array {0, 1, 2, 3, 4, 9, 14, 19} has
 *              U = 20 and runs with Mv = 16.  1 <= n < Mv: n may exceed m.
 *   lag table  for l = 0 .. Mv - 1 the pairs (i, j) with p_i - p_j = l in ascending i, c_l of them (built at create).
 *   per window R = the window's fp64 covariance of the m physical channels, after calibration and integration exactly as
 *              on a 1-D handle (both act on the physical R, before the mapping: the mapping is not linear, so an
 *              integrated co-array covariance is the map of the integrated R, not an average of maps);
 *              z_l = (1 / c_l) sum R_ij over the lag-l pairs in table order;
 *              T_ab = z_{a-b} for a >= b, conj(z_{b-a}) for a < b (Hermitian Toeplitz, Mv x Mv);
 *              R_ss = (1 / Mv) T T^H, each entry a sum over k ascending, computed for a >= b, the upper triangle its
 *              conjugate mirror, the diagonal real.  R_ss (= T^2 / Mv) has T's eigenvectors and is positive semi-definite,
 *              so the ascending eigensolver puts the noise subspace first even where a finite-sample T is indefinite.
 *   problem    R_ss is the window's R for every later stage and for the R and eigenvalue outputs of
 *              music_b200_process_device_ex ([W][Mv][Mv] and [W][Mv]).  The table is the steering table of the Mv-element
 *              ULA at l s, l < Mv, built by the set_geometry() table builder with M = Mv (bit-identical to a plain
 *              handle's set_geometry() on those positions; ROOTS and ESPRIT see a ULA).  get_table() returns [K][Mv].
 *              Angles follow the plain x-axis ULA conventions: ROOTS and ESPRIT give mirror-free angles; the grid modes
 *              on a line array carry the mirror peaks.
 *   caveat     the co-array model needs mutually uncorrelated sources.  Correlated or coherent sources break the Toeplitz
 *              structure: DML, WSF or IAA on a plain handle serve them.
 * Accepted: estimator MUSIC; peak modes TOP_BINS, LOCAL_MAXIMA, ROOTS, ESPRIT; refinement OFF or NEWTON (on the virtual
 * ULA's analytic steering); source rule FIXED; set_calibration() with m physical gains; set_integration(); the process
 * host / device / device_ex / counts / planar entries and the tracks entries under FIXED variance; the spectrum port, the
 * reducers, stage timing and get_table().  Refused with EINVAL, in either setting order: MVDR, Bartlett and IAA; DML, WSF
 * and MANIFOLD; MDL and AIC (the eigenvalues of R_ss are squares, so the Wishart-based criteria do not apply); JOINT
 * refinement; the CRB entries and tracking under CRB variance; the beamformer and the beams entries; calib_accumulate /
 * calib_solve and every calib_blind_* call (estimate the gains on a plain handle of the same receivers, then call
 * set_calibration() here); set_table() and set_geometry(); the sharded and gather entries.  create_multi() makes no
 * co-array handle.
 * A call never takes the fused kernels: per sub-batch the covariance of the m channels, the calibration and the
 * integration write a physical-R buffer beside the workspace, coarray_kernel maps it into the workspace R (timed in the
 * covariance slot of the stage timing), then the plain unfused stages run on Mv.
 * music_b200_create_coarray: argument checks (EINVAL) before device checks (ENODEVICE).
 * music_b200_set_geometry_coarray: the retune after an LO change - the virtual table rebuilt from a new step and
 * wavelength through the table double buffer, resetting integration and tracks like every retune.
 */
int music_b200_create_coarray(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution, const int32_t *positions,
                              const double step_xy[2], double wavelength, uint32_t mv, int device);
int music_b200_set_geometry_coarray(music_b200 *h, const double step_xy[2], double wavelength);
int music_b200_coarray_size(music_b200 *h, uint32_t *mv);

/* Copies the table currently in use (float[resolution][m][2]) back to host memory. */
int music_b200_get_table(music_b200 *h, float *table_c64);

/*
 * Replaces the body of baz_music_doa::work() (/root/reference/lib/baz_music_doa.cc:72-161)
 * for `nwindows` consecutive input items held in HOST memory (what the GNU Radio scheduler
 * hands to work(): input_items[0], output_items[0..2]).  Host<->device copies are done
 * inside (chunked, double-buffered).  levels / spectrum / bins may be NULL, mirroring
 * output_items.size() (:97-99, :148-149); NULL skips that work.
 * Pageable caller memory (GNU Radio's circular buffers, numpy arrays) of 1 MiB or more is pinned with cudaHostRegister
 * the first time it is seen and remembered in the handle (up to 16 ranges; released by destroy()), so that later calls
 * on the same buffers copy at the pinned rate; MUSIC_B200_HOSTREG=0 in the environment turns that off.
 */
int music_b200_process_host(music_b200 *h, const float *in_c64, uint32_t nwindows,
                            float *angles, float *levels, float *spectrum, int32_t *bins);

/*
 * Same computation with all buffers already resident in device memory (the streaming /
 * benchmark path, and the entry a device-resident upstream block would call).  Enqueued on
 * `stream` (a cudaStream_t, NULL = legacy default stream); does not synchronise.
 * d_in must be 16-byte aligned.
 * m = 4, n = 1 (and m = 8, n = 1 without the spectrum) run as ONE persistent kernel per call; consecutive calls of the
 * m = 4 kernel on one stream overlap their launch tails (programmatic dependent launch) while their results still
 * land in stream order.  d_spectrum != NULL (reference :120-121) keeps m = 4 / n = 1 on that kernel (its fp64 workers
 * write the spectrum); other shapes then take the three-kernel path.
 */
int music_b200_process_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows,
                              float *d_angles, float *d_levels, float *d_spectrum,
                              int32_t *d_bins, void *stream);

/*
 * process_device plus optional fp64 internals for stage-by-stage parity tests against the
 * oracle (any of them may be NULL):
 *   d_P64     [nwindows][resolution]  strength = 1/||G^H a||^2 before the float cast (:114-119)
 *   d_R       [nwindows][m][m][2]     covariance R = x x^H / N (:85)
 *   d_eigvals [nwindows][m]           ascending eigenvalues (:88-90)
 */
int music_b200_process_device_ex(music_b200 *h, const float *d_in_c64, uint32_t nwindows,
                                 float *d_angles, float *d_levels, float *d_spectrum,
                                 int32_t *d_bins, double *d_P64, double *d_R,
                                 double *d_eigvals, void *stream);

/*
 * process_host / process_device plus the per-window source counts (music_b200_set_source_rule):
 * counts / d_counts: int32 [nwindows] in host / device memory (may be NULL), in stream order on a multi-device handle.
 * Under the FIXED rule every count is n.  The planar and sharded entries honour the rule too, but return no counts.
 */
int music_b200_process_host_counts(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels,
                                   float *spectrum, int32_t *bins, int32_t *counts);
int music_b200_process_device_counts(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles,
                                     float *d_levels, float *d_spectrum, int32_t *d_bins, int32_t *d_counts, void *stream);

/* Number of CUDA kernels this handle has launched so far (bench.py's gpu_launches). */
uint64_t music_b200_launch_count(const music_b200 *h);

/*
 * Optional per-stage device timing for the benchmark's roofline leg.  While enabled, every
 * internal chunk records CUDA events on the launch stream around K1 (covariance), K2
 * (eigendecomposition), K3 (scan) and the top-n kernel.  get_stage_times() synchronises on
 * them, returns the accumulated milliseconds since the last call in ms4[0..3] and the number
 * of chunks in *chunks (may be NULL), then resets the accumulation.
 */
int music_b200_set_stage_timing(music_b200 *h, int enable);
int music_b200_get_stage_times(music_b200 *h, double *ms4, uint64_t *chunks);

/* Debug: copy the first max_ctas rows of the fused kernel's per-CTA trace (40 int64 per row; only when
 * the handle was created with MUSIC_B200_TRACE=1 in the environment).  The trace is a ring of 32
 * launches of 1024 rows: the l-th fused launch of the handle writes rows [(l % 32) * 1024, .. + grid). */
int music_b200_debug_fused_trace(music_b200 *h, long long *host_out, int max_ctas);

/* Debug: cumulative window counts of the fused M = 8 kernel - out2[0] solved by the principal-eigenvector (squaring) solver,
 * out2[1] by the Jacobi fallback. */
int music_b200_debug_fused8_stats(music_b200 *h, uint64_t *out2);

/* Last error text for this handle; h == NULL returns the last create() failure. */
const char *music_b200_last_error(const music_b200 *h);

void music_b200_destroy(music_b200 *h);

#ifdef __cplusplus
}
#endif
#endif /* MUSIC_B200_H */
