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
 * compute-capability 10.x GPU.
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
 *   roots      Aberth-Ehrlich iteration in fp64 (starting points on the unit circle, at most 100 steps).  Two roots that
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
 */
#define MUSIC_B200_PEAKS_TOP_BINS 0
#define MUSIC_B200_PEAKS_LOCAL_MAXIMA 1
#define MUSIC_B200_PEAKS_ROOTS 2
int music_b200_set_peak_mode(music_b200 *h, int mode, uint32_t exclusion_bins);

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
#define MUSIC_B200_REFINE_OFF 0
#define MUSIC_B200_REFINE_NEWTON 1
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
 */
#define MUSIC_B200_ESTIMATOR_MUSIC 0
#define MUSIC_B200_ESTIMATOR_MVDR 1
#define MUSIC_B200_ESTIMATOR_BARTLETT 2
int music_b200_set_estimator(music_b200 *h, int estimator, double loading);

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
