/* -*- c++ -*- */
/*
 * baz_music_doa.h - H100-native replacement for gr-baz's MUSIC DOA block.
 *
 * Same public surface as /root/reference/lib/baz_music_doa.h:29-60: class baz_music_doa :
 * gr::sync_block, friend factory baz_make_music_doa(m, n, nsamples, array_response,
 * resolution), work(), set_array_response(), the three typedefs.  What differs is private:
 * instead of Armadillo members the block owns an opaque `music_b200` handle (include/
 * music_b200.h) - all per-window arithmetic runs in the sm_90a CUDA library.  No Armadillo,
 * BLAS or LAPACK dependency remains.
 *
 * Build gating mirrors the reference's ARMADILLO_FOUND (CMakeLists-3.7.txt:195-202,
 * swig/baz_swig.i:560): compile this file only when CUDA was found (MUSIC_B200_FOUND).
 */
#ifndef INCLUDED_BAZ_MUSIC_DOA_H
#define INCLUDED_BAZ_MUSIC_DOA_H

#include <gnuradio/sync_block.h>
#include <gnuradio/thread/thread.h>
#include <boost/shared_ptr.hpp>
#include <complex>
#include <utility>
#include <vector>

struct music_b200; /* opaque, include/music_b200.h */

class baz_music_doa;
typedef boost::shared_ptr<baz_music_doa> baz_music_doa_sptr;

typedef std::vector<gr_complex> antenna_response_t;        /* one angle step: m element responses */
typedef std::vector<antenna_response_t> array_response_t;  /* [resolution][m] */
typedef std::pair<double, double> doa_t;                   /* (angle in degrees, strength) */

baz_music_doa_sptr baz_make_music_doa(unsigned int m, unsigned int n, unsigned int nsamples,
                                      const array_response_t &array_response, unsigned int resolution);
/* extension: a sparse linear array read through its difference co-array (include/music_b200.h,
 * music_b200_create_coarray): m physical elements at the integer positions p_0 = 0 < p_1 < ... times the step
 * step_xy = [s_x, s_y] metres, the wavelength, and the virtual size mv (0: the largest the array's lags fill, up to 16),
 * with up to mv - 1 sources (n may exceed m).  The block has the ports of baz_music_doa; set_coarray_geometry() is its
 * retune, and the setters the co-array handle refuses throw. */
baz_music_doa_sptr baz_make_music_doa_coarray(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution,
                                              const std::vector<int> &positions, const std::vector<double> &step_xy,
                                              double wavelength, unsigned int mv);

class baz_music_doa : public gr::sync_block
{
private:
    friend baz_music_doa_sptr baz_make_music_doa(unsigned int m, unsigned int n, unsigned int nsamples,
                                                 const array_response_t &array_response, unsigned int resolution);

    baz_music_doa(unsigned int m, unsigned int n, unsigned int nsamples, const array_response_t &array_response,
                  unsigned int resolution);
    friend baz_music_doa_sptr baz_make_music_doa_coarray(unsigned int m, unsigned int n, unsigned int nsamples,
                                                         unsigned int resolution, const std::vector<int> &positions,
                                                         const std::vector<double> &step_xy, double wavelength, unsigned int mv);
    /* around a handle already created (the co-array factory) */
    baz_music_doa(music_b200 *handle, unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution);

public:
    ~baz_music_doa();

    int work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items);

    void set_array_response(const array_response_t &array_response);
    /* extension: device-side table build from element positions [m][x, y] (metres) and the wavelength */
    void set_array_geometry(const std::vector<std::vector<double> > &positions_xy, double wavelength);
    /* extension: the retune of a co-array block (baz_make_music_doa_coarray) after an LO change: the step [s_x, s_y]
     * metres and the wavelength; resets integration and tracks */
    void set_coarray_geometry(const std::vector<double> &step_xy, double wavelength);
    /* extension: 0 = the reference's n largest bins (default), 1 = n largest local maxima > exclusion_bins apart,
     * 2 = root-MUSIC, 3 = LS-ESPRIT, each on a uniform linear array set by set_array_geometry() (exclusion_bins must be 0),
     * 4 = deterministic maximum likelihood (coherent sources, any table; exclusion_bins must be 0),
     * 5 = root-MUSIC by manifold separation on any planar array set by set_array_geometry() spanning <= ~4.4 wavelengths
     * (exclusion_bins must be 0), 6 = weighted subspace fitting (DML's search on the weighted signal subspace, any table;
     * exclusion_bins must be 0) */
    void set_peak_mode(int mode, unsigned int exclusion_bins);
    /* extension: 0 = n sources in every window (default), 1 = MDL, 2 = AIC estimate of 0..n sources per window */
    void set_source_rule(int rule);
    /* extension: true = refine every peak off the grid on the exact spectrum of the geometry set by
     * set_array_geometry() (bins stay the grid bins); false = grid angles (default) */
    void set_refine(bool enable);
    /* extension: the refine mode by number: 0 = off, 1 = Newton on the spectrum (as set_refine(true)), 2 = joint
     * Gauss-Newton refinement of all slots of a window under peak modes 4 and 6 (include/music_b200.h) */
    void set_refine_mode(int mode);
    /* extension: 0 = MUSIC (default), 1 = MVDR / Capon with diagonal loading loading * tr(R) / m, 2 = Bartlett
     * beamscan, 4 = IAA with diagonal loading loading * tr(R) / m (loading must be 0 for 0 and 2) */
    void set_estimator(int estimator, double loading);
    /* the IAA estimator's iteration count: 1 .. 64, default 15 */
    void set_iaa_iterations(int iterations);
    /* extension: beamformed source signals - 0 = off (default), 1 = delay-and-sum, 2 = MVDR, 3 = LCMV, with diagonal
     * loading loading * tr(R) / m for 2 and 3 (must be 0 for 0 and 1).  While it is on, work() also forms one beam per
     * filled peak slot of every item (include/music_b200.h), read back with last_beams(). */
    void set_beamformer(int rule, double loading);
    /* extension: receiver calibration (include/music_b200.h).  set_calibration(): the complex gain g_m of each element's
     * receiver chain; every later work() call corrects the covariance by 1 / g_m, in every mode (an empty vector clears
     * it).  calibration(): the gains in use (all 1 when none is set).  calibrate(): arms the block - the next nitems
     * items work() receives, from one dominant source at the known direction, are also accumulated (their outputs are
     * produced as usual); then the block solves for the gains (kind 1 = phase only, 2 = gain and phase, m >= 3) and
     * applies them.  last_calibration_residual(): the fit's relative off-diagonal residual, NaN when the solve failed
     * (the old gains are kept), or before any calibration finished.  Needs a table from set_array_geometry(). */
    void set_calibration(const std::vector<std::complex<double> > &gains);
    std::vector<std::complex<double> > calibration();
    void calibrate(double angle_deg, int kind, int nitems);
    double last_calibration_residual() const { return d_cal_residual; }
    /* extension: self-calibration without a known source (include/music_b200.h).  calibrate_blind(): arms the block like
     * calibrate() - the next nitems items (a multiple of segment) are also accumulated, every `segment` consecutive items
     * one segment covariance of nsources unknown emitters; then the block solves for the gains (32 starts, seed 0) and
     * applies them.  last_calibration_residual() then reads the solve's misfit (small when calibrated), NaN when the
     * solve failed (the old gains are kept).  Needs m >= 3 elements off one line and a table from set_array_geometry(). */
    void calibrate_blind(int nsources, int kind, int nitems, int segment);
    /* extension: covariance integration across work() calls (include/music_b200.h).  set_integration(): forgetting
     * factor 0 <= alpha < 1 (0, the default, is off); each item's estimate reads the exponentially weighted covariance of
     * the items since the last reset, across calls, and MDL / AIC count with the effective snapshot count.
     * reset_integration() restarts it at the next item; so do set_integration(), set_array_response(),
     * set_array_geometry() and set_calibration(). */
    void set_integration(double alpha);
    void reset_integration();
    /* extension: true = every work() call also returns the stochastic Cramer-Rao bound on the standard deviation of each
     * reported angle, in degrees (include/music_b200.h), read back with last_crb(); with the beamformer on, the bound and
     * the beams come from the same single call.  Needs a table from set_array_geometry(). */
    void set_crb(bool enable);
    /* extension: angle tracking across work() calls (include/music_b200.h).  variance MUSIC_B200_TRACK_OFF (default),
     * _FIXED or _CRB; the other arguments as music_b200_set_tracking().  While it is on, every work() call also returns
     * last_slot_track() [items][n] (the track id each slot's measurement updated or started, -1 for none),
     * last_track_ids() [items][max_tracks] (the confirmed track of every row, -1 for none) and last_track_state()
     * [items][max_tracks][3] (angle, rate in degrees per item, std of the angle), all from the same single call as the
     * bound and the beams.  set_tracking() and reset_tracks() drop every track; so do set_array_response() and
     * set_array_geometry(). */
    void set_tracking(int variance, double q, double rate_std0, double floor_deg, double crb_scale, double gate,
                      unsigned int confirm_hits, unsigned int confirm_window, unsigned int max_misses, unsigned int max_tracks);
    void reset_tracks();

    /* Integer peak-bin indices of the items produced by the last work() call, [items][n]
     * (not in the reference; -1 marks a slot the reference would leave at (0, 0)). */
    const std::vector<int> &last_bins() const { return d_bins; }
    /* Number of sources of each item produced by the last work() call, [items] (n unless set_source_rule() chose
     * MDL or AIC; slots at and beyond the count are left at (0, 0) with bin -1). */
    const std::vector<int> &last_counts() const { return d_counts; }
    /* Beams of the items produced by the last work() call while set_beamformer() is on, [items][n][nsamples / m]
     * (zeros for unfilled slots); empty while it is off. */
    const std::vector<gr_complex> &last_beams() const { return d_beams; }
    /* The bound of the items produced by the last work() call while set_crb() is on, [items][n] degrees (0 for unfilled
     * slots, NaN where the item's bound does not exist); empty while it is off. */
    const std::vector<float> &last_crb() const { return d_crb_out; }
    const std::vector<int> &last_slot_track() const { return d_slot_track; }
    const std::vector<int> &last_track_ids() const { return d_track_ids; }
    const std::vector<float> &last_track_state() const { return d_track_state; }

private:
    std::vector<float> flatten(const array_response_t &array_response) const;

    unsigned int d_m;
    unsigned int d_n;
    unsigned int d_nsamples;
    unsigned int d_resolution;
    music_b200 *d_handle;
    std::vector<int> d_bins;
    std::vector<int> d_counts;
    std::vector<gr_complex> d_beams;
    std::vector<float> d_crb_out;
    std::vector<int> d_slot_track, d_track_ids;
    std::vector<float> d_track_state;
    unsigned int d_track_rows; /* max_tracks while tracking is on, 0 while it is off */
    int d_source_rule;
    int d_beam_rule;
    bool d_crb;
    /* calibrate(): items still to accumulate (0: not armed), the source direction and the kind; the last residual */
    int d_cal_remaining;
    double d_cal_angle;
    int d_cal_kind;
    double d_cal_residual;
    /* calibrate_blind(): armed (d_cal_remaining and d_cal_kind serve it too), the source count, the segment length and
     * the items of a segment a work() call left incomplete */
    bool d_cal_blind;
    int d_cal_nsources;
    int d_cal_segment;
    std::vector<float> d_cal_pending;
    gr::thread::mutex d_mutex;
    void calibration_blind_step(const float *in, int noutput_items);
};

#endif /* INCLUDED_BAZ_MUSIC_DOA_H */
