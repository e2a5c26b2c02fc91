/* -*- c++ -*- */
/*
 * baz_music_doa_azel.h - (azimuth, elevation) MUSIC over a 3-D array geometry, as a gr::sync_block.
 *
 * Extension with no gr-baz counterpart: the planar arrays baz_music_doa serves can also measure elevation.  The block
 * owns an az-el handle of the CUDA library (music_b200_create_azel in include/music_b200.h, which defines the grid,
 * the table, both peak rules and the refinement).
 *   input  : one item of nsamples gr_complex per window (antennas sample-interleaved, as for baz_music_doa)
 *   outputs: 2..4 of azimuth (n floats), elevation (n floats), level (n floats), spectrum (n_el * n_az floats,
 *            elevation-major); unconnected trailing outputs are skipped
 */
#ifndef INCLUDED_BAZ_MUSIC_DOA_AZEL_H
#define INCLUDED_BAZ_MUSIC_DOA_AZEL_H

#include <gnuradio/sync_block.h>
#include <gnuradio/thread/thread.h>
#include <boost/shared_ptr.hpp>
#include <complex>
#include <vector>

struct music_b200; /* opaque, include/music_b200.h */

class baz_music_doa_azel;
typedef boost::shared_ptr<baz_music_doa_azel> baz_music_doa_azel_sptr;

/* positions_xyz: m element positions [x, y, z] in metres; el_lo / el_hi in degrees */
baz_music_doa_azel_sptr baz_make_music_doa_azel(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int n_az,
                                                unsigned int n_el, double el_lo, double el_hi,
                                                const std::vector<std::vector<double> > &positions_xyz, double wavelength);

class baz_music_doa_azel : public gr::sync_block
{
private:
    friend baz_music_doa_azel_sptr baz_make_music_doa_azel(unsigned int m, unsigned int n, unsigned int nsamples,
                                                           unsigned int n_az, unsigned int n_el, double el_lo, double el_hi,
                                                           const std::vector<std::vector<double> > &positions_xyz,
                                                           double wavelength);

    baz_music_doa_azel(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int n_az, unsigned int n_el,
                       double el_lo, double el_hi, const std::vector<std::vector<double> > &positions_xyz, double wavelength);

public:
    ~baz_music_doa_azel();

    int work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items);

    /* retune: element positions [m][x, y, z] (metres) and the wavelength; the table is built on the device */
    void set_array_geometry(const std::vector<std::vector<double> > &positions_xyz, double wavelength);
    /* 0 = the n largest bins (default), 1 = the n largest 2-D local maxima more than exclusion_bins apart */
    // mode 3 (MUSIC_B200_PEAKS_ESPRIT) on a planar lattice geometry: 2-D ESPRIT, gridless (azimuth, elevation) pairs
    // (include/music_b200.h); ROOTS, DML and MANIFOLD throw std::invalid_argument on this block
    void set_peak_mode(int mode, unsigned int exclusion_bins);
    /* 0 = n sources in every window (default), 1 = MDL, 2 = AIC estimate of 0..n sources per window */
    void set_source_rule(int rule);
    /* true = refine every peak off the grid on the exact spectrum of the geometry (bins stay the grid bins) */
    void set_refine(bool enable);
    /* 0 = MUSIC (default), 1 = MVDR with diagonal loading loading * tr(R) / m, 2 = Bartlett, 4 = IAA (loading 0 for 0 and 2) */
    void set_estimator(int estimator, double loading);
    /* the IAA estimator's iteration count: 1 .. 64, default 15 */
    void set_iaa_iterations(int iterations);
    /* receiver calibration, as for baz_music_doa; calibrate() takes the source's azimuth and elevation */
    void set_calibration(const std::vector<std::complex<double> > &gains);
    std::vector<std::complex<double> > calibration();
    void calibrate(double az_deg, double el_deg, int kind, int nitems);
    double last_calibration_residual() const { return d_cal_residual; }
    /* covariance integration across work() calls, as for baz_music_doa */
    void set_integration(double alpha);
    void reset_integration();
    /* the stochastic Cramer-Rao bound of every reported direction, as for baz_music_doa: last_crb() holds
     * [items][n][3] = std of the azimuth, std of the elevation (degrees), their correlation */
    void set_crb(bool enable);
    const std::vector<float> &last_crb() const { return d_crb_out; }
    /* angle tracking across work() calls, as for baz_music_doa: last_track_state() holds [items][max_tracks][6] = az,
     * its rate, el, its rate (degrees per item), std of the azimuth, std of the elevation */
    void set_tracking(int variance, double q, double rate_std0, double floor_deg, double crb_scale, double gate,
                      unsigned int confirm_hits, unsigned int confirm_window, unsigned int max_misses, unsigned int max_tracks);
    void reset_tracks();
    const std::vector<int> &last_slot_track() const { return d_slot_track; }
    const std::vector<int> &last_track_ids() const { return d_track_ids; }
    const std::vector<float> &last_track_state() const { return d_track_state; }

    /* flat peak bins b = i * n_az + k of the items produced by the last work() call, [items][n] (-1: unfilled slot) */
    const std::vector<int> &last_bins() const { return d_bins; }
    /* number of sources of each item produced by the last work() call, [items] */
    const std::vector<int> &last_counts() const { return d_counts; }

private:
    std::vector<double> flatten(const std::vector<std::vector<double> > &positions_xyz) const;

    unsigned int d_m;
    unsigned int d_n;
    music_b200 *d_handle;
    std::vector<int> d_bins;
    std::vector<int> d_counts;
    std::vector<float> d_crb_out;
    bool d_crb = false;
    std::vector<int> d_slot_track, d_track_ids;
    std::vector<float> d_track_state;
    unsigned int d_track_rows = 0; /* max_tracks while tracking is on, 0 while it is off */
    int d_cal_remaining;
    double d_cal_az, d_cal_el;
    int d_cal_kind;
    double d_cal_residual;
    gr::thread::mutex d_mutex;
};

#endif /* INCLUDED_BAZ_MUSIC_DOA_AZEL_H */
