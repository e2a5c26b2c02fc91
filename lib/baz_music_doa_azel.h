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
    void set_peak_mode(int mode, unsigned int exclusion_bins);
    /* 0 = n sources in every window (default), 1 = MDL, 2 = AIC estimate of 0..n sources per window */
    void set_source_rule(int rule);
    /* true = refine every peak off the grid on the exact spectrum of the geometry (bins stay the grid bins) */
    void set_refine(bool enable);
    /* 0 = MUSIC (default), 1 = MVDR with diagonal loading loading * tr(R) / m, 2 = Bartlett (loading 0 for 0 and 2) */
    void set_estimator(int estimator, double loading);

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
    gr::thread::mutex d_mutex;
};

#endif /* INCLUDED_BAZ_MUSIC_DOA_AZEL_H */
