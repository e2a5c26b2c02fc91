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

class baz_music_doa : public gr::sync_block
{
private:
    friend baz_music_doa_sptr baz_make_music_doa(unsigned int m, unsigned int n, unsigned int nsamples,
                                                 const array_response_t &array_response, unsigned int resolution);

    baz_music_doa(unsigned int m, unsigned int n, unsigned int nsamples, const array_response_t &array_response,
                  unsigned int resolution);

public:
    ~baz_music_doa();

    int work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items);

    void set_array_response(const array_response_t &array_response);
    /* extension: device-side table build from element positions [m][x, y] (metres) and the wavelength */
    void set_array_geometry(const std::vector<std::vector<double> > &positions_xy, double wavelength);
    /* extension: 0 = the reference's n largest bins (default), 1 = n largest local maxima > exclusion_bins apart,
     * 2 = root-MUSIC on a uniform linear array set by set_array_geometry() (exclusion_bins must be 0) */
    void set_peak_mode(int mode, unsigned int exclusion_bins);
    /* extension: 0 = n sources in every window (default), 1 = MDL, 2 = AIC estimate of 0..n sources per window */
    void set_source_rule(int rule);
    /* extension: true = refine every peak off the grid on the exact spectrum of the geometry set by
     * set_array_geometry() (bins stay the grid bins); false = grid angles (default) */
    void set_refine(bool enable);
    /* extension: 0 = MUSIC (default), 1 = MVDR / Capon with diagonal loading loading * tr(R) / m, 2 = Bartlett
     * beamscan (loading must be 0 for 0 and 2) */
    void set_estimator(int estimator, double loading);

    /* Integer peak-bin indices of the items produced by the last work() call, [items][n]
     * (not in the reference; -1 marks a slot the reference would leave at (0, 0)). */
    const std::vector<int> &last_bins() const { return d_bins; }
    /* Number of sources of each item produced by the last work() call, [items] (n unless set_source_rule() chose
     * MDL or AIC; slots at and beyond the count are left at (0, 0) with bin -1). */
    const std::vector<int> &last_counts() const { return d_counts; }

private:
    std::vector<float> flatten(const array_response_t &array_response) const;

    unsigned int d_m;
    unsigned int d_n;
    unsigned int d_nsamples;
    unsigned int d_resolution;
    music_b200 *d_handle;
    std::vector<int> d_bins;
    std::vector<int> d_counts;
    int d_source_rule;
    gr::thread::mutex d_mutex;
};

#endif /* INCLUDED_BAZ_MUSIC_DOA_H */
