/* -*- c++ -*- */
/*
 * baz_music_doa_channels.h - frequency-channelised direction finding as a gr::sync_block.
 *
 * Extension with no gr-baz counterpart: baz_music_doa forms one covariance over the whole sampled bandwidth.  This block
 * runs an FFT filter bank over each window and solves one problem per channel, each with a steering table built for that
 * channel's own wavelength, or combines the channels into one incoherent wideband MUSIC spectrum, or focuses every
 * channel's covariance onto the centre channel and solves one coherent wideband problem per window.  It owns a channel
 * handle of the CUDA library (music_b200_create_channels in include/music_b200.h, which has the definition).
 *   input  : one item of nsamples gr_complex per window (antennas sample-interleaved, as for baz_music_doa)
 *   outputs: 1..3 of angle, level, spectrum.  combine = 0 (separate): an item holds the chan_count channels of one
 *            window, chan_count * n / chan_count * n / chan_count * resolution floats, channel by channel;
 *            combine = 1 (incoherent) and 2 (coherent): n / n / resolution floats as for baz_music_doa.
 */
#ifndef INCLUDED_BAZ_MUSIC_DOA_CHANNELS_H
#define INCLUDED_BAZ_MUSIC_DOA_CHANNELS_H

#include <gnuradio/sync_block.h>
#include <gnuradio/thread/thread.h>
#include <boost/shared_ptr.hpp>
#include <vector>

struct music_b200; /* opaque, include/music_b200.h */

class baz_music_doa_channels;
typedef boost::shared_ptr<baz_music_doa_channels> baz_music_doa_channels_sptr;

/* taper: 0 = rectangular, 1 = Hann; combine: 0 = separate, 1 = incoherent, 2 = coherent; antenna_array: m positions [x, y] in units of
 * spacing metres; frequencies in Hz */
baz_music_doa_channels_sptr baz_make_music_doa_channels(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution,
                                                        unsigned int nfft, unsigned int chan_first, unsigned int chan_count, int taper,
                                                        int combine, const std::vector<std::vector<double> > &antenna_array,
                                                        double spacing, double centre_frequency, double sample_rate);

class baz_music_doa_channels : public gr::sync_block
{
private:
    friend baz_music_doa_channels_sptr baz_make_music_doa_channels(unsigned int m, unsigned int n, unsigned int nsamples,
                                                                   unsigned int resolution, unsigned int nfft, unsigned int chan_first,
                                                                   unsigned int chan_count, int taper, int combine,
                                                                   const std::vector<std::vector<double> > &antenna_array,
                                                                   double spacing, double centre_frequency, double sample_rate);

    baz_music_doa_channels(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution, unsigned int nfft,
                           unsigned int chan_first, unsigned int chan_count, int taper, int combine,
                           const std::vector<std::vector<double> > &antenna_array, double spacing, double centre_frequency,
                           double sample_rate);

public:
    ~baz_music_doa_channels();

    int work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items);

    /* retune: element positions [m][x, y] in metres, centre frequency and sample rate in Hz; one table per channel */
    void set_array_geometry(const std::vector<std::vector<double> > &positions_xy, double centre_frequency, double sample_rate);
    /* 0 = the n largest bins (default), 1 = the n largest local maxima more than exclusion_bins apart; coherent also
     * 2 = root-MUSIC, 3 = ESPRIT (uniform linear arrays), 4 = DML, 5 = root-MUSIC by manifold separation (any planar
     * array on the reference channel's geometry), 6 = WSF */
    void set_peak_mode(int mode, unsigned int exclusion_bins);
    /* 0 = n sources in every (window, channel) (default), 1 = MDL, 2 = AIC from the segments of each channel */
    void set_source_rule(int rule);
    /* 0 = MUSIC (default), 1 = MVDR with diagonal loading loading * tr(R) / m, 2 = Bartlett, 4 = IAA (loading 0 for 0 and 2) */
    void set_estimator(int estimator, double loading);
    /* the IAA estimator's iteration count: 1 .. 64, default 15 */
    void set_iaa_iterations(int iterations);

    /* coherent: fit the focusing matrices on grid bins (first_bin + i) mod resolution, i < bin_count */
    void set_focusing(unsigned int first_bin, unsigned int bin_count);
    /* coherent: each channel's focusing error ||T_c A_c - A_ref||_F / ||A_ref||_F, [chan_count] */
    std::vector<double> focusing_error();

    /* each channel's frequency offset from the centre frequency in Hz, [chan_count] */
    std::vector<double> channel_frequencies();
    /* peak bins of the items produced by the last work() call, [items][rows][n] (-1: unfilled slot); rows = chan_count
     * (separate) or 1 (incoherent, coherent) */
    const std::vector<int> &last_bins() const { return d_bins; }
    /* number of sources of each item of the last work() call: separate [items][chan_count], coherent [items], incoherent
     * none */
    const std::vector<int> &last_counts() const { return d_counts; }

private:
    unsigned int d_m, d_n, d_resolution, d_chan_count, d_rows;
    bool d_counted;  /* counts are reported (separate, coherent) */
    music_b200 *d_handle;
    std::vector<int> d_bins, d_counts;
    std::vector<float> d_stage;  /* the library's channel-major results, before they become window-major items */
    std::vector<int> d_istage;
    gr::thread::mutex d_mutex;
};

#endif /* INCLUDED_BAZ_MUSIC_DOA_CHANNELS_H */
