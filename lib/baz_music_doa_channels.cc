/* -*- c++ -*- */
/*
 * baz_music_doa_channels.cc - gr::sync_block front of frequency-channelised direction finding (include/music_b200.h,
 * music_b200_create_channels).  Conventions follow baz_music_doa.cc: bad parameters throw std::invalid_argument, CUDA
 * failures std::runtime_error; work() processes all noutput_items windows in one call; a banner on construction and
 * on retunes.
 */
#ifdef HAVE_CONFIG_H
#include "config.h"
#endif

#include <baz_music_doa_channels.h>

#include <gnuradio/io_signature.h>
#include <music_b200.h>

#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

baz_music_doa_channels_sptr baz_make_music_doa_channels(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution,
                                                        unsigned int nfft, unsigned int chan_first, unsigned int chan_count, int taper,
                                                        int combine, const std::vector<std::vector<double> > &antenna_array,
                                                        double spacing, double centre_frequency, double sample_rate)
{
    return baz_music_doa_channels_sptr(new baz_music_doa_channels(m, n, nsamples, resolution, nfft, chan_first, chan_count, taper, combine,
                                                                  antenna_array, spacing, centre_frequency, sample_rate));
}

static unsigned int rows_of(unsigned int chan_count, int combine) { return combine == MUSIC_B200_CHANNELS_SEPARATE ? chan_count : 1u; }

static std::vector<int> output_sizes(unsigned int rows, unsigned int n, unsigned int resolution)
{
    std::vector<int> s(2, (int)(rows * n * sizeof(float)));
    s.push_back((int)((size_t)rows * resolution * sizeof(float)));
    return s;
}

static int device_from_env()
{
    const char *e = getenv("BAZ_MUSIC_DOA_DEVICE"); /* as for baz_music_doa */
    return e ? atoi(e) : 0;
}

baz_music_doa_channels::baz_music_doa_channels(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution,
                                               unsigned int nfft, unsigned int chan_first, unsigned int chan_count, int taper, int combine,
                                               const std::vector<std::vector<double> > &antenna_array, double spacing,
                                               double centre_frequency, double sample_rate)
    : gr::sync_block("music_doa_channels", gr::io_signature::make(1, 1, nsamples * sizeof(gr_complex)),
                     gr::io_signature::makev(1, 3, output_sizes(rows_of(chan_count, combine), n, resolution))),
      d_m(m), d_n(n), d_resolution(resolution), d_chan_count(chan_count), d_rows(rows_of(chan_count, combine)),
      d_counted(combine != MUSIC_B200_CHANNELS_INCOHERENT), d_handle(NULL)
{
    const int rc = music_b200_create_channels(&d_handle, m, n, nsamples, resolution, nfft, chan_first, chan_count, taper, combine,
                                              device_from_env());
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa_channels: ") + music_b200_last_error(NULL));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_channels: ") + music_b200_last_error(NULL));

    fprintf(stderr, "[%s<%li>] MUSIC DOA channels: M: %d, N: %d, # samples: %d, angular resolution: %d, FFT: %d, channels: %d from bin %d\n",
            name().c_str(), unique_id(), m, n, nsamples, resolution, nfft, chan_count, chan_first);
    std::vector<std::vector<double> > pos(antenna_array);
    for (size_t i = 0; i < pos.size(); ++i)
        for (size_t c = 0; c < pos[i].size(); ++c) pos[i][c] *= spacing;
    try {
        set_array_geometry(pos, centre_frequency, sample_rate);
    } catch (...) {
        music_b200_destroy(d_handle);
        throw;
    }
}

baz_music_doa_channels::~baz_music_doa_channels() { music_b200_destroy(d_handle); }

void baz_music_doa_channels::set_array_geometry(const std::vector<std::vector<double> > &positions_xy, double centre_frequency,
                                                double sample_rate)
{
    if (positions_xy.size() != d_m) throw std::invalid_argument("music_doa_channels: positions_xy.size() != m");
    std::vector<double> flat;
    for (size_t i = 0; i < positions_xy.size(); ++i) {
        if (positions_xy[i].size() != 2) throw std::invalid_argument("music_doa_channels: each position must be [x, y]");
        flat.push_back(positions_xy[i][0]);
        flat.push_back(positions_xy[i][1]);
    }
    fprintf(stderr, "[%s<%li>] Updating array response\n", name().c_str(), unique_id());
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_geometry_channels(d_handle, flat.data(), centre_frequency, sample_rate);
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_channels::set_peak_mode(int mode, unsigned int exclusion_bins)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_peak_mode(d_handle, mode, exclusion_bins);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_channels::set_source_rule(int rule)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_source_rule(d_handle, rule);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_channels::set_estimator(int estimator, double loading)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_estimator(d_handle, estimator, loading);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
}

/* The IAA estimator's iteration count (1 .. 64, default 15), see include/music_b200.h. */
void baz_music_doa_channels::set_iaa_iterations(int iterations)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_iaa_iterations(d_handle, iterations);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_channels::set_focusing(unsigned int first_bin, unsigned int bin_count)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_focusing(d_handle, first_bin, bin_count);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
}

std::vector<double> baz_music_doa_channels::focusing_error()
{
    std::vector<double> e(d_chan_count);
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_get_focusing(d_handle, NULL, e.data());
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
    return e;
}

std::vector<double> baz_music_doa_channels::channel_frequencies()
{
    std::vector<double> f(d_chan_count);
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_channel_frequencies(d_handle, f.data());
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
    return f;
}

/* the library's channel-major rows [rows][W][per] -> window-major items [W][rows][per] */
template <class T>
static void to_items(const T *src, T *dst, size_t rows, size_t W, size_t per)
{
    for (size_t r = 0; r < rows; ++r)
        for (size_t w = 0; w < W; ++w)
            for (size_t i = 0; i < per; ++i) dst[(w * rows + r) * per + i] = src[(r * W + w) * per + i];
}

int baz_music_doa_channels::work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items)
{
    if (noutput_items <= 0) return 0;
    if (output_items.empty()) throw std::invalid_argument("music_doa_channels: the angle output must be connected");
    const float *in = static_cast<const float *>(input_items[0]);
    const size_t W = (size_t)noutput_items, rn = (size_t)d_rows * d_n, rk = (size_t)d_rows * d_resolution;
    const bool lvl = output_items.size() > 1, spec = output_items.size() > 2;

    gr::thread::scoped_lock guard(d_mutex);
    /* staging: angles, levels, then the spectrum rows; bins, then the counts (not under the incoherent rule) */
    d_stage.resize(W * (2 * rn + (spec ? rk : 0)));
    d_istage.resize(W * (rn + d_rows));
    float *s_ang = d_stage.data(), *s_lvl = s_ang + W * rn, *s_spec = s_lvl + W * rn;
    int *s_bins = d_istage.data(), *s_cnt = s_bins + W * rn;
    const int rc = music_b200_process_channels_host(d_handle, in, (uint32_t)W, s_ang, lvl ? s_lvl : NULL, spec ? s_spec : NULL, s_bins,
                                                    d_counted ? s_cnt : NULL, NULL);
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_channels: ") + music_b200_last_error(d_handle));
    to_items(s_ang, static_cast<float *>(output_items[0]), d_rows, W, d_n);
    if (lvl) to_items(s_lvl, static_cast<float *>(output_items[1]), d_rows, W, d_n);
    if (spec) to_items(s_spec, static_cast<float *>(output_items[2]), d_rows, W, d_resolution);
    d_bins.resize(W * rn);
    to_items(s_bins, d_bins.data(), d_rows, W, d_n);
    d_counts.clear();
    if (d_counted) {
        d_counts.resize(W * d_rows);
        to_items(s_cnt, d_counts.data(), d_rows, W, 1);
    }
    return noutput_items;
}
