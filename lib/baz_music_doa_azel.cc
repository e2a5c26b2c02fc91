/* -*- c++ -*- */
/*
 * baz_music_doa_azel.cc - gr::sync_block front of (azimuth, elevation) MUSIC (include/music_b200.h,
 * music_b200_create_azel).  Conventions follow baz_music_doa.cc: bad parameters throw std::invalid_argument, CUDA
 * failures std::runtime_error; work() processes all noutput_items windows in one call; a banner on construction and
 * on retunes.
 */
#ifdef HAVE_CONFIG_H
#include "config.h"
#endif

#include <baz_music_doa_azel.h>

#include <gnuradio/io_signature.h>
#include <music_b200.h>

#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

baz_music_doa_azel_sptr baz_make_music_doa_azel(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int n_az,
                                                unsigned int n_el, double el_lo, double el_hi,
                                                const std::vector<std::vector<double> > &positions_xyz, double wavelength)
{
    return baz_music_doa_azel_sptr(new baz_music_doa_azel(m, n, nsamples, n_az, n_el, el_lo, el_hi, positions_xyz, wavelength));
}

static std::vector<int> output_sizes(unsigned int n, unsigned int n_az, unsigned int n_el)
{
    std::vector<int> s(3, (int)(n * sizeof(float)));
    s.push_back((int)((size_t)n_az * n_el * sizeof(float)));
    return s;
}

static int device_from_env()
{
    const char *e = getenv("BAZ_MUSIC_DOA_DEVICE"); /* as for baz_music_doa */
    return e ? atoi(e) : 0;
}

baz_music_doa_azel::baz_music_doa_azel(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int n_az,
                                       unsigned int n_el, double el_lo, double el_hi,
                                       const std::vector<std::vector<double> > &positions_xyz, double wavelength)
    : gr::sync_block("music_doa_azel", gr::io_signature::make(1, 1, nsamples * sizeof(gr_complex)),
                     gr::io_signature::makev(2, 4, output_sizes(n, n_az, n_el))),
      d_m(m), d_n(n), d_handle(NULL)
{
    const std::vector<double> pos = flatten(positions_xyz);
    const int rc = music_b200_create_azel(&d_handle, m, n, nsamples, n_az, n_el, el_lo, el_hi, pos.data(), wavelength, device_from_env());
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(NULL));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_azel: ") + music_b200_last_error(NULL));

    fprintf(stderr, "[%s<%li>] MUSIC DOA az-el: M: %d, N: %d, # samples: %d, azimuth steps: %d, elevation steps: %d (%g .. %g deg)\n",
            name().c_str(), unique_id(), m, n, nsamples, n_az, n_el, el_lo, el_hi);
}

baz_music_doa_azel::~baz_music_doa_azel() { music_b200_destroy(d_handle); }

std::vector<double> baz_music_doa_azel::flatten(const std::vector<std::vector<double> > &positions_xyz) const
{
    if (positions_xyz.size() != d_m) throw std::invalid_argument("music_doa_azel: positions_xyz.size() != m");
    std::vector<double> flat;
    flat.reserve(3 * (size_t)d_m);
    for (size_t i = 0; i < positions_xyz.size(); ++i) {
        if (positions_xyz[i].size() != 3) throw std::invalid_argument("music_doa_azel: each position must be [x, y, z]");
        for (int c = 0; c < 3; ++c) flat.push_back(positions_xyz[i][c]);
    }
    return flat;
}

void baz_music_doa_azel::set_array_geometry(const std::vector<std::vector<double> > &positions_xyz, double wavelength)
{
    const std::vector<double> flat = flatten(positions_xyz);
    fprintf(stderr, "[%s<%li>] Updating array response\n", name().c_str(), unique_id());
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_geometry_azel(d_handle, flat.data(), wavelength);
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_azel::set_peak_mode(int mode, unsigned int exclusion_bins)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_peak_mode(d_handle, mode, exclusion_bins);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_azel::set_source_rule(int rule)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_source_rule(d_handle, rule);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_azel::set_refine(bool enable)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_refine(d_handle, enable ? MUSIC_B200_REFINE_NEWTON : MUSIC_B200_REFINE_OFF);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_azel::set_estimator(int estimator, double loading)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_estimator(d_handle, estimator, loading);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

int baz_music_doa_azel::work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items)
{
    if (noutput_items <= 0) return 0;
    if (output_items.size() < 2) throw std::invalid_argument("music_doa_azel: azimuth and elevation outputs must be connected");
    const float *in = static_cast<const float *>(input_items[0]);
    float *az = static_cast<float *>(output_items[0]);
    float *el = static_cast<float *>(output_items[1]);
    float *lvl = output_items.size() > 2 ? static_cast<float *>(output_items[2]) : NULL;
    float *spectrum = output_items.size() > 3 ? static_cast<float *>(output_items[3]) : NULL;

    gr::thread::scoped_lock guard(d_mutex);
    d_bins.resize((size_t)noutput_items * d_n);
    d_counts.resize((size_t)noutput_items);
    const int rc = music_b200_process_azel_host(d_handle, in, (uint32_t)noutput_items, az, el, lvl, spectrum, d_bins.data(), d_counts.data());
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
    return noutput_items;
}
