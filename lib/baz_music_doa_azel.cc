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

#include "calibration_step.h"

#include <cstdio>
#include <cstdlib>
#include <limits>
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
      d_m(m), d_n(n), d_handle(NULL), d_cal_remaining(0), d_cal_az(0.0), d_cal_el(0.0), d_cal_kind(MUSIC_B200_CALIB_GAIN_PHASE),
      d_cal_residual(std::numeric_limits<double>::quiet_NaN())
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

/* The IAA estimator's iteration count (1 .. 64, default 15), see include/music_b200.h. */
void baz_music_doa_azel::set_iaa_iterations(int iterations)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_iaa_iterations(d_handle, iterations);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

/* Extension (not in the reference): covariance integration across windows, see include/music_b200.h. */
void baz_music_doa_azel::set_integration(double alpha)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_integration(d_handle, alpha);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_azel::reset_integration()
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_reset_integration(d_handle);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

void baz_music_doa_azel::set_calibration(const std::vector<std::complex<double> > &gains)
{
    if (!gains.empty() && gains.size() != d_m) throw std::invalid_argument("music_doa_azel: gains.size() != m");
    std::vector<double> flat;
    for (size_t i = 0; i < gains.size(); ++i) {
        flat.push_back(gains[i].real());
        flat.push_back(gains[i].imag());
    }
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_calibration(d_handle, gains.empty() ? NULL : flat.data());
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
}

std::vector<std::complex<double> > baz_music_doa_azel::calibration()
{
    std::vector<double> flat(2 * (size_t)d_m);
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_get_calibration(d_handle, flat.data());
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
    std::vector<std::complex<double> > g(d_m);
    for (unsigned int i = 0; i < d_m; ++i) g[i] = std::complex<double>(flat[2 * i], flat[2 * i + 1]);
    return g;
}

void baz_music_doa_azel::calibrate(double az_deg, double el_deg, int kind, int nitems)
{
    if (nitems <= 0) throw std::invalid_argument("music_doa_azel: calibrate() needs nitems > 0");
    if (kind != MUSIC_B200_CALIB_PHASE && kind != MUSIC_B200_CALIB_GAIN_PHASE) throw std::invalid_argument("music_doa_azel: unknown calibration kind");
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_calib_reset(d_handle);
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
    d_cal_remaining = nitems;
    d_cal_az = az_deg;
    d_cal_el = el_deg;
    d_cal_kind = kind;
}

void baz_music_doa_azel::set_crb(bool enable)
{
    gr::thread::scoped_lock guard(d_mutex);
    d_crb = enable;
}

void baz_music_doa_azel::set_tracking(int variance, double q, double rate_std0, double floor_deg, double crb_scale, double gate,
                                      unsigned int confirm_hits, unsigned int confirm_window, unsigned int max_misses,
                                      unsigned int max_tracks)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_tracking(d_handle, variance, q, rate_std0, floor_deg, crb_scale, gate, confirm_hits, confirm_window,
                                           max_misses, max_tracks);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
    d_track_rows = variance == MUSIC_B200_TRACK_OFF ? 0 : max_tracks;
}

void baz_music_doa_azel::reset_tracks()
{
    const int rc = music_b200_reset_tracks(d_handle);
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
    d_crb_out.assign(d_crb ? (size_t)noutput_items * d_n * 3 : 0, 0.0f);
    d_slot_track.assign(d_track_rows ? (size_t)noutput_items * d_n : 0, 0);
    d_track_ids.assign((size_t)noutput_items * d_track_rows, 0);
    d_track_state.assign((size_t)noutput_items * d_track_rows * 6, 0.0f);
    int rc;
    if (d_track_rows)  /* one call for the tracks and the bound: two would advance the carries twice */
        rc = music_b200_process_azel_host_tracks(d_handle, in, (uint32_t)noutput_items, az, el, lvl, spectrum, d_bins.data(), d_counts.data(),
                                                 d_crb ? d_crb_out.data() : NULL, d_slot_track.data(), d_track_ids.data(),
                                                 d_track_state.data());
    else if (d_crb)
        rc = music_b200_process_azel_host_crb(d_handle, in, (uint32_t)noutput_items, az, el, lvl, spectrum, d_bins.data(), d_counts.data(),
                                              d_crb_out.data());
    else
        rc = music_b200_process_azel_host(d_handle, in, (uint32_t)noutput_items, az, el, lvl, spectrum, d_bins.data(), d_counts.data());
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa_azel: ") + music_b200_last_error(d_handle));
    calibration_step(d_handle, in, noutput_items, d_cal_remaining, d_cal_az, d_cal_el, d_cal_kind, d_cal_residual);
    return noutput_items;
}
