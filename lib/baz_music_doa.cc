/* -*- c++ -*- */
/*
 * baz_music_doa.cc - gr::sync_block front of the H100-native MUSIC DOA path.
 *
 * Drop-in for /root/reference/lib/baz_music_doa.cc.  The GNU Radio facing behaviour is kept:
 *   - io signatures: 1 input of nsamples*sizeof(gr_complex); 1..3 outputs of n*4, n*4,
 *     resolution*4 bytes                                      (reference :36-38)
 *   - stderr banners on construction and on table updates      (reference :52, :65)
 *   - optional ports: levels only if output 1 is connected, spectrum only if output 2 is
 *                                                              (reference :97-99, :148-149)
 * What changed, deliberately:
 *   - the reference's asserts (:45-50, :62-63, no-ops in its Release build) throw
 *     std::invalid_argument, the library's convention for bad parameters
 *     (e.g. /root/reference/lib/baz_additive_scrambler_bb.cc:59);
 *   - work() processes ALL noutput_items windows in one call and returns noutput_items (the
 *     reference returns 1, :160).  Legal for a sync_block, same per-window results, and the
 *     only way the GPU sees a batch;
 *   - with only output 0 connected the reference dereferences lvl == NULL (:147-154); here the
 *     level output is simply skipped.
 * All arithmetic (reference :74-155) happens behind the C ABI in include/music_b200.h.
 */
#ifdef HAVE_CONFIG_H
#include "config.h"
#endif

#include <baz_music_doa.h>

#include <gnuradio/io_signature.h>
#include <music_b200.h>

#include "calibration_step.h"

#include <cstdio>
#include <cstdlib>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>

baz_music_doa_sptr baz_make_music_doa(unsigned int m, unsigned int n, unsigned int nsamples,
                                      const array_response_t &array_response, unsigned int resolution)
{
    return baz_music_doa_sptr(new baz_music_doa(m, n, nsamples, array_response, resolution));
}

static int device_from_env()
{
    const char *e = getenv("BAZ_MUSIC_DOA_DEVICE"); /* device choice must not change the flowgraph/GRC params */
    return e ? atoi(e) : 0;
}

/* BAZ_MUSIC_DOA_DEVICES="0,1,2,3": one engine per listed GPU behind this ONE block - work() deals its windows
   round-robin to them (music_b200_create_multi), so an unchanged flowgraph uses every GPU and every PCIe link of the
   node.  Unset: the single device of BAZ_MUSIC_DOA_DEVICE. */
static std::vector<int> devices_from_env()
{
    std::vector<int> d;
    const char *e = getenv("BAZ_MUSIC_DOA_DEVICES");
    if (!e) return d;
    for (const char *p = e; *p;) {
        char *end = NULL;
        const long v = strtol(p, &end, 10);
        if (end == p) break;
        d.push_back((int)v);
        p = end;
        while (*p == ',' || *p == ' ') ++p;
    }
    return d;
}

baz_music_doa::baz_music_doa(unsigned int m, unsigned int n, unsigned int nsamples,
                             const array_response_t &array_response, unsigned int resolution)
    : gr::sync_block("music_doa", gr::io_signature::make(1, 1, nsamples * sizeof(gr_complex)),
                     gr::io_signature::make3(1, 3, n * sizeof(float), n * sizeof(float), resolution * sizeof(float))),
      d_m(m), d_n(n), d_nsamples(nsamples), d_resolution(resolution), d_handle(NULL), d_track_rows(0),
      d_source_rule(MUSIC_B200_SOURCES_FIXED), d_beam_rule(MUSIC_B200_BEAMS_OFF), d_crb(false), d_cal_remaining(0), d_cal_angle(0.0), d_cal_kind(MUSIC_B200_CALIB_GAIN_PHASE),
      d_cal_residual(std::numeric_limits<double>::quiet_NaN()), d_cal_blind(false), d_cal_nsources(1), d_cal_segment(1)
{
    if (array_response.size() != resolution) throw std::invalid_argument("music_doa: array_response.size() != resolution");
    const std::vector<float> table = flatten(array_response);
    const std::vector<int> devices = devices_from_env();
    const int rc = devices.empty() ? music_b200_create(&d_handle, m, n, nsamples, resolution, table.data(), device_from_env())
                                   : music_b200_create_multi(&d_handle, m, n, nsamples, resolution, table.data(), devices.data(), (int)devices.size());
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(NULL));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(NULL));

    fprintf(stderr, "[%s<%li>] MUSIC DOA: M: %d, N: %d, # samples: %d, angular resolution: %d\n", name().c_str(),
            unique_id(), m, n, nsamples, resolution);
}

/* Extension (not in the reference): a sparse linear array through its difference co-array, see include/music_b200.h. */
baz_music_doa_sptr baz_make_music_doa_coarray(unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution,
                                              const std::vector<int> &positions, const std::vector<double> &step_xy,
                                              double wavelength, unsigned int mv)
{
    if (positions.size() != m) throw std::invalid_argument("music_doa: positions.size() != m");
    if (step_xy.size() != 2) throw std::invalid_argument("music_doa: step_xy must be [s_x, s_y]");
    music_b200 *h = NULL;
    const int rc = music_b200_create_coarray(&h, m, n, nsamples, resolution, positions.data(), step_xy.data(), wavelength, mv,
                                             device_from_env());
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(NULL));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(NULL));
    return baz_music_doa_sptr(new baz_music_doa(h, m, n, nsamples, resolution));
}

baz_music_doa::baz_music_doa(music_b200 *handle, unsigned int m, unsigned int n, unsigned int nsamples, unsigned int resolution)
    : gr::sync_block("music_doa", gr::io_signature::make(1, 1, nsamples * sizeof(gr_complex)),
                     gr::io_signature::make3(1, 3, n * sizeof(float), n * sizeof(float), resolution * sizeof(float))),
      d_m(m), d_n(n), d_nsamples(nsamples), d_resolution(resolution), d_handle(handle), d_track_rows(0),
      d_source_rule(MUSIC_B200_SOURCES_FIXED), d_beam_rule(MUSIC_B200_BEAMS_OFF), d_crb(false), d_cal_remaining(0), d_cal_angle(0.0), d_cal_kind(MUSIC_B200_CALIB_GAIN_PHASE),
      d_cal_residual(std::numeric_limits<double>::quiet_NaN()), d_cal_blind(false), d_cal_nsources(1), d_cal_segment(1)
{
    uint32_t mv = 0;
    music_b200_coarray_size(d_handle, &mv);
    fprintf(stderr, "[%s<%li>] MUSIC DOA co-array: M: %d, virtual M: %u, N: %d, # samples: %d, angular resolution: %d\n", name().c_str(),
            unique_id(), m, mv, n, nsamples, resolution);
}

baz_music_doa::~baz_music_doa() { music_b200_destroy(d_handle); }

std::vector<float> baz_music_doa::flatten(const array_response_t &array_response) const
{
    std::vector<float> t;
    t.reserve((size_t)array_response.size() * d_m * 2);
    for (size_t k = 0; k < array_response.size(); ++k) {
        if (array_response[k].size() != d_m) throw std::invalid_argument("music_doa: array_response[k].size() != m");
        for (unsigned int i = 0; i < d_m; ++i) {
            t.push_back(array_response[k][i].real());
            t.push_back(array_response[k][i].imag());
        }
    }
    return t;
}

void baz_music_doa::set_array_response(const array_response_t &array_response)
{
    if (array_response.size() != d_resolution) throw std::invalid_argument("music_doa: array_response.size() != resolution");
    const std::vector<float> table = flatten(array_response);

    fprintf(stderr, "[%s<%li>] Updating array response\n", name().c_str(), unique_id());

    /* music_b200_set_table() is itself serialised against process_host(); the block-level lock
       keeps d_bins / scratch consistent with the reference's "one mutex" model (:67, :101). */
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_table(d_handle, table.data());
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

/* Extension (not in the reference): retune from the element positions; the table is built on the device
   (music_b200_set_geometry) and is bit-identical to calculate_antenna_array_response() + set_array_response()
   of /root/reference/python/music_doa_helper.py:32-46, :100-103. */
void baz_music_doa::set_array_geometry(const std::vector<std::vector<double> > &positions_xy, double wavelength)
{
    if (positions_xy.size() != d_m) throw std::invalid_argument("music_doa: positions_xy.size() != m");
    std::vector<double> flat;
    flat.reserve(2 * (size_t)d_m);
    for (size_t i = 0; i < positions_xy.size(); ++i) {
        if (positions_xy[i].size() != 2) throw std::invalid_argument("music_doa: each position must be [x, y]");
        flat.push_back(positions_xy[i][0]);
        flat.push_back(positions_xy[i][1]);
    }
    fprintf(stderr, "[%s<%li>] Updating array response\n", name().c_str(), unique_id());
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_geometry(d_handle, flat.data(), wavelength, NULL);
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

void baz_music_doa::set_coarray_geometry(const std::vector<double> &step_xy, double wavelength)
{
    if (step_xy.size() != 2) throw std::invalid_argument("music_doa: step_xy must be [s_x, s_y]");
    fprintf(stderr, "[%s<%li>] Updating array response\n", name().c_str(), unique_id());
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_geometry_coarray(d_handle, step_xy.data(), wavelength);
    if (rc == MUSIC_B200_EINVAL) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

/* Extension (not in the reference): opt-in local-maximum peak rule, see include/music_b200.h. */
void baz_music_doa::set_peak_mode(int mode, unsigned int exclusion_bins)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_peak_mode(d_handle, mode, exclusion_bins);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

/* Extension (not in the reference): per-window estimate of the number of sources, see include/music_b200.h. */
void baz_music_doa::set_source_rule(int rule)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_source_rule(d_handle, rule);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
    d_source_rule = rule;
}

/* Extension (not in the reference): off-grid peak refinement on the exact spectrum of the array geometry, see
   include/music_b200.h.  Needs a table installed with set_array_geometry(). */
void baz_music_doa::set_refine(bool enable) { set_refine_mode(enable ? MUSIC_B200_REFINE_NEWTON : MUSIC_B200_REFINE_OFF); }

/* The refine mode by number: OFF, NEWTON, or JOINT under the DML and WSF peak modes. */
void baz_music_doa::set_refine_mode(int mode)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_refine(d_handle, mode);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

/* Extension (not in the reference): the spectrum estimator - 0 MUSIC (default), 1 MVDR with diagonal loading
   `loading` * tr(R) / m, 2 Bartlett; see include/music_b200.h. */
void baz_music_doa::set_estimator(int estimator, double loading)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_estimator(d_handle, estimator, loading);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

/* The IAA estimator's iteration count (1 .. 64, default 15), see include/music_b200.h. */
void baz_music_doa::set_iaa_iterations(int iterations)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_iaa_iterations(d_handle, iterations);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

/* Extension (not in the reference): beamformed source signals, see include/music_b200.h. */
void baz_music_doa::set_beamformer(int rule, double loading)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_beamformer(d_handle, rule, loading);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
    d_beam_rule = rule;
}

/* Extension (not in the reference): receiver calibration, see include/music_b200.h. */
/* Extension (not in the reference): covariance integration across windows, see include/music_b200.h. */
void baz_music_doa::set_integration(double alpha)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_integration(d_handle, alpha);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

void baz_music_doa::reset_integration()
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_reset_integration(d_handle);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

/* Extension (not in the reference): the stochastic CRB of every reported angle, see include/music_b200.h. */
void baz_music_doa::set_crb(bool enable)
{
    gr::thread::scoped_lock guard(d_mutex);
    d_crb = enable;
}

/* Extension (not in the reference): angle tracking across work() calls, see include/music_b200.h. */
void baz_music_doa::set_tracking(int variance, double q, double rate_std0, double floor_deg, double crb_scale, double gate,
                                 unsigned int confirm_hits, unsigned int confirm_window, unsigned int max_misses, unsigned int max_tracks)
{
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_tracking(d_handle, variance, q, rate_std0, floor_deg, crb_scale, gate, confirm_hits, confirm_window,
                                           max_misses, max_tracks);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
    d_track_rows = variance == MUSIC_B200_TRACK_OFF ? 0 : max_tracks;
}

void baz_music_doa::reset_tracks()
{
    const int rc = music_b200_reset_tracks(d_handle);
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

void baz_music_doa::set_calibration(const std::vector<std::complex<double> > &gains)
{
    if (!gains.empty() && gains.size() != d_m) throw std::invalid_argument("music_doa: gains.size() != m");
    std::vector<double> flat;
    for (size_t i = 0; i < gains.size(); ++i) {
        flat.push_back(gains[i].real());
        flat.push_back(gains[i].imag());
    }
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_set_calibration(d_handle, gains.empty() ? NULL : flat.data());
    if (rc != MUSIC_B200_OK) throw std::invalid_argument(std::string("music_doa: ") + music_b200_last_error(d_handle));
}

std::vector<std::complex<double> > baz_music_doa::calibration()
{
    std::vector<double> flat(2 * (size_t)d_m);
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_get_calibration(d_handle, flat.data());
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(d_handle));
    std::vector<std::complex<double> > g(d_m);
    for (unsigned int i = 0; i < d_m; ++i) g[i] = std::complex<double>(flat[2 * i], flat[2 * i + 1]);
    return g;
}

void baz_music_doa::calibrate(double angle_deg, int kind, int nitems)
{
    if (nitems <= 0) throw std::invalid_argument("music_doa: calibrate() needs nitems > 0");
    if (kind != MUSIC_B200_CALIB_PHASE && kind != MUSIC_B200_CALIB_GAIN_PHASE) throw std::invalid_argument("music_doa: unknown calibration kind");
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_calib_reset(d_handle);
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(d_handle));
    d_cal_remaining = nitems;
    d_cal_angle = angle_deg;
    d_cal_kind = kind;
    d_cal_blind = false;
}

void baz_music_doa::calibrate_blind(int nsources, int kind, int nitems, int segment)
{
    if (segment <= 0 || nitems <= 0 || nitems % segment != 0)
        throw std::invalid_argument("music_doa: calibrate_blind() needs segment > 0 and nitems a positive multiple of segment");
    if (kind != MUSIC_B200_CALIB_PHASE && kind != MUSIC_B200_CALIB_GAIN_PHASE) throw std::invalid_argument("music_doa: unknown calibration kind");
    if (nsources <= 0) throw std::invalid_argument("music_doa: calibrate_blind() needs nsources > 0");
    gr::thread::scoped_lock guard(d_mutex);
    const int rc = music_b200_calib_blind_reset(d_handle);
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(d_handle));
    d_cal_remaining = nitems;
    d_cal_kind = kind;
    d_cal_blind = true;
    d_cal_nsources = nsources;
    d_cal_segment = segment;
    d_cal_pending.clear();
}

/* The armed self-calibration step at the end of work(): accumulate the whole segments of this call's armed items (a
 * segment split across calls waits in d_cal_pending); once all are in, solve, apply and record the misfit (NaN on
 * failure, with the old gains kept). */
void baz_music_doa::calibration_blind_step(const float *in, int noutput_items)
{
    if (d_cal_remaining <= 0) return;
    const int take = noutput_items < d_cal_remaining ? noutput_items : d_cal_remaining;
    d_cal_remaining -= take;
    const size_t item = (size_t)d_nsamples * 2;
    d_cal_pending.insert(d_cal_pending.end(), in, in + (size_t)take * item);
    const uint32_t whole = (uint32_t)(d_cal_pending.size() / item) / (uint32_t)d_cal_segment * (uint32_t)d_cal_segment;
    bool ok = whole == 0 || music_b200_calib_blind_accumulate_host(d_handle, d_cal_pending.data(), whole, (uint32_t)d_cal_segment) == MUSIC_B200_OK;
    d_cal_pending.erase(d_cal_pending.begin(), d_cal_pending.begin() + (ptrdiff_t)(whole * item));
    if (ok && d_cal_remaining > 0) return;
    std::vector<double> g(2 * MUSIC_B200_MAX_M);
    double stats[4];
    ok = ok && music_b200_calib_blind_solve(d_handle, (uint32_t)d_cal_nsources, d_cal_kind, 32, 0, g.data(), NULL, stats) == MUSIC_B200_OK &&
         music_b200_set_calibration(d_handle, g.data()) == MUSIC_B200_OK;
    d_cal_residual = ok ? stats[0] : std::numeric_limits<double>::quiet_NaN();
    d_cal_remaining = 0;
    d_cal_pending.clear();
}

int baz_music_doa::work(int noutput_items, gr_vector_const_void_star &input_items, gr_vector_void_star &output_items)
{
    if (noutput_items <= 0) return 0;
    const float *in = static_cast<const float *>(input_items[0]); /* gr_complex items, (re, im) pairs */
    float *out = static_cast<float *>(output_items[0]);
    float *lvl = output_items.size() > 1 ? static_cast<float *>(output_items[1]) : NULL;
    float *out_spectrum = output_items.size() > 2 ? static_cast<float *>(output_items[2]) : NULL;

    gr::thread::scoped_lock guard(d_mutex);
    d_bins.resize((size_t)noutput_items * d_n);
    d_beams.clear();
    d_crb_out.clear();
    d_slot_track.clear();
    d_track_ids.clear();
    d_track_state.clear();
    int rc;
    if (d_track_rows) {
        /* one call for the tracks, the bound and the beams: two would advance the integration and track carries twice */
        d_counts.resize((size_t)noutput_items);
        if (d_crb) d_crb_out.resize((size_t)noutput_items * d_n);
        if (d_beam_rule != MUSIC_B200_BEAMS_OFF) d_beams.resize((size_t)noutput_items * d_n * (d_nsamples / d_m));
        d_slot_track.resize((size_t)noutput_items * d_n);
        d_track_ids.resize((size_t)noutput_items * d_track_rows);
        d_track_state.resize((size_t)noutput_items * d_track_rows * 3);
        rc = music_b200_process_host_tracks(d_handle, in, (uint32_t)noutput_items, out, lvl, out_spectrum, d_bins.data(), d_counts.data(),
                                            NULL, d_beams.empty() ? NULL : reinterpret_cast<float *>(d_beams.data()),
                                            d_crb_out.empty() ? NULL : d_crb_out.data(), d_slot_track.data(), d_track_ids.data(),
                                            d_track_state.data());
    } else if (d_crb) {
        /* one call for the bound and the beams: two would advance the integration carry twice */
        d_counts.resize((size_t)noutput_items);
        d_crb_out.resize((size_t)noutput_items * d_n);
        if (d_beam_rule != MUSIC_B200_BEAMS_OFF) d_beams.resize((size_t)noutput_items * d_n * (d_nsamples / d_m));
        rc = music_b200_process_host_crb(d_handle, in, (uint32_t)noutput_items, out, lvl, out_spectrum, d_bins.data(), d_counts.data(),
                                         NULL, d_beams.empty() ? NULL : reinterpret_cast<float *>(d_beams.data()), d_crb_out.data());
    } else if (d_beam_rule != MUSIC_B200_BEAMS_OFF) {
        d_counts.resize((size_t)noutput_items);
        d_beams.resize((size_t)noutput_items * d_n * (d_nsamples / d_m));
        rc = music_b200_process_host_beams(d_handle, in, (uint32_t)noutput_items, out, lvl, out_spectrum, d_bins.data(), d_counts.data(),
                                           NULL, reinterpret_cast<float *>(d_beams.data()));
    } else if (d_source_rule == MUSIC_B200_SOURCES_FIXED) {
        rc = music_b200_process_host(d_handle, in, (uint32_t)noutput_items, out, lvl, out_spectrum, d_bins.data());
        d_counts.assign((size_t)noutput_items, (int)d_n);
    } else {
        d_counts.resize((size_t)noutput_items);
        rc = music_b200_process_host_counts(d_handle, in, (uint32_t)noutput_items, out, lvl, out_spectrum, d_bins.data(), d_counts.data());
    }
    if (rc != MUSIC_B200_OK) throw std::runtime_error(std::string("music_doa: ") + music_b200_last_error(d_handle));
    if (d_cal_blind) calibration_blind_step(in, noutput_items);
    else calibration_step(d_handle, in, noutput_items, d_cal_remaining, d_cal_angle, 0.0, d_cal_kind, d_cal_residual);
    return noutput_items;
}
