// music_b200.cu - C-ABI shim (include/music_b200.h) over the sm_90a (H100) MUSIC DOA kernels.
//
// Host-side responsibilities only: argument checks (the reference's constructor asserts,
// /root/reference/lib/baz_music_doa.cc:45-50, made real), device buffers, the steering-table
// double buffer (set_array_response semantics, :60-70), chunking and host<->device staging.
// No CPU compute path exists here: without an sm_90 device create() fails.
#include "../../include/music_b200.h"

#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "music_kernels.cuh"
#include "music_fused.cuh"
#include "music_covn.cuh"
#include "music_fused8.cuh"
#include "music_steer.cuh"
#include "music_planar.cuh"
#include "music_reduce.cuh"
#include "music_sources.cuh"
#include "music_refine.cuh"
#include "music_azel.cuh"
#include "music_estimators.cuh"
#include "music_iaa.cuh"
#include "music_roots.cuh"
#include "music_manifold.cuh"
#include "music_esprit.cuh"
#include "music_esprit2d.cuh"
#include "music_dml.cuh"
#include "music_wsf.cuh"
#include "music_beams.cuh"
#include "music_calib.cuh"
#include "music_calib_blind.cuh"
#include "music_integrate.cuh"
#include "music_crb.cuh"
#include "music_track.cuh"
#include "music_channels.cuh"
#include "music_focus.cuh"
#include "music_coarray.cuh"

using namespace music;

static_assert(CB_MAX_SEGMENTS == MUSIC_B200_CALIB_MAX_SEGMENTS, "one segment limit");

namespace {

std::mutex g_err_mutex;
std::string g_create_error;

cudaError_t pinned_alloc(void **p, size_t bytes) { return cudaHostAlloc(p, bytes, cudaHostAllocDefault); }

// The owner of one allocation of T elements made by Alloc and released by Free.  Every owner of a handle is destroyed
// while the handle's device is current (music_b200_destroy).
template <class T, cudaError_t (*Alloc)(void **, size_t), cudaError_t (*Free)(void *)>
class Owned {
public:
    Owned() = default;
    Owned(Owned &&o) noexcept { *this = std::move(o); }
    Owned &operator=(Owned &&o) noexcept
    {
        reset();
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        return *this;
    }
    ~Owned() { reset(); }
    // Holds at least n elements afterwards; the old block is freed before the new one is allocated, so a grow never
    // holds both.  The contents are not kept.  On failure the owner is empty.
    cudaError_t grow(size_t n)
    {
        if (n <= n_) return cudaSuccess;
        reset();
        void *p = nullptr;
        const cudaError_t e = Alloc(&p, n * sizeof(T));
        if (e == cudaSuccess) { p_ = static_cast<T *>(p); n_ = n; }
        return e;
    }
    size_t size() const { return n_; }
    T *get() const { return p_; }
    operator T *() const { return p_; }
private:
    void reset()
    {
        if (p_) Free(p_);
        p_ = nullptr;
        n_ = 0;
    }
    T *p_ = nullptr;
    size_t n_ = 0;
};

template <class T> using DevBuf = Owned<T, cudaMalloc, cudaFree>;
template <class T> using PinBuf = Owned<T, pinned_alloc, cudaFreeHost>;

// A view of one steering table; the buffers belong to its TableSlot.
struct DeviceTable {
    float *c64 = nullptr;   // [K][M] (re, im)
    double *soa = nullptr;  // [ntiles][2M+1][TILE]
    unsigned char *fz = nullptr;  // fused kernel's tensor-core screen layout (music_fused.cuh, M = 4 only)
    float *na_max = nullptr;      // max ||a||^2 over the table rows (screen threshold)
    bool screen_ok = true;        // the fused M = 4 kernel's fp32 screen bound holds for every row (screen_bounds_table)
    bool geometric = false;       // built by set_geometry() from `geo` (set_table() tables are not)
    RefineGeom geo = {};          // element positions and wavelength of a geometric table (peak refinement)
    AzelGeom ageo = {};           // the same for an az-el handle (music_b200_create_azel): [M][x, y, z] and the grid
    UlaGeom ula = {};             // whether `geo` is a uniform linear array the root mode accepts, and its p_0 and step
    LatticeGeom lat = {};         // whether `ageo` is a planar lattice the az-el ESPRIT mode accepts, and its steps
    uint32_t mf_L = 0;            // manifold order of `geo` (0: none built); above MF_MAX_L the mode refuses the table
    double mf_aperture = 0.0;     // largest element distance over lambda (the refusal's message)
    const double2 *mf_beta = nullptr;  // [pairs][mf_L + 1] manifold coefficients, in the slot's mf_beta
};

// One slot of the steering-table double buffer (retune()).  `tabs` holds C tables (C: the channel count on a channel
// handle, 1 on every other handle) as views into one c64 and one SoA allocation; it is empty until the slot is first
// used (alloc_slot).
struct TableSlot {
    std::vector<DeviceTable> tabs;
    DevBuf<float> c64;
    DevBuf<double> soa;
    DevBuf<unsigned char> fz;  // the fused M = 4 kernel's screen layout of tabs[0], on the handles that run that kernel
    DevBuf<float> na_max;
    bool shared = false;       // one table from set_table() (tabs[0]) serves every channel
    DevBuf<double2> foc_T;     // COHERENT channel handle: the focusing matrices T_c [C][m][m] of these tables
    std::vector<double> foc_err;  // and their focusing errors e_c
    DevBuf<double2> mf_beta;   // the manifold coefficients of the table the MANIFOLD mode reads (build_manifold)
};

// A non-owning view of a workspace slot's buffers, or of one channel's run of them (enqueue_channels)
struct WsView { double *R, *ev, *Vt, *P64; int32_t *cnt, *bins; double *wts; unsigned long long *n0; float *std; double *X; };

struct Workspace {
    DevBuf<double> R, ev, Vt, P64;
    DevBuf<int32_t> cnt;   // per-window source counts (source rule other than FIXED)
    DevBuf<int32_t> bins;  // [windows][n] peak bins for the refinement and the beams when the caller asked for none
    DevBuf<double> wts;    // [windows][n][m] complex beam weights when a beams call asked for none
    DevBuf<unsigned long long> n0;  // integration: the count since the reset at the sub-batch's first window
    DevBuf<float> std;     // [windows][sw] the CRB a tracks call under CRB variance reads when the caller asked for none
    DevBuf<double> X;      // [windows][m][m] complex: the WSF matrix the DML search reads (music_wsf.cuh)
    DevBuf<double> Rin;    // co-array handle: [windows][m_in][m_in] complex physical R, mapped into R (music_coarray.cuh)
    cudaEvent_t scan_done = nullptr;
    bool used = false;
    WsView view() const { return {R, ev, Vt, P64, cnt, bins, wts, n0, std, X}; }
};

// The modes set by set_peak_mode(), set_refine() and set_estimator(); check_modes() says which combine.
struct Modes {
    int peak = MUSIC_B200_PEAKS_TOP_BINS;
    uint32_t excl = 0;                       // exclusion_bins of the peak mode
    int refine = MUSIC_B200_REFINE_OFF;
    int est = MUSIC_B200_ESTIMATOR_MUSIC;
    double loading = 0.0;                    // MVDR and IAA diagonal loading
    int iaa_iter = IAA_DEFAULT_ITERATIONS;   // IAA iteration count (music_b200_set_iaa_iterations)
};

// Targets of the fused all-gather of the peak bins (SURVEY.md section 8e): with G > 0 this GPU's windows are the
// windows w = i * G + rank of a stream whose bins every GPU p receives in full, in peer[p].
struct Gather {
    int32_t *peer[MAX_PEERS] = {};
    int G = 0, rank = 0;
};

// The outputs of one call: device pointers (host pointers for the caller side of a host entry point), any of them NULL
// but `angles`, with the shape that lays out their rows.
struct Outputs {
    float *angles = nullptr;    // [W][n]; the azimuths on an az-el handle
    float *elev = nullptr;      // [W][n]: az-el handles only
    float *levels = nullptr;    // [W][n]
    float *spec = nullptr;      // [W][K]
    int32_t *bins = nullptr;    // [W][n]
    int32_t *counts = nullptr;  // [W]
    double *P64 = nullptr;      // [W][K]
    double *R = nullptr;        // [W][m][m] complex
    double *ev = nullptr;       // [W][m]
    double *wts = nullptr;      // [W][n][m] complex beam weights: beams entry points only
    float *beams = nullptr;     // [W][n][N] complex64 beams: beams entry points only
    float *std = nullptr;       // [W][sw] the CRB of every slot: crb and tracks entry points only
    int32_t *slot_track = nullptr;   // [W][n] the track each slot's measurement updated or started: tracks entries only
    int32_t *track_ids = nullptr;    // [W][T] the confirmed track of every carry row
    float *track_state = nullptr;    // [W][tsw / T] its state
    Gather gather;
    uint32_t n = 0, K = 0, m = 0, N = 0;
    uint32_t sw = 0;            // floats per window of std: n, 3 n on an az-el handle
    uint32_t T = 0, tsw = 0;    // carry rows of the tracker and floats per window of track_state: 3 T, 6 T on an az-el handle

    // the shape of h's calls and the all-gather h was attached to (music_b200_gather_attach)
    Outputs &shaped(const music_b200 *h);

    // the same outputs from window w0 of the call on
    Outputs at(size_t w0) const
    {
        Outputs o = *this;
        const auto skip = [w0](auto *&p, size_t row) { if (p) p += w0 * row; };
        skip(o.angles, n);
        skip(o.elev, n);
        skip(o.levels, n);
        skip(o.spec, K);
        skip(o.bins, n);
        skip(o.counts, 1);
        skip(o.P64, K);
        skip(o.R, (size_t)m * m * 2);
        skip(o.ev, m);
        skip(o.wts, (size_t)n * m * 2);
        skip(o.beams, (size_t)n * N * 2);
        skip(o.std, sw);
        skip(o.slot_track, n);
        skip(o.track_ids, T);
        skip(o.track_state, tsw);
        for (int p = 0; p < gather.G; ++p) skip(o.gather.peer[p], (size_t)gather.G * n);
        return o;
    }

    // the per-window outputs a host call stages through pinned memory (4-byte elements), with their elements per window
    struct Field { void *p; uint32_t per_win; };
    std::array<Field, 9> window_fields() const
    {
        return {{{angles, n}, {elev, n}, {levels, n}, {bins, n}, {counts, 1}, {std, sw}, {slot_track, n}, {track_ids, T},
                 {track_state, tsw}}};
    }

    // the rows of a beams call a host call stages through pinned memory, with their bytes per window
    struct Row { void *p; size_t bytes; };
    std::array<Row, 2> row_fields() const
    {
        return {{{wts, (size_t)n * m * 2 * sizeof(double)}, {beams, (size_t)n * N * 2 * sizeof(float)}}};
    }
};

// the buffers behind a staging slot's outputs, on the device or pinned (the spectrum is staged on the device only)
template <template <class> class Buf>
struct StagedOutputs {
    Buf<float> angles, elev, levels, spec, beams, std, track_state;
    Buf<int32_t> bins, counts, slot_track, track_ids;
    Buf<double> wts;

    Outputs view(const music_b200 *h) const
    {
        Outputs o;
        o.angles = angles; o.elev = elev; o.levels = levels; o.spec = spec;
        o.beams = beams; o.bins = bins; o.counts = counts; o.wts = wts; o.std = std;
        o.slot_track = slot_track; o.track_ids = track_ids; o.track_state = track_state;
        return o.shaped(h);
    }
};

// One staging stream of the host entry points: the input and output buffers of a chunk, and which windows of the call
// the pinned mirrors hold.  Device->host copies into caller memory would be synchronous when that memory is pageable
// (numpy arrays, GNU Radio buffers) and stall the enqueue of the next chunk's upload, hence the pinned mirrors.
struct HostSlot {
    DevBuf<float> in;
    StagedOutputs<DevBuf> dbuf;
    StagedOutputs<PinBuf> pbuf;
    Outputs dev;   // views of dbuf: device outputs (the spectrum only when a call asked for it)
    Outputs pin;   // views of pbuf: pinned host mirrors of dev's per-window outputs and of its beam and weight rows
    uint32_t w0 = 0, W = 0;  // W = 0: nothing pending
};

}  // namespace

struct music_b200 {
    uint32_t m = 0, n = 0, nsamples = 0, K = 0, N = 0;
    uint32_t m_in = 0;       // elements per input snapshot: m on every handle but a co-array handle, whose m is Mv
    int device = 0;
    int sm_count = 0;
    std::mutex mutex;        // serialises process_*() and set_table(), like d_mutex (:67, :101)
    std::mutex err_mutex;    // guards `error` alone: fail() may run before `mutex` is taken (argument checks)
    std::string error;
    std::atomic<uint64_t> launches{0};

    TableSlot tables[2];
    int cur_table = 0;
    DevBuf<double> steer_pos;      // device copy of the element positions (set_geometry)
    DevBuf<unsigned> steer_count;
    DevBuf<int> steer_list;
    DevBuf<float> steer_vals;
    Modes modes;
    int source_rule = MUSIC_B200_SOURCES_FIXED;  // set_source_rule()
    int beam_rule = MUSIC_B200_BEAMS_OFF;        // set_beamformer(): read by the beams entry points only
    double beam_loading = 0.0;
    // receiver calibration (music_b200_set_calibration): c_m = 1 / g_m applied to every window's R while `calib` is set
    bool calib = false;
    CalibVec cal_c = {};
    double cal_g[2 * MUSIC_B200_MAX_M] = {};  // the gains as set
    // the calibration accumulator (music_b200_calib_*; the served device of a multi-device handle): sum of the raw R
    // over cal_windows windows, the accumulate kernel's per-CTA partial sums and counter, the solve kernel's result
    DevBuf<double2> cal_acc, cal_part;
    DevBuf<unsigned> cal_ctr;
    DevBuf<double> cal_out;
    uint64_t cal_windows = 0;
    // the self-calibration accumulator (music_b200_calib_blind_*, music_calib_blind.cuh; the served device): per segment
    // the sum of the raw R of its windows (zeroed when allocated and at every reset), calib_accum_kernel's partial sums
    // and counter, and the window count of every segment accumulated so far
    DevBuf<double2> cb_acc, cb_part;
    DevBuf<unsigned> cb_ctr;
    std::vector<unsigned> cb_count;
    // the solve's device scratch (music_calib_blind.cuh), grown as the shapes of the solves need
    struct BlindWork {
        DevBuf<unsigned> cnt;
        DevBuf<double> Rw, ev, Vt, mag, Q, qev, qV, jp, J, out, angles;
        DevBuf<double2> Pi, phi;
        DevBuf<int> bins;
        DevBuf<CbState> st;
    } cb_work;
    // covariance integration (music_b200_set_integration, music_integrate.cuh), on while integ_alpha > 0: the carry S [m][m]
    // complex and the window count since the reset on the device, the tile scratch, and the event that orders each
    // sub-batch's integration after the previous one's, on whichever stream that ran.  integ_fresh: the next integration
    // starts from S = 0 and count 0.
    double integ_alpha = 0.0;
    bool integ_fresh = true, integ_used = false;
    DevBuf<double> integ_S, integ_tiles;
    DevBuf<unsigned long long> integ_cnt;
    cudaEvent_t integ_done = nullptr;
    // angle tracking (music_b200_set_tracking, music_track.cuh), on while trk_var is not OFF: the parameters, the carry
    // (rows, states and next_id) on the device, and the event that orders each sub-batch's tracking after the previous
    // one's, on whichever stream that ran.  trk_fresh: the next tracking sub-batch starts from empty rows and next_id 0.
    int trk_var = MUSIC_B200_TRACK_OFF;
    TrackParams trk = {};
    bool trk_fresh = true, trk_used = false;
    DevBuf<int32_t> trk_rows;
    DevBuf<double> trk_state;
    DevBuf<unsigned> trk_next;
    cudaEvent_t trk_done = nullptr;
    unsigned steer_guarded = 0;    // entries of the last built table re-evaluated with the host libm
    bool azel = false;             // music_b200_create_azel(): K = n_az * n_el rows, elevation-major (music_azel.cuh)
    AzelGrid grid = {};
    // channel handle (music_b200_create_channels, music_channels.cuh): the filter bank's shape and its twiddle and taper
    // tables; the C per-channel tables are in the table slots, and create_channels() installs none
    bool chan = false;
    ChanShape cshape = {};
    int chan_taper = MUSIC_B200_TAPER_RECT, chan_combine = MUSIC_B200_CHANNELS_SEPARATE;
    DevBuf<double2> chan_tw;
    DevBuf<double> chan_taper_d;
    int chan_ctas = 1;             // resident CTAs of chan_cov_kernel per SM at this shape
    double chan_fs = 0.0;          // sample rate of the last set_geometry_channels() (0: none yet)
    DevBuf<unsigned char> chan_arena;  // device staging of the channel host entry
    // COHERENT combine (music_focus.cuh): the focusing sector (count 0: the whole grid) and the set-up scratch; the
    // focusing matrices and errors are in the table slots
    uint32_t foc_first = 0, foc_count = 0;
    DevBuf<double> foc_lam;      // [C] the wavelengths of the slot being focused
    DevBuf<double2> foc_B;       // [C][m][m] B_c
    DevBuf<double> foc_e2;       // [C] squared focusing errors
    DevBuf<double2> foc_Rc;      // the filter bank's [C][W][m][m] covariances of a sub-batch (the workspace holds W windows)
    // co-array handle (music_b200_create_coarray, music_coarray.cuh): m_in physical elements, m = Mv virtual ones; the
    // lag table, and the physical R of each sub-batch in its workspace slot's Rin
    bool coarray = false;
    CoarrayLags co_lags = {};

    // fp64 workspace slots (R, eigenvalues, sorted eigenvectors, optional strengths) of the unfused path: one per
    // staging stream of the host entry points (slot 0 also serves the device entry points)
    Workspace ws[2];
    DevBuf<unsigned> work_ctr;         // persistent kernels: ring of self-resetting (window tickets, finished CTAs) pairs, CTR_RING per slot
    unsigned ctr_seq[2] = {0, 0};      // next ring entry per slot
    bool fused_spec = true;            // the spectrum port on the fused M = 4 kernel (MUSIC_B200_FUSED_SPEC=0: three-kernel path)
    bool pdl = true;                   // fused M = 4 kernel: programmatic dependent launch (MUSIC_B200_PDL=0 turns it off)
    cudaEvent_t fused_done = nullptr;  // orders persistent launches that share a ticket counter but not a stream
    bool fused_used[2] = {false, false};
    int eig_mode = 0;                 // fused kernels: 0 principal eigenvector by squaring (default), otherwise their Jacobi solver for every window (four lanes per window at M = 4, one warp at M = 8); MUSIC_B200_EIG=jacobi and the older spelling jacobi1 (2) both select it
    DevBuf<unsigned> f8_stats;        // fused M = 8 kernel: windows solved by squaring / by the Jacobi fallback
    int mma_fin_max = 2;              // fused kernel: no tensor-core pass starts once the tickets have run out and this many covariance warps are done (MUSIC_B200_MMA_FIN; 0: at ticket exhaustion, -1: fp64 drain only)
    DevBuf<long long> fused_trace;     // MUSIC_B200_TRACE=1: per-CTA clock64 trace of the fused kernel (tools/fused_trace.py)
    unsigned trace_seq = 0;            // next launch's slot in the trace ring (FZ_TRACE_LAUNCHES launches of FZ_TRACE_CTAS rows)
    bool fused = true;       // MUSIC_B200_FUSED=0 forces the three-kernel path
    // optional per-stage timing (bench.py's roofline leg): events around K1/K2/K3/top-n per chunk
    bool timing = false;
    std::vector<cudaEvent_t> tev;   // 5 events per timed chunk
    size_t tev_used = 0;

    // host path staging
    cudaStream_t streams[2] = {nullptr, nullptr};
    HostSlot stage[2];
    uint32_t host_chunk = 0;
    bool host_spec_alloc = false;
    bool host_beam_alloc = false;      // the staging slots hold beam and weight rows
    bool host_crb_alloc = false;       // the staging slots hold CRB rows
    uint32_t host_track_T = 0;         // the staging slots hold tracker rows for this many carry rows
    cudaStream_t last_fused_stream[2] = {nullptr, nullptr};  // per ticket counter: launches on one stream need no event

    // caller memory registered for DMA (cudaHostRegister), newest last: GNU Radio hands work() the same pageable
    // circular buffers over and over, so a range is pinned once and found again on every later call
    struct HostReg { uintptr_t base; size_t len; };
    std::vector<HostReg> hostregs;
    bool hostreg = true;   // MUSIC_B200_HOSTREG=0: never register (pageable copies go through the driver's staging)

    // multi-device handle (music_b200_create_multi): one child per device, windows dealt w -> child w mod G
    std::vector<music_b200 *> kids;

    // fused all-gather of the peak bins (music_b200_gather_*): peer-mapped buffers, epoch flags, and every IPC mapping of
    // a peer's buffer or flags this handle has opened
    DevBuf<int32_t> gather_buf;
    DevBuf<unsigned> gather_flags;
    size_t gather_cap = 0;
    Gather gather;
    unsigned *peer_flags[MAX_PEERS] = {};
    std::vector<void *> ipc_maps;
    unsigned gather_epoch = 0;

    ~music_b200()
    {
        for (int i = 0; i < 2; ++i) {
            if (streams[i]) cudaStreamDestroy(streams[i]);
            if (ws[i].scan_done) cudaEventDestroy(ws[i].scan_done);
        }
        if (fused_done) cudaEventDestroy(fused_done);
        if (integ_done) cudaEventDestroy(integ_done);
        if (trk_done) cudaEventDestroy(trk_done);
        for (cudaEvent_t e : tev) cudaEventDestroy(e);
    }
};

namespace {

Outputs &Outputs::shaped(const music_b200 *h)
{
    n = h->n;
    K = h->K;
    m = h->m;
    N = h->N;
    sw = h->azel ? 3 * h->n : h->n;
    T = h->trk.T;
    tsw = (h->azel ? 6 : 3) * T;
    gather = h->gather;
    return *this;
}

int fail(music_b200 *h, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (h) {
        std::lock_guard<std::mutex> g(h->err_mutex);
        h->error = buf;
    } else {
        std::lock_guard<std::mutex> g(g_err_mutex);
        g_create_error = buf;
    }
    return code;
}

#define CU(h, expr)                                                                             \
    do {                                                                                        \
        cudaError_t e_ = (expr);                                                                \
        if (e_ != cudaSuccess)                                                                  \
            return fail((h), e_ == cudaErrorMemoryAllocation ? MUSIC_B200_ENOMEM : MUSIC_B200_ECUDA, \
                        "%s failed: %s", #expr, cudaGetErrorString(e_));                        \
    } while (0)

// Table rows are padded (||a||^2 = +inf) to whole TILE-row tiles.
uint32_t table_tiles(uint32_t K) { return (uint32_t)((K + TILE - 1) / TILE); }
size_t soa_doubles(uint32_t K, uint32_t M) { return (size_t)table_tiles(K) * (2 * M + 1) * TILE; }

// derived layouts (fp64 SoA tiles, TF32 hi/lo MMA fragments) of the c64 table already in t.c64
int finish_table(music_b200 *h, DeviceTable &t, cudaStream_t st)
{
    const int ntiles = (int)table_tiles(h->K);
    prep_table_kernel<<<ntiles, TILE, 0, st>>>(reinterpret_cast<const float2 *>(t.c64), t.soa, (int)h->K, (int)h->m);
    h->launches++;
    if (t.fz) {
        const int threads = (FZ_NDEC + fused_tiles((int)h->K)) * (FZ_BINS / 16) * 32;
        CU(h, cudaMemsetAsync(t.na_max, 0, sizeof(float), st));
        prep_table_tc_kernel<<<(threads + 255) / 256, 256, 0, st>>>(t.c64, t.fz, t.na_max, (int)h->K);
        h->launches++;
    }
    CU(h, cudaGetLastError());
    CU(h, cudaStreamSynchronize(st));
    return MUSIC_B200_OK;
}

// Whether the fused M = 4 kernel's tensor-core screen can bound a [K][4] complex64 table (music_fused.cuh, "Screen
// error bound"): the bound is relative to each row's fl32(||a||^2), so that value and every fp32 quantity of the screen
// must be finite and far from the subnormal range.  Rows of zeros are exact in the screen (d~ = 0) and pass.  A table
// that fails (a calibrated table scaled near the float32 limits) runs on the kernel's all-fp64 drain instead: same
// results, without the tensor-core passes.
bool screen_bounds_table(const float *tab, uint32_t K)
{
    const double lo = 0x1p-100, hi = 0x1p100;
    for (uint32_t k = 0; k < K; ++k) {
        const float *row = tab + (size_t)k * 8;
        double na = 0.0;
        bool zero = true;
        for (int i = 0; i < 4; ++i) {
            na = std::fma((double)row[2 * i], (double)row[2 * i], std::fma((double)row[2 * i + 1], (double)row[2 * i + 1], na));
            zero = zero && row[2 * i] == 0.f && row[2 * i + 1] == 0.f;
        }
        const double f = (double)(float)na;
        if (!zero && !(f >= lo && f <= hi)) return false;  // NaN fails too
    }
    return true;
}

int upload_table(music_b200 *h, DeviceTable &t, const float *table_c64, cudaStream_t st)
{
    t.geometric = false;
    t.lat = {};
    t.screen_ok = h->m != 4 || screen_bounds_table(table_c64, h->K);
    CU(h, cudaMemcpyAsync(t.c64, table_c64, (size_t)h->K * h->m * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
    return finish_table(h, t, st);
}

// The root mode's ULA condition (include/music_b200.h) on positions [M][x, y]: s = (p_{M-1} - p_0) / (M - 1), |s| > 0,
// every element within 1e-6 |s| of p_0 + m s, |s| <= (lambda / 2)(1 + 1e-12).
UlaGeom ula_geometry(const double *pos, int M, double lambda)
{
    UlaGeom u = {};
    u.p0[0] = pos[0];
    u.p0[1] = pos[1];
    u.s[0] = (pos[2 * (M - 1)] - pos[0]) / (M - 1);
    u.s[1] = (pos[2 * (M - 1) + 1] - pos[1]) / (M - 1);
    const double sa = std::hypot(u.s[0], u.s[1]);
    double dev = 0.0;
    for (int m = 0; m < M; ++m)
        dev = std::max(dev, std::hypot(pos[2 * m] - (u.p0[0] + m * u.s[0]), pos[2 * m + 1] - (u.p0[1] + m * u.s[1])));
    u.ula = sa > 0.0 && dev <= 1e-6 * sa && sa <= 0.5 * lambda * (1.0 + 1e-12);
    return u;
}

// The peak modes that take their angles from the geometry instead of the table: ROOTS and ESPRIT (uniform linear
// arrays) and MANIFOLD (any planar array)
bool gridless_mode(int peak)
{
    return peak == MUSIC_B200_PEAKS_ROOTS || peak == MUSIC_B200_PEAKS_ESPRIT || peak == MUSIC_B200_PEAKS_MANIFOLD;
}

bool coherent(const music_b200 *h) { return h->chan && h->chan_combine == MUSIC_B200_CHANNELS_COHERENT; }

// EINVAL naming `what` on a co-array handle, which does not serve it (include/music_b200.h lists what it serves)
int refuse_coarray(music_b200 *h, const char *what)
{
    return h->coarray ? fail(h, MUSIC_B200_EINVAL, "%s is not built for co-array handles", what) : MUSIC_B200_OK;
}

// The independent looks behind each covariance: the N snapshots of a window, on a channel handle its J segments, and
// behind a focused covariance the J segments of all C channels.
uint32_t snapshots(const music_b200 *h)
{
    return !h->chan ? h->N : coherent(h) ? (uint32_t)(h->cshape.J * h->cshape.C) : (uint32_t)h->cshape.J;
}

// Whether handle h can run with modes p; if not, records why and returns EINVAL.  With a table t, also whether p can run
// on it: the gridless ULA peak modes need a ULA geometry, the manifold mode a geometric table of order <= MF_MAX_L, the
// az-el ESPRIT mode a planar lattice with n <= d_max, the refinement a geometric table.  Tables are checked on handles that
// hold one (single-device handles, and the children of a multi-device handle).
int check_modes(music_b200 *h, const Modes &p, const DeviceTable *t)
{
    const bool subspace_fit = p.peak == MUSIC_B200_PEAKS_DML || p.peak == MUSIC_B200_PEAKS_WSF;
    if (p.peak != MUSIC_B200_PEAKS_TOP_BINS && p.peak != MUSIC_B200_PEAKS_LOCAL_MAXIMA && !gridless_mode(p.peak) && !subspace_fit)
        return fail(h, MUSIC_B200_EINVAL, "unknown peak mode %d", p.peak);
    if (p.excl >= h->K) return fail(h, MUSIC_B200_EINVAL, "exclusion_bins must be < resolution");
    if (p.refine != MUSIC_B200_REFINE_OFF && p.refine != MUSIC_B200_REFINE_NEWTON && p.refine != MUSIC_B200_REFINE_JOINT)
        return fail(h, MUSIC_B200_EINVAL, "unknown refine mode %d", p.refine);
    const bool iaa = p.est == MUSIC_B200_ESTIMATOR_IAA;
    if (p.est != MUSIC_B200_ESTIMATOR_MUSIC && p.est != MUSIC_B200_ESTIMATOR_MVDR && p.est != MUSIC_B200_ESTIMATOR_BARTLETT && !iaa)
        return fail(h, MUSIC_B200_EINVAL, "unknown estimator %d", p.est);
    if (!std::isfinite(p.loading) || p.loading < 0.0) return fail(h, MUSIC_B200_EINVAL, "loading must be finite and >= 0 (got %g)", p.loading);
    if (p.est != MUSIC_B200_ESTIMATOR_MVDR && !iaa && p.loading != 0.0)
        return fail(h, MUSIC_B200_EINVAL, "diagonal loading applies to MVDR and IAA only (got %g)", p.loading);
    if (h->coarray) {
        // R_ss is a covariance of the virtual array only under the co-array model, whose noise subspace MUSIC reads
        if (p.est != MUSIC_B200_ESTIMATOR_MUSIC)
            return fail(h, MUSIC_B200_EINVAL, "a co-array handle takes the MUSIC estimator only (MVDR, Bartlett and IAA are not built on "
                                              "the co-array covariance)");
        if (subspace_fit || p.peak == MUSIC_B200_PEAKS_MANIFOLD)
            return fail(h, MUSIC_B200_EINVAL, "a co-array handle takes the TOP_BINS, LOCAL_MAXIMA, ROOTS and ESPRIT peak modes only "
                                              "(DML, WSF and MANIFOLD are not built on the co-array covariance)");
        if (p.refine == MUSIC_B200_REFINE_JOINT) return fail(h, MUSIC_B200_EINVAL, "a co-array handle takes refinement OFF or NEWTON");
    }
    if (iaa && p.refine != MUSIC_B200_REFINE_OFF)
        return fail(h, MUSIC_B200_EINVAL, "the IAA estimator takes refinement OFF (refinement of IAA peaks is not built)");
    if (p.est == MUSIC_B200_ESTIMATOR_MVDR && p.loading == 0.0 && snapshots(h) <= h->m)
        return fail(h, MUSIC_B200_EINVAL, "MVDR without diagonal loading needs more snapshots than antennas (N = %u, m = %u): R is singular",
                    snapshots(h), h->m);
    if (h->chan && !coherent(h)) {
        // per channel only the grid modes are built (include/music_b200.h lists the rest as not built)
        if (p.peak != MUSIC_B200_PEAKS_TOP_BINS && p.peak != MUSIC_B200_PEAKS_LOCAL_MAXIMA)
            return fail(h, MUSIC_B200_EINVAL, "a channel handle takes the TOP_BINS and LOCAL_MAXIMA peak modes only (ROOTS, ESPRIT, "
                                              "MANIFOLD, DML and WSF per channel are not built)");
        if (p.refine != MUSIC_B200_REFINE_OFF) return fail(h, MUSIC_B200_EINVAL, "peak refinement is not built for channel handles");
        if (h->chan_combine == MUSIC_B200_CHANNELS_INCOHERENT && p.est != MUSIC_B200_ESTIMATOR_MUSIC)
            return fail(h, MUSIC_B200_EINVAL, "the INCOHERENT combine is defined for the MUSIC estimator only");
    }
    if (gridless_mode(p.peak)) {
        const bool mf = p.peak == MUSIC_B200_PEAKS_MANIFOLD;
        const char *name = p.peak == MUSIC_B200_PEAKS_ROOTS ? "root" : mf ? "manifold" : "ESPRIT";
        if (p.excl != 0) return fail(h, MUSIC_B200_EINVAL, "the %s peak mode takes exclusion_bins = 0", name);
        if (h->azel && p.peak != MUSIC_B200_PEAKS_ESPRIT)
            return fail(h, MUSIC_B200_EINVAL, "the %s peak mode is not supported on an az-el handle", name);
        if (p.est != MUSIC_B200_ESTIMATOR_MUSIC) return fail(h, MUSIC_B200_EINVAL, "the %s peak mode needs the MUSIC estimator", name);
        if (p.refine != MUSIC_B200_REFINE_OFF) return fail(h, MUSIC_B200_EINVAL, "the %s peak mode needs refinement off", name);
        if (t && h->azel && !(t->geometric && t->lat.ok))
            return fail(h, MUSIC_B200_EINVAL, "the ESPRIT peak mode on an az-el handle needs a table built by "
                                              "music_b200_set_geometry_azel() from a planar lattice array (Mx x My elements "
                                              "in row-major order, one z, steps <= lambda / 2) (call set_geometry_azel(), or "
                                              "another peak mode)");
        if (t && h->azel && h->n > (uint32_t)esp2_dmax(t->lat))
            return fail(h, MUSIC_B200_EINVAL, "the ESPRIT peak mode on this %d x %d lattice resolves at most %d sources (n = %u)",
                        t->lat.mx, t->lat.my, esp2_dmax(t->lat), h->n);
        if (t && mf && !t->geometric)
            return fail(h, MUSIC_B200_EINVAL, "the manifold peak mode needs a table built by music_b200_set_geometry() (call "
                                              "set_geometry(), or another peak mode)");
        if (t && mf && t->mf_L > (uint32_t)MF_MAX_L)
            return fail(h, MUSIC_B200_EINVAL, "the manifold peak mode needs an aperture of about 4.4 wavelengths or less: this "
                                              "geometry spans %.4g wavelengths (order %u > %d)", t->mf_aperture, t->mf_L, MF_MAX_L);
        if (t && !mf && !h->azel && !(t->geometric && t->ula.ula))
            return fail(h, MUSIC_B200_EINVAL, "the %s peak mode needs a table built by music_b200_set_geometry() from a uniform linear "
                                              "array with spacing <= lambda / 2 (call set_geometry(), or another peak mode)", name);
    }
    if (subspace_fit) {
        // any 1-D table: DML and WSF read table rows only
        const char *name = p.peak == MUSIC_B200_PEAKS_DML ? "DML" : "WSF";
        if (p.excl != 0) return fail(h, MUSIC_B200_EINVAL, "the %s peak mode takes exclusion_bins = 0", name);
        if (h->azel) return fail(h, MUSIC_B200_EINVAL, "the %s peak mode is not supported on an az-el handle", name);
        if (p.est != MUSIC_B200_ESTIMATOR_MUSIC) return fail(h, MUSIC_B200_EINVAL, "the %s peak mode needs the MUSIC estimator", name);
        if (p.refine == MUSIC_B200_REFINE_NEWTON)
            return fail(h, MUSIC_B200_EINVAL, "the %s peak mode takes refinement OFF or JOINT (NEWTON refines the MUSIC objective)", name);
    }
    if (p.refine == MUSIC_B200_REFINE_JOINT) {
        if (!subspace_fit)
            return fail(h, MUSIC_B200_EINVAL, "JOINT refinement needs the DML or WSF peak mode (NEWTON refines the grid modes)");
        if (h->chan) return fail(h, MUSIC_B200_EINVAL, "JOINT refinement is not built for channel handles");
    }
    if (t && p.refine != MUSIC_B200_REFINE_OFF && !t->geometric)
        return fail(h, MUSIC_B200_EINVAL, "peak refinement needs a table built by music_b200_set_geometry(); the current one came from "
                                          "set_table() (call set_geometry(), or set_refine(OFF))");
    return MUSIC_B200_OK;
}

const TableSlot &cur_slot(const music_b200 *h) { return h->tables[h->cur_table]; }

// Whether the current slot holds a table.  A channel handle has none until its first retune, a multi-device handle none
// at all (its children hold the copies).
bool has_table(const music_b200 *h) { return !cur_slot(h).tabs.empty(); }

// the current table channel c scans with (c = 0 on a handle without channels)
const DeviceTable &table(const music_b200 *h, int c = 0)
{
    const TableSlot &s = cur_slot(h);
    return s.tabs[s.shared ? 0 : c];
}

// The current table of a handle that holds one.  On a channel handle: the reference channel's (what a focused covariance
// is matched against).
const DeviceTable *own_table(const music_b200 *h) { return has_table(h) ? &table(h, h->chan ? h->cshape.C / 2 : 0) : nullptr; }

// The handle that serves an entry point which a multi-device handle does not spread over its devices: device 0.
music_b200 *served(music_b200 *h) { return h && !h->kids.empty() ? h->kids[0] : h; }

// Applies a setting to every device of a multi-device handle (to none on a single-device handle); the first child that
// refuses it reports its error on h.
template <class F>
int for_each_child(music_b200 *h, F apply)
{
    for (music_b200 *c : h->kids)
        if (const int rc = apply(c)) return fail(h, rc, "%s", music_b200_last_error(c));
    return MUSIC_B200_OK;
}

// Steering table built on the device from the element positions (music_steer.cuh), then patched at the
// few entries whose float32 rounding could depend on the libm in use.
int build_table(music_b200 *h, DeviceTable &t, const double *pos_xy, double lambda, cudaStream_t st)
{
    const int K = (int)h->K, M = (int)h->m;
    t.geometric = false;
    t.screen_ok = true;  // unit-modulus rows: ||a||^2 = M
    CU(h, h->steer_pos.grow(2 * MUSIC_B200_MAX_M));
    CU(h, h->steer_count.grow(1));
    CU(h, h->steer_list.grow(STEER_GUARD_CAP));
    CU(h, h->steer_vals.grow(2 * STEER_GUARD_CAP));
    CU(h, cudaMemcpyAsync(h->steer_pos, pos_xy, sizeof(double) * 2 * M, cudaMemcpyHostToDevice, st));
    CU(h, cudaMemsetAsync(h->steer_count, 0, sizeof(unsigned), st));
    steer_table_kernel<<<(K * M + 255) / 256, 256, 0, st>>>(h->steer_pos, lambda, K, M, reinterpret_cast<float2 *>(t.c64),
                                                           h->steer_count, h->steer_list);
    h->launches++;
    CU(h, cudaGetLastError());
    unsigned cnt = 0;
    CU(h, cudaMemcpyAsync(&cnt, h->steer_count, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    h->steer_guarded = cnt;
    if (cnt > (unsigned)STEER_GUARD_CAP) {
        // more boundary cases than the list holds (a degenerate geometry, e.g. all elements at the origin, makes
        // every entry exactly (1, 0)): evaluate every entry the literal way
        std::vector<float> full((size_t)K * M * 2);
        for (int k = 0; k < K; ++k)
            for (int a = 0; a < M; ++a) steer_entry_host(pos_xy, lambda, K, k, a, &full[2 * ((size_t)k * M + a)], &full[2 * ((size_t)k * M + a) + 1]);
        CU(h, cudaMemcpyAsync(t.c64, full.data(), full.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        CU(h, cudaStreamSynchronize(st));
    } else if (cnt) {
        std::vector<int> list(cnt);
        CU(h, cudaMemcpyAsync(list.data(), h->steer_list, sizeof(int) * cnt, cudaMemcpyDeviceToHost, st));
        CU(h, cudaStreamSynchronize(st));
        std::vector<float> vals(2 * (size_t)cnt);
        for (unsigned i = 0; i < cnt; ++i) steer_entry_host(pos_xy, lambda, K, list[i] / M, list[i] % M, &vals[2 * i], &vals[2 * i + 1]);
        CU(h, cudaMemcpyAsync(h->steer_vals, vals.data(), vals.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        steer_patch_kernel<<<(cnt + 255) / 256, 256, 0, st>>>(reinterpret_cast<float2 *>(t.c64), h->steer_list,
                                                            reinterpret_cast<const float2 *>(h->steer_vals.get()), (int)cnt);
        h->launches++;
        CU(h, cudaGetLastError());
        CU(h, cudaStreamSynchronize(st));  // vals is a local
    }
    const int rc = finish_table(h, t, st);
    if (rc) return rc;
    t.geometric = true;
    for (int i = 0; i < 2 * M; ++i) t.geo.pos[i] = pos_xy[i];
    t.geo.lambda = lambda;
    t.ula = ula_geometry(pos_xy, M, lambda);
    return MUSIC_B200_OK;
}

// The manifold order and coefficients (music_manifold.cuh) of the geometric table t into slot s: the table the MANIFOLD
// peak mode reads, a plain handle's or a COHERENT channel handle's reference channel's.  Built at every such retune, so
// a slot's table and coefficients always come from one geometry.  A geometry above the order cap keeps its order (for
// the refusal) and no coefficients.
int build_manifold(music_b200 *h, TableSlot &s, DeviceTable &t)
{
    const int M = (int)h->m;
    t.mf_beta = nullptr;
    if (!manifold_coeffs_host(t.geo.pos, M, t.geo.lambda, &t.mf_L, nullptr, &t.mf_aperture)) return MUSIC_B200_OK;
    std::vector<double> beta((size_t)M * (M - 1) / 2 * (t.mf_L + 1) * 2);
    manifold_coeffs_host(t.geo.pos, M, t.geo.lambda, &t.mf_L, beta.data(), nullptr);
    CU(h, s.mf_beta.grow(beta.size() / 2));
    CU(h, cudaMemcpy(s.mf_beta, beta.data(), beta.size() * sizeof(double), cudaMemcpyHostToDevice));
    t.mf_beta = s.mf_beta;
    return MUSIC_B200_OK;
}

// Steering table of an az-el handle, built on the device from the element positions [M][x, y, z] (music_azel.cuh).
// No host patching: the table is defined to within one float32 ulp, not bit for bit.
int build_table_azel(music_b200 *h, DeviceTable &t, const double *pos_xyz, double lambda, cudaStream_t st)
{
    const int K = (int)h->K, M = (int)h->m;
    t.geometric = false;
    AzelGeom g = {};
    for (int i = 0; i < 3 * M; ++i) g.pos[i] = pos_xyz[i];
    g.lambda = lambda;
    g.grid = h->grid;
    azel_table_kernel<<<(K * M + 255) / 256, 256, 0, st>>>(g, M, reinterpret_cast<float2 *>(t.c64));
    h->launches++;
    CU(h, cudaGetLastError());
    const int rc = finish_table(h, t, st);
    if (rc) return rc;
    t.geometric = true;
    t.ageo = g;
    t.lat = azel_lattice(pos_xyz, M, lambda);
    return MUSIC_B200_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
EncodeTiledFn encode_tiled_fn()
{
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return nullptr;
        return reinterpret_cast<EncodeTiledFn>(p);
    }();
    return fn;
}

// Inside the chunk loops of the host entry points an error must not skip the common tail (stream syncs, slot
// reset): record it in rc and leave the loop instead of returning.
#define CU_BREAK(h, rc, expr)                                                                    \
    {                                                                                            \
        cudaError_t e_ = (expr);                                                                 \
        if (e_ != cudaSuccess) {                                                                 \
            rc = fail((h), e_ == cudaErrorMemoryAllocation ? MUSIC_B200_ENOMEM : MUSIC_B200_ECUDA, \
                      "%s failed: %s", #expr, cudaGetErrorString(e_));                           \
            break;                                                                               \
        }                                                                                        \
    }

constexpr unsigned CTR_RING = 256;  // ticket-counter pairs per slot (see ticket_counter)

enum class Path { Unfused, Fused4, Fused8 };
enum class Scan { None, Peak1, Grid };                     // scan_peak1_kernel, scan_kernel
enum class Peaks { None, TopN, Local, Local2D, Roots, Esprit, Esprit2D, Manifold, Dml };  // topn, topn_local, topn_local2d, roots, esprit, esprit2d, manifold, dml kernels

// What one call runs, from the handle's modes, the requested outputs and the input form (plan_call).
struct Plan {
    Path path = Path::Unfused;   // Fused8 still runs unfused when its tensor map cannot be encoded
    // the unfused path, per sub-batch:
    bool eig = false, count = false, mvdr = false;  // eigensolver, source count, MVDR preparation
    Scan scan = Scan::None;
    bool argmax = false, p64 = false, spec = false;  // template flags of scan_kernel
    int est = MUSIC_B200_ESTIMATOR_MUSIC;            // the form of scan_kernel and the refined objective
    Peaks peaks = Peaks::None;
    bool decode = false, refine = false;             // az-el bin decode; peak refinement (the az-el kind after a decode)
    bool wsf = false, joint = false;                 // the WSF matrix after the eigensolver; JOINT refinement after the peaks
    bool beams = false;                              // beam weights (+ beams) after the peaks: the beams entry points
    bool crb = false;                                // the CRB of every slot after the peaks (and beams): the crb entries
    bool track = false;                              // then the tracker (music_track.cuh): the tracks entries
    bool calib = false;                              // correct R after the covariance (and the beam weights) by the calibration
    bool integ = false;                              // then integrate R across windows (music_b200_set_integration)
    bool ws_p64 = false, ws_counts = false, ws_bins = false, ws_wts = false, ws_std = false;  // workspace buffers the kernels write
    bool combine = false;                            // channel handle, INCOHERENT: one spectrum per window from all channels
};

Plan plan_call(const music_b200 *h, const Outputs &o, const PlanarStreams *planar, unsigned hop)
{
    const Modes &md = h->modes;
    const bool fixed_n = h->source_rule == MUSIC_B200_SOURCES_FIXED;
    const bool music_est = md.est == MUSIC_B200_ESTIMATOR_MUSIC;
    const bool local = md.peak == MUSIC_B200_PEAKS_LOCAL_MAXIMA;
    const bool gridless = gridless_mode(md.peak);
    const bool wsf = md.peak == MUSIC_B200_PEAKS_WSF;
    const bool dml = md.peak == MUSIC_B200_PEAKS_DML || wsf;  // WSF runs the DML search on its matrix X
    Plan p;
    // The fused kernels find the principal eigenvector only, not every eigenvalue a source count needs nor the noise
    // eigenvectors the peak refinement needs; they compute the MUSIC spectrum only.  Planar streams can take the M = 4
    // kernel when the 16-byte granularity of its bulk copies allows it.
    bool planar_fusable = !planar || (hop % 2 == 0 && h->N % 2 == 0);
    for (uint32_t r = 0; planar && r < h->m_in; ++r) planar_fusable = planar_fusable && (reinterpret_cast<uintptr_t>(planar->p[r]) & 15u) == 0;
    // A beams call needs R, which the fused kernels keep in registers: it runs the unfused plan of a call that asks for R.
    const bool beams = o.wts || o.beams;
    const bool track = o.slot_track != nullptr;
    // a co-array handle never fuses: the fused kernels read the input with M = m, and its input has m_in elements
    const bool fusable = h->fused && !h->chan && !h->azel && !h->coarray && music_est && fixed_n && md.refine == MUSIC_B200_REFINE_OFF &&
                         md.peak == MUSIC_B200_PEAKS_TOP_BINS && h->n == 1 && !o.P64 && !o.R && !o.ev && !beams && !o.std && !track &&
                         !h->calib && h->integ_alpha == 0.0;
    if (fusable && h->m == 4 && planar_fusable && (!o.spec || h->fused_spec)) p.path = Path::Fused4;
    else if (fusable && h->m == 8 && !planar && !o.spec && h->N >= 128 && h->N % 2 == 0) p.path = Path::Fused8;

    // MVDR and Bartlett need the eigensolver only to count sources or when the caller asked for the eigenvalues; DML
    // (which reads R only) also for the MUSIC spectrum or P64; WSF always (X is built from the eigenvectors)
    p.eig = (music_est && (!dml || o.spec || o.P64)) || !fixed_n || o.ev || wsf;
    p.count = !fixed_n;
    p.mvdr = md.est == MUSIC_B200_ESTIMATOR_MVDR;
    p.est = md.est;
    // IAA writes P64 and leaves the peaks to the grid peak rules
    p.argmax = h->n == 1 && !local && !gridless && !dml && md.est != MUSIC_B200_ESTIMATOR_IAA;
    p.spec = o.spec != nullptr;
    if (music_est && (gridless || dml)) {
        // the grid spectrum only when the caller asked for it; the angles come from the root, ESPRIT or DML kernel
        p.scan = o.spec || o.P64 ? Scan::Grid : Scan::None;
        p.p64 = p.scan == Scan::Grid;
    } else if (music_est && p.argmax && !o.P64 && !o.spec && (h->m == 4 || h->m == 8 || h->m == 16)) {
        p.scan = Scan::Peak1;
    } else {
        p.scan = Scan::Grid;
        p.p64 = !p.argmax || o.P64;
    }
    if (gridless) p.peaks = md.peak == MUSIC_B200_PEAKS_ROOTS ? Peaks::Roots : md.peak != MUSIC_B200_PEAKS_ESPRIT ? Peaks::Manifold
                            : h->azel ? Peaks::Esprit2D : Peaks::Esprit;
    else if (dml) p.peaks = Peaks::Dml;
    else if (!p.argmax) p.peaks = local && h->azel ? Peaks::Local2D : local ? Peaks::Local : Peaks::TopN;
    p.decode = h->azel && p.peaks != Peaks::Esprit2D;  // the 2-D ESPRIT kernel writes both angles itself
    p.refine = md.refine == MUSIC_B200_REFINE_NEWTON;
    p.joint = md.refine == MUSIC_B200_REFINE_JOINT;
    p.wsf = wsf;
    p.ws_p64 = p.p64 && !o.P64;
    p.ws_counts = p.count;
    p.beams = beams;
    p.track = track;
    p.crb = o.std != nullptr || (track && h->trk_var == MUSIC_B200_TRACK_CRB);
    p.calib = h->calib;
    p.integ = h->integ_alpha > 0.0;
    p.ws_bins = p.decode || p.refine || p.joint || ((beams || p.crb || track) && !o.bins);
    p.ws_wts = beams && !o.wts;
    p.ws_std = p.crb && !o.std;
    if (h->chan && h->chan_combine == MUSIC_B200_CHANNELS_INCOHERENT) {
        // every channel's scan writes its fp64 strengths into the workspace; the combine kernel writes the spectrum and
        // the peak rule (also for n = 1) reads the combined strengths
        p.combine = true;
        p.scan = Scan::Grid;
        p.argmax = false;
        p.p64 = p.ws_p64 = true;
        p.spec = false;
        p.peaks = local ? Peaks::Local : Peaks::TopN;
    }
    return p;
}

// Windows per sub-batch bounding one workspace slot to ~384 MiB.
uint32_t max_sub_windows(const music_b200 *h, const Plan &p)
{
    const size_t per_win = (size_t)h->m * h->m * 2 * 8 * 2 + h->m * 8 + (p.ws_p64 ? (size_t)h->K * 8 : 0) +
                           (p.ws_counts ? sizeof(int32_t) : 0) + (p.ws_bins ? h->n * sizeof(int32_t) : 0) +
                           (p.ws_wts ? (size_t)h->n * h->m * 2 * sizeof(double) : 0) +
                           (p.ws_std ? (size_t)(h->azel ? 3 : 1) * h->n * sizeof(float) : 0) +
                           (p.wsf ? (size_t)h->m * h->m * 2 * sizeof(double) : 0) +
                           (h->coarray ? (size_t)h->m_in * h->m_in * 2 * sizeof(double) : 0);
    // A SEPARATE / INCOHERENT channel handle's workspace holds C pseudo-windows per window; a COHERENT one holds the
    // windows, and the channel buffer beside it the C covariances of each.
    const size_t C = h->chan ? (size_t)h->cshape.C : 1;
    size_t c = coherent(h) ? ((size_t)384 << 20) / (per_win + C * h->m * h->m * sizeof(double2)) : ((size_t)384 << 20) / (per_win * C);
    c = std::max<size_t>(SCAN_B, std::min<size_t>(c, 1u << 20));
    return (uint32_t)(c / SCAN_B * SCAN_B);
}

int ensure_slot(music_b200 *h, Workspace &ws, uint32_t windows, const Plan &p)
{
    bool idle = !ws.used;
    const auto grow = [&](auto &buf, size_t elems) -> int {
        if (elems <= buf.size()) return MUSIC_B200_OK;
        // the slot may still be in use by an earlier call on another stream
        if (!idle) CU(h, cudaEventSynchronize(ws.scan_done));
        idle = true;
        CU(h, buf.grow(elems));
        return MUSIC_B200_OK;
    };
    const size_t w = windows, mm = (size_t)h->m * h->m * 2;
    if (const int rc = grow(ws.R, w * mm)) return rc;
    if (const int rc = grow(ws.Vt, w * mm)) return rc;
    if (const int rc = grow(ws.ev, w * h->m)) return rc;
    if (const int rc = grow(ws.P64, p.ws_p64 ? w * h->K : 0)) return rc;
    if (const int rc = grow(ws.cnt, p.ws_counts ? w : 0)) return rc;
    if (const int rc = grow(ws.bins, p.ws_bins ? w * h->n : 0)) return rc;
    if (const int rc = grow(ws.n0, p.integ ? 1 : 0)) return rc;
    if (const int rc = grow(ws.std, p.ws_std ? w * (h->azel ? 3 : 1) * h->n : 0)) return rc;
    if (const int rc = grow(ws.X, p.wsf ? w * mm : 0)) return rc;
    if (const int rc = grow(ws.Rin, h->coarray ? w * h->m_in * h->m_in * 2 : 0)) return rc;
    return grow(ws.wts, p.ws_wts ? w * h->n * h->m * 2 : 0);
}

// Runtime M -> the M template argument of the scan kernels: 4, 8 and 16 are specialised, every other M runs the
// generic instantiation (0).  f receives std::integral_constant<int, MT>.
template <class F>
void with_scan_m(uint32_t M, F f)
{
    switch (M) {
    case 4: f(std::integral_constant<int, 4>()); break;
    case 8: f(std::integral_constant<int, 8>()); break;
    case 16: f(std::integral_constant<int, 16>()); break;
    default: f(std::integral_constant<int, 0>()); break;
    }
}

template <bool A, bool P, bool S>
struct ScanFlags {
    static constexpr bool argmax = A, p64 = P, spec = S;
};

// The six (argmax, p64, spec) instantiations of scan_kernel per form: without the arg-max the peak rule
// reads P64, so P64 is written.  f receives the matching ScanFlags.
template <class F>
void with_scan_flags(const Plan &p, F f)
{
    if (p.argmax && !p.p64 && !p.spec) f(ScanFlags<true, false, false>());
    else if (p.argmax && !p.p64 && p.spec) f(ScanFlags<true, false, true>());
    else if (p.argmax && p.p64 && !p.spec) f(ScanFlags<true, true, false>());
    else if (p.argmax && p.p64 && p.spec) f(ScanFlags<true, true, true>());
    else if (!p.argmax && p.p64 && !p.spec) f(ScanFlags<false, true, false>());
    else if (!p.argmax && p.p64 && p.spec) f(ScanFlags<false, true, true>());
}

template <int F, bool C>
struct ScanForm {
    static constexpr int form = F;
    static constexpr bool counts = C;
};

// The (FORM, COUNTS) instantiations of scan_kernel: the estimator's strength, and for MUSIC whether the scan reads the
// per-window source counts (cnt).  f receives the matching ScanForm.
template <class F>
void with_scan_form(const Plan &p, const int32_t *cnt, F f)
{
    if (p.est == MUSIC_B200_ESTIMATOR_MVDR) f(ScanForm<EST_MVDR, false>());
    else if (p.est == MUSIC_B200_ESTIMATOR_BARTLETT) f(ScanForm<EST_BARTLETT, false>());
    else if (cnt) f(ScanForm<EST_MUSIC, true>());
    else f(ScanForm<EST_MUSIC, false>());
}

// IAA (music_iaa.cuh) of W windows from ws.R against table tb: P64 [W][K], and the float spectrum when spec != NULL
void launch_iaa(music_b200 *h, const WsView &ws, uint32_t W, double *p64, float *spec, const DeviceTable &tb, cudaStream_t st)
{
    const int M = (int)h->m;
    with_scan_m(h->m, [&](auto mt) {
        constexpr int MT = decltype(mt)::value;
        const auto go = [&](auto tt) {
            constexpr int T = decltype(tt)::value;
            const size_t smem = iaa_smem_doubles(M, T) * sizeof(double);
            iaa_kernel<MT, T><<<(W + T - 1) / T, IAA_THREADS, smem, st>>>(tb.soa, ws.R, M, (int)h->K, (int)W, h->modes.iaa_iter,
                                                                         h->modes.loading, p64, spec);
        };
        if constexpr (MT != 0) go(std::integral_constant<int, iaa_windows(MT)>());
        else if (M > 8) go(std::integral_constant<int, iaa_windows(16)>());
        else go(std::integral_constant<int, iaa_windows(2)>());
    });
    h->launches++;
}

// K3, the grid scan of W windows the plan chose against table tb, into the outputs o of these windows.  cnt: the
// per-window source counts (NULL under the FIXED rule).  scan_kernel stages per window the eigenvectors (MUSIC), the g_j of mvdr_prep_kernel
// (MVDR) or R (Bartlett).
void launch_scan(music_b200 *h, const Plan &p, const WsView &ws, uint32_t W, const Outputs &o, const PeakOut &po,
                 const int32_t *cnt, const DeviceTable &tb, cudaStream_t st)
{
    if (p.scan == Scan::None) return;
    if (p.est == MUSIC_B200_ESTIMATOR_IAA) {
        launch_iaa(h, ws, W, o.P64 ? o.P64 : ws.P64, o.spec, tb, st);
        return;
    }
    const double *soa = tb.soa;
    const double *V = p.est == MUSIC_B200_ESTIMATOR_BARTLETT ? ws.R : ws.Vt;
    float *d_spec = o.spec;
    double *d_p64 = o.P64 ? o.P64 : ws.P64;
    const int M = (int)h->m, n = (int)h->n, K = (int)h->K, grid = (W + SCAN_B - 1) / SCAN_B;
    const size_t smem = (size_t)SCAN_B * M * M * 2 * sizeof(double);
    with_scan_m(h->m, [&](auto mt) {
        constexpr int MT = decltype(mt)::value;
        if (p.scan == Scan::Peak1) {
            if constexpr (MT != 0) scan_peak1_kernel<MT><<<grid, TILE, 0, st>>>(soa, ws.Vt, K, (int)W, po, cnt);  // (planned for M = 4, 8, 16 only)
            return;
        }
        with_scan_form(p, cnt, [&](auto fm) {
            with_scan_flags(p, [&](auto f) {
                using Fm = decltype(fm);
                using Fl = decltype(f);
                scan_kernel<MT, Fm::form, Fl::argmax, Fl::p64, Fl::spec, Fm::counts>
                    <<<grid, TILE, smem, st>>>(soa, V, M, n, K, (int)W, po, d_spec, d_p64, cnt);
            });
        });
    });
    h->launches++;
}

cudaEvent_t *timing_events(music_b200 *h)
{
    if (!h->timing) return nullptr;
    if (h->tev_used + 5 > h->tev.size()) {
        for (int i = 0; i < 5; ++i) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return nullptr;
            h->tev.push_back(e);
        }
    }
    cudaEvent_t *p = h->tev.data() + h->tev_used;
    h->tev_used += 5;
    return p;
}

// Ticket counter pair `slot` (0 / 1) for a persistent kernel about to be launched on `st`.  The counters re-arm
// themselves at the end of a launch, so launches that share a pair must not overlap: on one stream that is stream
// order; when the stream changes, the new stream first waits for everything enqueued on the previous one.
unsigned *ticket_counter(music_b200 *h, int slot, cudaStream_t st)
{
    slot &= 1;
    if (h->fused_used[slot] && h->last_fused_stream[slot] != st) {
        if (cudaEventRecord(h->fused_done, h->last_fused_stream[slot]) != cudaSuccess ||
            cudaStreamWaitEvent(st, h->fused_done, 0) != cudaSuccess) {
            cudaGetLastError();        // e.g. the previous stream no longer exists
            cudaDeviceSynchronize();
        }
    }
    h->fused_used[slot] = true;
    h->last_fused_stream[slot] = st;
    // Every launch draws its own pair from the slot's ring: with programmatic dependent launch the CTAs of launch k + 1
    // run next to those of launch k (the fused M = 4 kernel: in the other half of each SM), so the two must not share
    // tickets.  A pair is reused CTR_RING launches later; launches on one stream overlap only with their neighbours (a
    // launch's CTAs leave only after the previous launch has finished), so fewer than CTR_RING launches are ever resident together.
    const unsigned e = h->ctr_seq[slot]++ % CTR_RING;
    return h->work_ctr + 2 * ((size_t)slot * CTR_RING + e);
}

// K1: covariance of W windows of m_in elements into ws.R, on `st`.
void launch_cov(music_b200 *h, const WsView &ws, const float *d_in, uint32_t W, cudaStream_t st, int ctr_slot)
{
    const int M = (int)h->m_in, N = (int)h->N;
    if (M == 4) {
        // persistent, one CTA per SM, per-warp TMA ring (see cov4_tma_kernel)
        const int grid = std::min<int>(h->sm_count, (int)((W + COV_WARPS - 1) / COV_WARPS));
        cov4_tma_kernel<<<grid, COV_WARPS * 32, COV_SMEM, st>>>(d_in, ws.R, (int)W, N);
        h->launches++;
        return;
    }
    if ((M == 8 || M == 16) && N >= 128 && N % (16 / M) == 0 && encode_tiled_fn()) {
        // TMA-tiled, window staged once per group of warps (music_covn.cuh)
        CUtensorMap tm;
        // rows of 128 bytes (SPR snapshots each): with SWIZZLE_128B a narrower inner box would be padded to the span
        const int SPR = 16 / M;  // snapshots per 128-byte row
        const cuuint64_t gdim[3] = {32u, (cuuint64_t)(N / SPR), (cuuint64_t)W};
        const cuuint64_t gstr[2] = {128u, (cuuint64_t)(8 * M) * (cuuint64_t)N};
        const cuuint32_t box[3] = {32u, (cuuint32_t)(M == 8 ? 32 * CovNJobs<8>::STEPS * 8 * 8 / 128 : 32 * CovNJobs<16>::STEPS * 8 * 16 / 128), 1u};  // one stage
        const cuuint32_t estr[3] = {1u, 1u, 1u};
        const CUresult cr = encode_tiled_fn()(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float *>(d_in), gdim, gstr, box, estr,
                                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                              CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr == CUDA_SUCCESS) {
            constexpr int groups8 = CN_WARPS / CovNJobs<8>::J, groups16 = CN_WARPS / CovNJobs<16>::J;
            const int groups = M == 8 ? groups8 : groups16;
            const int grid = std::min<int>(h->sm_count, (int)((W + groups - 1) / groups));
            unsigned *ctr = ticket_counter(h, ctr_slot, st);
            if (M == 8) covN_tma_kernel<8><<<grid, CN_WARPS * 32, CN_SMEM, st>>>(tm, ws.R, (int)W, N, ctr);
            else covN_tma_kernel<16><<<grid, CN_WARPS * 32, CN_SMEM, st>>>(tm, ws.R, (int)W, N, ctr);
            h->launches++;
            return;
        }
        // (encode failed: the tile kernels below)
    }
    if (M % 4 == 0) {
        const int T = M / 4;
        const int wpb = 8;
        {
            const long long items = (long long)W * T;
            cov_tile_kernel<false><<<(unsigned)((items + wpb - 1) / wpb), wpb * 32, 0, st>>>(d_in, ws.R, (int)W, N, M);
            h->launches++;
        }
        if (T > 1) {
            const long long items = (long long)W * (T * (T - 1) / 2);
            cov_tile_kernel<true><<<(unsigned)((items + wpb - 1) / wpb), wpb * 32, 0, st>>>(d_in, ws.R, (int)W, N, M);
            h->launches++;
        }
    } else {
        const int E = M * (M + 1) / 2;
        const int S = 256 / E;
        cov_generic_kernel<<<W, 256, (size_t)S * E * 2 * sizeof(double), st>>>(d_in, ws.R, (int)W, N, M);
        h->launches++;
    }
}

// The peak kernels' view of the outputs o (already moved to the batch's first window by Outputs::at)
PeakOut make_peak_out(const Outputs &o)
{
    PeakOut po;
    po.angles = o.angles; po.levels = o.levels; po.bins = o.bins;
    po.npeer = o.gather.G; po.rank = o.gather.rank; po.n = (int)o.n;
    for (int p = 0; p < MAX_PEERS; ++p) po.peer[p] = p < o.gather.G ? o.gather.peer[p] : nullptr;
    return po;
}

// the epoch flags a call gathering into g raises at its peers (only those of music_b200_gather_attach exist)
GatherFlags make_gather_flags(const music_b200 *h, const Gather &g)
{
    GatherFlags gf;
    for (int p = 0; p < MAX_PEERS; ++p) gf.peer[p] = p < g.G ? h->peer_flags[p] : nullptr;
    gf.epoch = (g.G > 0 && h->peer_flags[0]) ? h->gather_epoch : 0u;
    return gf;
}

// raises this GPU's epoch flag at every peer once everything before it on the stream is done (unfused paths; the
// fused kernel signals from its last CTA)
__global__ void gather_signal_kernel(const GatherFlags gf, int npeer, int rank)
{
    if ((int)threadIdx.x < npeer) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(gf.peer[threadIdx.x] + rank), "r"(gf.epoch) : "memory");
    }
}

// consumer side: returns when every peer's flag in THIS GPU's array has reached `epoch`
__global__ void gather_wait_kernel(const unsigned *flags, int npeer, unsigned epoch)
{
    if ((int)threadIdx.x < npeer) {
        unsigned v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
            if ((int)(v - epoch) >= 0) break;
            __nanosleep(200);
        } while (true);
    }
}

// The beam weights of W windows from ws.R, the angles and bins po holds, into o.wts (or the workspace), then the beams
// of the W windows at d_in into o.beams when the caller asked for them (music_beams.cuh).  With a calibration set the
// weights are taken back to raw-input coordinates before the beams are formed (music_calib.cuh).
void launch_beams(music_b200 *h, const Plan &p, const WsView &ws, uint32_t W, const Outputs &o, const PeakOut &po, const float *d_in,
                  cudaStream_t st)
{
    const DeviceTable &tb = table(h);
    const int M = (int)h->m, n = (int)h->n, N = (int)h->N;
    double *wts = o.wts ? o.wts : ws.wts;
    beam_weights_kernel<<<(W + BEAM_WARPS - 1) / BEAM_WARPS, BEAM_WARPS * 32, 0, st>>>(
        ws.R, po.angles, po.bins, reinterpret_cast<const float2 *>(tb.c64), M, n, (int)W, h->beam_rule, h->beam_loading, tb.geometric,
        tb.geo, wts);
    h->launches++;
    if (p.calib) {
        const size_t e = (size_t)W * n * M;
        calib_weights_kernel<<<(unsigned)((e + CALIB_THREADS - 1) / CALIB_THREADS), CALIB_THREADS, 0, st>>>(wts, M, n, (int)W, h->cal_c);
        h->launches++;
    }
    if (!o.beams) return;
    const int spans = (N + BEAM_SPAN - 1) / BEAM_SPAN;
    const size_t smem = beam_apply_smem(M, n);
    with_scan_m(h->m, [&](auto mt) {
        constexpr int MT = decltype(mt)::value;
        beam_apply_kernel<MT><<<(unsigned)((size_t)W * spans), BEAM_SPAN, smem, st>>>(d_in, wts, M, n, N, spans, o.beams);
    });
    h->launches++;
}

// The CRB of every filled slot of W windows from ws.R and the angles (and elevations) and bins po holds, into std
// (music_crb.cuh); under integration N_eff per window from the sub-batch's count ws.n0.
void launch_crb(music_b200 *h, const Plan &p, const WsView &ws, uint32_t W, const Outputs &o, const PeakOut &po, uint32_t nsnap,
                float *std, cudaStream_t st)
{
    const DeviceTable &tb = table(h);
    const unsigned long long *n0 = p.integ ? ws.n0 : nullptr;
    if (h->azel)
        crb_kernel<true><<<W, 32, 0, st>>>(ws.R, po.angles, o.elev, po.bins, n0, (int)h->m, (int)h->n, (int)W, (int)nsnap,
                                           h->integ_alpha, tb.geo, tb.ageo, std);
    else
        crb_kernel<false><<<W, 32, 0, st>>>(ws.R, po.angles, nullptr, po.bins, n0, (int)h->m, (int)h->n, (int)W, (int)nsnap,
                                            h->integ_alpha, tb.geo, tb.ageo, std);
    h->launches++;
}

// The tracker over W windows from the angles (and elevations) and bins po holds and the CRB in std (read under CRB
// variance), into o's slot_track, track_ids and track_state (music_track.cuh): one CTA, after the previous sub-batch's
// tracking on whichever stream that ran, so the carry goes from one sub-batch to the next in enqueue order.
int launch_track(music_b200 *h, uint32_t W, const Outputs &o, const PeakOut &po, const float *std, cudaStream_t st)
{
    if (h->trk_used) CU(h, cudaStreamWaitEvent(st, h->trk_done, 0));
    if (h->azel)
        track_kernel<2><<<1, 32, 0, st>>>(po.angles, o.elev, po.bins, std, (int)h->n, (int)W, h->trk, h->trk_fresh, h->trk_rows,
                                          h->trk_state, h->trk_next, o.slot_track, o.track_ids, o.track_state);
    else
        track_kernel<1><<<1, 32, 0, st>>>(po.angles, nullptr, po.bins, std, (int)h->n, (int)W, h->trk, h->trk_fresh, h->trk_rows,
                                          h->trk_state, h->trk_next, o.slot_track, o.track_ids, o.track_state);
    h->launches++;
    CU(h, cudaGetLastError());
    CU(h, cudaEventRecord(h->trk_done, st));
    h->trk_fresh = false;
    h->trk_used = true;
    return MUSIC_B200_OK;
}

// K2 of W windows from ws.R as planned: the eigensolver, the source count from `nsnap` snapshots (into ws.cnt and, when
// given, counts_out) and the MVDR preparation.  Returns the per-window counts the later stages read (NULL under FIXED).
const int32_t *launch_eig_stage(music_b200 *h, const Plan &p, const WsView &ws, uint32_t W, int32_t *counts_out, uint32_t nsnap,
                                cudaStream_t st)
{
    const int M = (int)h->m;
    if (p.eig) {
        const int grid = (W + 127) / 128;
        switch (M) {
        case 4: eig_kernel<4, true><<<grid, 128, 0, st>>>(ws.R, ws.ev, ws.Vt, M, (int)W); break;
        case 8: eig_coop_kernel<8><<<(W + EIGC_WARPS - 1) / EIGC_WARPS, EIGC_WARPS * 32, 0, st>>>(ws.R, ws.ev, ws.Vt, (int)W); break;
        case 12: eig_coop_kernel<12><<<(W + EIGC_WARPS - 1) / EIGC_WARPS, EIGC_WARPS * 32, 0, st>>>(ws.R, ws.ev, ws.Vt, (int)W); break;
        case 16: eig_coop_kernel<16><<<(W + EIGC_WARPS - 1) / EIGC_WARPS, EIGC_WARPS * 32, 0, st>>>(ws.R, ws.ev, ws.Vt, (int)W); break;
        default:
            if (M <= 8) eig_kernel<8, false><<<grid, 128, 0, st>>>(ws.R, ws.ev, ws.Vt, M, (int)W);
            else eig_kernel<MAXM, false><<<grid, 128, 0, st>>>(ws.R, ws.ev, ws.Vt, M, (int)W);
            break;
        }
        h->launches++;
    }
    // per-window model order from the eigenvalues just written (timed with the eigensolver)
    const int32_t *cnt = nullptr;
    if (p.count) {
        if (p.integ)  // N_eff of each window's integrated covariance in place of the snapshot count
            source_count_neff_kernel<<<(W + 127) / 128, 128, 0, st>>>(ws.ev, M, (int)h->n, (int)nsnap, h->source_rule, (int)W, h->integ_alpha,
                                                                    ws.n0, ws.cnt, counts_out);
        else
            source_count_kernel<<<(W + 127) / 128, 128, 0, st>>>(ws.ev, M, (int)h->n, (int)nsnap, h->source_rule, (int)W, ws.cnt, counts_out);
        h->launches++;
        cnt = ws.cnt;
    }
    // WSF: the weighted signal-subspace matrix X into ws.X (timed with the eigensolver)
    if (p.wsf) {
        const size_t e = (size_t)W * M * M;
        wsf_x_kernel<<<(unsigned)((e + WSF_X_THREADS - 1) / WSF_X_THREADS), WSF_X_THREADS, 0, st>>>(ws.ev, ws.Vt, cnt, M, (int)h->n,
                                                                                                  (int)W, ws.X);
        h->launches++;
    }
    // MVDR: the rows of L^-1 of R + delta I into ws.Vt (timed with the eigensolver)
    if (p.mvdr) {
        mvdr_prep_kernel<<<(W + PREP_WARPS - 1) / PREP_WARPS, PREP_WARPS * 32, 0, st>>>(ws.R, ws.Vt, M, (int)W, h->modes.loading);
        h->launches++;
    }
    return cnt;
}

// The 1-D grid peak rules (TopN, Local) of W windows on the fp64 strengths p64
void launch_grid_peaks(music_b200 *h, Peaks peaks, const double *p64, uint32_t W, const PeakOut &po, const int32_t *cnt, cudaStream_t st)
{
    if (peaks == Peaks::Local) topn_local_kernel<<<(W + 7) / 8, 256, 0, st>>>(p64, (int)h->n, (int)h->K, (int)W, (int)h->modes.excl, po, cnt);
    else topn_kernel<<<(W + 7) / 8, 256, 0, st>>>(p64, (int)h->n, (int)h->K, (int)W, po, cnt);
}

// K2 (+ source count from `nsnap` looks) + K3 (+ peak rule) of W windows from ws.R against table tb into the outputs o
// (of these W windows), on `st`, as planned.  tev (optional) = timing events [1..4].  An az-el handle's peak bins are decoded into (azimuth, elevation)
// after the peak rule.  With refinement on, the refine kernel follows (timed with the peak rule) and reads the bins
// written before it: from the caller's array, or from the workspace when the caller asked for none.  A beams call
// then forms the weights and beams of the windows at d_in, a CRB call the bound of every slot and a tracks call the
// tracker's outputs (all timed with the peak rule as well).
int launch_eig_scan(music_b200 *h, const Plan &p, const WsView &ws, uint32_t W, const Outputs &o, const DeviceTable &tb, uint32_t nsnap,
                    cudaStream_t st, cudaEvent_t *tev, const float *d_in = nullptr)
{
    const int M = (int)h->m;
    PeakOut po = make_peak_out(o);
    if (p.ws_bins && !po.bins) po.bins = ws.bins;
    const int32_t *cnt = launch_eig_stage(h, p, ws, W, o.counts, nsnap, st);
    if (tev) cudaEventRecord(tev[2], st);
    launch_scan(h, p, ws, W, o, po, cnt, tb, st);
    double *p64 = o.P64 ? o.P64 : ws.P64;  // what the peak rules read
    if (tev) cudaEventRecord(tev[3], st);
    const int excl = (int)h->modes.excl;
    switch (p.peaks) {
    case Peaks::Roots:
        roots_kernel<<<W, ROOTS_THREADS, 0, st>>>(ws.Vt, cnt, M, (int)h->n, (int)h->K, tb.geo, tb.ula, po);
        break;
    case Peaks::Esprit:
        esprit_kernel<<<(W + ESPRIT_WARPS - 1) / ESPRIT_WARPS, ESPRIT_WARPS * 32, 0, st>>>(ws.Vt, cnt, M, (int)h->n, (int)h->K, (int)W,
                                                                                        tb.geo, tb.ula, po);
        break;
    case Peaks::Esprit2D:
        esprit2d_kernel<<<(W + ESP2_WARPS - 1) / ESP2_WARPS, ESP2_WARPS * 32, 0, st>>>(ws.Vt, cnt, M, (int)h->n, (int)W, tb.ageo,
                                                                                    tb.lat, po, o.elev);
        break;
    case Peaks::Manifold:
        manifold_kernel<<<W, manifold_threads((int)tb.mf_L), 0, st>>>(ws.Vt, cnt, M, (int)h->n, (int)h->K, tb.geo, tb.mf_beta,
                                                                       (int)tb.mf_L, po);
        break;
    case Peaks::Dml:
        // M = 16 runs the runtime-M instantiation (its loops have the same 16-entry bound): the fixed-M one spills
        with_scan_m(h->m, [&](auto mt) {
            constexpr int MT = decltype(mt)::value == 16 ? 0 : decltype(mt)::value;
            dml_kernel<MT><<<W, DML_THREADS, 0, st>>>(p.wsf ? ws.X : ws.R, ws.R, tb.soa, cnt, M, (int)h->n, (int)h->K, po);
        });
        break;
    case Peaks::Local2D: topn_local2d_kernel<<<W, AZEL_LM_THREADS, 0, st>>>(p64, (int)h->n, h->grid.n_az, h->grid.n_el, excl, po, cnt); break;
    case Peaks::Local:
    case Peaks::TopN: launch_grid_peaks(h, p.peaks, p64, W, po, cnt, st); break;
    case Peaks::None: break;
    }
    if (p.peaks != Peaks::None) h->launches++;
    if (p.decode) {
        const int slots = (int)(W * h->n);
        azel_decode_kernel<<<(slots + 255) / 256, 256, 0, st>>>(po.bins, slots, h->grid, po.angles, o.elev);
        h->launches++;
    }
    if (p.refine) {
        const int slots = (int)(W * h->n), rgrid = (slots + REFINE_THREADS - 1) / REFINE_THREADS;
        // the vectors the refined objective is built from: noise eigenvectors (MUSIC), rows of L^-1 (MVDR), R (Bartlett)
        const double *rv = p.est == MUSIC_B200_ESTIMATOR_BARTLETT ? ws.R : ws.Vt;
#define REFINE_CASE(E)                                                                                                         \
        if (p.decode)                                                                                                          \
            refine_azel_kernel<E><<<rgrid, REFINE_THREADS, 0, st>>>(rv, cnt, po.bins, M, (int)h->n, (int)W, tb.ageo, po.angles, o.elev, \
                                                                    po.levels);                                                \
        else                                                                                                                   \
            refine_peaks_kernel<E><<<rgrid, REFINE_THREADS, 0, st>>>(rv, cnt, po.bins, M, (int)h->n, (int)h->K, (int)W, tb.geo,   \
                                                                     po.angles, po.levels);
        if (p.est == MUSIC_B200_ESTIMATOR_MVDR) { REFINE_CASE(EST_MVDR) }
        else if (p.est == MUSIC_B200_ESTIMATOR_BARTLETT) { REFINE_CASE(EST_BARTLETT) }
        else { REFINE_CASE(EST_MUSIC) }
#undef REFINE_CASE
        h->launches++;
    }
    if (p.joint) {
        const int n = (int)h->n;
        joint_kernel<<<W, 32, (size_t)joint_smem_elems(M, n) * sizeof(double2), st>>>(ws.R, p.wsf ? ws.ev : nullptr, ws.Vt, cnt, po.bins,
                                                                                      M, n, (int)h->K, tb.geo, po.angles, po.levels);
        h->launches++;
    }
    if (p.beams) launch_beams(h, p, ws, W, o, po, d_in, st);
    float *std = o.std ? o.std : ws.std;
    if (p.crb) launch_crb(h, p, ws, W, o, po, nsnap, std, st);
    if (p.track)
        if (const int rc = launch_track(h, W, o, po, std, st)) return rc;
    if (tev) cudaEventRecord(tev[4], st);
    if (o.R)
        CU(h, cudaMemcpyAsync(o.R, ws.R, (size_t)W * M * M * 2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (o.ev)
        CU(h, cudaMemcpyAsync(o.ev, ws.ev, (size_t)W * M * sizeof(double), cudaMemcpyDeviceToDevice, st));
    CU(h, cudaGetLastError());
    return MUSIC_B200_OK;
}

// K1 on planar streams (music_planar.cuh): windows first .. first + W - 1 of the call
void launch_cov_planar(music_b200 *h, const WsView &ws, const PlanarStreams &S, unsigned long long first_snapshot,
                       unsigned hop, uint32_t W, cudaStream_t st)
{
    const int M = (int)h->m_in, N = (int)h->N, T = (M + 3) / 4, wpb = 8;
    cov_planar_kernel<false><<<(unsigned)(((long long)W * T + wpb - 1) / wpb), wpb * 32, 0, st>>>(S, first_snapshot, hop, ws.R, (int)W, N, M);
    h->launches++;
    if (T > 1) {
        const long long items = (long long)W * (T * (T - 1) / 2);
        cov_planar_kernel<true><<<(unsigned)((items + wpb - 1) / wpb), wpb * 32, 0, st>>>(S, first_snapshot, hop, ws.R, (int)W, N, M);
        h->launches++;
    }
}

// The integration of the W covariances in R (music_integrate.cuh) on `st`, after the previous sub-batch's integration on
// whichever stream that ran: the handle's carry goes from one sub-batch to the next in enqueue order, which is window
// order within a call (the host entries' chunks alternate between two streams) and call order across calls.
int launch_integrate(music_b200 *h, const WsView &ws, uint32_t W, cudaStream_t st)
{
    const int E = (int)(2 * h->m_in * h->m_in), ntiles = (int)((W + INTEG_T - 1) / INTEG_T);
    const size_t elems = (size_t)ntiles * E;
    if (elems > h->integ_tiles.size()) {
        if (h->integ_used) CU(h, cudaEventSynchronize(h->integ_done));  // the last integration may still read the scratch
        CU(h, h->integ_tiles.grow(elems));
    }
    if (h->integ_used) CU(h, cudaStreamWaitEvent(st, h->integ_done, 0));
    if (h->integ_fresh) {
        CU(h, cudaMemsetAsync(h->integ_S, 0, (size_t)E * sizeof(double), st));
        CU(h, cudaMemsetAsync(h->integ_cnt, 0, sizeof(unsigned long long), st));
        h->integ_fresh = false;
    }
    double *R = ws.R;
    const double a = h->integ_alpha;
    const uint32_t last = W - (uint32_t)(ntiles - 1) * INTEG_T;
    const unsigned blocks = (unsigned)((elems + INTEG_THREADS - 1) / INTEG_THREADS);
    integ_tiles_kernel<<<blocks, INTEG_THREADS, 0, st>>>(R, h->integ_tiles, E, (int)W, a);
    integ_carry_kernel<<<E, INTEG_SCAN_THREADS, 0, st>>>(h->integ_tiles, h->integ_S, h->integ_cnt, ws.n0, E, (int)W,
                                                         std::pow(a, (double)INTEG_T), std::pow(a, (double)last));
    integ_apply_kernel<<<blocks, INTEG_THREADS, 0, st>>>(R, h->integ_tiles, ws.n0, E, (int)W, a);
    h->launches += 3;
    CU(h, cudaGetLastError());
    CU(h, cudaEventRecord(h->integ_done, st));
    h->integ_used = true;
    return MUSIC_B200_OK;
}

// Enqueue `nwindows` windows on `st`: one persistent fused launch where the shape allows it, otherwise the unfused
// kernels in sub-batches of at most max_sub_windows(), which bounds the workspace slot `slot` (0 / 1) they run in.
// out: the outputs of the call; counts (may be NULL) receives the per-window source counts, under the FIXED rule n each.
int enqueue_device(music_b200 *h, const float *d_in, uint32_t nwindows, const Outputs &out, cudaStream_t st, int slot,
                   const PlanarStreams *planar = nullptr, unsigned hop = 0)
{
    if (nwindows == 0) return MUSIC_B200_OK;
    if ((!planar && !d_in) || !out.angles) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 and d_angles must not be NULL");
    if (h->azel && !out.elev) return fail(h, MUSIC_B200_EINVAL, "an az-el handle needs the elevation output");
    if (!planar && (reinterpret_cast<uintptr_t>(d_in) & 15u) != 0) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 must be 16-byte aligned");
    if (const int rc = check_modes(h, h->modes, &table(h))) return rc;
    if (out.slot_track && h->trk_var == MUSIC_B200_TRACK_OFF)
        return fail(h, MUSIC_B200_EINVAL, "tracking is off (call music_b200_set_tracking() with FIXED or CRB variance)");
    if ((out.std || (out.slot_track && h->trk_var == MUSIC_B200_TRACK_CRB)) && !table(h).geometric)
        return fail(h, MUSIC_B200_EINVAL, "the CRB needs a table built by music_b200_set_geometry%s(); the current one came from "
                                          "set_table(), which has no geometry", h->azel ? "_azel" : "");
    if (h->source_rule == MUSIC_B200_SOURCES_FIXED && out.counts) {
        fill_counts_kernel<<<(nwindows + 255) / 256, 256, 0, st>>>(out.counts, (int)h->n, (int)nwindows);
        h->launches++;
        CU(h, cudaGetLastError());
    }
    const Plan plan = plan_call(h, out, planar, hop);
    if (plan.path == Path::Fused4) {
        // whole call in one persistent launch (music_fused.cuh); no workspace involved
        cudaEvent_t *tev = timing_events(h);
        if (tev) cudaEventRecord(tev[0], st);
        const int grid = std::min<int>(h->sm_count, (int)((nwindows + FZ_COV_WARPS - 1) / FZ_COV_WARPS));
        unsigned *ctr = ticket_counter(h, slot, st);
        const DeviceTable &tb = table(h);
        const PeakOut po = make_peak_out(out);
        const GatherFlags gf = make_gather_flags(h, out.gather);
        // Programmatic dependent launch: when the previous operation on `st` is another launch of this kernel, the new
        // CTAs are placed at once in the free half of every SM (every CTA signals launch_dependents at its start; the grid,
        // at most one CTA per SM, leaves the other half free) instead of after the whole grid has drained; the kernel
        // orders its own output writes behind the previous grid (fused_emit).  After any other kind of operation the launch
        // is an ordinary stream-ordered one.
        cudaLaunchConfig_t lc = {};
        lc.gridDim = dim3((unsigned)grid); lc.blockDim = dim3(FZ_THREADS); lc.dynamicSmemBytes = FZ_SMEM; lc.stream = st;
        cudaLaunchAttribute la[1];
        la[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        la[0].val.programmaticStreamSerializationAllowed = 1;
        lc.attrs = la; lc.numAttrs = h->pdl ? 1 : 0;
        const int W_i = (int)nwindows, N_i = (int)h->N, K_i = (int)h->K;
        const bool tr = h->fused_trace != nullptr;  // MUSIC_B200_TRACE=1: the instantiation with the clock64 trace
        // each launch writes its own slot of the trace ring, so launches that are resident together do not mix their rows
        long long *trace = tr ? h->fused_trace + (size_t)(h->trace_seq++ % FZ_TRACE_LAUNCHES) * FZ_TRACE_CTAS * FZ_TRACE : nullptr;
        const unsigned char *fz = tb.fz;
        const float *c64 = tb.c64, *na_max = tb.na_max;
        const int mma_fin = tb.screen_ok ? h->mma_fin_max : -1;  // a table the screen cannot bound: fp64 drain only
        cudaError_t le;
        if (planar) {
            auto kern = tr ? music4_fused_kernel<true, true> : music4_fused_kernel<true, false>;
            le = cudaLaunchKernelEx(&lc, kern, (const float *)nullptr, *planar, 0ull, (unsigned)hop, fz, c64, na_max, W_i, N_i, K_i, po, ctr,
                                    trace, h->eig_mode, gf, mma_fin, out.spec);
        } else {
            auto kern = tr ? music4_fused_kernel<false, true> : music4_fused_kernel<false, false>;
            le = cudaLaunchKernelEx(&lc, kern, d_in, PlanarStreams{}, 0ull, 0u, fz, c64, na_max, W_i, N_i, K_i, po, ctr, trace,
                                    h->eig_mode, gf, mma_fin, out.spec);
        }
        CU(h, le);
        h->launches++;
        if (tev) for (int i = 1; i < 5; ++i) cudaEventRecord(tev[i], st);
        CU(h, cudaGetLastError());
        return MUSIC_B200_OK;
    }
    if (plan.path == Path::Fused8 && encode_tiled_fn()) {
        // M = 8: whole call in one persistent launch (music_fused8.cuh); R and the eigenvectors stay in shared memory
        CUtensorMap tm;
        const cuuint64_t gdim[3] = {32u, (cuuint64_t)(h->N / 2), (cuuint64_t)nwindows};  // 128-byte rows of two snapshots
        const cuuint64_t gstr[2] = {128u, (cuuint64_t)64 * (cuuint64_t)h->N};
        const cuuint32_t box[3] = {32u, (cuuint32_t)(F8_STAGE / 128), 1u};
        const cuuint32_t estr[3] = {1u, 1u, 1u};
        if (encode_tiled_fn()(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float *>(d_in), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS) {
            cudaEvent_t *tev = timing_events(h);
            if (tev) cudaEventRecord(tev[0], st);
            const int grid = std::min<int>(h->sm_count, (int)((nwindows + F8_WARPS - 1) / F8_WARPS));
            unsigned *ctr = ticket_counter(h, slot, st);
            music8_fused_kernel<<<grid, F8_WARPS * 32, F8_SMEM, st>>>(tm, table(h).soa, (int)nwindows, (int)h->N, (int)h->K,
                                                                     make_peak_out(out), ctr, make_gather_flags(h, out.gather),
                                                                     h->eig_mode ? 1 : 0, h->f8_stats);
            h->launches++;
            if (tev) for (int i = 1; i < 5; ++i) cudaEventRecord(tev[i], st);
            CU(h, cudaGetLastError());
            return MUSIC_B200_OK;
        }
        // (the tensor map could not be encoded: the unfused kernels below)
    }
    const uint32_t sub = std::min((nwindows + SCAN_B - 1) / SCAN_B * SCAN_B, max_sub_windows(h, plan));
    Workspace &ws = h->ws[slot];
    int rc = ensure_slot(h, ws, sub, plan);
    if (rc) return rc;
    if (ws.used) CU(h, cudaStreamWaitEvent(st, ws.scan_done, 0));  // the slot's last user may have run on another stream
    const WsView v = ws.view();
    // the input side (covariance, calibration, integration) works on the m_in elements of a snapshot: on a co-array
    // handle in the slot's physical-R buffer, which coarray_kernel then maps into the workspace R
    WsView vin = v;
    if (h->coarray) vin.R = ws.Rin;
    for (uint32_t w0 = 0; w0 < nwindows; w0 += sub) {
        const uint32_t W = std::min(sub, nwindows - w0);
        cudaEvent_t *tev = timing_events(h);
        if (tev) cudaEventRecord(tev[0], st);
        if (planar) launch_cov_planar(h, vin, *planar, (unsigned long long)w0 * hop, hop, W, st);
        else launch_cov(h, vin, d_in + (size_t)w0 * h->nsamples * 2, W, st, slot);
        if (plan.calib) {
            // the receiver correction of R, inside the covariance slot of the stage timing
            const size_t e = (size_t)W * h->m_in * h->m_in;
            calib_apply_kernel<<<(unsigned)((e + CALIB_THREADS - 1) / CALIB_THREADS), CALIB_THREADS, 0, st>>>(vin.R, (int)h->m_in, (int)W, h->cal_c);
            h->launches++;
        }
        if (plan.integ) {
            // the integration across windows, also inside the covariance slot
            rc = launch_integrate(h, vin, W, st);
            if (rc) return rc;
        }
        if (h->coarray) {
            // R_ss of the virtual array into the workspace R, inside the covariance slot
            coarray_kernel<<<(W + CO_WARPS - 1) / CO_WARPS, CO_WARPS * 32, 0, st>>>(reinterpret_cast<const double2 *>(vin.R), (int)h->m_in,
                                                                                (int)W, h->co_lags, reinterpret_cast<double2 *>(v.R));
            h->launches++;
        }
        if (tev) cudaEventRecord(tev[1], st);
        rc = launch_eig_scan(h, plan, v, W, out.at(w0), table(h), h->N, st, tev,
                             planar ? nullptr : d_in + (size_t)w0 * h->nsamples * 2);
        if (rc) return rc;
        CU(h, cudaEventRecord(ws.scan_done, st));
        ws.used = true;
    }
    const GatherFlags gf = make_gather_flags(h, out.gather);
    if (gf.epoch) {
        gather_signal_kernel<<<1, 32, 0, st>>>(gf, out.gather.G, out.gather.rank);
        h->launches++;
    }
    return MUSIC_B200_OK;
}

// A channel handle's call (music_channels.cuh): `nwindows` windows on `st` in sub-batches through workspace slot 0, which
// holds a sub-batch of W windows as C * W pseudo-windows, channel-major [C][W].  The filter bank writes every channel's
// R in one launch; eigensolver, source count (from the J segments) and MVDR preparation run once over all C * W
// pseudo-windows; scan and peak rule run once per channel on that channel's contiguous run, with that channel's table,
// straight into the channel's block of the caller's channel-major outputs `out` ([C][nwindows] rows under SEPARATE,
// [nwindows] rows under INCOHERENT).  R_out (may be NULL): [C][nwindows][m][m] complex fp64.
// Under COHERENT the filter bank writes the C * W covariances into the handle's channel buffer (foc_Rc), the focus kernel
// folds them into W focused ones in the workspace, which is sized for W windows, and the plain unfused stages run once
// over them, on the reference channel's table, with J * C looks; outputs and R_out have
// [nwindows] rows.
int enqueue_channels(music_b200 *h, const float *d_in, uint32_t nwindows, const Outputs &out, double *R_out, cudaStream_t st)
{
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!d_in || !out.angles) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 and d_angles must not be NULL");
    if ((reinterpret_cast<uintptr_t>(d_in) & 15u) != 0) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 must be 16-byte aligned");
    if (!has_table(h)) return fail(h, MUSIC_B200_EINVAL, "no array response yet: call music_b200_set_geometry_channels() or music_b200_set_table()");
    const bool separate = h->chan_combine == MUSIC_B200_CHANNELS_SEPARATE, focus = coherent(h);
    const ChanShape &cs = h->cshape;
    const int ref = cs.C / 2;
    if (const int rc = check_modes(h, h->modes, focus ? &table(h, ref) : nullptr)) return rc;
    if (h->chan_combine == MUSIC_B200_CHANNELS_INCOHERENT && out.counts)
        return fail(h, MUSIC_B200_EINVAL, "the INCOHERENT combine reports no counts: counts must be NULL");
    const uint32_t C = (uint32_t)cs.C;
    if (h->source_rule == MUSIC_B200_SOURCES_FIXED && out.counts) {
        const size_t e = (size_t)(separate ? C : 1) * nwindows;
        fill_counts_kernel<<<(unsigned)((e + 255) / 256), 256, 0, st>>>(out.counts, (int)h->n, (int)e);
        h->launches++;
        CU(h, cudaGetLastError());
    }
    const Plan plan = plan_call(h, out, nullptr, 0);
    const uint32_t sub = std::min((nwindows + SCAN_B - 1) / SCAN_B * SCAN_B, max_sub_windows(h, plan));
    Workspace &ws = h->ws[0];
    if (const int rc = ensure_slot(h, ws, focus ? sub : sub * C, plan)) return rc;
    const size_t foc_elems = (size_t)sub * C * h->m * h->m;
    if (focus && foc_elems > h->foc_Rc.size()) {
        if (ws.used) CU(h, cudaEventSynchronize(ws.scan_done));  // the last call may still read it on another stream
        CU(h, h->foc_Rc.grow(foc_elems));
    }
    if (ws.used) CU(h, cudaStreamWaitEvent(st, ws.scan_done, 0));
    const WsView v = ws.view();
    const size_t mm2 = (size_t)h->m * h->m * 2, K = h->K;
    const size_t smem = chan_smem(cs.M, cs.F, cs.B, cs.Cg).total;
    for (uint32_t w0 = 0; w0 < nwindows; w0 += sub) {
        const uint32_t W = std::min(sub, nwindows - w0);
        cudaEvent_t *tev = timing_events(h);
        if (tev) cudaEventRecord(tev[0], st);
        const int grid = (int)std::min<uint32_t>(W, (uint32_t)(h->sm_count * h->chan_ctas));
        double *Rc = focus ? reinterpret_cast<double *>(h->foc_Rc.get()) : v.R;
        chan_cov_kernel<<<grid, CHAN_THREADS, smem, st>>>(d_in + (size_t)w0 * h->nsamples * 2, Rc, (int)W, cs, h->chan_tw, h->chan_taper_d);
        h->launches++;
        if (focus) {
            // R_foc into the workspace, inside the covariance slot of the stage timing; then one plain problem per window
            const int M = (int)h->m, wt = focus_windows(M);
            chan_focus_kernel<<<(W + wt - 1) / wt, focus_threads(M), 0, st>>>(h->foc_Rc, reinterpret_cast<double2 *>(v.R), (int)W, (int)C,
                                                                            M, ref, cur_slot(h).foc_T);
            h->launches++;
            if (tev) cudaEventRecord(tev[1], st);
            Outputs o = out.at(w0);
            o.R = R_out ? R_out + (size_t)w0 * mm2 : nullptr;
            if (const int rc = launch_eig_scan(h, plan, v, W, o, table(h, ref), snapshots(h), st, tev)) return rc;
            CU(h, cudaEventRecord(ws.scan_done, st));
            ws.used = true;
            continue;
        }
        if (tev) cudaEventRecord(tev[1], st);
        const int32_t *cnt = launch_eig_stage(h, plan, v, C * W, nullptr, (uint32_t)cs.J, st);
        if (cnt && out.counts)
            CU(h, cudaMemcpy2DAsync(out.counts + w0, (size_t)nwindows * sizeof(int32_t), cnt, (size_t)W * sizeof(int32_t), (size_t)W * sizeof(int32_t), C,
                                    cudaMemcpyDeviceToDevice, st));
        if (tev) cudaEventRecord(tev[2], st);
        // channel c's run of the workspace, and its block of the outputs from window w0 on
        const auto run = [&](uint32_t c) {
            WsView r = v;
            r.R += (size_t)c * W * mm2;
            r.Vt += (size_t)c * W * mm2;
            if (r.P64) r.P64 += (size_t)c * W * K;
            return r;
        };
        const auto block = [&](uint32_t c) { return separate ? out.at((size_t)c * nwindows + w0) : Outputs().shaped(h); };
        for (uint32_t c = 0; c < C; ++c) {
            const Outputs o = block(c);
            launch_scan(h, plan, run(c), W, o, make_peak_out(o), cnt ? cnt + (size_t)c * W : nullptr, table(h, (int)c), st);
        }
        if (tev) cudaEventRecord(tev[3], st);
        if (plan.combine) {
            const size_t WK = (size_t)W * K;
            chan_combine_kernel<<<(unsigned)((WK + 255) / 256), 256, 0, st>>>(v.P64, (int)C, WK, out.spec ? out.spec + (size_t)w0 * K : nullptr);
            launch_grid_peaks(h, plan.peaks, v.P64, W, make_peak_out(out.at(w0)), nullptr, st);
            h->launches += 2;
        } else if (plan.peaks != Peaks::None) {
            for (uint32_t c = 0; c < C; ++c) {
                const Outputs o = block(c);
                launch_grid_peaks(h, plan.peaks, o.P64 ? o.P64 : run(c).P64, W, make_peak_out(o), cnt ? cnt + (size_t)c * W : nullptr, st);
                h->launches++;
            }
        }
        if (tev) cudaEventRecord(tev[4], st);
        if (R_out)
            CU(h, cudaMemcpy2DAsync(R_out + (size_t)w0 * mm2, (size_t)nwindows * mm2 * sizeof(double), v.R, (size_t)W * mm2 * sizeof(double),
                                    (size_t)W * mm2 * sizeof(double), C, cudaMemcpyDeviceToDevice, st));
        CU(h, cudaGetLastError());
        CU(h, cudaEventRecord(ws.scan_done, st));
        ws.used = true;
    }
    return MUSIC_B200_OK;
}

struct NvtxRange {  // SURVEY.md section 5 tracing hook: ranges show up in nsys / ncu timelines, free when no tool is attached
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

// Drops every range of ours that overlaps [ptr, ptr + bytes) without holding all of it.  A registration covers whole
// pages, so it can take in the first or last page of a neighbouring buffer; the driver refuses a copy from or to memory
// that is registered only in part, so a caller range a copy touches must lie inside one registration or outside all.
void release_straddling(music_b200 *h, const void *ptr, size_t bytes)
{
    if (!ptr || bytes == 0) return;
    const uintptr_t a = reinterpret_cast<uintptr_t>(ptr), e = a + bytes;
    for (size_t i = 0; i < h->hostregs.size();) {
        const music_b200::HostReg &g = h->hostregs[i];
        if (g.base < e && a < g.base + g.len && !(g.base <= a && e <= g.base + g.len)) {
            cudaHostUnregister(reinterpret_cast<void *>(g.base));
            h->hostregs.erase(h->hostregs.begin() + i);
        } else {
            ++i;
        }
    }
}

// Makes [ptr, ptr + bytes) DMA-able if it is ordinary pageable memory: page-aligned cudaHostRegister, remembered in
// the handle (at most 16 ranges, oldest evicted).  Memory that is already pinned (cudaHostAlloc, registered by the
// caller) or that cannot be registered is left alone - the copies then take the driver's staged path.
void host_register(music_b200 *h, const void *ptr, size_t bytes, bool read_only)
{
    if (!h->hostreg || !ptr || bytes < ((size_t)1 << 20)) return;
    const uintptr_t a = reinterpret_cast<uintptr_t>(ptr), page = 4096;
    const uintptr_t lo = a & ~(page - 1), hi = (a + bytes + page - 1) & ~(page - 1);
    for (size_t i = 0; i < h->hostregs.size(); ++i)
        if (h->hostregs[i].base <= lo && hi <= h->hostregs[i].base + h->hostregs[i].len) return;  // already ours
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, ptr) == cudaSuccess) {
        if (at.type != cudaMemoryTypeUnregistered) return;  // pinned by the caller (or not host memory at all)
    } else {
        cudaGetLastError();
    }
    NvtxRange r("music_b200: cudaHostRegister");
    // ranges of ours that overlap the new one (a circular buffer seen at a shifted offset): drop them first
    for (size_t i = 0; i < h->hostregs.size();) {
        const music_b200::HostReg &g = h->hostregs[i];
        if (g.base < hi && lo < g.base + g.len) {
            cudaHostUnregister(reinterpret_cast<void *>(g.base));
            h->hostregs.erase(h->hostregs.begin() + i);
        } else {
            ++i;
        }
    }
    cudaError_t e = cudaHostRegister(reinterpret_cast<void *>(lo), hi - lo, cudaHostRegisterPortable | (read_only ? cudaHostRegisterReadOnly : 0));
    if (e != cudaSuccess && read_only) {
        cudaGetLastError();
        e = cudaHostRegister(reinterpret_cast<void *>(lo), hi - lo, cudaHostRegisterPortable);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();  // not registrable (e.g. a read-only mapping): pageable copies still work
        return;
    }
    if (h->hostregs.size() >= 16) {
        cudaHostUnregister(reinterpret_cast<void *>(h->hostregs.front().base));
        h->hostregs.erase(h->hostregs.begin());
    }
    h->hostregs.push_back(music_b200::HostReg{lo, (size_t)(hi - lo)});
}

int ensure_host_staging(music_b200 *h, uint32_t chunk, bool spec, bool beams, bool crb, uint32_t track_T)
{
    if (chunk <= h->host_chunk && (!spec || h->host_spec_alloc) && (!beams || h->host_beam_alloc) && (!crb || h->host_crb_alloc) &&
        track_T <= h->host_track_T)
        return MUSIC_B200_OK;
    spec = spec || h->host_spec_alloc;
    beams = beams || h->host_beam_alloc;
    crb = crb || h->host_crb_alloc;
    track_T = std::max(track_T, h->host_track_T);
    const uint32_t cap = std::max(chunk, h->host_chunk);
    // every old buffer is freed before the first new one is allocated
    for (HostSlot &sl : h->stage) sl = HostSlot();
    h->host_chunk = 0;
    h->host_spec_alloc = h->host_beam_alloc = h->host_crb_alloc = false;
    h->host_track_T = 0;
    const size_t wn = (size_t)cap * h->n;
    const auto alloc = [&](auto &b) -> int {
        CU(h, b.angles.grow(wn));
        CU(h, b.levels.grow(wn));
        CU(h, b.bins.grow(wn));
        CU(h, b.counts.grow(cap));
        if (beams) {
            CU(h, b.wts.grow(wn * h->m * 2));
            CU(h, b.beams.grow(wn * h->N * 2));
        }
        if (h->azel) CU(h, b.elev.grow(wn));
        if (crb) CU(h, b.std.grow(h->azel ? 3 * wn : wn));
        if (track_T) {
            CU(h, b.slot_track.grow(wn));
            CU(h, b.track_ids.grow((size_t)cap * track_T));
            CU(h, b.track_state.grow((size_t)cap * track_T * (h->azel ? 6 : 3)));
        }
        return MUSIC_B200_OK;
    };
    for (HostSlot &sl : h->stage) {
        CU(h, sl.in.grow((size_t)cap * h->nsamples * 2));
        if (spec) CU(h, sl.dbuf.spec.grow((size_t)cap * h->K));
        if (const int rc = alloc(sl.dbuf)) return rc;
        if (const int rc = alloc(sl.pbuf)) return rc;
        sl.dev = sl.dbuf.view(h);
        sl.pin = sl.pbuf.view(h);
    }
    h->host_chunk = cap;
    h->host_spec_alloc = spec;
    h->host_beam_alloc = beams;
    h->host_crb_alloc = crb;
    h->host_track_T = track_T;
    return MUSIC_B200_OK;
}

// Results of the chunk last computed in staging slot s: pinned mirrors -> the caller's outputs dst (the slot's stream
// is idle).  The chunk holds the windows w = (w0 + i) * G + g of the call (G = 1, g = 0 on a single-device handle).
void flush_host_slot(music_b200 *h, int s, const Outputs &dst, uint32_t G, uint32_t g)
{
    HostSlot &sl = h->stage[s];
    if (!sl.W) return;
    const auto from = sl.pin.window_fields(), to = dst.window_fields();
    for (size_t f = 0; f < to.size(); ++f) {
        if (!to[f].p) continue;
        const size_t row = to[f].per_win * sizeof(float);  // bytes of one window
        char *d = static_cast<char *>(to[f].p);
        const char *src = static_cast<const char *>(from[f].p);
        if (G == 1) {
            memcpy(d + sl.w0 * row, src, sl.W * row);
        } else {
            for (uint32_t i = 0; i < sl.W; ++i) memcpy(d + ((size_t)(sl.w0 + i) * G + g) * row, src + i * row, row);
        }
    }
    const auto rfrom = sl.pin.row_fields(), rto = dst.row_fields();
    for (size_t f = 0; f < rto.size(); ++f) {
        if (!rto[f].p) continue;
        const size_t row = rto[f].bytes;
        char *d = static_cast<char *>(rto[f].p);
        const char *src = static_cast<const char *>(rfrom[f].p);
        if (G == 1) {
            memcpy(d + sl.w0 * row, src, sl.W * row);
        } else {
            for (uint32_t i = 0; i < sl.W; ++i) memcpy(d + ((size_t)(sl.w0 + i) * G + g) * row, src + i * row, row);
        }
    }
    sl.W = 0;
}

// device -> pinned mirrors of slot s, for the outputs dst asks for (asynchronous on st whatever memory dst lives in)
int download_host_slot(music_b200 *h, int s, uint32_t w0, uint32_t W, const Outputs &dst, cudaStream_t st)
{
    HostSlot &sl = h->stage[s];
    const auto want = dst.window_fields(), from = sl.dev.window_fields(), to = sl.pin.window_fields();
    for (size_t f = 0; f < want.size(); ++f)
        if (want[f].p) CU(h, cudaMemcpyAsync(to[f].p, from[f].p, (size_t)W * want[f].per_win * sizeof(float), cudaMemcpyDeviceToHost, st));
    const auto rwant = dst.row_fields(), rfrom = sl.dev.row_fields(), rto = sl.pin.row_fields();
    for (size_t f = 0; f < rwant.size(); ++f)
        if (rwant[f].p) CU(h, cudaMemcpyAsync(rto[f].p, rfrom[f].p, (size_t)W * rwant[f].bytes, cudaMemcpyDeviceToHost, st));
    sl.w0 = w0;
    sl.W = W;
    return MUSIC_B200_OK;
}

// the outputs every process entry point takes; the entries that have more set them on the result
Outputs caller_outputs(float *angles, float *levels, float *spec, int32_t *bins)
{
    Outputs o;
    o.angles = angles;
    o.levels = levels;
    o.spec = spec;
    o.bins = bins;
    return o;
}

// The input of a host entry point: interleaved windows, or one stream per antenna with windows `hop` snapshots apart.
struct HostInput {
    const float *windows = nullptr;
    const float *const *streams = nullptr;
    unsigned hop = 0;
};

// The chunk loop of the host entry points, from caller memory through the staging slots into the caller's outputs dst.
// Lanes: the handle itself, or the per-device children of a multi-device handle (interleaved input only); lane g takes
// the windows w = i * G + g (round-robin at window granularity, SURVEY.md section 8e) - every lane feeds its own PCIe
// link.  Each of a lane's two copy streams computes in its own workspace slot and with its own ticket counter, so H2D,
// kernels and D2H of consecutive chunks overlap freely (the path is PCIe-bound by ~100x).
int stage_host(music_b200 *h, const HostInput &in, uint32_t nwindows, const Outputs &dst)
{
    music_b200 *self[1] = {h};
    music_b200 *const *lanes = h->kids.empty() ? self : h->kids.data();
    const uint32_t G = h->kids.empty() ? 1u : (uint32_t)h->kids.size();
    const size_t N = h->N, win_bytes = (size_t)h->nsamples * 2 * sizeof(float);
    const uint32_t per_lane = (nwindows + G - 1) / G;
    // chunk: ~32 MiB of input per copy, so that H2D of chunk i+1 overlaps compute of chunk i (with the spectrum port
    // connected a window also returns K floats, with beams n * N complex64 and n * m complex fp64: bound the chunk by
    // the larger of the input and the output), and at most half the call while a chunk still fills whole scan CTAs
    const size_t out_bytes = (dst.spec ? (size_t)h->K * sizeof(float) : 0) + (dst.beams ? (size_t)h->n * N * 2 * sizeof(float) : 0) +
                             (dst.wts ? (size_t)h->n * h->m * 2 * sizeof(double) : 0);
    const size_t per_win = std::max(win_bytes, out_bytes);
    const bool beams = dst.beams || dst.wts;
    const uint32_t base = (uint32_t)std::max<size_t>(SCAN_B, ((size_t)32 << 20) / per_win);
    const uint32_t half = (per_lane + 1) / 2 > SCAN_B ? (per_lane + 1) / 2 : per_lane;
    // Staging holds `host_chunk` windows of m * N samples per slot.  Planar, a chunk of C windows needs m * ((C - 1) *
    // hop + N) of them: the staging is sized for at least one window when hop > N and the chunk fitted into it.
    const uint32_t staged = in.streams ? (uint32_t)std::max<size_t>(base, ((size_t)in.hop + N - 1) / N + 1) : std::max<uint32_t>(1, std::min(base, half));
    int rc = MUSIC_B200_OK;
    for (uint32_t l = 0; l < G && rc == MUSIC_B200_OK; ++l) {
        music_b200 *c = lanes[l];
        if (cudaSetDevice(c->device) != cudaSuccess) { rc = fail(h, MUSIC_B200_ECUDA, "cudaSetDevice(%d) failed", c->device); break; }
        c->stage[0].W = c->stage[1].W = 0;  // nothing pending from an earlier (possibly failed) call
        rc = ensure_host_staging(c, staged, dst.spec != nullptr, beams, dst.std != nullptr, dst.slot_track ? c->trk.T : 0);
        if (rc && c != h) fail(h, rc, "%s", std::string(c->error).c_str());
        for (HostSlot &sl : c->stage) {  // the tracker's row count may have changed since the staging was allocated
            sl.dev.shaped(c);
            sl.pin.shaped(c);
        }
    }
    const size_t cap = lanes[0]->host_chunk;
    const uint32_t chunk = in.streams ? std::max<uint32_t>(1, std::min((uint32_t)std::min<size_t>(cap, 1 + (cap * N - N) / in.hop), half)) : staged;
    for (uint32_t it = 0; rc == MUSIC_B200_OK && (uint64_t)it * chunk < per_lane; ++it) {
        const int s = (int)(it & 1);
        for (uint32_t l = 0; l < G && rc == MUSIC_B200_OK; ++l) {
            music_b200 *c = lanes[l];
            HostSlot &sl = c->stage[s];
            const uint32_t Wl = l < nwindows ? (nwindows - l + G - 1) / G : 0;  // windows of this lane
            const uint32_t i0 = it * chunk;
            if (i0 >= Wl) continue;
            const uint32_t W = std::min(chunk, Wl - i0);
            cudaStream_t st = c->streams[s];
            CU_BREAK(h, rc, cudaSetDevice(c->device));
            if (it >= 2) {
                CU_BREAK(h, rc, cudaStreamSynchronize(st));  // slot buffers free again (its D2H finished)
                flush_host_slot(c, s, dst, G, l);
            }
            PlanarStreams S = {};
            {
                NvtxRange r("music_b200: H2D");
                if (in.streams) {
                    const size_t seg = (size_t)(W - 1) * in.hop + N;  // snapshots of each stream this chunk touches
                    for (uint32_t a = 0; a < h->m_in && rc == MUSIC_B200_OK; ++a) {
                        float *d = sl.in + (size_t)a * seg * 2;
                        CU_BREAK(h, rc, cudaMemcpyAsync(d, in.streams[a] + (size_t)i0 * in.hop * 2, seg * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
                        S.p[a] = reinterpret_cast<const float2 *>(d);
                    }
                } else {
                    const float *src = in.windows + ((size_t)i0 * G + l) * h->nsamples * 2;
                    if (G == 1) { CU_BREAK(h, rc, cudaMemcpyAsync(sl.in, src, (size_t)W * win_bytes, cudaMemcpyHostToDevice, st)); }
                    else { CU_BREAK(h, rc, cudaMemcpy2DAsync(sl.in, win_bytes, src, (size_t)G * win_bytes, win_bytes, W, cudaMemcpyHostToDevice, st)); }
                }
            }
            if (rc) break;
            {
                NvtxRange r("music_b200: kernels");
                Outputs o = sl.dev;  // the staging buffers of the outputs the caller asked for
                o.gather = c->gather;
                if (!dst.spec) o.spec = nullptr;
                if (!dst.counts) o.counts = nullptr;
                if (!dst.wts) o.wts = nullptr;
                if (!dst.beams) o.beams = nullptr;
                if (!dst.std) o.std = nullptr;
                if (!dst.slot_track) o.slot_track = nullptr;
                if (!dst.track_ids) { o.track_ids = nullptr; o.track_state = nullptr; }
                rc = enqueue_device(c, in.streams ? nullptr : sl.in.get(), W, o, st, s, in.streams ? &S : nullptr, in.hop);
                if (rc && c != h) fail(h, rc, "%s", std::string(c->error).c_str());
                if (rc) break;
            }
            NvtxRange r("music_b200: D2H");
            rc = download_host_slot(c, s, i0, W, dst, st);
            if (rc && c != h) fail(h, rc, "%s", std::string(c->error).c_str());
            if (rc) break;
            if (dst.spec) {
                float *d = dst.spec + ((size_t)i0 * G + l) * h->K;
                const size_t row = (size_t)h->K * sizeof(float);
                if (G == 1) { CU_BREAK(h, rc, cudaMemcpyAsync(d, sl.dev.spec, (size_t)W * row, cudaMemcpyDeviceToHost, st)); }
                else { CU_BREAK(h, rc, cudaMemcpy2DAsync(d, (size_t)G * row, sl.dev.spec, row, row, W, cudaMemcpyDeviceToHost, st)); }
            }
        }
    }
    // common tail, also after an error: every stream idle, nothing left pending in the slots
    cudaError_t e_sync = cudaSuccess;
    for (uint32_t l = 0; l < G; ++l) {
        music_b200 *c = lanes[l];
        cudaSetDevice(c->device);
        for (int s = 0; s < 2; ++s) {
            const cudaError_t e = cudaStreamSynchronize(c->streams[s]);
            if (e != cudaSuccess && e_sync == cudaSuccess) e_sync = e;
        }
    }
    if (rc == MUSIC_B200_OK && e_sync != cudaSuccess) rc = fail(h, MUSIC_B200_ECUDA, "stream sync failed: %s", cudaGetErrorString(e_sync));
    for (uint32_t l = 0; l < G; ++l) {
        music_b200 *c = lanes[l];
        if (rc == MUSIC_B200_OK) {
            flush_host_slot(c, 0, dst, G, l);
            flush_host_slot(c, 1, dst, G, l);
        } else {
            c->stage[0].W = c->stage[1].W = 0;  // nothing valid to hand out
        }
    }
    return rc;
}


// The device part of create() / create_azel(), after their argument checks: device checks, buffers, the first table
// (uploaded, or for an az-el handle (azel != NULL) built from its element positions, wavelength and grid).
// The filter bank of a channel handle: twiddles and taper on the device, the group split, the kernel's shared memory.
int init_channels(music_b200 *h)
{
    ChanShape &cs = h->cshape;
    std::vector<double2> tw(cs.F / 2);
    std::vector<double> taper(cs.F);
    cs.denom = (double)cs.J * chan_tables_host(cs.F, h->chan_taper, tw.data(), taper.data());
    cs.B = chan_batch(cs.M, cs.F, cs.J);
    cs.Cg = chan_group_size(cs.M, cs.F, cs.B, cs.C);
    cs.groups = (cs.C + cs.Cg - 1) / cs.Cg;
    CU(h, h->chan_tw.grow(tw.size()));
    CU(h, h->chan_taper_d.grow(taper.size()));
    CU(h, cudaMemcpy(h->chan_tw, tw.data(), tw.size() * sizeof(double2), cudaMemcpyHostToDevice));
    CU(h, cudaMemcpy(h->chan_taper_d, taper.data(), taper.size() * sizeof(double), cudaMemcpyHostToDevice));
    const size_t smem = chan_smem(cs.M, cs.F, cs.B, cs.Cg).total;
    CU(h, cudaFuncSetAttribute(chan_cov_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CHAN_SMEM_MAX));
    CU(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->chan_ctas, chan_cov_kernel, CHAN_THREADS, smem));
    if (h->chan_ctas < 1) return fail(h, MUSIC_B200_ECUDA, "chan_cov_kernel does not fit an SM with %zu bytes of shared memory", smem);
    return MUSIC_B200_OK;
}

// The buffers of table slot s, allocated the first time the slot is filled
int alloc_slot(music_b200 *h, TableSlot &s)
{
    if (!s.tabs.empty()) return MUSIC_B200_OK;
    const size_t C = h->chan ? (size_t)h->cshape.C : 1, c64 = (size_t)h->K * h->m * 2, soa = soa_doubles(h->K, h->m);
    CU(h, s.c64.grow(C * c64));
    CU(h, s.soa.grow(C * soa));
    if (h->m == 4 && !h->azel && !h->chan && !h->coarray) {  // the fused M = 4 kernel's screen layout; no other handle runs that kernel
        CU(h, s.fz.grow(fused_table_bytes((int)h->K)));
        CU(h, s.na_max.grow(1));
    }
    if (coherent(h)) CU(h, s.foc_T.grow(C * h->m * h->m));
    s.tabs.resize(C);
    for (size_t c = 0; c < C; ++c) {
        s.tabs[c].c64 = s.c64 + c * c64;
        s.tabs[c].soa = s.soa + c * soa;
    }
    s.tabs[0].fz = s.fz;
    s.tabs[0].na_max = s.na_max;
    return MUSIC_B200_OK;
}

// A retune: fills the idle table slot and makes it current only when `fill` succeeded.  Work enqueued by earlier calls
// may still read the current slot on a caller stream, so it is never rewritten; the idle slot was current before the
// last retune, and the device is synchronised once to be sure it is idle - retunes are rare.
template <class F>
int retune(music_b200 *h, F fill)
{
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaDeviceSynchronize());
    const int idle = h->cur_table ^ 1;
    if (const int rc = alloc_slot(h, h->tables[idle])) return rc;
    if (const int rc = fill(h->tables[idle])) return rc;
    h->cur_table = idle;
    h->integ_fresh = true;  // the integrated covariances described the old manifold
    h->trk_fresh = true;    // and the tracks its directions
    return MUSIC_B200_OK;
}

// The checks every create entry point makes first, the reference's constructor asserts (lib/baz_music_doa.cc:45-50,
// + n >= 1, n < m, see header)
int check_create(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples)
{
    if (!out) return fail(nullptr, MUSIC_B200_EINVAL, "out must not be NULL");
    *out = nullptr;
    if (m == 0 || m > MUSIC_B200_MAX_M) return fail(nullptr, MUSIC_B200_EINVAL, "m must be in 1..%d (got %u)", MUSIC_B200_MAX_M, m);
    if (n == 0 || n >= m) return fail(nullptr, MUSIC_B200_EINVAL, "need 1 <= n < m (got n=%u, m=%u)", n, m);
    if (nsamples == 0 || nsamples % m != 0) return fail(nullptr, MUSIC_B200_EINVAL, "nsamples must be a positive multiple of m (got %u)", nsamples);
    return MUSIC_B200_OK;
}

// The settings music_b200_create_coarray() checked: the physical element count, the lag table and the first virtual table
struct CoarrayDef {
    uint32_t m_in;
    CoarrayLags lags;
    double pos[2 * MAXM];  // the virtual ULA l s, l < Mv
    double lambda;
};

int create_on_device(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution, const float *table_c64,
                     int device, const AzelGeom *azel, const music_b200 *chan = nullptr, const CoarrayDef *co = nullptr)
{
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, MUSIC_B200_ENODEVICE, "no CUDA device (%s); this library has no CPU path", e == cudaSuccess ? "count 0" : cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(nullptr, MUSIC_B200_ENODEVICE, "device %d out of range (0..%d)", device, ndev - 1);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess)
        return fail(nullptr, MUSIC_B200_ECUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, MUSIC_B200_ENODEVICE, "device %d is sm_%d%d; this build targets sm_90a only", device, prop.major, prop.minor);

    music_b200 *h = new (std::nothrow) music_b200();
    if (!h) return fail(nullptr, MUSIC_B200_ENOMEM, "out of host memory");
    h->m = m; h->n = n; h->nsamples = nsamples; h->K = resolution;
    h->m_in = co ? co->m_in : m;
    h->N = nsamples / h->m_in;
    h->device = device; h->sm_count = prop.multiProcessorCount;
    if (co) {
        h->coarray = true;
        h->co_lags = co->lags;
    }
    if (azel) {
        h->azel = true;
        h->grid = azel->grid;
    }
    if (chan) {  // the channel settings create_channels() checked
        h->chan = true;
        h->cshape = chan->cshape;
        h->chan_taper = chan->chan_taper;
        h->chan_combine = chan->chan_combine;
    }

    int rc = MUSIC_B200_OK;
    auto init = [&]() -> int {
        CU(h, cudaSetDevice(device));
        for (int i = 0; i < 2; ++i) {
            CU(h, cudaStreamCreateWithFlags(&h->streams[i], cudaStreamNonBlocking));
            CU(h, cudaEventCreateWithFlags(&h->ws[i].scan_done, cudaEventDisableTiming));
        }
        // scan kernels with M = 16 need 32 KiB dynamic smem (< 48 KiB default), nothing to opt in.
        if (const char *e = getenv("MUSIC_B200_FUSED")) h->fused = atoi(e) != 0;
        if (const char *e = getenv("MUSIC_B200_EIG")) h->eig_mode = !strcmp(e, "jacobi") ? 1 : !strcmp(e, "jacobi1") ? 2 : 0;
        if (const char *e = getenv("MUSIC_B200_PDL")) h->pdl = atoi(e) != 0;
        if (const char *e = getenv("MUSIC_B200_FUSED_SPEC")) h->fused_spec = atoi(e) != 0;
        if (const char *e = getenv("MUSIC_B200_MMA_FIN")) h->mma_fin_max = std::max(-1, std::min(FZ_COV_WARPS, atoi(e)));
        CU(h, cudaFuncSetAttribute(covN_tma_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CN_SMEM));
        CU(h, cudaFuncSetAttribute(covN_tma_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CN_SMEM));
        CU(h, cudaFuncSetAttribute(music8_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F8_SMEM));
        CU(h, h->f8_stats.grow(2));
        CU(h, cudaMemset(h->f8_stats, 0, 2 * sizeof(unsigned)));
        CU(h, cudaEventCreateWithFlags(&h->fused_done, cudaEventDisableTiming));
        CU(h, h->work_ctr.grow(2 * CTR_RING * 2));  // self-resetting (tickets, finished CTAs) pairs
        CU(h, cudaMemset(h->work_ctr, 0, 2 * CTR_RING * 2 * sizeof(unsigned)));
        if (const char *e = getenv("MUSIC_B200_HOSTREG")) h->hostreg = atoi(e) != 0;
        if (getenv("MUSIC_B200_TRACE")) {
            const size_t tb = (size_t)FZ_TRACE_LAUNCHES * FZ_TRACE_CTAS * FZ_TRACE;
            CU(h, h->fused_trace.grow(tb));
            CU(h, cudaMemset(h->fused_trace, 0, tb * sizeof(long long)));
        }
        // the fused M = 4 kernel runs two CTAs per SM: all of the SM's unified L1 / shared memory goes to shared memory
        for (const void *k : {(const void *)music4_fused_kernel<false, false>, (const void *)music4_fused_kernel<true, false>,
                              (const void *)music4_fused_kernel<false, true>, (const void *)music4_fused_kernel<true, true>}) {
            CU(h, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FZ_SMEM));
            CU(h, cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
        }
        CU(h, cudaFuncSetAttribute(cov4_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)COV_SMEM));
        // IAA (music_iaa.cuh): each instance opts in to the largest dynamic shared memory of the M it serves
        CU(h, cudaFuncSetAttribute(iaa_kernel<4, iaa_windows(4)>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(iaa_smem_max(4, 4, iaa_windows(4)) * sizeof(double))));
        CU(h, cudaFuncSetAttribute(iaa_kernel<8, iaa_windows(8)>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(iaa_smem_max(8, 8, iaa_windows(8)) * sizeof(double))));
        CU(h, cudaFuncSetAttribute(iaa_kernel<16, iaa_windows(16)>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(iaa_smem_max(16, 16, iaa_windows(16)) * sizeof(double))));
        CU(h, cudaFuncSetAttribute(iaa_kernel<0, iaa_windows(2)>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(iaa_smem_max(2, 8, iaa_windows(2)) * sizeof(double))));
        CU(h, cudaFuncSetAttribute(iaa_kernel<0, iaa_windows(16)>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)(iaa_smem_max(9, 16, iaa_windows(16)) * sizeof(double))));
        if (chan) return init_channels(h);  // a channel handle takes its first tables at its first retune
        if (const int rc = alloc_slot(h, h->tables[0])) return rc;
        DeviceTable &t = h->tables[0].tabs[0];
        if (co) return build_table(h, t, co->pos, co->lambda, h->streams[0]);
        return azel ? build_table_azel(h, t, azel->pos, azel->lambda, h->streams[0]) : upload_table(h, t, table_c64, h->streams[0]);
    };
    rc = init();
    if (rc != MUSIC_B200_OK) {
        fail(nullptr, rc, "%s", std::string(h->error).c_str());
        music_b200_destroy(h);
        return rc;
    }
    *out = h;
    return MUSIC_B200_OK;
}

}  // namespace

extern "C" {

int music_b200_version(void) { return 2; }

const char *music_b200_last_error(const music_b200 *h)
{
    static thread_local std::string copy;  // the returned text stays valid until this thread's next call
    if (h) {
        music_b200 *hm = const_cast<music_b200 *>(h);
        std::lock_guard<std::mutex> g(hm->err_mutex);
        copy = hm->error;
        return copy.c_str();
    }
    std::lock_guard<std::mutex> g(g_err_mutex);
    copy = g_create_error;
    return copy.c_str();
}

uint64_t music_b200_launch_count(const music_b200 *h)
{
    if (!h) return 0;
    uint64_t n = h->launches.load();
    for (const music_b200 *c : h->kids) n += c->launches.load();
    return n;
}

int music_b200_debug_fused_trace(music_b200 *h, long long *host_out, int max_ctas)
{
    h = served(h);
    if (!h || !host_out || !h->fused_trace) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaDeviceSynchronize());
    CU(h, cudaMemcpy(host_out, h->fused_trace, (size_t)std::min(max_ctas, FZ_TRACE_LAUNCHES * FZ_TRACE_CTAS) * FZ_TRACE * sizeof(long long),
                     cudaMemcpyDeviceToHost));
    return MUSIC_B200_OK;
}

int music_b200_debug_fused8_stats(music_b200 *h, uint64_t *out2)
{
    h = served(h);
    if (!h || !out2 || !h->f8_stats) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    unsigned v[2];
    CU(h, cudaMemcpy(v, h->f8_stats, sizeof v, cudaMemcpyDeviceToHost));
    out2[0] = v[0];
    out2[1] = v[1];
    return MUSIC_B200_OK;
}

int music_b200_set_stage_timing(music_b200 *h, int enable)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    h->timing = enable != 0;
    h->tev_used = 0;
    return MUSIC_B200_OK;
}

int music_b200_get_stage_times(music_b200 *h, double *ms4, uint64_t *chunks)
{
    h = served(h);
    if (!h || !ms4) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    for (int i = 0; i < 4; ++i) ms4[i] = 0.0;
    const size_t nch = h->tev_used / 5;
    for (size_t c = 0; c < nch; ++c) {
        cudaEvent_t *e = h->tev.data() + 5 * c;
        CU(h, cudaEventSynchronize(e[4]));
        for (int i = 0; i < 4; ++i) {
            float ms = 0.f;
            CU(h, cudaEventElapsedTime(&ms, e[i], e[i + 1]));
            ms4[i] += ms;
        }
    }
    if (chunks) *chunks = nch;
    h->tev_used = 0;
    return MUSIC_B200_OK;
}

int music_b200_create(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution,
                      const float *table_c64, int device)
{
    if (const int rc = check_create(out, m, n, nsamples)) return rc;
    if (resolution == 0) return fail(nullptr, MUSIC_B200_EINVAL, "resolution must be > 0");
    if (!table_c64) return fail(nullptr, MUSIC_B200_EINVAL, "array response table must not be NULL");

    return create_on_device(out, m, n, nsamples, resolution, table_c64, device, nullptr);
}

int music_b200_set_table(music_b200 *h, const float *table_c64)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!table_c64) return fail(h, MUSIC_B200_EINVAL, "array response table must not be NULL");
    if (const int rc = refuse_coarray(h, "set_table (the virtual table is set by music_b200_set_geometry_coarray)")) return rc;
    std::lock_guard<std::mutex> g(h->mutex);
    if (!h->kids.empty())  // multi-device handle: every device holds a full copy of the table (SURVEY.md section 8e)
        return for_each_child(h, [&](music_b200 *c) { return music_b200_set_table(c, table_c64); });
    if (coherent(h))
        return fail(h, MUSIC_B200_EINVAL, "the COHERENT combine focuses geometric tables: one measured table gives no focusing "
                                          "(call music_b200_set_geometry_channels())");
    // on a channel handle one measured table serves every channel (the narrowband assumption)
    return retune(h, [&](TableSlot &s) {
        s.shared = true;
        return upload_table(h, s.tabs[0], table_c64, h->streams[0]);
    });
}

int music_b200_process_planar_device(music_b200 *h, const float *const *d_streams, uint32_t hop, uint32_t nwindows,
                                     float *d_angles, float *d_levels, float *d_spectrum, int32_t *d_bins, void *stream)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "planar input is not supported on an az-el handle");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "planar input is not built for channel handles");
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!d_streams) return fail(h, MUSIC_B200_EINVAL, "d_streams must not be NULL");
    if (hop == 0) return fail(h, MUSIC_B200_EINVAL, "hop must be >= 1 snapshot");
    PlanarStreams S = {};
    for (uint32_t r = 0; r < h->m_in; ++r) {
        if (!d_streams[r] || (reinterpret_cast<uintptr_t>(d_streams[r]) & 7u) != 0)
            return fail(h, MUSIC_B200_EINVAL, "antenna stream %u must be a non-NULL, 8-byte aligned device pointer", r);
        S.p[r] = reinterpret_cast<const float2 *>(d_streams[r]);
    }
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    Outputs o = caller_outputs(d_angles, d_levels, d_spectrum, d_bins);
    return enqueue_device(h, nullptr, nwindows, o.shaped(h), static_cast<cudaStream_t>(stream), 0, &S, hop);
}

int music_b200_process_planar_host(music_b200 *h, const float *const *streams, uint32_t hop, uint32_t nwindows,
                                   float *angles, float *levels, float *spectrum, int32_t *bins)
{
    music_b200 *const top = h;  // the handle process_host registers caller memory on
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "planar input is not supported on an az-el handle");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "planar input is not built for channel handles");
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!streams || !angles) return fail(h, MUSIC_B200_EINVAL, "streams and angles must not be NULL");
    if (hop == 0) return fail(h, MUSIC_B200_EINVAL, "hop must be >= 1 snapshot");
    for (uint32_t r = 0; r < h->m_in; ++r)
        if (!streams[r]) return fail(h, MUSIC_B200_EINVAL, "antenna stream %u must not be NULL", r);
    // the chunk copies read the streams (and write the spectrum) straight from and to caller memory
    const auto release = [&](music_b200 *owner) {
        const size_t stream_bytes = ((size_t)(nwindows - 1) * hop + h->N) * 2 * sizeof(float);
        for (uint32_t r = 0; r < h->m_in; ++r) release_straddling(owner, streams[r], stream_bytes);
        if (spectrum) release_straddling(owner, spectrum, (size_t)nwindows * h->K * sizeof(float));
    };
    if (top != h) {
        std::lock_guard<std::mutex> gt(top->mutex);
        release(top);
    }
    std::lock_guard<std::mutex> g(h->mutex);
    if (top == h) release(h);
    CU(h, cudaSetDevice(h->device));
    HostInput in;
    in.streams = streams;
    in.hop = hop;
    Outputs dst = caller_outputs(angles, levels, spectrum, bins);
    return stage_host(h, in, nwindows, dst.shaped(h));
}

int music_b200_reduce_angles_device(music_b200 *h, const float *d_angles, const float *d_levels, uint32_t nwindows, int weighted,
                                    float *d_mean_deg, float *d_resultant, float *d_weight_sum, void *stream)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (!d_angles || !d_mean_deg) return fail(h, MUSIC_B200_EINVAL, "d_angles and d_mean_deg must not be NULL");
    if (weighted && !d_levels) return fail(h, MUSIC_B200_EINVAL, "level weighting needs d_levels");
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    reduce_angles_kernel<<<h->n, REDUCE_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(d_angles, d_levels, (int)nwindows, (int)h->n,
                                                                                      weighted ? 1 : 0, d_mean_deg, d_resultant, d_weight_sum);
    h->launches++;
    CU(h, cudaGetLastError());
    return MUSIC_B200_OK;
}

int music_b200_reduce_spectrum_device(music_b200 *h, const float *d_spectrum, uint32_t nwindows, float *d_mean, void *stream)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (!d_spectrum || !d_mean) return fail(h, MUSIC_B200_EINVAL, "d_spectrum and d_mean must not be NULL");
    if (nwindows == 0) return fail(h, MUSIC_B200_EINVAL, "nwindows must be >= 1");
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    reduce_spectrum_kernel<<<(h->K + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(d_spectrum, (int)nwindows, (int)h->K, d_mean);
    h->launches++;
    CU(h, cudaGetLastError());
    return MUSIC_B200_OK;
}

// host-buffer conveniences: upload, reduce, download (GUI-rate calls; not a throughput path)
int music_b200_reduce_angles_host(music_b200 *h, const float *angles, const float *levels, uint32_t nwindows, int weighted,
                                  float *mean_deg, float *resultant, float *weight_sum)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (!angles || !mean_deg) return fail(h, MUSIC_B200_EINVAL, "angles and mean_deg must not be NULL");
    if (weighted && !levels) return fail(h, MUSIC_B200_EINVAL, "level weighting needs levels");
    DevBuf<float> d_a, d_l, d_o;
    const size_t ne = (size_t)nwindows * h->n, nb = ne * sizeof(float);
    {
        std::lock_guard<std::mutex> g(h->mutex);
        CU(h, cudaSetDevice(h->device));
        if (d_a.grow(std::max<size_t>(ne, 1)) != cudaSuccess || d_o.grow(3 * h->n) != cudaSuccess ||
            (levels && d_l.grow(std::max<size_t>(ne, 1)) != cudaSuccess))
            return fail(h, MUSIC_B200_ENOMEM, "cudaMalloc failed for the reducer buffers");
        cudaMemcpy(d_a, angles, nb, cudaMemcpyHostToDevice);
        if (levels) cudaMemcpy(d_l, levels, nb, cudaMemcpyHostToDevice);
    }
    int rc = music_b200_reduce_angles_device(h, d_a, d_l, nwindows, weighted, d_o, d_o + h->n, d_o + 2 * h->n, nullptr);
    if (rc == MUSIC_B200_OK) {
        std::vector<float> out(3 * h->n);
        const cudaError_t e = cudaMemcpy(out.data(), d_o, out.size() * sizeof(float), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) rc = fail(h, MUSIC_B200_ECUDA, "reducer failed: %s", cudaGetErrorString(e));
        else {
            for (uint32_t i = 0; i < h->n; ++i) {
                mean_deg[i] = out[i];
                if (resultant) resultant[i] = out[h->n + i];
                if (weight_sum) weight_sum[i] = out[2 * h->n + i];
            }
        }
    }
    return rc;
}

int music_b200_reduce_spectrum_host(music_b200 *h, const float *spectrum, uint32_t nwindows, float *mean)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (!spectrum || !mean) return fail(h, MUSIC_B200_EINVAL, "spectrum and mean must not be NULL");
    if (nwindows == 0) return fail(h, MUSIC_B200_EINVAL, "nwindows must be >= 1");
    DevBuf<float> d_s, d_m;
    const size_t ne = (size_t)nwindows * h->K;
    {
        std::lock_guard<std::mutex> g(h->mutex);
        CU(h, cudaSetDevice(h->device));
        if (d_s.grow(ne) != cudaSuccess || d_m.grow(h->K) != cudaSuccess)
            return fail(h, MUSIC_B200_ENOMEM, "cudaMalloc failed for the reducer buffers");
        cudaMemcpy(d_s, spectrum, ne * sizeof(float), cudaMemcpyHostToDevice);
    }
    int rc = music_b200_reduce_spectrum_device(h, d_s, nwindows, d_m, nullptr);
    if (rc == MUSIC_B200_OK) {
        const cudaError_t e = cudaMemcpy(mean, d_m, h->K * sizeof(float), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) rc = fail(h, MUSIC_B200_ECUDA, "reducer failed: %s", cudaGetErrorString(e));
    }
    return rc;
}

int music_b200_set_peak_mode(music_b200 *h, int mode, uint32_t exclusion_bins)
{
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    Modes p = h->modes;
    p.peak = mode;
    p.excl = exclusion_bins;
    if (const int rc = check_modes(h, p, gridless_mode(mode) ? own_table(h) : nullptr)) return rc;
    if (const int rc = for_each_child(h, [&](music_b200 *c) { return music_b200_set_peak_mode(c, mode, exclusion_bins); })) return rc;
    h->modes = p;
    return MUSIC_B200_OK;
}

int music_b200_set_geometry(music_b200 *h, const double *positions_xy, double wavelength, uint32_t *guarded)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "an az-el handle takes music_b200_set_geometry_azel()");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "a channel handle takes music_b200_set_geometry_channels()");
    if (h->coarray) return fail(h, MUSIC_B200_EINVAL, "a co-array handle takes music_b200_set_geometry_coarray()");
    if (!positions_xy) return fail(h, MUSIC_B200_EINVAL, "element positions must not be NULL");
    if (!(wavelength > 0.0) || !std::isfinite(wavelength)) return fail(h, MUSIC_B200_EINVAL, "wavelength must be positive and finite");
    for (uint32_t i = 0; i < 2 * h->m; ++i)
        if (!std::isfinite(positions_xy[i])) return fail(h, MUSIC_B200_EINVAL, "element positions must be finite");
    std::lock_guard<std::mutex> g(h->mutex);
    if (!h->kids.empty())
        return for_each_child(h, [&](music_b200 *c) { return music_b200_set_geometry(c, positions_xy, wavelength, guarded); });
    if (const int rc = retune(h, [&](TableSlot &s) {
            const int rb = build_table(h, s.tabs[0], positions_xy, wavelength, h->streams[0]);
            return rb ? rb : build_manifold(h, s, s.tabs[0]);
        }))
        return rc;
    if (guarded) *guarded = h->steer_guarded;
    return MUSIC_B200_OK;
}

void music_b200_steer_entry_host(const double *positions_xy, double wavelength, uint32_t resolution, uint32_t step,
                                 uint32_t antenna, float *re_im)
{
    steer_entry_host(positions_xy, wavelength, (int)resolution, (int)step, (int)antenna, &re_im[0], &re_im[1]);
}

int music_b200_manifold_coeffs_host(const double *positions_xy, uint32_t m, double wavelength, uint32_t *L, double *beta)
{
    if (!positions_xy || !L) return fail(nullptr, MUSIC_B200_EINVAL, "positions_xy and L must not be NULL");
    if (m == 0 || m > MUSIC_B200_MAX_M) return fail(nullptr, MUSIC_B200_EINVAL, "m must be in 1..%d (got %u)", MUSIC_B200_MAX_M, m);
    if (!(wavelength > 0.0) || !std::isfinite(wavelength)) return fail(nullptr, MUSIC_B200_EINVAL, "wavelength must be positive and finite");
    for (uint32_t i = 0; i < 2 * m; ++i)
        if (!std::isfinite(positions_xy[i])) return fail(nullptr, MUSIC_B200_EINVAL, "element positions must be finite");
    double ap = 0.0;
    if (!manifold_coeffs_host(positions_xy, (int)m, wavelength, L, beta, &ap))
        return fail(nullptr, MUSIC_B200_EINVAL, "the geometry spans %.4g wavelengths: manifold order %u > %d", ap, *L, MF_MAX_L);
    return MUSIC_B200_OK;
}

int music_b200_get_table(music_b200 *h, float *table_c64)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!table_c64) return fail(h, MUSIC_B200_EINVAL, "output table must not be NULL");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "a channel handle has one table per channel: music_b200_get_table_channel()");
    h = served(h);
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaMemcpy(table_c64, table(h).c64, (size_t)h->K * h->m * 2 * sizeof(float), cudaMemcpyDeviceToHost));
    return MUSIC_B200_OK;
}

}  // extern "C"

namespace {

// the 1-D device entry points: outputs o in device memory
int process_device_impl(music_b200 *h, const float *d_in_c64, uint32_t nwindows, Outputs o, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->kids.empty()) {
        // multi-device handle: the call goes to the child on whose device the input lives
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, d_in_c64) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
            cudaGetLastError();
            return fail(h, MUSIC_B200_EINVAL, "d_in_c64 is not a device pointer");
        }
        for (music_b200 *c : h->kids)
            if (c->device == at.device) {
                const int rc = process_device_impl(c, d_in_c64, nwindows, o, stream);
                if (rc) fail(h, rc, "%s", music_b200_last_error(c));
                return rc;
            }
        return fail(h, MUSIC_B200_EINVAL, "d_in_c64 lives on device %d, which this handle does not own", at.device);
    }
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "an az-el handle takes music_b200_process_azel_device()");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "a channel handle takes music_b200_process_channels_device()");
    std::lock_guard<std::mutex> g(h->mutex);
    NvtxRange range("music_b200_process_device");
    CU(h, cudaSetDevice(h->device));
    if (h->gather.G > 0) {
        if ((size_t)nwindows * h->gather.G * h->n > h->gather_cap) return fail(h, MUSIC_B200_EINVAL, "gather buffer holds %zu entries, the call needs %zu", h->gather_cap, (size_t)nwindows * h->gather.G * h->n);
        ++h->gather_epoch;
    }
    return enqueue_device(h, d_in_c64, nwindows, o.shaped(h), static_cast<cudaStream_t>(stream), 0);
}

// the host entry points: outputs dst in host memory (dst.elev: an az-el handle's elevations)
int process_host_impl(music_b200 *h, const float *in_c64, uint32_t nwindows, Outputs dst)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel && !dst.elev) return fail(h, MUSIC_B200_EINVAL, "an az-el handle takes music_b200_process_azel_host()");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "a channel handle takes music_b200_process_channels_host()");
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!in_c64 || !dst.angles) return fail(h, MUSIC_B200_EINVAL, "in_c64 and angles must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    // under the FIXED rule every count is n: nothing to compute or copy
    if (dst.counts && h->source_rule == MUSIC_B200_SOURCES_FIXED) {
        for (uint32_t w = 0; w < nwindows; ++w) dst.counts[w] = (int32_t)h->n;
        dst.counts = nullptr;
    }
    NvtxRange range("music_b200_process_host");
    // pageable caller memory (GNU Radio's circular buffers, numpy arrays) is pinned once and found again on later calls
    CU(h, cudaSetDevice(served(h)->device));
    const size_t in_bytes = (size_t)nwindows * h->nsamples * 2 * sizeof(float), spec_bytes = (size_t)nwindows * h->K * sizeof(float);
    host_register(h, in_c64, in_bytes, true);
    if (dst.spec) host_register(h, dst.spec, spec_bytes, false);
    // the two ranges the chunk copies touch directly, after both registrations (one may have dropped the other)
    release_straddling(h, in_c64, in_bytes);
    if (dst.spec) release_straddling(h, dst.spec, spec_bytes);
    HostInput in;
    in.windows = in_c64;
    return stage_host(h, in, nwindows, dst.shaped(h));
}

}  // namespace

extern "C" {

int music_b200_process_device_ex(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles,
                                 float *d_levels, float *d_spectrum, int32_t *d_bins, double *d_P64, double *d_R,
                                 double *d_eigvals, void *stream)
{
    Outputs o = caller_outputs(d_angles, d_levels, d_spectrum, d_bins);
    o.P64 = d_P64;
    o.R = d_R;
    o.ev = d_eigvals;
    return process_device_impl(h, d_in_c64, nwindows, o, stream);
}

int music_b200_process_device_counts(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles,
                                     float *d_levels, float *d_spectrum, int32_t *d_bins, int32_t *d_counts, void *stream)
{
    Outputs o = caller_outputs(d_angles, d_levels, d_spectrum, d_bins);
    o.counts = d_counts;
    return process_device_impl(h, d_in_c64, nwindows, o, stream);
}

int music_b200_process_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles,
                              float *d_levels, float *d_spectrum, int32_t *d_bins, void *stream)
{
    return music_b200_process_device_ex(h, d_in_c64, nwindows, d_angles, d_levels, d_spectrum, d_bins, nullptr, nullptr,
                                        nullptr, stream);
}

int music_b200_process_host(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels,
                            float *spectrum, int32_t *bins)
{
    return process_host_impl(h, in_c64, nwindows, caller_outputs(angles, levels, spectrum, bins));
}

int music_b200_process_host_counts(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels,
                                   float *spectrum, int32_t *bins, int32_t *counts)
{
    Outputs o = caller_outputs(angles, levels, spectrum, bins);
    o.counts = counts;
    return process_host_impl(h, in_c64, nwindows, o);
}

namespace {

// the checks every beams entry point makes before it runs: a beamformer set, an output asked for, the alignment
int check_beams_call(music_b200 *h, const void *weights, const void *beams)
{
    if (const int rc = refuse_coarray(h, "the beams entry")) return rc;
    if (h->beam_rule == MUSIC_B200_BEAMS_OFF)
        return fail(h, MUSIC_B200_EINVAL, "no beamformer set (call music_b200_set_beamformer() with DAS, MVDR or LCMV)");
    if (!weights && !beams) return fail(h, MUSIC_B200_EINVAL, "weights and beams must not both be NULL");
    if ((reinterpret_cast<uintptr_t>(beams) & 7u) != 0) return fail(h, MUSIC_B200_EINVAL, "beams must be 8-byte aligned");
    if ((reinterpret_cast<uintptr_t>(weights) & 15u) != 0) return fail(h, MUSIC_B200_EINVAL, "weights must be 16-byte aligned");
    return MUSIC_B200_OK;
}

}  // namespace

int music_b200_set_beamformer(music_b200 *h, int rule, double loading)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "the beamformer is not supported on an az-el handle");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "wideband beams are not built: a channel handle takes no beamformer");
    if (rule != MUSIC_B200_BEAMS_OFF)
        if (const int rc = refuse_coarray(h, "the beamformer")) return rc;
    if (rule != MUSIC_B200_BEAMS_OFF && rule != MUSIC_B200_BEAMS_DAS && rule != MUSIC_B200_BEAMS_MVDR && rule != MUSIC_B200_BEAMS_LCMV)
        return fail(h, MUSIC_B200_EINVAL, "unknown beamformer %d", rule);
    if (!std::isfinite(loading) || loading < 0.0) return fail(h, MUSIC_B200_EINVAL, "loading must be finite and >= 0 (got %g)", loading);
    if (loading != 0.0 && (rule == MUSIC_B200_BEAMS_OFF || rule == MUSIC_B200_BEAMS_DAS))
        return fail(h, MUSIC_B200_EINVAL, "diagonal loading applies to MVDR and LCMV beams only (got %g)", loading);
    if ((rule == MUSIC_B200_BEAMS_MVDR || rule == MUSIC_B200_BEAMS_LCMV) && loading == 0.0 && h->N <= h->m)
        return fail(h, MUSIC_B200_EINVAL, "MVDR and LCMV beams without diagonal loading need more snapshots than antennas (N = %u, m = %u): R is singular",
                    h->N, h->m);
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = for_each_child(h, [&](music_b200 *c) { return music_b200_set_beamformer(c, rule, loading); })) return rc;
    h->beam_rule = rule;
    h->beam_loading = loading;
    return MUSIC_B200_OK;
}

int music_b200_process_device_beams(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles, float *d_levels,
                                    float *d_spectrum, int32_t *d_bins, int32_t *d_counts, double *d_weights, float *d_beams, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (const int rc = check_beams_call(h, d_weights, d_beams)) return rc;
    Outputs o = caller_outputs(d_angles, d_levels, d_spectrum, d_bins);
    o.counts = d_counts;
    o.wts = d_weights;
    o.beams = d_beams;
    return process_device_impl(h, d_in_c64, nwindows, o, stream);
}

int music_b200_process_host_beams(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels, float *spectrum,
                                  int32_t *bins, int32_t *counts, double *weights, float *beams)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (const int rc = check_beams_call(h, weights, beams)) return rc;
    Outputs o = caller_outputs(angles, levels, spectrum, bins);
    o.counts = counts;
    o.wts = weights;
    o.beams = beams;
    return process_host_impl(h, in_c64, nwindows, o);
}

/* ---- the stochastic CRB of every slot (music_crb.cuh) ---- */
namespace {

// the checks every crb entry point makes before it runs: the output asked for and aligned, and the beams checks when
// the call asks for weights or beams
int check_crb_call(music_b200 *h, const void *out, const void *weights, const void *beams)
{
    if (const int rc = refuse_coarray(h, "the CRB")) return rc;
    if (!out) return fail(h, MUSIC_B200_EINVAL, "the CRB output must not be NULL");
    if ((reinterpret_cast<uintptr_t>(out) & 3u) != 0) return fail(h, MUSIC_B200_EINVAL, "the CRB output must be 4-byte aligned");
    if (weights || beams) return check_beams_call(h, weights, beams);
    return MUSIC_B200_OK;
}

}  // namespace

int music_b200_process_device_crb(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles, float *d_levels,
                                  float *d_spectrum, int32_t *d_bins, int32_t *d_counts, double *d_weights, float *d_beams,
                                  float *d_std, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (const int rc = check_crb_call(h, d_std, d_weights, d_beams)) return rc;
    Outputs o = caller_outputs(d_angles, d_levels, d_spectrum, d_bins);
    o.counts = d_counts;
    o.wts = d_weights;
    o.beams = d_beams;
    o.std = d_std;
    return process_device_impl(h, d_in_c64, nwindows, o, stream);
}

int music_b200_process_host_crb(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels, float *spectrum,
                                int32_t *bins, int32_t *counts, double *weights, float *beams, float *std_out)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "an az-el handle takes music_b200_process_azel_host_crb()");
    if (const int rc = check_crb_call(h, std_out, weights, beams)) return rc;
    Outputs o = caller_outputs(angles, levels, spectrum, bins);
    o.counts = counts;
    o.wts = weights;
    o.beams = beams;
    o.std = std_out;
    return process_host_impl(h, in_c64, nwindows, o);
}

/* ---- angle tracking (music_track.cuh) ---- */
namespace {

// the checks every tracks entry point makes before it runs: tracking on, slot_track asked for, track ids and states both
// or neither, every tracker output aligned, and the CRB entry's checks on the rest when std is given (the CRB, weights
// and beams may all be NULL)
int check_track_call(music_b200 *h, const void *std, const void *weights, const void *beams, const int32_t *slot_track,
                     const int32_t *track_ids, const float *track_state)
{
    if (h->trk_var == MUSIC_B200_TRACK_OFF)
        return fail(h, MUSIC_B200_EINVAL, "tracking is off (call music_b200_set_tracking() with FIXED or CRB variance)");
    if (!slot_track) return fail(h, MUSIC_B200_EINVAL, "slot_track must not be NULL");
    if (!track_ids != !track_state) return fail(h, MUSIC_B200_EINVAL, "track_ids and track_state are given both or neither");
    if (std)
        if (const int rc = refuse_coarray(h, "the CRB")) return rc;
    for (const void *q : {(const void *)slot_track, (const void *)track_ids, (const void *)track_state, std})
        if ((reinterpret_cast<uintptr_t>(q) & 3u) != 0) return fail(h, MUSIC_B200_EINVAL, "the tracker outputs and the CRB must be 4-byte aligned");
    if (weights || beams) return check_beams_call(h, weights, beams);
    return MUSIC_B200_OK;
}

Outputs with_tracks(Outputs o, int32_t *slot_track, int32_t *track_ids, float *track_state)
{
    o.slot_track = slot_track;
    o.track_ids = track_ids;
    o.track_state = track_state;
    return o;
}

}  // namespace

int music_b200_process_device_tracks(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles, float *d_levels,
                                     float *d_spectrum, int32_t *d_bins, int32_t *d_counts, double *d_weights, float *d_beams,
                                     float *d_std, int32_t *d_slot_track, int32_t *d_track_ids, float *d_track_state, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "an az-el handle takes music_b200_process_azel_device_tracks()");
    if (const int rc = check_track_call(h, d_std, d_weights, d_beams, d_slot_track, d_track_ids, d_track_state)) return rc;
    Outputs o = caller_outputs(d_angles, d_levels, d_spectrum, d_bins);
    o.counts = d_counts;
    o.wts = d_weights;
    o.beams = d_beams;
    o.std = d_std;
    return process_device_impl(h, d_in_c64, nwindows, with_tracks(o, d_slot_track, d_track_ids, d_track_state), stream);
}

int music_b200_process_host_tracks(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels, float *spectrum,
                                   int32_t *bins, int32_t *counts, double *weights, float *beams, float *std_out, int32_t *slot_track,
                                   int32_t *track_ids, float *track_state)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "an az-el handle takes music_b200_process_azel_host_tracks()");
    if (const int rc = check_track_call(h, std_out, weights, beams, slot_track, track_ids, track_state)) return rc;
    Outputs o = caller_outputs(angles, levels, spectrum, bins);
    o.counts = counts;
    o.wts = weights;
    o.beams = beams;
    o.std = std_out;
    return process_host_impl(h, in_c64, nwindows, with_tracks(o, slot_track, track_ids, track_state));
}

/* ---- receiver calibration (music_calib.cuh) ---- */
int music_b200_set_calibration(music_b200 *h, const double *gains)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "per-channel calibration is not built: a channel handle takes no calibration");
    CalibVec cv = {};
    if (gains) {
        for (uint32_t m = 0; m < h->m_in; ++m) {
            const double gr = gains[2 * m], gi = gains[2 * m + 1];
            if (!std::isfinite(gr) || !std::isfinite(gi)) return fail(h, MUSIC_B200_EINVAL, "gain %u is not finite", m);
            // c = 1 / g = conj(g) / |g|^2 in fp64
            const double d = gr * gr + gi * gi;
            cv.c[m] = make_double2(gr / d, -gi / d);
            if (!(d > 0.0) || !std::isfinite(cv.c[m].x) || !std::isfinite(cv.c[m].y))
                return fail(h, MUSIC_B200_EINVAL, "gain %u must have a modulus > 0 whose inverse is finite", m);
        }
    }
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = for_each_child(h, [&](music_b200 *c) { return music_b200_set_calibration(c, gains); })) return rc;
    h->calib = gains != nullptr;
    h->cal_c = cv;
    h->integ_fresh = true;  // the carry is kept in corrected coordinates
    for (uint32_t i = 0; i < 2 * h->m_in; ++i) h->cal_g[i] = gains ? gains[i] : (i % 2 == 0 ? 1.0 : 0.0);
    return MUSIC_B200_OK;
}

int music_b200_get_calibration(music_b200 *h, double *gains)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!gains) return fail(h, MUSIC_B200_EINVAL, "gains must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    for (uint32_t i = 0; i < 2 * h->m_in; ++i) gains[i] = h->calib ? h->cal_g[i] : (i % 2 == 0 ? 1.0 : 0.0);
    return MUSIC_B200_OK;
}

}  // extern "C"

/* ---- covariance integration across windows (music_integrate.cuh) ---- */
namespace {

// the handles whose windows form one stream on one device: every other handle refuses integration
int check_integration(music_b200 *h)
{
    if (!h->kids.empty())
        return fail(h, MUSIC_B200_EINVAL, "integration is not built for multi-device handles (their windows are dealt round-robin "
                                          "over the devices)");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "per-channel integration is not built: a channel handle takes no integration");
    if (h->gather_buf)
        return fail(h, MUSIC_B200_EINVAL, "integration is not built for a handle with a bins all-gather (its windows are one "
                                          "rank's share of a stream)");
    return MUSIC_B200_OK;
}

}  // namespace

extern "C" {

int music_b200_set_integration(music_b200 *h, double alpha)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!std::isfinite(alpha) || alpha < 0.0 || alpha >= 1.0)
        return fail(h, MUSIC_B200_EINVAL, "the forgetting factor must be finite with 0 <= alpha < 1 (got %g)", alpha);
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = check_integration(h)) return rc;
    if (alpha > 0.0 && !h->integ_done) {
        CU(h, cudaSetDevice(h->device));
        CU(h, h->integ_S.grow(2 * (size_t)h->m_in * h->m_in));
        CU(h, h->integ_cnt.grow(1));
        CU(h, cudaEventCreateWithFlags(&h->integ_done, cudaEventDisableTiming));
    }
    h->integ_alpha = alpha;
    h->integ_fresh = true;
    return MUSIC_B200_OK;
}

int music_b200_reset_integration(music_b200 *h)
{
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = check_integration(h)) return rc;
    h->integ_fresh = true;
    return MUSIC_B200_OK;
}

}  // extern "C"

/* ---- angle tracking (music_track.cuh) ---- */
namespace {

// the handles whose windows form one stream on one device, as for the integration: every other handle refuses tracking
int check_tracking(music_b200 *h)
{
    if (!h->kids.empty())
        return fail(h, MUSIC_B200_EINVAL, "tracking is not built for multi-device handles (their windows are dealt round-robin "
                                          "over the devices)");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "per-channel tracking is not built: a channel handle takes no tracking");
    if (h->gather_buf)
        return fail(h, MUSIC_B200_EINVAL, "tracking is not built for a handle with a bins all-gather (its windows are one "
                                          "rank's share of a stream)");
    return MUSIC_B200_OK;
}

}  // namespace

extern "C" {

int music_b200_set_tracking(music_b200 *h, int variance, double q, double rate_std0, double floor_deg, double crb_scale,
                            double gate, uint32_t confirm_hits, uint32_t confirm_window, uint32_t max_misses, uint32_t max_tracks)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (variance != MUSIC_B200_TRACK_OFF && variance != MUSIC_B200_TRACK_FIXED && variance != MUSIC_B200_TRACK_CRB)
        return fail(h, MUSIC_B200_EINVAL, "unknown measurement variance %d", variance);
    const auto nonneg = [](double v) { return std::isfinite(v) && v >= 0.0; };
    if (!nonneg(q) || !nonneg(rate_std0) || !nonneg(floor_deg))
        return fail(h, MUSIC_B200_EINVAL, "q, rate_std0 and floor_deg must be finite and >= 0 (got %g, %g, %g)", q, rate_std0, floor_deg);
    if (!std::isfinite(gate) || !(gate > 0.0)) return fail(h, MUSIC_B200_EINVAL, "the gate must be finite and > 0 (got %g)", gate);
    if (variance == MUSIC_B200_TRACK_FIXED && !(floor_deg > 0.0))
        return fail(h, MUSIC_B200_EINVAL, "FIXED variance needs floor_deg > 0");
    if (variance == MUSIC_B200_TRACK_CRB && !(std::isfinite(crb_scale) && crb_scale > 0.0))
        return fail(h, MUSIC_B200_EINVAL, "CRB variance needs a finite crb_scale > 0 (got %g)", crb_scale);
    if (confirm_hits < 1 || confirm_hits > confirm_window || confirm_window > 64)
        return fail(h, MUSIC_B200_EINVAL, "need 1 <= confirm_hits <= confirm_window <= 64 (got %u, %u)", confirm_hits, confirm_window);
    if (max_misses < 1) return fail(h, MUSIC_B200_EINVAL, "max_misses must be >= 1");
    if (max_tracks < 1 || max_tracks > MUSIC_B200_TRACK_MAX_ROWS)
        return fail(h, MUSIC_B200_EINVAL, "max_tracks must be in 1..%d (got %u)", MUSIC_B200_TRACK_MAX_ROWS, max_tracks);
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = check_tracking(h)) return rc;
    if (variance == MUSIC_B200_TRACK_CRB)
        if (const int rc = refuse_coarray(h, "tracking under CRB variance")) return rc;
    if (variance == MUSIC_B200_TRACK_CRB && !table(h).geometric)
        return fail(h, MUSIC_B200_EINVAL, "CRB variance needs a table built by music_b200_set_geometry%s(); the current one came "
                                          "from set_table(), which has no geometry", h->azel ? "_azel" : "");
    if (variance != MUSIC_B200_TRACK_OFF && !h->trk_done) {
        CU(h, cudaSetDevice(h->device));
        CU(h, h->trk_rows.grow((size_t)MUSIC_B200_TRACK_MAX_ROWS * TRK_ROW_INTS));
        CU(h, h->trk_state.grow((size_t)MUSIC_B200_TRACK_MAX_ROWS * track_state_len(2)));
        CU(h, h->trk_next.grow(1));
        CU(h, cudaEventCreateWithFlags(&h->trk_done, cudaEventDisableTiming));
    }
    TrackParams tp = {};
    tp.crb = variance == MUSIC_B200_TRACK_CRB;
    tp.q = q; tp.rate0 = rate_std0; tp.floor = floor_deg; tp.crb_scale = crb_scale; tp.gate = gate;
    tp.confirm_hits = (int)confirm_hits; tp.confirm_window = (int)confirm_window; tp.max_misses = (int)max_misses;
    tp.T = (int)max_tracks;
    h->trk_var = variance;
    h->trk = tp;
    h->trk_fresh = true;
    return MUSIC_B200_OK;
}

int music_b200_reset_tracks(music_b200 *h)
{
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = check_tracking(h)) return rc;
    h->trk_fresh = true;
    return MUSIC_B200_OK;
}

int music_b200_get_tracks(music_b200 *h, int32_t *rows, double *state, uint32_t *next_id)
{
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    const size_t T = (size_t)h->trk.T, sl = (size_t)track_state_len(h->azel ? 2 : 1);
    if (h->trk_fresh || !h->trk_used) {
        // the carry a reset leaves: every row empty
        for (size_t r = 0; r < T; ++r) {
            if (rows) {
                rows[r * TRK_ROW_INTS] = -1;
                for (int k = 1; k < TRK_ROW_INTS; ++k) rows[r * TRK_ROW_INTS + k] = 0;
            }
            if (state) for (size_t k = 0; k < sl; ++k) state[r * sl + k] = 0.0;
        }
        if (next_id) *next_id = 0;
        return MUSIC_B200_OK;
    }
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaEventSynchronize(h->trk_done));
    if (rows) CU(h, cudaMemcpy(rows, h->trk_rows, T * TRK_ROW_INTS * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (state) CU(h, cudaMemcpy(state, h->trk_state, T * sl * sizeof(double), cudaMemcpyDeviceToHost));
    if (next_id) CU(h, cudaMemcpy(next_id, h->trk_next, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return MUSIC_B200_OK;
}

}  // extern "C"

namespace {

// the accumulator, partial sums, counter and result buffer of a served handle (zeroed on first use)
int ensure_calib_buffers(music_b200 *h)
{
    if (h->cal_out) return MUSIC_B200_OK;  // (allocated last)
    const size_t mm = (size_t)h->m * h->m;
    CU(h, h->cal_acc.grow(mm));
    CU(h, h->cal_part.grow((size_t)CALIB_ACC_MAX_CTAS * mm));
    CU(h, h->cal_ctr.grow(1));
    CU(h, h->cal_out.grow(CALIB_OUT));
    CU(h, cudaMemset(h->cal_acc, 0, mm * sizeof(double2)));
    CU(h, cudaMemset(h->cal_ctr, 0, sizeof(unsigned)));
    CU(h, cudaDeviceSynchronize());  // the memsets ran on the legacy stream; the kernels run on non-blocking ones
    h->cal_windows = 0;
    return MUSIC_B200_OK;
}

// Adds the raw covariance of nwindows windows at d_in (device memory of h, served and locked) to the accumulator, on
// st: the covariance kernels in sub-batches through workspace slot 0, each followed by calib_accum_kernel.
int calib_accumulate(music_b200 *h, const float *d_in, uint32_t nwindows, cudaStream_t st)
{
    if (nwindows == 0) return MUSIC_B200_OK;
    if (const int rc = ensure_calib_buffers(h)) return rc;
    Plan plan;  // R only
    const uint32_t sub = std::min((nwindows + SCAN_B - 1) / SCAN_B * SCAN_B, max_sub_windows(h, plan));
    Workspace &ws = h->ws[0];
    if (const int rc = ensure_slot(h, ws, sub, plan)) return rc;
    if (ws.used) CU(h, cudaStreamWaitEvent(st, ws.scan_done, 0));
    for (uint32_t w0 = 0; w0 < nwindows; w0 += sub) {
        const uint32_t W = std::min(sub, nwindows - w0);
        launch_cov(h, ws.view(), d_in + (size_t)w0 * h->nsamples * 2, W, st, 0);
        const int wpc = calib_acc_wpc((int)W);
        calib_accum_kernel<<<(W + wpc - 1) / wpc, CALIB_THREADS, 0, st>>>(ws.R, (int)h->m, (int)W, wpc, h->cal_part, h->cal_ctr, h->cal_acc);
        h->launches++;
        CU(h, cudaGetLastError());
        CU(h, cudaEventRecord(ws.scan_done, st));
        ws.used = true;
    }
    h->cal_windows += nwindows;
    return MUSIC_B200_OK;
}

}  // namespace

extern "C" {

int music_b200_calib_reset(music_b200 *h)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "per-channel calibration is not built: a channel handle takes no calibration");
    if (const int rc = refuse_coarray(h, "calibration estimation (estimate the gains on a plain handle, then set_calibration)")) return rc;
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    if (const int rc = ensure_calib_buffers(h)) return rc;
    CU(h, cudaDeviceSynchronize());  // accumulate calls still in flight on any stream
    CU(h, cudaMemset(h->cal_acc, 0, (size_t)h->m * h->m * sizeof(double2)));
    CU(h, cudaDeviceSynchronize());
    h->cal_windows = 0;
    return MUSIC_B200_OK;
}

int music_b200_calib_accumulate_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, void *stream)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "per-channel calibration is not built: a channel handle takes no calibration");
    if (const int rc = refuse_coarray(h, "calibration estimation (estimate the gains on a plain handle, then set_calibration)")) return rc;
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!d_in_c64) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 must not be NULL");
    if ((reinterpret_cast<uintptr_t>(d_in_c64) & 15u) != 0) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 must be 16-byte aligned");
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    return calib_accumulate(h, d_in_c64, nwindows, static_cast<cudaStream_t>(stream));
}

int music_b200_calib_accumulate_host(music_b200 *h, const float *in_c64, uint32_t nwindows)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "per-channel calibration is not built: a channel handle takes no calibration");
    if (const int rc = refuse_coarray(h, "calibration estimation (estimate the gains on a plain handle, then set_calibration)")) return rc;
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!in_c64) return fail(h, MUSIC_B200_EINVAL, "in_c64 must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    // chunks of ~32 MiB through one pinned and one device buffer on the handle's first stream (not a throughput path; the
    // pinned copy makes the transfer independent of how the caller's memory is, or partly is, registered)
    const size_t win_bytes = (size_t)h->nsamples * 2 * sizeof(float);
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>(nwindows, ((size_t)32 << 20) / win_bytes));
    const size_t chunk_floats = (size_t)chunk * h->nsamples * 2;
    DevBuf<float> d;
    PinBuf<float> pin;
    cudaStream_t st = h->streams[0];
    int rc = MUSIC_B200_OK;
    if (d.grow(chunk_floats) != cudaSuccess || pin.grow(chunk_floats) != cudaSuccess)
        rc = fail(h, MUSIC_B200_ENOMEM, "cannot allocate the calibration staging buffers");
    for (uint32_t w0 = 0; w0 < nwindows && rc == MUSIC_B200_OK; w0 += chunk) {
        const uint32_t W = std::min(chunk, nwindows - w0);
        CU_BREAK(h, rc, cudaStreamSynchronize(st));  // the previous chunk's upload has left the pinned buffer
        memcpy(pin, in_c64 + (size_t)w0 * h->nsamples * 2, W * win_bytes);
        CU_BREAK(h, rc, cudaMemcpyAsync(d, pin, W * win_bytes, cudaMemcpyHostToDevice, st));
        rc = calib_accumulate(h, d, W, st);
    }
    const cudaError_t e = cudaStreamSynchronize(st);
    if (rc == MUSIC_B200_OK && e != cudaSuccess) rc = fail(h, MUSIC_B200_ECUDA, "stream sync failed: %s", cudaGetErrorString(e));
    return rc;
}

int music_b200_calib_solve(music_b200 *h, double az_deg, double el_deg, int kind, double *gains, double *stats)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "per-channel calibration is not built: a channel handle takes no calibration");
    if (const int rc = refuse_coarray(h, "calibration estimation (estimate the gains on a plain handle, then set_calibration)")) return rc;
    if (!gains) return fail(h, MUSIC_B200_EINVAL, "gains must not be NULL");
    if (kind != MUSIC_B200_CALIB_PHASE && kind != MUSIC_B200_CALIB_GAIN_PHASE) return fail(h, MUSIC_B200_EINVAL, "unknown calibration kind %d", kind);
    if (kind == MUSIC_B200_CALIB_GAIN_PHASE && h->m < 3)
        return fail(h, MUSIC_B200_EINVAL, "gain and phase calibration needs m >= 3 (with two elements the magnitudes cannot be "
                                          "identified; use MUSIC_B200_CALIB_PHASE)");
    if (!std::isfinite(az_deg) || !std::isfinite(el_deg)) return fail(h, MUSIC_B200_EINVAL, "the source direction must be finite");
    if (!h->azel && el_deg != 0.0) return fail(h, MUSIC_B200_EINVAL, "a 1-D handle takes el_deg = 0 (got %g)", el_deg);
    std::lock_guard<std::mutex> g(h->mutex);
    const DeviceTable &tb = table(h);
    if (!tb.geometric)
        return fail(h, MUSIC_B200_EINVAL, "calibration needs a table built from the array geometry (set_geometry / set_geometry_azel); "
                                          "the current one came from set_table()");
    if (h->cal_windows == 0) return fail(h, MUSIC_B200_EINVAL, "no calibration windows accumulated");
    CalibSource src = {};
    for (uint32_t m = 0; m < h->m; ++m) {
        src.pos[3 * m] = h->azel ? tb.ageo.pos[3 * m] : tb.geo.pos[2 * m];
        src.pos[3 * m + 1] = h->azel ? tb.ageo.pos[3 * m + 1] : tb.geo.pos[2 * m + 1];
        src.pos[3 * m + 2] = h->azel ? tb.ageo.pos[3 * m + 2] : 0.0;
    }
    src.lambda = h->azel ? tb.ageo.lambda : tb.geo.lambda;
    src.az = az_deg * STEER_DEG2RAD;
    src.el = el_deg * STEER_DEG2RAD;
    src.azel = h->azel;
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaDeviceSynchronize());  // every accumulate call, on whatever stream, has landed
    cudaStream_t st = h->streams[0];
    calib_solve_kernel<<<1, 32, 0, st>>>(h->cal_acc, (double)h->cal_windows, (int)h->m, src, kind, h->cal_out);
    h->launches++;
    CU(h, cudaGetLastError());
    double out[CALIB_OUT];
    CU(h, cudaMemcpyAsync(out, h->cal_out, sizeof out, cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    switch ((int)out[2 * MAXM + 2]) {
    case CALIB_OK: break;
    case CALIB_NOPOWER: return fail(h, MUSIC_B200_EINVAL, "calibration failed: the accumulated covariance has no power on its diagonal");
    case CALIB_DEAD: return fail(h, MUSIC_B200_EINVAL, "calibration failed: an element has zero gain (a dead channel)");
    default: return fail(h, MUSIC_B200_EINVAL, "calibration failed: a non-finite value in the accumulated covariance or the fit");
    }
    for (uint32_t i = 0; i < 2 * h->m; ++i) gains[i] = out[i];
    if (stats) {
        stats[0] = out[2 * MAXM];
        stats[1] = out[2 * MAXM + 1];
    }
    return MUSIC_B200_OK;
}

}  // extern "C"

namespace {

// Refusals shared by the self-calibration entry points: az-el and channel handles are out of its scope.
int check_blind_handle(music_b200 *h)
{
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "self-calibration is not built for channel handles");
    if (const int rc = refuse_coarray(h, "self-calibration (estimate the gains on a plain handle, then set_calibration)")) return rc;
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "self-calibration is not built for az-el handles");
    return MUSIC_B200_OK;
}

// the per-segment sums, partial sums and counter of a served handle (zeroed on first use)
int ensure_blind_buffers(music_b200 *h)
{
    if (h->cb_ctr) return MUSIC_B200_OK;  // (allocated last)
    const size_t mm = (size_t)h->m * h->m;
    CU(h, h->cb_acc.grow((size_t)CB_MAX_SEGMENTS * mm));
    CU(h, h->cb_part.grow((size_t)CALIB_ACC_MAX_CTAS * mm));
    CU(h, h->cb_ctr.grow(1));
    CU(h, cudaMemset(h->cb_acc, 0, (size_t)CB_MAX_SEGMENTS * mm * sizeof(double2)));
    CU(h, cudaMemset(h->cb_ctr, 0, sizeof(unsigned)));
    CU(h, cudaDeviceSynchronize());  // the memsets ran on the legacy stream; the kernels run on non-blocking ones
    h->cb_count.clear();
    return MUSIC_B200_OK;
}

// nwindows windows in segments of `segment` (validated by the caller): nwindows a multiple of segment, room for the
// segments in the accumulator
int check_blind_accumulate(music_b200 *h, uint32_t nwindows, uint32_t segment)
{
    if (segment == 0) return fail(h, MUSIC_B200_EINVAL, "segment must be >= 1");
    if (nwindows % segment != 0) return fail(h, MUSIC_B200_EINVAL, "nwindows (%u) must be a multiple of segment (%u)", nwindows, segment);
    if (h->cb_count.size() + nwindows / segment > (size_t)CB_MAX_SEGMENTS)
        return fail(h, MUSIC_B200_EINVAL, "more than %d self-calibration segments", CB_MAX_SEGMENTS);
    return MUSIC_B200_OK;
}

// Adds the segments of nwindows windows at d_in (device memory of h, served and locked) to the accumulator, on st: the
// covariance kernels in sub-batches of whole segments through workspace slot 0, then calib_accum_kernel once per segment
// into that segment's sum.  A segment's sum depends on its windows alone, however the windows are split across calls.
int calib_blind_accumulate(music_b200 *h, const float *d_in, uint32_t nwindows, uint32_t segment, cudaStream_t st)
{
    if (const int rc = ensure_blind_buffers(h)) return rc;
    if (const int rc = check_blind_accumulate(h, nwindows, segment)) return rc;
    Plan plan;  // R only
    const uint32_t sub = std::max(segment, std::min(nwindows, max_sub_windows(h, plan)) / segment * segment);
    Workspace &ws = h->ws[0];
    if (const int rc = ensure_slot(h, ws, (sub + SCAN_B - 1) / SCAN_B * SCAN_B, plan)) return rc;
    if (ws.used) CU(h, cudaStreamWaitEvent(st, ws.scan_done, 0));
    const size_t mm = (size_t)h->m * h->m;
    const int wpc = calib_acc_wpc((int)segment);
    for (uint32_t w0 = 0; w0 < nwindows; w0 += sub) {
        const uint32_t W = std::min(sub, nwindows - w0);
        launch_cov(h, ws.view(), d_in + (size_t)w0 * h->nsamples * 2, W, st, 0);
        for (uint32_t j = 0; j < W / segment; ++j) {
            calib_accum_kernel<<<(segment + wpc - 1) / wpc, CALIB_THREADS, 0, st>>>(ws.R + (size_t)j * segment * mm * 2, (int)h->m,
                                                                                   (int)segment, wpc, h->cb_part, h->cb_ctr,
                                                                                   h->cb_acc + h->cb_count.size() * mm);
            h->launches++;
            h->cb_count.push_back(segment);
        }
        CU(h, cudaGetLastError());
        CU(h, cudaEventRecord(ws.scan_done, st));
        ws.used = true;
    }
    return MUSIC_B200_OK;
}

// whether the element positions [M][x, y] lie on one line (all coincident included): tests/calib_blind_oracle.py
bool collinear(const double *pos, uint32_t M)
{
    int f = 0;
    double L2 = 0.0;
    for (uint32_t m = 0; m < M; ++m) {
        const double dx = pos[2 * m] - pos[0], dy = pos[2 * m + 1] - pos[1], l = dx * dx + dy * dy;
        if (l > L2) { L2 = l; f = (int)m; }
    }
    if (L2 == 0.0) return true;
    const double fx = pos[2 * f] - pos[0], fy = pos[2 * f + 1] - pos[1];
    double c = 0.0;
    for (uint32_t m = 0; m < M; ++m) c = std::max(c, std::fabs((pos[2 * m] - pos[0]) * fy - (pos[2 * m + 1] - pos[1]) * fx));
    return c <= 1e-9 * L2;
}

}  // namespace

extern "C" {

int music_b200_calib_blind_reset(music_b200 *h)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (const int rc = check_blind_handle(h)) return rc;
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    if (const int rc = ensure_blind_buffers(h)) return rc;
    CU(h, cudaDeviceSynchronize());  // accumulate calls still in flight on any stream
    CU(h, cudaMemset(h->cb_acc, 0, h->cb_count.size() * h->m * h->m * sizeof(double2)));
    CU(h, cudaDeviceSynchronize());
    h->cb_count.clear();
    return MUSIC_B200_OK;
}

int music_b200_calib_blind_accumulate_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, uint32_t segment, void *stream)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (const int rc = check_blind_handle(h)) return rc;
    if (segment == 0) return fail(h, MUSIC_B200_EINVAL, "segment must be >= 1");
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!d_in_c64) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 must not be NULL");
    if ((reinterpret_cast<uintptr_t>(d_in_c64) & 15u) != 0) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 must be 16-byte aligned");
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    return calib_blind_accumulate(h, d_in_c64, nwindows, segment, static_cast<cudaStream_t>(stream));
}

int music_b200_calib_blind_accumulate_host(music_b200 *h, const float *in_c64, uint32_t nwindows, uint32_t segment)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (const int rc = check_blind_handle(h)) return rc;
    if (segment == 0) return fail(h, MUSIC_B200_EINVAL, "segment must be >= 1");
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!in_c64) return fail(h, MUSIC_B200_EINVAL, "in_c64 must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    if (const int rc = ensure_blind_buffers(h)) return rc;
    if (const int rc = check_blind_accumulate(h, nwindows, segment)) return rc;
    // chunks of whole segments, ~32 MiB or one segment, through one pinned and one device buffer on the handle's first
    // stream, as calib_accumulate_host does
    const size_t win_bytes = (size_t)h->nsamples * 2 * sizeof(float);
    const uint32_t chunk = std::max<uint32_t>(segment, (uint32_t)std::min<size_t>(nwindows, ((size_t)32 << 20) / win_bytes) / segment * segment);
    const size_t chunk_floats = (size_t)chunk * h->nsamples * 2;
    DevBuf<float> d;
    PinBuf<float> pin;
    cudaStream_t st = h->streams[0];
    int rc = MUSIC_B200_OK;
    if (d.grow(chunk_floats) != cudaSuccess || pin.grow(chunk_floats) != cudaSuccess)
        rc = fail(h, MUSIC_B200_ENOMEM, "cannot allocate the self-calibration staging buffers");
    for (uint32_t w0 = 0; w0 < nwindows && rc == MUSIC_B200_OK; w0 += chunk) {
        const uint32_t W = std::min(chunk, nwindows - w0);
        CU_BREAK(h, rc, cudaStreamSynchronize(st));  // the previous chunk's upload has left the pinned buffer
        memcpy(pin, in_c64 + (size_t)w0 * h->nsamples * 2, W * win_bytes);
        CU_BREAK(h, rc, cudaMemcpyAsync(d, pin, W * win_bytes, cudaMemcpyHostToDevice, st));
        rc = calib_blind_accumulate(h, d, W, segment, st);
    }
    const cudaError_t e = cudaStreamSynchronize(st);
    if (rc == MUSIC_B200_OK && e != cudaSuccess) rc = fail(h, MUSIC_B200_ECUDA, "stream sync failed: %s", cudaGetErrorString(e));
    return rc;
}

int music_b200_calib_blind_solve(music_b200 *h, uint32_t d, int kind, uint32_t starts, uint64_t seed, double *gains, double *angles,
                                 double *stats)
{
    h = served(h);
    if (!h) return MUSIC_B200_EINVAL;
    if (const int rc = check_blind_handle(h)) return rc;
    if (!gains) return fail(h, MUSIC_B200_EINVAL, "gains must not be NULL");
    if (kind != MUSIC_B200_CALIB_PHASE && kind != MUSIC_B200_CALIB_GAIN_PHASE) return fail(h, MUSIC_B200_EINVAL, "unknown calibration kind %d", kind);
    if (h->m < 3) return fail(h, MUSIC_B200_EINVAL, "self-calibration needs m >= 3 (got %u)", h->m);
    if (d < 1 || d > h->m - 2) return fail(h, MUSIC_B200_EINVAL, "self-calibration needs 1 <= d <= m - 2 (got d = %u, m = %u)", d, h->m);
    if (starts < 1 || starts > (uint32_t)CB_MAX_STARTS) return fail(h, MUSIC_B200_EINVAL, "starts must be in 1 .. %d (got %u)", CB_MAX_STARTS, starts);
    std::lock_guard<std::mutex> g(h->mutex);
    const DeviceTable &tb = table(h);
    if (!tb.geometric)
        return fail(h, MUSIC_B200_EINVAL, "self-calibration needs a table built from the array geometry (set_geometry); the current one "
                                          "came from set_table()");
    if (collinear(tb.geo.pos, h->m))
        return fail(h, MUSIC_B200_EINVAL, "self-calibration needs elements off one line (on a line a phase ramp along it cannot be told "
                                          "from a shift of every direction)");
    if (h->K > (uint32_t)CB_MAX_K) return fail(h, MUSIC_B200_EINVAL, "self-calibration scans tables of at most %d rows (K = %u)", CB_MAX_K, h->K);
    const uint32_t S = (uint32_t)h->cb_count.size();
    if (S == 0) return fail(h, MUSIC_B200_EINVAL, "no self-calibration segments accumulated");
    const int M = (int)h->m, MM = M * M, P = (int)starts, D = (int)d, K = (int)h->K;
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaDeviceSynchronize());  // every accumulate call, on whatever stream, has landed
    auto &b = h->cb_work;
    CU(h, b.cnt.grow(S));
    CU(h, b.Rw.grow((size_t)S * MM * 2));
    CU(h, b.ev.grow((size_t)S * M));
    CU(h, b.Vt.grow((size_t)S * MM * 2));
    CU(h, b.mag.grow(M));
    CU(h, b.Q.grow((size_t)P * MM * 2));
    CU(h, b.qev.grow((size_t)P * M));
    CU(h, b.qV.grow((size_t)P * MM * 2));
    CU(h, b.jp.grow((size_t)P * S));
    CU(h, b.J.grow(P));
    CU(h, b.out.grow(CB_OUT));
    CU(h, b.angles.grow((size_t)S * D));
    CU(h, b.Pi.grow((size_t)S * MM));
    CU(h, b.phi.grow((size_t)P * M));
    CU(h, b.bins.grow((size_t)P * S * D));
    CU(h, b.st.grow(1));
    cudaStream_t st = h->streams[0];
    CU(h, cudaMemcpyAsync(b.cnt, h->cb_count.data(), S * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    Plan eig;
    eig.eig = true;
    const auto solve_eig = [&](double *R, double *ev, double *Vt, uint32_t W) {
        launch_eig_stage(h, eig, WsView{R, ev, Vt, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, W, nullptr, 0, st);
    };
    // magnitudes, whitened segments, their noise projectors, the starts
    cb_prep_kernel<<<1, CB_THREADS, 0, st>>>(h->cb_acc, b.cnt, M, (int)S, b.Rw, b.mag, b.st);
    solve_eig(b.Rw, b.ev, b.Vt, S);
    cb_proj_kernel<<<(unsigned)(((size_t)S * MM + CB_THREADS - 1) / CB_THREADS), CB_THREADS, 0, st>>>(b.Vt, M, M - D, (int)S, b.Pi);
    cb_init_kernel<<<(P * M + 255) / 256, 256, 0, st>>>(b.phi, M, P, seed, b.st);
    h->launches += 3;
    CU(h, cudaGetLastError());
    const size_t smem = (size_t)K * sizeof(double);
    const auto scan_kernel = M <= 4 ? cb_scan_kernel<4> : M <= 8 ? cb_scan_kernel<8> : cb_scan_kernel<MAXM>;
    CU(h, cudaFuncSetAttribute(scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const auto iteration = [&](bool polish) -> int {
        scan_kernel<<<polish ? S : (unsigned)P * S, CB_THREADS, smem, st>>>(tb.soa, K, M, D, (int)S, b.Vt, b.phi, polish, b.st, b.bins, b.jp);
        cb_q_kernel<<<polish ? 1 : P, CB_THREADS, 0, st>>>(tb.soa, M, D, (int)S, b.Pi, b.bins, b.jp, polish, b.st, b.Q, b.J);
        solve_eig(b.Q, b.qev, b.qV, polish ? 1 : P);
        cb_update_kernel<<<polish ? 1 : (P + 127) / 128, polish ? 32 : 128, 0, st>>>(b.qV, M, P, polish, b.st, b.phi);
        h->launches += 3;
        CU(h, cudaGetLastError());
        return MUSIC_B200_OK;
    };
    for (int t = 0; t < CB_T1; ++t)
        if (const int rc = iteration(false)) return rc;
    cb_select_kernel<<<1, 1, 0, st>>>(b.J, P, b.st);
    h->launches++;
    for (int t = 0; t < CB_T2; ++t)
        if (const int rc = iteration(true)) return rc;
    cb_out_kernel<<<1, CB_THREADS, 0, st>>>(b.phi, b.mag, b.bins, b.J, M, (int)S, D, K, kind == MUSIC_B200_CALIB_PHASE, b.st, b.out, b.angles);
    h->launches++;
    CU(h, cudaGetLastError());
    double out[CB_OUT];
    std::vector<double> ang((size_t)S * D);
    CU(h, cudaMemcpyAsync(out, b.out, sizeof out, cudaMemcpyDeviceToHost, st));
    CU(h, cudaMemcpyAsync(ang.data(), b.angles, ang.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    if (out[2 * MAXM + 3] == CB_NONFINITE_INPUT)
        return fail(h, MUSIC_B200_EINVAL, "self-calibration failed: a non-finite value in the segment covariances, or an element without power");
    if (out[2 * MAXM + 3] != CB_OK)
        return fail(h, MUSIC_B200_EINVAL, "self-calibration failed: the fit is not finite (an eigenvector component of Q vanished)");
    for (int i = 0; i < 2 * M; ++i) gains[i] = out[i];
    if (angles) std::copy(ang.begin(), ang.end(), angles);
    if (stats) {
        stats[0] = out[2 * MAXM];
        stats[1] = out[2 * MAXM + 1];
        stats[2] = out[2 * MAXM + 2];
        stats[3] = (double)S;
    }
    return MUSIC_B200_OK;
}

int music_b200_set_source_rule(music_b200 *h, int rule)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (rule != MUSIC_B200_SOURCES_FIXED && rule != MUSIC_B200_SOURCES_MDL && rule != MUSIC_B200_SOURCES_AIC)
        return fail(h, MUSIC_B200_EINVAL, "unknown source rule %d", rule);
    if (rule != MUSIC_B200_SOURCES_FIXED && h->coarray)
        return fail(h, MUSIC_B200_EINVAL, "a co-array handle takes the FIXED source rule only (the eigenvalues of R_ss are squares: "
                                          "MDL and AIC do not apply)");
    if (rule != MUSIC_B200_SOURCES_FIXED && snapshots(h) <= h->m)
        return fail(h, MUSIC_B200_EINVAL, "MDL / AIC need more snapshots than antennas (N = %u, m = %u)", snapshots(h), h->m);
    if (rule != MUSIC_B200_SOURCES_FIXED && h->chan && h->chan_combine == MUSIC_B200_CHANNELS_INCOHERENT)
        return fail(h, MUSIC_B200_EINVAL, "the INCOHERENT combine is defined for the FIXED source rule only");
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = for_each_child(h, [&](music_b200 *c) { return music_b200_set_source_rule(c, rule); })) return rc;
    h->source_rule = rule;
    return MUSIC_B200_OK;
}

int music_b200_set_refine(music_b200 *h, int mode)
{
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    Modes p = h->modes;
    p.refine = mode;
    if (const int rc = check_modes(h, p, mode != MUSIC_B200_REFINE_OFF ? own_table(h) : nullptr)) return rc;
    if (const int rc = for_each_child(h, [&](music_b200 *c) { return music_b200_set_refine(c, mode); })) return rc;
    h->modes = p;
    return MUSIC_B200_OK;
}

int music_b200_set_estimator(music_b200 *h, int estimator, double loading)
{
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    Modes p = h->modes;
    p.est = estimator;
    p.loading = loading;
    if (const int rc = check_modes(h, p, nullptr)) return rc;
    if (const int rc = for_each_child(h, [&](music_b200 *c) { return music_b200_set_estimator(c, estimator, loading); })) return rc;
    h->modes = p;
    return MUSIC_B200_OK;
}

static_assert(IAA_MAX_ITERATIONS == MUSIC_B200_IAA_MAX_ITERATIONS && IAA_DEFAULT_ITERATIONS == MUSIC_B200_IAA_DEFAULT_ITERATIONS,
              "the IAA iteration bounds of music_iaa.cuh and the header");

int music_b200_set_iaa_iterations(music_b200 *h, int iterations)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (iterations < 1 || iterations > IAA_MAX_ITERATIONS)
        return fail(h, MUSIC_B200_EINVAL, "the IAA iteration count must be 1 .. %d (got %d)", IAA_MAX_ITERATIONS, iterations);
    std::lock_guard<std::mutex> g(h->mutex);
    if (const int rc = for_each_child(h, [&](music_b200 *c) { return music_b200_set_iaa_iterations(c, iterations); })) return rc;
    h->modes.iaa_iter = iterations;
    return MUSIC_B200_OK;
}

int music_b200_create_multi(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution,
                            const float *table_c64, const int *devices, int ndev)
{
    if (!out) return fail(nullptr, MUSIC_B200_EINVAL, "out must not be NULL");
    *out = nullptr;
    if (!devices || ndev < 1 || ndev > MAX_PEERS) return fail(nullptr, MUSIC_B200_EINVAL, "need 1..%d devices (got %d)", MAX_PEERS, ndev);
    for (int i = 0; i < ndev; ++i)
        for (int j = 0; j < i; ++j)
            if (devices[i] == devices[j]) return fail(nullptr, MUSIC_B200_EINVAL, "device %d listed twice", devices[i]);
    music_b200 *h = new (std::nothrow) music_b200();
    if (!h) return fail(nullptr, MUSIC_B200_ENOMEM, "out of host memory");
    h->m = m; h->m_in = m; h->n = n; h->nsamples = nsamples; h->K = resolution; h->N = m ? nsamples / m : 0;
    h->device = devices[0];
    if (const char *e = getenv("MUSIC_B200_HOSTREG")) h->hostreg = atoi(e) != 0;
    for (int i = 0; i < ndev; ++i) {
        music_b200 *c = nullptr;
        const int rc = music_b200_create(&c, m, n, nsamples, resolution, table_c64, devices[i]);  // (sets the create error text)
        if (rc != MUSIC_B200_OK) {
            music_b200_destroy(h);
            return rc;
        }
        h->kids.push_back(c);
    }
    // peer access between every pair (the sharded device entry stores peak bins straight into the peers' buffers)
    for (int i = 0; i < ndev; ++i) {
        cudaSetDevice(devices[i]);
        for (int j = 0; j < ndev; ++j) {
            if (i == j) continue;
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, devices[i], devices[j]) == cudaSuccess && can) {
                const cudaError_t e = cudaDeviceEnablePeerAccess(devices[j], 0);
                if (e != cudaSuccess) cudaGetLastError();  // already enabled is fine
            }
        }
    }
    *out = h;
    return MUSIC_B200_OK;
}

int music_b200_device_count(const music_b200 *h) { return h ? (h->kids.empty() ? 1 : (int)h->kids.size()) : 0; }

/* ---- fused all-gather of the peak bins across processes (one GPU per process) ---- */
int music_b200_gather_create(music_b200 *h, uint32_t total_windows, unsigned char *ipc_handles /* [2][64] */)
{
    if (!h || !ipc_handles) return MUSIC_B200_EINVAL;
    if (!h->kids.empty()) return fail(h, MUSIC_B200_EINVAL, "gather_create applies to single-device handles (a multi-device handle gathers in process_device_sharded)");
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "the bins all-gather is not supported on an az-el handle");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "the bins all-gather is not built for channel handles");
    if (const int rc = refuse_coarray(h, "the bins all-gather")) return rc;
    std::lock_guard<std::mutex> g(h->mutex);
    CU(h, cudaSetDevice(h->device));
    if (h->gather_buf) return fail(h, MUSIC_B200_EINVAL, "gather buffer already created");
    if (h->integ_alpha > 0.0) return fail(h, MUSIC_B200_EINVAL, "the bins all-gather is not built for an integrating handle (set_integration(0) first)");
    if (h->trk_var != MUSIC_B200_TRACK_OFF)
        return fail(h, MUSIC_B200_EINVAL, "the bins all-gather is not built for a tracking handle (set_tracking(OFF) first)");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    const size_t elems = (size_t)total_windows * h->n;
    // the handle takes the buffers once both exist and are shared: a failure leaves it without a gather buffer
    DevBuf<int32_t> buf;
    DevBuf<unsigned> flags;
    CU(h, buf.grow(std::max<size_t>(elems, 1)));
    CU(h, flags.grow(MAX_PEERS));
    CU(h, cudaMemset(buf, 0xff, buf.size() * sizeof(int32_t)));
    CU(h, cudaMemset(flags, 0, MAX_PEERS * sizeof(unsigned)));
    cudaIpcMemHandle_t hb, hf;
    CU(h, cudaIpcGetMemHandle(&hb, buf));
    CU(h, cudaIpcGetMemHandle(&hf, flags));
    memcpy(ipc_handles, &hb, 64);
    memcpy(ipc_handles + 64, &hf, 64);
    h->gather_buf = std::move(buf);
    h->gather_flags = std::move(flags);
    h->gather_cap = elems;
    return MUSIC_B200_OK;
}

int music_b200_gather_attach(music_b200 *h, int nranks, int rank, const unsigned char *all_handles /* [nranks][2][64] */)
{
    if (!h || !all_handles) return MUSIC_B200_EINVAL;
    if (nranks < 1 || nranks > MAX_PEERS || rank < 0 || rank >= nranks) return fail(h, MUSIC_B200_EINVAL, "need 1 <= nranks <= %d and 0 <= rank < nranks", MAX_PEERS);
    if (h->azel) return fail(h, MUSIC_B200_EINVAL, "the bins all-gather is not supported on an az-el handle");
    if (h->chan) return fail(h, MUSIC_B200_EINVAL, "the bins all-gather is not built for channel handles");
    if (const int rc = refuse_coarray(h, "the bins all-gather")) return rc;
    std::lock_guard<std::mutex> g(h->mutex);
    if (!h->gather_buf) return fail(h, MUSIC_B200_EINVAL, "call gather_create first");
    CU(h, cudaSetDevice(h->device));
    for (int p = 0; p < nranks; ++p) {
        if (p == rank) {
            h->gather.peer[p] = h->gather_buf;
            h->peer_flags[p] = h->gather_flags;
            continue;
        }
        cudaIpcMemHandle_t hb, hf;
        memcpy(&hb, all_handles + (size_t)p * 128, 64);
        memcpy(&hf, all_handles + (size_t)p * 128 + 64, 64);
        // each mapping is recorded as soon as it is open, so that music_b200_destroy() closes it whatever fails next
        void *pb = nullptr, *pf = nullptr;
        CU(h, cudaIpcOpenMemHandle(&pb, hb, cudaIpcMemLazyEnablePeerAccess));
        h->ipc_maps.push_back(pb);
        CU(h, cudaIpcOpenMemHandle(&pf, hf, cudaIpcMemLazyEnablePeerAccess));
        h->ipc_maps.push_back(pf);
        h->gather.peer[p] = static_cast<int32_t *>(pb);
        h->peer_flags[p] = static_cast<unsigned *>(pf);
    }
    h->gather.G = nranks;
    h->gather.rank = rank;
    h->gather_epoch = 0;
    return MUSIC_B200_OK;
}

int music_b200_gather_wait(music_b200 *h, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    if (h->gather.G <= 0 || !h->gather_flags) return fail(h, MUSIC_B200_EINVAL, "no gather attached");
    CU(h, cudaSetDevice(h->device));
    gather_wait_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(h->gather_flags, h->gather.G, h->gather_epoch);
    h->launches++;
    CU(h, cudaGetLastError());
    return MUSIC_B200_OK;
}

const int32_t *music_b200_gather_buffer(const music_b200 *h) { return h ? h->gather_buf.get() : nullptr; }

int music_b200_gather_read(music_b200 *h, int32_t *host_out, uint32_t count)
{
    if (!h || !host_out) return MUSIC_B200_EINVAL;
    std::lock_guard<std::mutex> g(h->mutex);
    if (!h->gather_buf || count > h->gather_cap) return fail(h, MUSIC_B200_EINVAL, "gather buffer holds %zu entries", h->gather_cap);
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaMemcpy(host_out, h->gather_buf, (size_t)count * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return MUSIC_B200_OK;
}

/* ---- one call, G devices, inputs resident: shard g holds the windows w = i * G + g ---- */
int music_b200_process_device_sharded(music_b200 *h, const float *const *d_in_c64, uint32_t nwindows_total, float *const *d_angles,
                                      float *const *d_levels, int32_t *const *d_bins_all, void *const *streams)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->kids.empty()) return fail(h, MUSIC_B200_EINVAL, "process_device_sharded needs a handle from music_b200_create_multi");
    if (!d_in_c64 || !d_angles) return fail(h, MUSIC_B200_EINVAL, "d_in_c64 and d_angles must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    NvtxRange range("music_b200_process_device_sharded");
    const int G = (int)h->kids.size();
    int rc = MUSIC_B200_OK;
    for (int l = 0; l < G && rc == MUSIC_B200_OK; ++l) {
        music_b200 *c = h->kids[l];
        const uint32_t Wl = (uint32_t)l < nwindows_total ? (nwindows_total - l + G - 1) / G : 0;
        if (!Wl) continue;
        CU_BREAK(h, rc, cudaSetDevice(c->device));
        Outputs o = caller_outputs(d_angles[l], d_levels ? d_levels[l] : nullptr, nullptr, nullptr);
        o.shaped(c);
        if (d_bins_all) {
            // the scan epilogue of shard l stores its peak bins at stream position w = i * G + l of EVERY device's array
            o.gather.G = G;
            o.gather.rank = l;
            for (int p = 0; p < G; ++p) o.gather.peer[p] = d_bins_all[p];
        }
        rc = enqueue_device(c, d_in_c64[l], Wl, o, streams ? static_cast<cudaStream_t>(streams[l]) : nullptr, 0);
        if (rc) fail(h, rc, "%s", std::string(c->error).c_str());
    }
    return rc;
}

/* ---- (azimuth, elevation) MUSIC (music_azel.cuh) ---- */
namespace {

// positions_xyz [m][3] and the wavelength: finite, wavelength > 0
int check_azel_geometry(music_b200 *h, uint32_t m, const double *positions_xyz, double wavelength)
{
    if (!positions_xyz) return fail(h, MUSIC_B200_EINVAL, "element positions must not be NULL");
    if (!(wavelength > 0.0) || !std::isfinite(wavelength)) return fail(h, MUSIC_B200_EINVAL, "wavelength must be positive and finite");
    for (uint32_t i = 0; i < 3 * m; ++i)
        if (!std::isfinite(positions_xyz[i])) return fail(h, MUSIC_B200_EINVAL, "element positions must be finite");
    return MUSIC_B200_OK;
}

}  // namespace

int music_b200_create_azel(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t n_az, uint32_t n_el,
                           double el_lo_deg, double el_hi_deg, const double *positions_xyz, double wavelength, int device)
{
    if (const int rc = check_create(out, m, n, nsamples)) return rc;
    if (n_az == 0 || n_el == 0) return fail(nullptr, MUSIC_B200_EINVAL, "n_az and n_el must be > 0");
    if ((uint64_t)n_az * n_el > MUSIC_B200_AZEL_MAX_BINS)
        return fail(nullptr, MUSIC_B200_EINVAL, "n_az * n_el must be at most %u (got %llu)", (unsigned)MUSIC_B200_AZEL_MAX_BINS, (unsigned long long)n_az * n_el);
    if (!(el_lo_deg >= -90.0 && el_lo_deg <= el_hi_deg && el_hi_deg <= 90.0))
        return fail(nullptr, MUSIC_B200_EINVAL, "need -90 <= el_lo <= el_hi <= 90 degrees (got %g, %g)", el_lo_deg, el_hi_deg);
    if (n_el >= 2 && !(el_lo_deg < el_hi_deg)) return fail(nullptr, MUSIC_B200_EINVAL, "n_el >= 2 needs el_lo < el_hi");
    const int rc = check_azel_geometry(nullptr, m, positions_xyz, wavelength);
    if (rc) return rc;
    AzelGeom g = {};
    for (uint32_t i = 0; i < 3 * m; ++i) g.pos[i] = positions_xyz[i];
    g.lambda = wavelength;
    g.grid = {(int)n_az, (int)n_el, el_lo_deg, el_hi_deg};
    return create_on_device(out, m, n, nsamples, n_az * n_el, nullptr, device, &g);
}

int music_b200_set_geometry_azel(music_b200 *h, const double *positions_xyz, double wavelength)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->azel) return fail(h, MUSIC_B200_EINVAL, "set_geometry_azel needs a handle from music_b200_create_azel");
    const int rc = check_azel_geometry(h, h->m, positions_xyz, wavelength);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(h->mutex);
    return retune(h, [&](TableSlot &s) { return build_table_azel(h, s.tabs[0], positions_xyz, wavelength, h->streams[0]); });
}

int music_b200_azel_lattice_host(const double *positions_xyz, uint32_t m, double wavelength, int *mx, int *my, double s[4])
{
    if (!positions_xyz || !mx || !my || !s) return fail(nullptr, MUSIC_B200_EINVAL, "positions_xyz, mx, my and s must not be NULL");
    if (m == 0 || m > MUSIC_B200_MAX_M) return fail(nullptr, MUSIC_B200_EINVAL, "m must be in 1..%d (got %u)", MUSIC_B200_MAX_M, m);
    if (const int rc = check_azel_geometry(nullptr, m, positions_xyz, wavelength)) return rc;
    const LatticeGeom g = azel_lattice(positions_xyz, (int)m, wavelength);
    if (!g.ok) return fail(nullptr, MUSIC_B200_EINVAL, "the positions are not a planar lattice with steps <= lambda / 2");
    *mx = g.mx;
    *my = g.my;
    s[0] = g.s1[0], s[1] = g.s1[1], s[2] = g.s2[0], s[3] = g.s2[1];
    return MUSIC_B200_OK;
}

namespace {

// The az-el device entry named `entry`, after its own checks: outputs o (the azimuths in o.angles, the elevations in
// o.elev) in device memory.  process_azel_host_impl: the same for the host entries, outputs in host memory.
int process_azel_device_impl(music_b200 *h, const char *entry, const float *d_in_c64, uint32_t nwindows, Outputs o, void *stream)
{
    if (!h->azel) return fail(h, MUSIC_B200_EINVAL, "%s needs a handle from music_b200_create_azel", entry);
    if (nwindows && (!o.angles || !o.elev)) return fail(h, MUSIC_B200_EINVAL, "d_azimuth and d_elevation must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    NvtxRange range(entry);
    CU(h, cudaSetDevice(h->device));
    return enqueue_device(h, d_in_c64, nwindows, o.shaped(h), static_cast<cudaStream_t>(stream), 0);
}

int process_azel_host_impl(music_b200 *h, const char *entry, const float *in_c64, uint32_t nwindows, Outputs o)
{
    if (!h->azel) return fail(h, MUSIC_B200_EINVAL, "%s needs a handle from music_b200_create_azel", entry);
    if (nwindows && !o.elev) return fail(h, MUSIC_B200_EINVAL, "elevation must not be NULL");
    return process_host_impl(h, in_c64, nwindows, o);
}

// the outputs of the az-el entries
Outputs azel_outputs(float *azimuth, float *elevation, float *levels, float *spectrum, int32_t *bins, int32_t *counts, float *crb)
{
    Outputs o = caller_outputs(azimuth, levels, spectrum, bins);
    o.elev = elevation;
    o.counts = counts;
    o.std = crb;
    return o;
}

}  // namespace

int music_b200_process_azel_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_azimuth, float *d_elevation,
                                   float *d_levels, float *d_spectrum, int32_t *d_bins, int32_t *d_counts, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    return process_azel_device_impl(h, "music_b200_process_azel_device", d_in_c64, nwindows,
                                    azel_outputs(d_azimuth, d_elevation, d_levels, d_spectrum, d_bins, d_counts, nullptr), stream);
}

int music_b200_process_azel_host(music_b200 *h, const float *in_c64, uint32_t nwindows, float *azimuth, float *elevation,
                                 float *levels, float *spectrum, int32_t *bins, int32_t *counts)
{
    if (!h) return MUSIC_B200_EINVAL;
    return process_azel_host_impl(h, "music_b200_process_azel_host", in_c64, nwindows,
                                  azel_outputs(azimuth, elevation, levels, spectrum, bins, counts, nullptr));
}

int music_b200_process_azel_device_crb(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_azimuth, float *d_elevation,
                                       float *d_levels, float *d_spectrum, int32_t *d_bins, int32_t *d_counts, float *d_crb, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel)
        if (const int rc = check_crb_call(h, d_crb, nullptr, nullptr)) return rc;
    return process_azel_device_impl(h, "music_b200_process_azel_device_crb", d_in_c64, nwindows,
                                    azel_outputs(d_azimuth, d_elevation, d_levels, d_spectrum, d_bins, d_counts, d_crb), stream);
}

int music_b200_process_azel_host_crb(music_b200 *h, const float *in_c64, uint32_t nwindows, float *azimuth, float *elevation,
                                     float *levels, float *spectrum, int32_t *bins, int32_t *counts, float *crb)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel)
        if (const int rc = check_crb_call(h, crb, nullptr, nullptr)) return rc;
    return process_azel_host_impl(h, "music_b200_process_azel_host_crb", in_c64, nwindows,
                                  azel_outputs(azimuth, elevation, levels, spectrum, bins, counts, crb));
}

int music_b200_process_azel_device_tracks(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_azimuth,
                                          float *d_elevation, float *d_levels, float *d_spectrum, int32_t *d_bins, int32_t *d_counts,
                                          float *d_crb, int32_t *d_slot_track, int32_t *d_track_ids, float *d_track_state, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel)
        if (const int rc = check_track_call(h, d_crb, nullptr, nullptr, d_slot_track, d_track_ids, d_track_state)) return rc;
    return process_azel_device_impl(h, "music_b200_process_azel_device_tracks", d_in_c64, nwindows,
                                    with_tracks(azel_outputs(d_azimuth, d_elevation, d_levels, d_spectrum, d_bins, d_counts, d_crb),
                                                d_slot_track, d_track_ids, d_track_state),
                                    stream);
}

int music_b200_process_azel_host_tracks(music_b200 *h, const float *in_c64, uint32_t nwindows, float *azimuth, float *elevation,
                                        float *levels, float *spectrum, int32_t *bins, int32_t *counts, float *crb, int32_t *slot_track,
                                        int32_t *track_ids, float *track_state)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (h->azel)
        if (const int rc = check_track_call(h, crb, nullptr, nullptr, slot_track, track_ids, track_state)) return rc;
    return process_azel_host_impl(h, "music_b200_process_azel_host_tracks", in_c64, nwindows,
                                  with_tracks(azel_outputs(azimuth, elevation, levels, spectrum, bins, counts, crb), slot_track,
                                              track_ids, track_state));
}

/* ---- frequency-channelised direction finding (music_channels.cuh) ---- */
int music_b200_create_channels(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution, uint32_t nfft,
                               uint32_t chan_first, uint32_t chan_count, int taper, int combine, int device)
{
    if (const int rc = check_create(out, m, n, nsamples)) return rc;
    if (resolution == 0) return fail(nullptr, MUSIC_B200_EINVAL, "resolution must be > 0");
    if (nfft < (uint32_t)CHAN_MIN_F || nfft > (uint32_t)CHAN_MAX_F || (nfft & (nfft - 1)) != 0)
        return fail(nullptr, MUSIC_B200_EINVAL, "nfft must be a power of two in %d..%d (got %u)", CHAN_MIN_F, CHAN_MAX_F, nfft);
    if ((nsamples / m) % nfft != 0)
        return fail(nullptr, MUSIC_B200_EINVAL, "nfft must divide the %u snapshots of a window (got %u)", nsamples / m, nfft);
    if (chan_count == 0 || chan_count > nfft || chan_first >= nfft)
        return fail(nullptr, MUSIC_B200_EINVAL, "need 1 <= chan_count <= nfft and chan_first < nfft (got first=%u, count=%u)", chan_first, chan_count);
    if (taper != MUSIC_B200_TAPER_RECT && taper != MUSIC_B200_TAPER_HANN) return fail(nullptr, MUSIC_B200_EINVAL, "unknown taper %d", taper);
    if (combine != MUSIC_B200_CHANNELS_SEPARATE && combine != MUSIC_B200_CHANNELS_INCOHERENT && combine != MUSIC_B200_CHANNELS_COHERENT)
        return fail(nullptr, MUSIC_B200_EINVAL, "unknown combine rule %d", combine);
    music_b200 spec;
    ChanShape &cs = spec.cshape;
    cs.M = (int)m;
    cs.N = (int)(nsamples / m);
    cs.F = (int)nfft;
    for (cs.logF = 0; (1u << cs.logF) < nfft; ++cs.logF) {}
    cs.J = cs.N / cs.F;
    cs.first = (int)chan_first;
    cs.C = (int)chan_count;
    spec.chan_taper = taper;
    spec.chan_combine = combine;
    return create_on_device(out, m, n, nsamples, resolution, nullptr, device, nullptr, &spec);
}

namespace {

// frequency offset of channel c in units of the sample rate: s(b_c) / F
double channel_offset(const ChanShape &cs, int c)
{
    const int b = (cs.first + c) & (cs.F - 1);
    return (double)(b < cs.F / 2 ? b : b - cs.F) / (double)cs.F;
}

// The focusing matrices and errors of table slot s (music_focus.cuh) from its channel tables' geometry and the
// handle's sector: B_c on the device, the polar factors on the host, then the errors on the device.  On EINVAL (a
// singular B_c) the slot's matrices are left as they were.
int build_focusing(music_b200 *h, TableSlot &s, cudaStream_t st)
{
    const int C = h->cshape.C, M = (int)h->m, ref = C / 2;
    const size_t MM = (size_t)M * M;
    CU(h, h->foc_B.grow((size_t)C * MM));
    CU(h, h->foc_lam.grow(C));
    CU(h, h->foc_e2.grow(C));
    FocusGeom g = {};
    for (int i = 0; i < 2 * M; ++i) g.pos[i] = s.tabs[0].geo.pos[i];
    g.M = M; g.K = (int)h->K; g.C = C; g.ref = ref;
    g.first = (int)h->foc_first;
    g.count = h->foc_count ? (int)h->foc_count : (int)h->K;
    std::vector<double> lam(C);
    for (int c = 0; c < C; ++c) lam[c] = s.tabs[c].geo.lambda;
    CU(h, cudaMemcpyAsync(h->foc_lam, lam.data(), C * sizeof(double), cudaMemcpyHostToDevice, st));
    focus_setup_kernel<<<C, FOCUS_THREADS, 0, st>>>(g, h->foc_lam, nullptr, h->foc_B, nullptr);
    h->launches++;
    CU(h, cudaGetLastError());
    std::vector<std::complex<double>> B((size_t)C * MM), T((size_t)C * MM, std::complex<double>(0.0, 0.0));
    CU(h, cudaMemcpyAsync(B.data(), h->foc_B, B.size() * sizeof(double2), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));
    for (int c = 0; c < C; ++c) {
        if (c == ref) {
            for (int i = 0; i < M; ++i) T[(size_t)c * MM + (size_t)i * M + i] = 1.0;
            continue;
        }
        if (!focus_polar(M, B.data() + (size_t)c * MM, T.data() + (size_t)c * MM))
            return fail(h, MUSIC_B200_EINVAL, "the focusing matrix of channel %d is singular on this sector (sigma_min <= %g sigma_max): "
                                              "widen the sector", c, FOCUS_SINGULAR);
    }
    CU(h, cudaMemcpyAsync(s.foc_T, T.data(), T.size() * sizeof(double2), cudaMemcpyHostToDevice, st));
    focus_setup_kernel<<<C, FOCUS_THREADS, 0, st>>>(g, h->foc_lam, s.foc_T, nullptr, h->foc_e2);
    h->launches++;
    CU(h, cudaGetLastError());
    std::vector<double> e2(C);
    CU(h, cudaMemcpyAsync(e2.data(), h->foc_e2, C * sizeof(double), cudaMemcpyDeviceToHost, st));
    CU(h, cudaStreamSynchronize(st));  // T and e2 are locals
    s.foc_err.assign(C, 0.0);
    for (int c = 0; c < C; ++c)
        if (c != ref) s.foc_err[c] = std::sqrt(e2[c]) / std::sqrt((double)M * g.count);
    return MUSIC_B200_OK;
}

}  // namespace

int music_b200_set_geometry_channels(music_b200 *h, const double *positions_xy, double centre_frequency_hz, double sample_rate_hz)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->chan) return fail(h, MUSIC_B200_EINVAL, "set_geometry_channels needs a handle from music_b200_create_channels");
    if (!positions_xy) return fail(h, MUSIC_B200_EINVAL, "element positions must not be NULL");
    for (uint32_t i = 0; i < 2 * h->m; ++i)
        if (!std::isfinite(positions_xy[i])) return fail(h, MUSIC_B200_EINVAL, "element positions must be finite");
    if (!(sample_rate_hz > 0.0) || !std::isfinite(sample_rate_hz)) return fail(h, MUSIC_B200_EINVAL, "the sample rate must be positive and finite");
    if (!std::isfinite(centre_frequency_hz) || !(centre_frequency_hz > 0.5 * sample_rate_hz))
        return fail(h, MUSIC_B200_EINVAL, "the centre frequency must be finite and above half the sample rate (every channel frequency must be > 0)");
    std::lock_guard<std::mutex> g(h->mutex);
    const int rc = retune(h, [&](TableSlot &s) {
        for (int c = 0; c < h->cshape.C; ++c) {
            const double f_c = sample_rate_hz * channel_offset(h->cshape, c);
            const double lambda = 299792458.0 / (centre_frequency_hz + f_c);
            if (const int rb = build_table(h, s.tabs[c], positions_xy, lambda, h->streams[0])) return rb;
        }
        s.shared = false;
        if (!coherent(h)) return MUSIC_B200_OK;
        if (const int rb = build_manifold(h, s, s.tabs[h->cshape.C / 2])) return rb;
        return build_focusing(h, s, h->streams[0]);
    });
    if (rc == MUSIC_B200_OK) h->chan_fs = sample_rate_hz;
    return rc;
}

int music_b200_channel_frequencies(music_b200 *h, double *offsets_hz)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->chan) return fail(h, MUSIC_B200_EINVAL, "channel_frequencies needs a handle from music_b200_create_channels");
    if (!offsets_hz) return fail(h, MUSIC_B200_EINVAL, "offsets_hz must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    if (h->chan_fs == 0.0) return fail(h, MUSIC_B200_EINVAL, "no sample rate yet: call music_b200_set_geometry_channels()");
    for (int c = 0; c < h->cshape.C; ++c) offsets_hz[c] = h->chan_fs * channel_offset(h->cshape, c);
    return MUSIC_B200_OK;
}

int music_b200_get_table_channel(music_b200 *h, uint32_t channel, float *table_c64)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->chan) return fail(h, MUSIC_B200_EINVAL, "get_table_channel needs a handle from music_b200_create_channels");
    if (!table_c64) return fail(h, MUSIC_B200_EINVAL, "output table must not be NULL");
    if (channel >= (uint32_t)h->cshape.C) return fail(h, MUSIC_B200_EINVAL, "channel %u out of range (0..%d)", channel, h->cshape.C - 1);
    std::lock_guard<std::mutex> g(h->mutex);
    if (!has_table(h)) return fail(h, MUSIC_B200_EINVAL, "no array response yet: call music_b200_set_geometry_channels() or music_b200_set_table()");
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaMemcpy(table_c64, table(h, (int)channel).c64, (size_t)h->K * h->m * 2 * sizeof(float), cudaMemcpyDeviceToHost));
    return MUSIC_B200_OK;
}

int music_b200_set_focusing(music_b200 *h, uint32_t first_bin, uint32_t bin_count)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!coherent(h)) return fail(h, MUSIC_B200_EINVAL, "set_focusing needs a channel handle with the COHERENT combine");
    if (bin_count == 0 || bin_count > h->K || first_bin >= h->K)
        return fail(h, MUSIC_B200_EINVAL, "need 1 <= bin_count <= resolution and first_bin < resolution (got first=%u, count=%u)", first_bin,
                    bin_count);
    std::lock_guard<std::mutex> g(h->mutex);
    const uint32_t first0 = h->foc_first, count0 = h->foc_count;
    h->foc_first = first_bin;
    h->foc_count = bin_count;
    if (!has_table(h)) return MUSIC_B200_OK;  // the next set_geometry_channels() focuses on this sector
    // a retune to the current slot's channel tables with new matrices
    const TableSlot &cur = cur_slot(h);
    const int rc = retune(h, [&](TableSlot &s) {
        CU(h, cudaMemcpy(s.c64, cur.c64, cur.c64.size() * sizeof(float), cudaMemcpyDeviceToDevice));
        CU(h, cudaMemcpy(s.soa, cur.soa, cur.soa.size() * sizeof(double), cudaMemcpyDeviceToDevice));
        if (cur.mf_beta.size()) {
            CU(h, s.mf_beta.grow(cur.mf_beta.size()));
            CU(h, cudaMemcpy(s.mf_beta, cur.mf_beta, cur.mf_beta.size() * sizeof(double2), cudaMemcpyDeviceToDevice));
        }
        for (size_t c = 0; c < s.tabs.size(); ++c) {
            DeviceTable t = cur.tabs[c];  // geometry, ULA test and flags; the slot's own buffers
            t.c64 = s.tabs[c].c64;
            t.soa = s.tabs[c].soa;
            if (t.mf_beta) t.mf_beta = s.mf_beta;
            s.tabs[c] = t;
        }
        s.shared = false;
        return build_focusing(h, s, h->streams[0]);
    });
    if (rc) {
        h->foc_first = first0;
        h->foc_count = count0;
    }
    return rc;
}

int music_b200_get_focusing(music_b200 *h, double *T, double *err)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!coherent(h)) return fail(h, MUSIC_B200_EINVAL, "get_focusing needs a channel handle with the COHERENT combine");
    std::lock_guard<std::mutex> g(h->mutex);
    if (!has_table(h)) return fail(h, MUSIC_B200_EINVAL, "no focusing yet: call music_b200_set_geometry_channels()");
    CU(h, cudaSetDevice(h->device));
    const TableSlot &s = cur_slot(h);
    const size_t C = (size_t)h->cshape.C;
    if (T) CU(h, cudaMemcpy(T, s.foc_T, C * h->m * h->m * sizeof(double2), cudaMemcpyDeviceToHost));
    if (err)
        for (size_t c = 0; c < C; ++c) err[c] = s.foc_err[c];
    return MUSIC_B200_OK;
}

int music_b200_process_channels_device(music_b200 *h, const float *d_in_c64, uint32_t nwindows, float *d_angles, float *d_levels,
                                       float *d_spectrum, int32_t *d_bins, int32_t *d_counts, double *d_R, void *stream)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->chan) return fail(h, MUSIC_B200_EINVAL, "process_channels_device needs a handle from music_b200_create_channels");
    std::lock_guard<std::mutex> g(h->mutex);
    NvtxRange range("music_b200_process_channels_device");
    CU(h, cudaSetDevice(h->device));
    Outputs o = caller_outputs(d_angles, d_levels, d_spectrum, d_bins);
    o.counts = d_counts;
    return enqueue_channels(h, d_in_c64, nwindows, o.shaped(h), d_R, static_cast<cudaStream_t>(stream));
}

int music_b200_process_channels_host(music_b200 *h, const float *in_c64, uint32_t nwindows, float *angles, float *levels, float *spectrum,
                                     int32_t *bins, int32_t *counts, double *R)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->chan) return fail(h, MUSIC_B200_EINVAL, "process_channels_host needs a handle from music_b200_create_channels");
    if (nwindows == 0) return MUSIC_B200_OK;
    if (!in_c64 || !angles) return fail(h, MUSIC_B200_EINVAL, "in_c64 and angles must not be NULL");
    std::lock_guard<std::mutex> g(h->mutex);
    NvtxRange range("music_b200_process_channels_host");
    CU(h, cudaSetDevice(h->device));
    // Chunks of windows through one device arena on the handle's first stream: the input, then each output in the
    // chunk's own channel-major layout [rows][chunk], copied into the caller's [rows][nwindows] arrays row by row.
    const size_t C = (size_t)h->cshape.C, rows = h->chan_combine == MUSIC_B200_CHANNELS_SEPARATE ? C : 1;
    const size_t r_rows = coherent(h) ? 1 : C;  // R: the focused covariance of each window, or every channel's
    const size_t n = h->n, K = h->K, mm2 = (size_t)h->m * h->m * 2, win_bytes = (size_t)h->nsamples * 2 * sizeof(float);
    struct Piece { void *host; size_t nrows, row_bytes; bool want; size_t off; };  // row_bytes: of one window
    Piece pc[6] = {{angles, rows, n * sizeof(float), true, 0},      {levels, rows, n * sizeof(float), levels != nullptr, 0},
                   {bins, rows, n * sizeof(int32_t), bins != nullptr, 0}, {counts, rows, sizeof(int32_t), counts != nullptr, 0},
                   {spectrum, rows, K * sizeof(float), spectrum != nullptr, 0}, {R, r_rows, mm2 * sizeof(double), R != nullptr, 0}};
    size_t per_win = win_bytes;
    for (const Piece &p : pc) per_win += p.want ? p.nrows * p.row_bytes : 0;
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>(nwindows, ((size_t)64 << 20) / per_win));
    const auto align = [](size_t b) { return (b + 255) / 256 * 256; };
    size_t need = align((size_t)chunk * win_bytes);
    for (Piece &p : pc) {
        p.off = need;
        if (p.want) need += align(p.nrows * p.row_bytes * chunk);
    }
    if (need > h->chan_arena.size()) {
        CU(h, cudaDeviceSynchronize());
        CU(h, h->chan_arena.grow(need));
    }
    cudaStream_t st = h->streams[0];
    int rc = MUSIC_B200_OK;
    for (uint32_t w0 = 0; w0 < nwindows && rc == MUSIC_B200_OK; w0 += chunk) {
        const uint32_t W = std::min(chunk, nwindows - w0);
        float *d_in = reinterpret_cast<float *>(h->chan_arena.get());
        CU_BREAK(h, rc, cudaMemcpyAsync(d_in, in_c64 + (size_t)w0 * h->nsamples * 2, (size_t)W * win_bytes, cudaMemcpyHostToDevice, st));
        const auto dev = [&](int i) { return pc[i].want ? h->chan_arena + pc[i].off : nullptr; };
        Outputs o = caller_outputs(reinterpret_cast<float *>(dev(0)), reinterpret_cast<float *>(dev(1)), reinterpret_cast<float *>(dev(4)),
                                   reinterpret_cast<int32_t *>(dev(2)));
        o.counts = reinterpret_cast<int32_t *>(dev(3));
        rc = enqueue_channels(h, d_in, W, o.shaped(h), reinterpret_cast<double *>(dev(5)), st);
        if (rc) break;
        for (int i = 0; i < 6 && rc == MUSIC_B200_OK; ++i) {
            const Piece &p = pc[i];
            if (!p.want) continue;
            CU_BREAK(h, rc, cudaMemcpy2DAsync(static_cast<char *>(p.host) + (size_t)w0 * p.row_bytes, (size_t)nwindows * p.row_bytes, dev(i),
                                              (size_t)W * p.row_bytes, (size_t)W * p.row_bytes, p.nrows, cudaMemcpyDeviceToHost, st));
        }
        if (rc) break;
        CU_BREAK(h, rc, cudaStreamSynchronize(st));  // the arena is free for the next chunk
    }
    const cudaError_t e = cudaStreamSynchronize(st);
    if (rc == MUSIC_B200_OK && e != cudaSuccess) rc = fail(h, MUSIC_B200_ECUDA, "stream sync failed: %s", cudaGetErrorString(e));
    return rc;
}

/* ---- sparse linear arrays through the difference co-array (music_coarray.cuh) ---- */
namespace {

// the step vector and wavelength of a co-array handle: finite, wavelength > 0, 0 < |s| <= (wavelength / 2)(1 + 1e-12)
int check_coarray_step(music_b200 *h, const double *step_xy, double wavelength)
{
    if (!step_xy) return fail(h, MUSIC_B200_EINVAL, "step_xy must not be NULL");
    if (!(wavelength > 0.0) || !std::isfinite(wavelength)) return fail(h, MUSIC_B200_EINVAL, "wavelength must be positive and finite");
    if (!std::isfinite(step_xy[0]) || !std::isfinite(step_xy[1])) return fail(h, MUSIC_B200_EINVAL, "the step must be finite");
    const double s = std::hypot(step_xy[0], step_xy[1]);
    if (!(s > 0.0) || s > 0.5 * wavelength * (1.0 + 1e-12))
        return fail(h, MUSIC_B200_EINVAL, "need 0 < |step| <= wavelength / 2 (got |step| = %g, wavelength = %g)", s, wavelength);
    return MUSIC_B200_OK;
}

// the virtual ULA: element l at l s, l < mv
void coarray_positions(const double *step_xy, uint32_t mv, double *pos)
{
    for (uint32_t l = 0; l < mv; ++l) {
        pos[2 * l] = (double)l * step_xy[0];
        pos[2 * l + 1] = (double)l * step_xy[1];
    }
}

}  // namespace

int music_b200_create_coarray(music_b200 **out, uint32_t m, uint32_t n, uint32_t nsamples, uint32_t resolution, const int32_t *positions,
                              const double step_xy[2], double wavelength, uint32_t mv, int device)
{
    if (!out) return fail(nullptr, MUSIC_B200_EINVAL, "out must not be NULL");
    *out = nullptr;
    if (m < 2 || m > MUSIC_B200_MAX_M) return fail(nullptr, MUSIC_B200_EINVAL, "a co-array handle needs 2 <= m <= %d (got %u)", MUSIC_B200_MAX_M, m);
    if (!positions) return fail(nullptr, MUSIC_B200_EINVAL, "positions must not be NULL");
    if (positions[0] != 0) return fail(nullptr, MUSIC_B200_EINVAL, "positions must start at p_0 = 0 (got %d)", positions[0]);
    for (uint32_t i = 1; i < m; ++i)
        if (positions[i] <= positions[i - 1]) return fail(nullptr, MUSIC_B200_EINVAL, "positions must be strictly ascending (p_%u = %d)", i, positions[i]);
    if (nsamples == 0 || nsamples % m != 0) return fail(nullptr, MUSIC_B200_EINVAL, "nsamples must be a positive multiple of m (got %u)", nsamples);
    if (resolution == 0) return fail(nullptr, MUSIC_B200_EINVAL, "resolution must be > 0");
    if (const int rc = check_coarray_step(nullptr, step_xy, wavelength)) return rc;
    // the hole-free extent U, counted up to MAXM + 1: only min(U, MAXM) matters
    bool has[MAXM + 1] = {};
    for (uint32_t i = 0; i < m; ++i)
        for (uint32_t j = 0; j <= i; ++j) {
            const long long d = (long long)positions[i] - positions[j];
            if (d <= MAXM) has[d] = true;
        }
    uint32_t U = 0;
    while (U <= (uint32_t)MAXM && has[U]) ++U;
    const uint32_t cap = std::min<uint32_t>(U, MAXM);
    if (mv == 0) mv = cap;
    if (mv < 2 || mv > cap)
        return fail(nullptr, MUSIC_B200_EINVAL, "need 2 <= mv <= min(U, %d) = %u, U the hole-free extent of the lags (got mv = %u)", MAXM, cap, mv);
    if (n == 0 || n >= mv) return fail(nullptr, MUSIC_B200_EINVAL, "need 1 <= n < mv (got n=%u, mv=%u)", n, mv);
    CoarrayDef co = {};
    co.m_in = m;
    co.lambda = wavelength;
    co.lags.mv = (int)mv;
    int q = 0;
    for (uint32_t l = 0; l < mv; ++l) {
        co.lags.start[l] = (unsigned char)q;
        for (uint32_t i = 0; i < m; ++i)
            for (uint32_t j = 0; j <= i; ++j)
                if ((long long)positions[i] - positions[j] == (long long)l) {
                    co.lags.pi[q] = (unsigned char)i;
                    co.lags.pj[q] = (unsigned char)j;
                    ++q;
                }
    }
    co.lags.start[mv] = (unsigned char)q;
    coarray_positions(step_xy, mv, co.pos);
    return create_on_device(out, mv, n, nsamples, resolution, nullptr, device, nullptr, nullptr, &co);
}

int music_b200_set_geometry_coarray(music_b200 *h, const double step_xy[2], double wavelength)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->coarray) return fail(h, MUSIC_B200_EINVAL, "set_geometry_coarray needs a handle from music_b200_create_coarray");
    if (const int rc = check_coarray_step(h, step_xy, wavelength)) return rc;
    double pos[2 * MAXM];
    coarray_positions(step_xy, h->m, pos);
    std::lock_guard<std::mutex> g(h->mutex);
    return retune(h, [&](TableSlot &s) { return build_table(h, s.tabs[0], pos, wavelength, h->streams[0]); });
}

int music_b200_coarray_size(music_b200 *h, uint32_t *mv)
{
    if (!h) return MUSIC_B200_EINVAL;
    if (!h->coarray) return fail(h, MUSIC_B200_EINVAL, "coarray_size needs a handle from music_b200_create_coarray");
    if (!mv) return fail(h, MUSIC_B200_EINVAL, "mv must not be NULL");
    *mv = h->m;
    return MUSIC_B200_OK;
}

void music_b200_destroy(music_b200 *h)
{
    if (!h) return;
    for (music_b200 *c : h->kids) music_b200_destroy(c);
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (const music_b200::HostReg &r : h->hostregs) cudaHostUnregister(reinterpret_cast<void *>(r.base));
    for (void *p : h->ipc_maps) cudaIpcCloseMemHandle(p);
    cudaGetLastError();
    delete h;  // the streams, events and buffers with it, on the device made current above
}

}  // extern "C"
