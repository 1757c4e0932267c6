// host.cu -- host side of the C ABI declared in include/rnnoise.h: table construction, model upload,
// the batch handle that owns the per-stream device state, and the per-frame launch sequence
//   hp_filter -> pitch -> analysis -> rnn -> synthesis
// which together are DenoiseState::process_frame (src/denoise.rs:95-116) for n_streams streams.
#include <array>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <algorithm>
#include <type_traits>
#include <utility>
#include <variant>
#include <vector>

#include "../../include/rnnoise.h"
#include "abi.hpp"
#include "common.cuh"
#include "model.hpp"
#include "owners.hpp"

using namespace nnb;

struct RNNModel {
    HostModel m;
};

namespace {

thread_local std::string g_err;
std::atomic<unsigned long long> g_launches{0};

}  // namespace

// ---- the conventions of every C-ABI entry point (abi.hpp) ---------------------------------------------------------
namespace nnb {

int fail(const std::string& what, cudaError_t e) {
    g_err = what;
    if (e != cudaSuccess) {
        g_err += ": ";
        g_err += cudaGetErrorString(e);
    }
    return -1;
}

void count_launches(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

int open_device(int device, int* chosen) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return fail("no CUDA device available (this library has no CPU fallback)", e);
    if (device < 0) CK(cudaGetDevice(&device));
    if (device >= ndev) return fail("device index out of range");
    *chosen = device;
    return 0;
}

int check_streams(int total, const int* streams, int n, const char* holder) {
    if (n < 0) return fail("negative number of streams");
    if (!streams) return n <= total ? 0 : fail(std::string("more streams than the ") + holder + " holds");
    std::vector<char> seen((size_t)total, 0);
    for (int i = 0; i < n; i++) {
        const int s = streams[i];
        if (s < 0 || s >= total) return fail("stream index " + std::to_string(s) + " out of range");
        if (seen[(size_t)s]) return fail("stream index " + std::to_string(s) + " given twice");
        seen[(size_t)s] = 1;
    }
    return 0;
}

int wait_for_caller(cudaStream_t s, cudaStream_t us, cudaEvent_t ev) {
    if (!us) return 0;
    CK(cudaEventRecord(ev, us));
    CK(cudaStreamWaitEvent(s, ev, 0));
    return 0;
}

int resume_caller(cudaStream_t s, cudaStream_t us, cudaEvent_t ev) {
    if (!us) {
        CK(cudaStreamSynchronize(s));
        return 0;
    }
    CK(cudaEventRecord(ev, s));
    CK(cudaStreamWaitEvent(us, ev, 0));
    return 0;
}

}  // namespace nnb

namespace nnb {

// ---- tables (src/lib.rs:99-136) -------------------------------------------------
const int kEband5ms[NB_BANDS] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 34, 40, 48, 60, 78, 100};

void build_tables(DeviceTables* t) {
    std::memset(t, 0, sizeof(*t));
    const double pi = 3.14159265358979323846264338327950288;
    for (int i = 0; i < FRAME_SIZE; i++) {
        double s = std::sin(0.5 * pi * ((double)i + 0.5) / (double)FRAME_SIZE);
        float w = (float)std::sin(0.5 * pi * s * s);
        t->window[i] = w;
        t->window[WINDOW_SIZE - i - 1] = w;
    }
    for (int i = 0; i < FRAME_SIZE; i++) t->ramp[i] = (float)(i + 1) / 480.0f;
    volatile float acc = 0.0f;  // f32 sequential sum (src/lib.rs:116)
    for (int i = 0; i < WINDOW_SIZE; i++) acc = acc + t->window[i] * t->window[i];
    t->wnorm = 1.0f / acc;
    for (int i = 0; i < NB_BANDS; i++)
        for (int j = 0; j < NB_BANDS; j++) {
            float v = (float)std::cos(((double)i + 0.5) * (double)j * pi / (double)NB_BANDS);
            if (j == 0) v *= std::sqrt(0.5f);
            t->dct[i * NB_BANDS + j] = v;
        }
    for (int k = 0; k <= 480; k++)
        t->tw960[k] = make_float2((float)std::cos(-2.0 * pi * (double)k / 960.0), (float)std::sin(-2.0 * pi * (double)k / 960.0));
    for (int i = 0; i < NB_BANDS; i++) t->band_start[i] = kEband5ms[i] << 2;
    for (int i = 0; i < NB_BANDS - 1; i++) {
        int band_size = (kEband5ms[i + 1] - kEband5ms[i]) << 2;
        for (int j = 0; j < band_size; j++) {
            int idx = (kEband5ms[i] << 2) + j;
            t->band_frac[idx] = (float)j / (float)band_size;
            t->band_of[idx] = i;
        }
    }
    // tables of the warp-per-stream spectral kernels
    for (int k1 = 0; k1 < 15; k1++)
        for (int b = 0; b < 32; b++) {
            const double ang = -2.0 * pi * (double)(b * k1) / 480.0;
            t->twl[k1][b] = make_float2((float)std::cos(ang), (float)std::sin(ang));
        }
    {
        int l = 0;
        for (int sgi = 0; sgi < NB_BANDS - 1; sgi++) {
            const int first = t->band_start[sgi], size = t->band_start[sgi + 1] - first;
            const int nl = size <= 16 ? 1 : (size <= 32 ? 2 : (size <= 48 ? 3 : 4));
            for (int q = 0; q < nl; q++) {
                const int lo = first + (int)((long)size * q / nl), hi = first + (int)((long)size * (q + 1) / nl);
                if (l >= 32 || hi - lo > BP_MAXBINS) {
                    fprintf(stderr, "nnnoiseless_b200: band partition broken\n");
                    abort();
                }
                // rotations found by a local search over the 64-bit shared-memory bank model (22 walk steps x 2 half-warps:
                // 48 wavefronts instead of 188 without rotation; 38 is the floor)
                static const int kRot[32] = {2, 1, 0, 0, 3, 0, 1, 0, 6, 5, 4, 0, 1, 6, 3, 0, 9, 2, 0, 12, 2, 1, 15, 3, 15, 3, 2, 2, 21, 19, 12, 4};
                t->bp_seg[l] = (int16_t)sgi;
                t->bp_b0[l] = (int16_t)lo;
                t->bp_n[l] = (int16_t)(hi - lo);
                t->bp_rot[l] = (int16_t)(kRot[l] % (hi - lo));
                t->bp_off[l] = (int16_t)(lo - first);
                t->bp_inv[l] = 1.0f / (float)size;
                l++;
            }
        }
        if (l != 32) {
            fprintf(stderr, "nnnoiseless_b200: band partition uses %d lanes\n", l);
            abort();
        }
    }
}

}  // namespace nnb

// ---- the batch handle -----------------------------------------------------------------------------------
constexpr int kNumKernels = 5;
const char* const kKernelNames[kNumKernels] = {"hp_filter", "pitch", "analysis", "rnn", "synthesis"};
constexpr int kEvRing = 16;  // events are recycled after 16 frames (PIPE_DEPTH << 16)

// Which model each row of a frame runs on (DESIGN.md 7c): one model for all rows, or rows grouped by model into tiles.
struct ModelRoute {
    int uniform = 0;                  // the model of every row, or -1: several models, see the tile table
    std::vector<int> h_rows;          // host images of the two tables
    std::vector<ModelTile> h_tiles;
    DeviceMem rows, tiles;            // device tables (ModelTiles)
};
using StateMem = std::array<DeviceMem, 11>;  // owners of the eleven persistent fields of a BatchBuffers (each_state_field)
struct LinkGroup {                            // a group of linked streams (rnnoise_batch_link_streams)
    int mode;                                 // RNNOISE_LINK_MAX or RNNOISE_LINK_MEAN
    std::vector<int> members;                 // ascending
};

struct RNNoiseBatch {
    int device = 0;
    int n_streams = 0;
    // Frame pipeline: stage i of every frame runs on st[i], so K_i(f) -> K_i(f+1) is stream order; K_{i-1}(f) ->
    // K_i(f) and the back-pressure K_4(f - PIPE_DEPTH) -> K_0(f) are events.  At small batches one kernel cannot
    // fill 132 SMs; overlapping the five stages of up to four consecutive frames does.
    Stream st[kNumKernels];
    int n_stages = kNumKernels;  // stages per frame: the denoise path's five, or a trainer's four (its last stage ends a frame)
    Stream c_in, c_out;          // host-API copy streams
    Event ev[kNumKernels][kEvRing];
    Event ev_in[kEvRing], ev_call;
    BatchBuffers buf{};  // persistent state + set 0 of the intermediates
    StateMem state_mem;  // owners of buf's persistent state
    std::vector<DeviceMem> fixed;  // owners of buf's intermediates, d_tab, pitch_stats and d_first_bad
    DeviceTables* d_tab = nullptr;
    int pitch_exact = 0;  // NNB_PITCH_EXACT=1: every stream takes the pitch kernel's order-exact recomputation paths (2: coarse only, 3: ladder only)
    // Two frame counters; without subset calls they are equal.
    unsigned long long seq = 0;    // frames issued, full-batch or subset: intermediate set seq % PIPE_DEPTH, event ring, back-pressure
    unsigned long long phase = 0;  // full-batch frames: ring slot phase % HIST_SLOTS of the batch's own streams
    bool taps_subset = false;      // the most recent frame was a subset frame: its intermediates do not describe the batch's rows
    // Split frames (rnnoise_batch_analyze_device / _synthesize_device): frames seq - pending .. seq - 1 are analyzed and
    // not yet synthesized.  Their intermediates stay in their sets, so pending <= PIPE_DEPTH.
    int pending = 0;
    // Window frames (rnnoise_batch_analyze_window_device / _synthesize_window_device): frames seq - window .. seq - 1 are
    // analyzed and not yet synthesized.  Their spectra are in the caller's context records, so `window` has no bound;
    // window and pending are never both > 0.
    int window = 0;
    bool taps_split = false;       // the most recent frame was a split frame: its features and gains are the caller's
    int tail_stage = 0, tail_e = 0;  // stage and event-ring index of the stage issue_frame issued last
    // host-call staging: kStageSlots frames of device memory, recycled while a call of any length streams through
    // (sized for the sample type in use only: float or int16)
    DeviceMem stage_in, stage_out, stage_vad;
    Event ev_out[8];  // D2H copy of the frame that last used staging slot k
    int slot_ev[8];   // event-ring index of the frame that last used staging slot k
    // per-stream state records (state.cu): the gather / scatter kernels run on st[0], ahead of the next frame's stage 0
    HostModel model;                        // the batch's model, for rnnoise_clone; its GRU widths fix the record format
    DeviceMem idx;                          // stream indices of the most recent state call
    DeviceMem rec_stage;                    // records of host-memory calls
    int* d_first_bad = nullptr;             // validation of device-resident records
    Event ev_state;                         // end of the most recent state call on st[0]
    // subset calls (rnnoise_batch_process_streams_*): the listed streams' persistent state is gathered into rows 0..n-1 of
    // the work state, advanced there by the unchanged frame kernels, and scattered back
    BatchBuffers work{};                    // persistent buffers only (intermediates: the batch's own sets); n_streams = rows in use
    StateMem work_mem;                      // owners of work's buffers, grown to the high-water n
    unsigned long long work_frames = 0;     // frames of the current subset call issued so far: work ring slot (phase + work_frames) % 8
    // model table (rnnoise_batch_add_model; DESIGN.md 7c): models of the batch model's geometry, model 0 = `model`.  Their
    // images for the batch's GRU kernel lie `mtab_stride` bytes apart in mtab, and all of them share model 0's descriptor.
    std::vector<int> model_acts;            // activation codes of each model, packed as ModelTile::acts
    DeviceMem mtab;
    size_t mtab_bytes = 0;                  // bytes of each image
    size_t mtab_stride = 0;                 // mtab_bytes rounded up to 256
    // The GRU kernel, chosen at creation: wgmma when model 0 fits its budget, else (or with NNB_RNN_MMA=1) mma.sync.
    // Model 0's descriptor for it, in offset form.
    std::variant<DeviceModelTc, DeviceModelMma> gru0;
    std::vector<int> stream_model;          // host mirror: the model of every stream
    ModelRoute route;                       // full-batch frames
    ModelRoute work_route;                  // frames of the current subset call (rows = work rows)
    // stream controls (rnnoise_batch_set_stream_controls; DESIGN.md 7m): host mirror of every stream's parameters (the
    // gate state lives on the device only, in buf.gate).  A stream is live from a set of anything but the defaults
    // until its parameters are the defaults and a reset or set has zeroed its gate state; frames take the synthesis
    // kernel with controls only while some stream is live.
    std::vector<RNNoiseStreamControls> stream_ctl;
    std::vector<char> ctl_live;
    int n_ctl_live = 0;
    // stream links (rnnoise_batch_link_streams; DESIGN.md 7n): every group by its lowest member, and for every stream its
    // group's lowest member (itself when unlinked) and mode (0 when unlinked).  Full-batch fused frames take the linked
    // synthesis kernel with link_tab (the batch's LinkTable, common.cuh) while some group exists; a link call marks it
    // stale, and the next full-batch fused frame rebuilds and uploads it first.  A subset call takes work_link, its work
    // rows' table, while it lists some linked stream.  Neither table is stream state: gather, scatter and reset leave
    // them alone.
    std::map<int, LinkGroup> groups;
    std::vector<int> link_group, link_mode;
    bool links_stale = false;
    DeviceMem link_tab, work_link;
    std::vector<int> h_link, h_work_link;  // the tables' host images: the copies' sources stay alive until the next upload
    bool work_linked = false;
};
constexpr int kStageSlots = 8;  // >= PIPE_DEPTH frames in the kernels + frames in the two copy engines

// used by resample_stream.cu
namespace nnb {
int batch_device(const RNNoiseBatch* b) { return b->device; }
int batch_check_no_pending(const RNNoiseBatch* b);
int batch_check_whole_groups(const RNNoiseBatch* b, const int* streams, int n);
}  // namespace nnb

namespace {

int model_acts(const HostModel& m) {
    const int a[6] = {m.input_dense.act, m.vad_gru.act, m.noise_gru.act, m.denoise_gru.act, m.denoise_output.act, m.vad_output.act};
    int acts = 0;
    for (int i = 0; i < 6; i++) acts |= a[i] << (4 * i);
    return acts;
}

// The eleven persistent per-stream fields of BatchBuffers: f(member, elements per stream, reset).  gru_state takes the
// state size, at least one element, so a model without GRU neurons still has a state array.  reset is false for the
// stream controls' parameters, which a reset keeps (all zero when allocated: the defaults).
template <typename F>
void each_state_field(const RNNoiseBatch* b, F f) {
    f(&BatchBuffers::hist, HIST_CAP, true);
    f(&BatchBuffers::hp_mem, 2, true);
    f(&BatchBuffers::synth_mem, FRAME_SIZE, true);
    f(&BatchBuffers::ceps_mem, CEPS_MEM * NB_BANDS, true);
    f(&BatchBuffers::ceps_id, 1, true);
    f(&BatchBuffers::last_period, 1, true);
    f(&BatchBuffers::last_gain, 1, true);
    f(&BatchBuffers::gru_state, std::max(b->model.state_size(), 1), true);
    f(&BatchBuffers::lastg, NB_BANDS, true);
    f(&BatchBuffers::ctl, 1, false);
    f(&BatchBuffers::gate, 1, true);
}

// The ten per-frame intermediates of BatchBuffers: f(member, elements per stream) of one of the PIPE_DEPTH sets.
template <typename F>
void each_frame_field(F f) {
    f(&BatchBuffers::X, FREQ_SIZE);
    f(&BatchBuffers::P, NB_BINS_BANDED);
    f(&BatchBuffers::ex, NB_BANDS);
    f(&BatchBuffers::ep, NB_BANDS);
    f(&BatchBuffers::exp, NB_BANDS);
    f(&BatchBuffers::features, NB_FEATURES);
    f(&BatchBuffers::silence, 1);
    f(&BatchBuffers::pitch, 1);
    f(&BatchBuffers::gains, NB_BANDS);
    f(&BatchBuffers::vad, 1);
}

// intermediates of frame f live in set f % PIPE_DEPTH
BatchBuffers view(const RNNoiseBatch* b, unsigned long long f) {
    BatchBuffers v = b->buf;
    const size_t k = (size_t)(f % PIPE_DEPTH), B = (size_t)b->n_streams;
    each_frame_field([&](auto m, size_t per) { v.*m += k * B * per; });
    return v;
}

// a frame of a subset call: intermediates of set f % PIPE_DEPTH (rows 0..n-1), persistent state of the work rows
BatchBuffers work_view(const RNNoiseBatch* b, unsigned long long f) {
    BatchBuffers v = view(b, f);
    v.n_streams = b->work.n_streams;
    each_state_field(b, [&](auto m, size_t, bool) { v.*m = b->work.*m; });
    return v;
}

int sync_all(RNNoiseBatch* b) {
    for (int i = 0; i < kNumKernels; i++) CK(cudaStreamSynchronize(b->st[i]));
    CK(cudaStreamSynchronize(b->c_in));
    CK(cudaStreamSynchronize(b->c_out));
    return 0;
}

// The one growth rule of the buffers a batch reuses from call to call: nothing if m holds `bytes` already; else, once
// nothing in flight can read it, the old allocation is freed before the new one is made, so peak memory stays at the
// larger of the two.
int grow(RNNoiseBatch* b, DeviceMem* m, size_t bytes) {
    if (m->bytes() >= bytes) return 0;
    if (sync_all(b)) return -1;
    m->reset();
    CK(m->alloc(bytes));
    return 0;
}

// The persistent fields of `rows` streams in *u, owned by *mem: each field grows to its size and is zeroed when it is
// allocated.  Rows and ring positions the frame kernels never read are then defined.
int grow_state(RNNoiseBatch* b, BatchBuffers* u, StateMem* mem, size_t rows) {
    int i = 0, rc = 0;
    each_state_field(b, [&](auto m, size_t per, bool) {
        using T = std::remove_pointer_t<std::remove_reference_t<decltype(u->*m)>>;
        DeviceMem& d = (*mem)[i++];
        const size_t bytes = rows * per * sizeof(T);
        if (rc == 0 && d.bytes() < bytes) {
            rc = grow(b, &d, bytes);
            const cudaError_t e = rc ? cudaSuccess : cudaMemsetAsync(d.get(), 0, bytes, b->st[0]);
            if (e != cudaSuccess) rc = fail("zeroing the stream state", e);
        }
        u->*m = d.get<T>();
    });
    return rc;
}

bool default_controls(const RNNoiseStreamControls& c) {
    return std::isinf(c.atten_lim_db) && c.atten_lim_db > 0 && c.gate_threshold == 0.0f && c.gate_closed_gain == 0.0f &&
           c.gate_hold_frames == 0 && c.gate_hold_left == 0 && c.gate_closed == 0;
}

void set_ctl_live(RNNoiseBatch* b, size_t s, bool live) {
    b->n_ctl_live += (int)live - (int)b->ctl_live[s];
    b->ctl_live[s] = live;
}

// after a reset of stream s: its gate state is zero, its parameters kept
void reset_ctl_live(RNNoiseBatch* b, size_t s) {
    RNNoiseStreamControls c = b->stream_ctl[s];
    c.gate_hold_left = c.gate_closed = 0;
    set_ctl_live(b, s, !default_controls(c));
}

int zero_state(RNNoiseBatch* b) {
    const size_t B = (size_t)b->n_streams, D = PIPE_DEPTH;
    BatchBuffers& u = b->buf;
    if (sync_all(b)) return -1;
    cudaStream_t s = b->st[0];
    cudaError_t e = cudaSuccess;
    auto zero = [&](auto* p, size_t count) { if (e == cudaSuccess) e = cudaMemsetAsync(p, 0, count * sizeof(*p), s); };
    each_state_field(b, [&](auto m, size_t per, bool reset) {
        if (reset) zero(u.*m, B * per);
    });
    zero(u.gains, D * B * NB_BANDS);
    zero(u.vad, D * B);
    zero(u.silence, D * B);
    zero(u.pitch, D * B);
    zero(u.features, D * B * NB_FEATURES);
    if (e != cudaSuccess) return fail("zeroing the stream state", e);
    b->seq = b->phase = 0;
    b->taps_subset = b->taps_split = false;
    b->pending = b->window = 0;
    for (size_t r = 0; r < B; r++) reset_ctl_live(b, r);
    CK(cudaStreamSynchronize(s));
    return 0;
}

// Picks the batch's GRU kernel and uploads model 0, packed for that kernel only, as entry 0 of the model table.  The
// table has room for one more model; its capacity doubles whenever rnnoise_batch_add_model finds it full.
int init_model_table(RNNoiseBatch* b, const HostModel& hm) {
    const char* e = getenv("NNB_RNN_MMA");
    std::vector<unsigned char> img;
    if ((e && e[0] == '1') || !pack_model(hm, &b->gru0.emplace<DeviceModelTc>(), &img)) pack_model(hm, &b->gru0.emplace<DeviceModelMma>(), &img);
    b->mtab_bytes = img.size();
    b->mtab_stride = (img.size() + 255) & ~(size_t)255;
    CK(b->mtab.alloc(b->mtab_stride * 2));
    CK(cudaMemcpyAsync(b->mtab.get(), img.data(), img.size(), cudaMemcpyHostToDevice, b->st[0]));
    CK(cudaStreamSynchronize(b->st[0]));
    return 0;
}

int batch_init(RNNoiseBatch* b, const HostModel& hm, int n_streams, int device) {
    if (open_device(device, &device)) return -1;
    if (n_streams <= 0) return fail("n_streams must be positive");
    CK(cudaSetDevice(device));
    b->device = device;
    b->n_streams = n_streams;
    for (int i = 0; i < kNumKernels; i++) CK(cudaStreamCreateWithFlags(b->st[i].put(), cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(b->c_in.put(), cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(b->c_out.put(), cudaStreamNonBlocking));
    for (int i = 0; i < kNumKernels; i++)
        for (int k = 0; k < kEvRing; k++) CK(cudaEventCreateWithFlags(b->ev[i][k].put(), cudaEventDisableTiming));
    for (int k = 0; k < kEvRing; k++) CK(cudaEventCreateWithFlags(b->ev_in[k].put(), cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(b->ev_call.put(), cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(b->ev_state.put(), cudaEventDisableTiming));
    for (int k = 0; k < kStageSlots; k++) CK(cudaEventCreateWithFlags(b->ev_out[k].put(), cudaEventDisableTiming));
    b->model = hm;
    b->model_acts.assign(1, model_acts(hm));
    b->stream_model.assign((size_t)n_streams, 0);
    b->stream_ctl.assign((size_t)n_streams, RNNoiseStreamControls{INFINITY, 0.0f, 0.0f, 0, 0, 0});
    b->ctl_live.assign((size_t)n_streams, 0);
    b->link_group.resize((size_t)n_streams);
    for (int i = 0; i < n_streams; i++) b->link_group[(size_t)i] = i;
    b->link_mode.assign((size_t)n_streams, 0);
    const size_t B = (size_t)n_streams, D = PIPE_DEPTH;
    BatchBuffers& u = b->buf;
    u.n_streams = n_streams;
    if (init_model_table(b, hm)) return -1;
    {
        const char* e3 = getenv("NNB_PITCH_EXACT");
        b->pitch_exact = !e3 ? 0 : (e3[0] == '1' ? 3 : (e3[0] == '2' ? 1 : (e3[0] == '3' ? 2 : 0)));
    }
    if (grow_state(b, &u, &b->state_mem, B)) return -1;
    cudaError_t ae = cudaSuccess;
    each_frame_field([&](auto m, size_t per) {
        if (ae == cudaSuccess) ae = dalloc(&b->fixed, &(u.*m), D * B * per);
    });
    if (ae != cudaSuccess) return fail("intermediates of " + std::to_string(n_streams) + " streams", ae);
    CK(dalloc(&b->fixed, &b->d_tab, 1));
    CK(dalloc(&b->fixed, &u.pitch_stats, 3));
    CK(dalloc(&b->fixed, &b->d_first_bad, 1));
    CK(cudaMemsetAsync(u.pitch_stats, 0, 3 * sizeof(unsigned long long), b->st[0]));
    const std::unique_ptr<DeviceTables> ht(new DeviceTables());
    build_tables(ht.get());
    cudaError_t ce = cudaMemcpyAsync(b->d_tab, ht.get(), sizeof(DeviceTables), cudaMemcpyHostToDevice, b->st[0]);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(b->st[0]);
    if (ce != cudaSuccess) return fail("table upload", ce);
    return zero_state(b);
}

// Deletes a batch once its streams that exist have finished: the destructors free what it owns, with its device
// selected.  Reports no error.
struct BatchRelease {
    void operator()(RNNoiseBatch* b) const {
        DeviceGuard guard(b->device);
        for (int i = 0; i < kNumKernels; i++)
            if (b->st[i]) cudaStreamSynchronize(b->st[i]);
        if (b->c_in) cudaStreamSynchronize(b->c_in);
        if (b->c_out) cudaStreamSynchronize(b->c_out);
        delete b;
    }
};
using BatchPtr = std::unique_ptr<RNNoiseBatch, BatchRelease>;

// A batch on `device` (< 0: the current device), which stays the caller's current device; null on an error.
BatchPtr create_batch(const HostModel& hm, int n_streams, int device) {
    BatchPtr b(new (std::nothrow) RNNoiseBatch());
    if (!b) {
        fail("out of memory");
        return nullptr;
    }
    int prev_dev = -1;
    cudaGetDevice(&prev_dev);  // batch_init selects the batch's device; the caller's current device is restored below
    const int rc = batch_init(b.get(), hm, n_streams, device);
    if (prev_dev >= 0) cudaSetDevice(prev_dev);
    if (rc != 0) b.reset();
    return b;
}

// host-call staging: kStageSlots frames of the sample type in use
int ensure_stage(RNNoiseBatch* b, bool pcm) {
    const size_t frames = (size_t)kStageSlots * b->n_streams, bytes = frames * FRAME_SIZE * (pcm ? sizeof(short) : sizeof(float));
    return grow(b, &b->stage_in, bytes) || grow(b, &b->stage_out, bytes) || grow(b, &b->stage_vad, frames * sizeof(float)) ? -1 : 0;
}

// One denoise frame's device I/O.  in/out are float samples or 16-bit PCM: fmt bit 0 = int16 input, bit 1 = int16 output
// (element strides either way).  vad: one value per row of the frame, may be NULL.
constexpr int kFmtF32 = 0, kFmtPcmIn = 1, kFmtPcmOut = 2, kFmtPcm = 3;
struct FrameIO {
    void* out;
    const void* in;
    int fmt;
    float* vad;
    long stream_stride, sample_stride;

    // frame t of a call whose frames lie frame_stride elements apart and have `rows` vad values each
    FrameIO at(int t, long frame_stride, int rows) const {
        const size_t esz_in = (fmt & kFmtPcmIn) ? sizeof(short) : sizeof(float), esz_out = (fmt & kFmtPcmOut) ? sizeof(short) : sizeof(float);
        return {(char*)out + (size_t)t * frame_stride * esz_out, (const char*)in + (size_t)t * frame_stride * esz_in, fmt,
                vad ? vad + (size_t)t * rows : nullptr, stream_stride, sample_stride};
    }
};

// the pcm16 argument of the strided and subset device calls, range-checked by the caller
int pcm16_fmt(int pcm16) {
    static const int to_fmt[4] = {kFmtF32, kFmtPcm, kFmtPcmOut, kFmtPcmIn};
    return to_fmt[pcm16];
}

// The five stages of a denoise frame: hp_filter -> pitch -> analysis -> rnn -> synthesis.
// The GRU stage of a frame: every row on model k (image k of the table, model k's activation codes), or the rows
// grouped by model over the route's tile table.
int launch_rnn(const RNNoiseBatch* b, const BatchBuffers& v, const ModelRoute& r, cudaStream_t s) {
    const size_t k = (size_t)std::max(r.uniform, 0);
    const unsigned char* img = b->mtab.get<unsigned char>() + k * b->mtab_stride;
    const ModelTiles mt{r.tiles.get<ModelTile>(), r.rows.get<int>(), (int)r.h_tiles.size(), (uint32_t)b->mtab_stride};
    const ModelTiles* tiles = r.uniform >= 0 ? nullptr : &mt;
    CK(std::visit([&](const auto& m0) { return launch_gru(v, m0, img, b->model_acts[k], tiles, s); }, b->gru0));
    return 0;
}

struct DenoiseStages {
    const RNNoiseBatch* b;
    FrameIO io;
    bool work = false;  // the frame advances a subset call's work rows
    // a split frame: the caller's features [B] (row stride feature_stride) and silence flags [B] (may be NULL), written by
    // analysis; the caller's raw gains, read by synthesis.  NULL: the frame's own set.
    float* features = nullptr;
    long feature_stride = 0;
    int* silence = nullptr;
    const float* gains = nullptr;
    long gain_stride = 0;
    // a saving split frame: stream s's context record at ctx + s * ctx_stride records, stored just before synthesis.  A
    // window frame (window): the record analysis writes the spectra to and synthesis reads them from.
    void* ctx = nullptr;
    long ctx_stride = 0;
    bool window = false;

    // the rows' link table for a fused frame's synthesis, or NULL: no row is linked (split and window frames ignore it)
    const int4* link() const {
        if (work) return b->work_linked ? b->work_link.get<int4>() : nullptr;
        return b->groups.empty() ? nullptr : b->link_tab.get<int4>();
    }

    int operator()(int i, const BatchBuffers& v, int slot, cudaStream_t s) const {
        switch (i) {
            case 0: CK(launch_hp_filter(v, io.in, (io.fmt & kFmtPcmIn) != 0, io.stream_stride, io.sample_stride, slot, s)); break;
            case 1: CK(launch_pitch(v, slot, b->pitch_exact, s)); break;
            case 2: CK(launch_analysis_warp(v, b->d_tab, slot, s, features, feature_stride, silence, window ? ctx : nullptr, ctx_stride)); break;
            case 3:
                if (launch_rnn(b, v, work ? b->work_route : b->route, s)) return -1;
                break;
            default:
                if (ctx && !window) {
                    CK(launch_synth_context(v, gains, gain_stride, ctx, ctx_stride, s));
                    count_launches(1);
                }
                CK(launch_synthesis_warp(v, b->d_tab, io.out, (io.fmt & kFmtPcmOut) != 0, io.stream_stride, io.sample_stride, io.vad, s,
                                         gains, gain_stride, window ? ctx : nullptr, ctx_stride, b->n_ctl_live > 0, link()));
                break;
        }
        return 0;
    }
};

// The stages [first, last) of one frame that one issue_frame issues (last < 0: through the batch's last stage).  first ==
// 0 starts a new frame; first > 0 resumes the oldest pending frame (window: the oldest owed window frame), after its
// stage `after`.
struct StageRange {
    int first = 0, last = -1, after = -1;
    bool window = false;
};
constexpr StageRange kFused{}, kAnalyze{0, 3, -1}, kSynthesize{4, 5, 2}, kAnalyzeWindow{0, 3, -1, true}, kSynthesizeWindow{4, 5, 2, true};

// Issues stages r.first .. r.last - 1 of one frame: launch(i, v, slot, s) launches stage i of the batch's n_stages on
// stream s, for the frame's buffers v and history ring slot.  Stage i runs on st[i], after the frame's previous stage i-1
// (r.after for the range's first stage; event ev[.][frame % kEvRing]).  A new frame's stage 0 runs after in_ready
// (optional) and after the last stage of frame seq - PIPE_DEPTH, whose intermediate set it reuses: with split frames
// pending, that frame's last stage has been issued because at most PIPE_DEPTH frames are pending.  The first fused or
// split frame after window frames waits the same way: every owed window frame has been synthesized by then, so stage 4
// of frame seq - PIPE_DEPTH has been issued and recorded.  A resumed frame's first stage runs after in_ready.
// A new window frame waits on stage 2 (analysis) of frame seq - PIPE_DEPTH instead, whose stage 4 may not be issued yet:
// the set of a window frame holds only what stages 0-2 use (its pitch; X, P, the band energies and the silence flag go
// to the caller's record, the features to the caller), and the history ring slot it overwrites was last read by the
// analysis of frame seq - PIPE_DEPTH - 1 at the latest, as with fused frames.  The synthesis of window frame f waits on
// ev[2][f % kEvRing]; with more than kEvRing frames owed that event has since been recorded again by the analysis of a
// later frame on the same stream, which follows frame f's analysis: the wait stays correct, only conservative.
// work_rows: the frame advances the work rows of a subset call, whose ring continues the batch's phase.
// one (optional): every stage runs on this stream instead.  The caller orders it after the batch's earlier work and later
// work after it; the ring events are recorded all the same.  tev (optional): timing events around the stages, tev[i]
// before stage i and tev[last] after the range.
template <typename Launch>
int issue_frame(RNNoiseBatch* b, const Launch& launch, bool work_rows, cudaEvent_t in_ready, cudaStream_t one = nullptr,
                const Event* tev = nullptr, StageRange r = kFused) {
    const int n = b->n_stages, last = r.last < 0 ? n : r.last;
    int& owed = r.window ? b->window : b->pending;
    const unsigned long long back = r.first > 0 ? (unsigned long long)owed : 0;  // a resumed frame: the oldest owed one
    const unsigned long long f = b->seq - back;
    const int e = (int)(f % kEvRing);
    const int slot = (int)(((work_rows ? b->phase + b->work_frames : b->phase) - back) % HIST_SLOTS);
    const BatchBuffers v = work_rows ? work_view(b, f) : view(b, f);
    auto S = [&](int i) { return one ? one : b->st[i]; };
    if (in_ready) CK(cudaStreamWaitEvent(S(r.first), in_ready, 0));
    if (r.first == 0 && f >= (unsigned long long)PIPE_DEPTH)
        CK(cudaStreamWaitEvent(S(0), b->ev[r.window ? 2 : n - 1][(int)((f - PIPE_DEPTH) % kEvRing)], 0));
    for (int i = r.first; i < last; i++) {
        const int prev = i > r.first ? i - 1 : r.after;
        if (!one && prev >= 0) CK(cudaStreamWaitEvent(S(i), b->ev[prev][e], 0));
        if (tev) CK(cudaEventRecord(tev[i], S(i)));
        if (launch(i, v, slot, S(i))) return -1;
        CK(cudaEventRecord(b->ev[i][e], S(i)));
    }
    if (tev) CK(cudaEventRecord(tev[last], S(last - 1)));
    g_launches.fetch_add((unsigned long long)(last - r.first), std::memory_order_relaxed);
    b->tail_stage = last - 1;
    b->tail_e = e;
    if (r.first > 0) {
        owed--;
        return 0;
    }
    b->seq++;
    if (work_rows) b->work_frames++;
    else b->phase++;
    b->taps_subset = work_rows;
    b->taps_split = last < n;
    if (last < n) owed++;
    return 0;
}

// Join: make `s` wait for everything issued so far on the stage streams.  Only called with no split or window frame owed:
// the last stage of the newest frame has then been issued and its event recorded.
int join_into(RNNoiseBatch* b, cudaStream_t s) {
    if (b->seq == 0) return 0;
    // the last stage follows every earlier kernel of its frame; earlier frames precede it in stream order per stage
    CK(cudaStreamWaitEvent(s, b->ev[b->n_stages - 1][(int)((b->seq - 1) % kEvRing)], 0));
    return 0;
}

// Calls that would run between a pending or owed frame's analysis and its synthesis are refused.
int check_no_pending(const RNNoiseBatch* b) {
    if (b->pending > 0)
        return fail(std::to_string(b->pending) + " split frame(s) pending: rnnoise_batch_synthesize_device finishes them first");
    if (b->window > 0)
        return fail(std::to_string(b->window) + " window frame(s) owed: rnnoise_batch_synthesize_window_device finishes them first");
    return 0;
}

// Split and window frames are never mixed.
int check_no_window(const RNNoiseBatch* b) {
    if (b->window == 0) return 0;
    return fail(std::to_string(b->window) + " window frame(s) owed: split frames wait until rnnoise_batch_synthesize_window_device "
                "finishes them");
}

}  // namespace

int nnb::batch_check_no_pending(const RNNoiseBatch* b) { return check_no_pending(b); }

namespace {

int subset_begin(RNNoiseBatch* b, const int* streams, int n, cudaStream_t us);
int subset_end(RNNoiseBatch* b, const int* streams, int n);
}  // namespace
int refresh_links(RNNoiseBatch* b);
int check_whole_groups(const RNNoiseBatch* b, const int* streams, int n);
namespace {

// A call of n_frames frames through device buffers; frame(t, in_ready) issues frame t.  The frames run after the work
// queued so far on the caller's stream `us`; then `us` continues behind them, or without a stream the call returns when
// they have finished.  subset: the listed streams are gathered into the work rows before the frames and scattered back
// after them.
template <typename Frame>
int device_call(RNNoiseBatch* b, cudaStream_t us, int n_frames, const Frame& frame, bool subset = false, const int* streams = nullptr,
                int n = 0) {
    cudaEvent_t ready = nullptr;
    if (subset) {
        if (subset_begin(b, streams, n, us)) return -1;
    } else if (us) {  // work queued on the caller's stream (e.g. the producer of `in`) must finish first
        CK(cudaEventRecord(b->ev_call, us));
        ready = b->ev_call;
    }
    for (int t = 0; t < n_frames; t++)
        if (frame(t, t == 0 ? ready : nullptr)) return -1;
    if (subset) return subset_end(b, streams, n) ? -1 : resume_caller(b->st[0], us, b->ev_state);
    // the stage issued last follows the call's earlier stages (events) and its stream's earlier kernels (stream order)
    if (us) CK(cudaStreamWaitEvent(us, b->ev[b->tail_stage][b->tail_e], 0));
    else CK(cudaStreamSynchronize(b->st[b->tail_stage]));
    return 0;
}

// copy(v, B) reads the intermediates v of the most recent full-batch frame of the batch's B streams, after every frame
// issued so far has finished.
template <typename Copy>
int read_taps(RNNoiseBatch* b, const Copy& copy) {
    if (!b) return fail("null batch");
    ON_DEVICE(b->device);
    if (check_no_pending(b)) return -1;
    if (b->taps_subset) return fail("the most recent frame was a subset frame: taps describe full-batch frames only");
    if (b->taps_split) return fail("the most recent frame was a split frame: taps describe fused full-batch frames only");
    if (sync_all(b)) return -1;
    return copy(view(b, b->seq ? b->seq - 1 : 0), (size_t)b->n_streams);
}

}  // namespace

// ============================================================================================== C ABI
extern "C" {

const char* rnnoise_last_error(void) { return g_err.c_str(); }
unsigned long long rnnoise_kernel_launches(void) { return g_launches.load(); }

RNNModel* rnnoise_model_from_bytes(const unsigned char* bytes, size_t len) {
    std::unique_ptr<RNNModel> m(new (std::nothrow) RNNModel());
    if (!m) return nullptr;
    if (!bytes || !HostModel::parse(bytes, len, &m->m)) {
        fail("model bytes rejected (src/rnn.rs:116-232 validation)");
        return nullptr;
    }
    return m.release();
}

RNNModel* rnnoise_model_from_text(const char* text, size_t len) {
    std::unique_ptr<RNNModel> m(new (std::nothrow) RNNModel());
    if (!m) return nullptr;
    if (!text || !HostModel::parse_text(text, len, &m->m)) {
        fail("text model rejected");
        return nullptr;
    }
    return m.release();
}

RNNModel* rnnoise_model_from_file(FILE* file) {
    if (!file) return nullptr;
    std::vector<unsigned char> data;
    unsigned char chunk[65536];
    size_t n;
    bool err = false;
    while ((n = fread(chunk, 1, sizeof chunk, file)) > 0) data.insert(data.end(), chunk, chunk + n);
    if (ferror(file)) err = true;
    fclose(file);  // the reference takes the FILE over and closes it (src/capi.rs:93-94)
    if (err) return nullptr;
    return rnnoise_model_from_bytes(data.data(), data.size());
}

void rnnoise_model_free(RNNModel* model) { delete model; }

size_t rnnoise_model_bytes(const RNNModel* model, unsigned char* buf, size_t cap) {
    const HostModel& m = model ? model->m : HostModel::builtin();
    if (buf && cap >= m.bytes.size()) std::memcpy(buf, m.bytes.data(), m.bytes.size());
    return m.bytes.size();
}

RNNoiseBatch* rnnoise_batch_create(const RNNModel* model, int n_streams, int device) {
    return create_batch(model ? model->m : HostModel::builtin(), n_streams, device).release();
}

void rnnoise_batch_destroy(RNNoiseBatch* b) {
    if (b) BatchRelease()(b);
}

int rnnoise_batch_streams(const RNNoiseBatch* b) { return b ? b->n_streams : 0; }

int rnnoise_batch_reset(RNNoiseBatch* b) {
    if (!b) return fail("null batch");
    ON_DEVICE(b->device);
    return zero_state(b);
}

static int process_device_impl(RNNoiseBatch* b, const FrameIO& io, int n_frames, long frame_stride, void* cuda_stream) {
    if (!b || !io.out || !io.in) return fail("null argument");
    if (check_no_pending(b)) return -1;
    if (io.sample_stride < 1) return fail("sample_stride must be >= 1");
    if (n_frames < 0) return fail("negative n_frames");
    if (n_frames == 0) return 0;
    ON_DEVICE(b->device);
    if (refresh_links(b)) return -1;
    return device_call(b, (cudaStream_t)cuda_stream, n_frames, [&](int t, cudaEvent_t ready) {
        return issue_frame(b, DenoiseStages{b, io.at(t, frame_stride, b->n_streams)}, false, ready);
    });
}

int rnnoise_batch_process_device(RNNoiseBatch* b, float* out, const float* in, float* vad, int n_frames, long stream_stride,
                                 long frame_stride, void* cuda_stream) {
    return process_device_impl(b, {out, in, kFmtF32, vad, stream_stride, 1}, n_frames, frame_stride, cuda_stream);
}

int rnnoise_batch_process_device_pcm16(RNNoiseBatch* b, short* out, const short* in, float* vad, int n_frames, long stream_stride,
                                       long frame_stride, void* cuda_stream) {
    return process_device_impl(b, {out, in, kFmtPcm, vad, stream_stride, 1}, n_frames, frame_stride, cuda_stream);
}

int rnnoise_batch_process_device_strided(RNNoiseBatch* b, void* out, const void* in, int pcm16, float* vad, int n_frames, long stream_stride,
                                         long sample_stride, long frame_stride, void* cuda_stream) {
    if (pcm16 < 0 || pcm16 > 3) return fail("pcm16 must be 0..3");
    return process_device_impl(b, {out, in, pcm16_fmt(pcm16), vad, stream_stride, sample_stride}, n_frames, frame_stride, cuda_stream);
}

// ---- split frames: the caller's network between analysis and synthesis (DESIGN.md 7h) ----
static_assert(RNNOISE_MAX_PENDING_FRAMES == PIPE_DEPTH, "a pending frame keeps its intermediate set");
static_assert(CX_FLOATS * 4 == RNNOISE_SYNTH_CONTEXT_BYTES, "record layout");

int rnnoise_batch_pending_frames(const RNNoiseBatch* b) { return b ? b->pending : 0; }

// The checks both halves of a split frame share; 1: nothing to do, 0: go ahead, -1: error (nothing has run).
static int split_check(RNNoiseBatch* b, const void* samples, const void* per_band, int pcm16, int n_frames, long sample_stride) {
    if (!b) return fail("null batch");
    if (b->n_stages != kNumKernels) return fail("split frames need a denoise batch");
    if (!samples || !per_band) return fail("null argument");
    if (pcm16 != 0 && pcm16 != 1) return fail("pcm16 must be 0 (float) or 1 (int16)");
    if (sample_stride < 1) return fail("sample_stride must be >= 1");
    if (n_frames < 0) return fail("negative n_frames");
    return n_frames == 0 ? 1 : 0;
}

int rnnoise_batch_analyze_device(RNNoiseBatch* b, const void* in, int pcm16, float* features, int* silence, int n_frames,
                                 long stream_stride, long sample_stride, long frame_stride, long feature_stream_stride,
                                 long feature_frame_stride, void* cuda_stream) {
    const int rc = split_check(b, in, features, pcm16, n_frames, sample_stride);
    if (rc) return rc < 0 ? -1 : 0;
    if (check_no_window(b)) return -1;
    if (b->pending + n_frames > RNNOISE_MAX_PENDING_FRAMES)
        return fail("analyzing " + std::to_string(n_frames) + " frame(s) with " + std::to_string(b->pending) +
                    " pending would exceed RNNOISE_MAX_PENDING_FRAMES = " + std::to_string(RNNOISE_MAX_PENDING_FRAMES));
    ON_DEVICE(b->device);
    const size_t esz = pcm16 ? sizeof(short) : sizeof(float);
    return device_call(b, (cudaStream_t)cuda_stream, n_frames, [&](int t, cudaEvent_t ready) {
        DenoiseStages st{b, {nullptr, (const char*)in + (size_t)t * frame_stride * esz, pcm16 ? kFmtPcmIn : kFmtF32, nullptr, stream_stride,
                             sample_stride}};
        st.features = features + (size_t)t * feature_frame_stride;
        st.feature_stride = feature_stream_stride;
        st.silence = silence ? silence + (size_t)t * b->n_streams : nullptr;
        return issue_frame(b, st, false, ready, nullptr, nullptr, kAnalyze);
    });
}

// ctx (may be NULL): the saving call's context records, frame t's at ctx + t * ctx_frame_stride records
static int synthesize_impl(RNNoiseBatch* b, void* out, int pcm16, const float* gains, int n_frames, long stream_stride, long sample_stride,
                           long frame_stride, long gain_stream_stride, long gain_frame_stride, void* ctx, long ctx_stream_stride,
                           long ctx_frame_stride, void* cuda_stream) {
    const int rc = split_check(b, out, gains, pcm16, n_frames, sample_stride);
    if (rc) return rc < 0 ? -1 : 0;
    if (check_no_window(b)) return -1;
    if (n_frames > b->pending)
        return fail("synthesizing " + std::to_string(n_frames) + " frame(s) with " + std::to_string(b->pending) + " pending");
    ON_DEVICE(b->device);
    const size_t esz = pcm16 ? sizeof(short) : sizeof(float);
    return device_call(b, (cudaStream_t)cuda_stream, n_frames, [&](int t, cudaEvent_t ready) {
        DenoiseStages st{b, {(char*)out + (size_t)t * frame_stride * esz, nullptr, pcm16 ? kFmtPcmOut : kFmtF32, nullptr, stream_stride,
                             sample_stride}};
        st.gains = gains + (size_t)t * gain_frame_stride;
        st.gain_stride = gain_stream_stride;
        if (ctx) {
            st.ctx = (unsigned char*)ctx + (size_t)t * ctx_frame_stride * RNNOISE_SYNTH_CONTEXT_BYTES;
            st.ctx_stride = ctx_stream_stride;
        }
        return issue_frame(b, st, false, ready, nullptr, nullptr, kSynthesize);
    });
}

int rnnoise_batch_synthesize_device(RNNoiseBatch* b, void* out, int pcm16, const float* gains, int n_frames, long stream_stride,
                                    long sample_stride, long frame_stride, long gain_stream_stride, long gain_frame_stride, void* cuda_stream) {
    return synthesize_impl(b, out, pcm16, gains, n_frames, stream_stride, sample_stride, frame_stride, gain_stream_stride, gain_frame_stride,
                           nullptr, 0, 0, cuda_stream);
}

int rnnoise_batch_synthesize_saving_device(RNNoiseBatch* b, float* out, const float* gains, int n_frames, long stream_stride,
                                           long sample_stride, long frame_stride, long gain_stream_stride, long gain_frame_stride, void* ctx,
                                           long ctx_stream_stride, long ctx_frame_stride, void* cuda_stream) {
    if (!ctx) return fail("null argument");
    if (reinterpret_cast<uintptr_t>(ctx) & 15) return fail("ctx must be 16-byte aligned");
    if (b && n_frames > 0 && !rows_disjoint(b->n_streams, n_frames, ctx_stream_stride, ctx_frame_stride, 1))
        return fail("context strides overlap records");
    return synthesize_impl(b, out, 0, gains, n_frames, stream_stride, sample_stride, frame_stride, gain_stream_stride, gain_frame_stride, ctx,
                           ctx_stream_stride, ctx_frame_stride, cuda_stream);
}

// ---- window frames: split frames of any length, through the caller's context records (DESIGN.md 7j) ----
int rnnoise_batch_window_frames(const RNNoiseBatch* b) { return b ? b->window : 0; }

// The checks both window calls share: split_check's, then the records' and the mode's.  1: nothing to do, 0: go ahead,
// -1: error (nothing has run).
static int window_check(RNNoiseBatch* b, const void* samples, const void* per_band, int pcm16, int n_frames, long sample_stride,
                        const void* ctx, long ctx_stream_stride, long ctx_frame_stride) {
    const int rc = split_check(b, samples, per_band, pcm16, n_frames, sample_stride);
    if (rc < 0) return -1;
    if (!ctx) return fail("null argument");
    if (reinterpret_cast<uintptr_t>(ctx) & 15) return fail("ctx must be 16-byte aligned");
    if (rc) return 1;
    if (!rows_disjoint(b->n_streams, n_frames, ctx_stream_stride, ctx_frame_stride, 1)) return fail("context strides overlap records");
    if (b->pending > 0)
        return fail(std::to_string(b->pending) + " split frame(s) pending: window frames wait until rnnoise_batch_synthesize_device "
                    "finishes them");
    return 0;
}

int rnnoise_batch_analyze_window_device(RNNoiseBatch* b, const void* in, int pcm16, float* features, int* silence, int n_frames,
                                        long stream_stride, long sample_stride, long frame_stride, long feature_stream_stride,
                                        long feature_frame_stride, void* ctx, long ctx_stream_stride, long ctx_frame_stride,
                                        void* cuda_stream) {
    const int rc = window_check(b, in, features, pcm16, n_frames, sample_stride, ctx, ctx_stream_stride, ctx_frame_stride);
    if (rc) return rc < 0 ? -1 : 0;
    ON_DEVICE(b->device);
    const size_t esz = pcm16 ? sizeof(short) : sizeof(float);
    return device_call(b, (cudaStream_t)cuda_stream, n_frames, [&](int t, cudaEvent_t ready) {
        DenoiseStages st{b, {nullptr, (const char*)in + (size_t)t * frame_stride * esz, pcm16 ? kFmtPcmIn : kFmtF32, nullptr, stream_stride,
                             sample_stride}};
        st.features = features + (size_t)t * feature_frame_stride;
        st.feature_stride = feature_stream_stride;
        st.silence = silence ? silence + (size_t)t * b->n_streams : nullptr;
        st.ctx = (unsigned char*)ctx + (size_t)t * ctx_frame_stride * RNNOISE_SYNTH_CONTEXT_BYTES;
        st.ctx_stride = ctx_stream_stride;
        st.window = true;
        return issue_frame(b, st, false, ready, nullptr, nullptr, kAnalyzeWindow);
    });
}

int rnnoise_batch_synthesize_window_device(RNNoiseBatch* b, void* out, int pcm16, const float* gains, int n_frames, long stream_stride,
                                           long sample_stride, long frame_stride, long gain_stream_stride, long gain_frame_stride, void* ctx,
                                           long ctx_stream_stride, long ctx_frame_stride, void* cuda_stream) {
    const int rc = window_check(b, out, gains, pcm16, n_frames, sample_stride, ctx, ctx_stream_stride, ctx_frame_stride);
    if (rc) return rc < 0 ? -1 : 0;
    if (n_frames > b->window)
        return fail("synthesizing " + std::to_string(n_frames) + " window frame(s) with " + std::to_string(b->window) + " owed");
    ON_DEVICE(b->device);
    const size_t esz = pcm16 ? sizeof(short) : sizeof(float);
    return device_call(b, (cudaStream_t)cuda_stream, n_frames, [&](int t, cudaEvent_t ready) {
        DenoiseStages st{b, {(char*)out + (size_t)t * frame_stride * esz, nullptr, pcm16 ? kFmtPcmOut : kFmtF32, nullptr, stream_stride,
                             sample_stride}};
        st.gains = gains + (size_t)t * gain_frame_stride;
        st.gain_stride = gain_stream_stride;
        st.ctx = (unsigned char*)ctx + (size_t)t * ctx_frame_stride * RNNOISE_SYNTH_CONTEXT_BYTES;
        st.ctx_stride = ctx_stream_stride;
        st.window = true;
        return issue_frame(b, st, false, ready, nullptr, nullptr, kSynthesizeWindow);
    });
}

const char* rnnoise_kernel_name(int i) { return (i >= 0 && i < kNumKernels) ? kKernelNames[i] : nullptr; }

int rnnoise_batch_profile_step(RNNoiseBatch* b, float* out, const float* in, float* vad, long stream_stride, void* cuda_stream,
                               float* ms, int cap) {
    if (!b || !out || !in || !ms) return fail("null argument");
    if (cap < kNumKernels) return fail("ms[] too small");
    if (check_no_pending(b)) return -1;
    ON_DEVICE(b->device);
    if (refresh_links(b) || sync_all(b)) return -1;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : b->st[0];
    Event ev[kNumKernels + 1];
    for (int i = 0; i <= kNumKernels; i++) CK(cudaEventCreate(ev[i].put()));
    int rc = issue_frame(b, DenoiseStages{b, {out, in, kFmtF32, vad, stream_stride, 1}}, false, nullptr, st, ev);
    if (rc == 0) {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) rc = fail("profile_step sync", e);
    }
    if (rc == 0)
        for (int i = 0; i < kNumKernels; i++) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
    return rc == 0 ? kNumKernels : rc;
}

// Host buffers: frame t is copied in on c_in, processed on the stage streams, copied out on c_out; copies of
// neighbouring frames overlap the kernels (true overlap needs page-locked host memory).  The device staging is a ring
// of kStageSlots frames whatever the length of the call: slot k is refilled as soon as the high-pass kernel of the
// frame that used it has consumed its input, and rewritten by the synthesis kernel as soon as that frame's D2H copy
// has finished -- so the copy/compute pipeline depth does not depend on n_frames and a call of any length needs the
// same memory.  16-bit PCM is consumed and produced by the kernels directly (half the bytes over PCIe and HBM).
// subset: the frames advance the work state's rows (a subset call's gather has been issued), B = its row count.
static int process_host_impl(RNNoiseBatch* b, void* out, const void* in, bool pcm, float* vad, int n_frames, bool subset = false) {
    if (ensure_stage(b, pcm) || (!subset && refresh_links(b))) return -1;
    const size_t B = (size_t)(subset ? b->work.n_streams : b->n_streams), fs = B * FRAME_SIZE;
    const size_t esz = pcm ? sizeof(short) : sizeof(float);
    char* din = b->stage_in.get<char>();
    char* dout = b->stage_out.get<char>();
    const int last = b->n_stages - 1;
    // everything issued earlier on the stage streams may still be reading/writing the staging buffers
    if (join_into(b, b->c_in)) return -1;
    for (int t = 0; t < n_frames; t++) {
        const int e = (int)(b->seq % kEvRing), k = t % kStageSlots;
        if (t >= kStageSlots) {
            // input slot: consumed by the first kernel of the frame that used it; output slot: drained by its D2H copy
            CK(cudaStreamWaitEvent(b->c_in, b->ev[0][b->slot_ev[k]], 0));
            CK(cudaStreamWaitEvent(b->st[last], b->ev_out[k], 0));
        }
        CK(cudaMemcpyAsync(din + k * fs * esz, (const char*)in + (size_t)t * fs * esz, fs * esz, cudaMemcpyHostToDevice, b->c_in));
        CK(cudaEventRecord(b->ev_in[e], b->c_in));
        const FrameIO io{dout + k * fs * esz, din + k * fs * esz, pcm ? kFmtPcm : kFmtF32, b->stage_vad.get<float>() + (size_t)k * B, FRAME_SIZE, 1};
        if (issue_frame(b, DenoiseStages{b, io, subset}, subset, b->ev_in[e])) return -1;
        CK(cudaStreamWaitEvent(b->c_out, b->ev[last][e], 0));
        CK(cudaMemcpyAsync((char*)out + (size_t)t * fs * esz, dout + k * fs * esz, fs * esz, cudaMemcpyDeviceToHost, b->c_out));
        if (vad) CK(cudaMemcpyAsync(vad + (size_t)t * B, b->stage_vad.get<float>() + (size_t)k * B, B * sizeof(float), cudaMemcpyDeviceToHost, b->c_out));
        CK(cudaEventRecord(b->ev_out[k], b->c_out));
        b->slot_ev[k] = e;
    }
    CK(cudaStreamSynchronize(b->c_out));
    CK(cudaStreamSynchronize(b->c_in));
    return 0;
}

int rnnoise_batch_process_host(RNNoiseBatch* b, float* out, const float* in, float* vad, int n_frames) {
    if (!b || !out || !in) return fail("null argument");
    if (check_no_pending(b)) return -1;
    if (n_frames <= 0) return n_frames == 0 ? 0 : fail("negative n_frames");
    ON_DEVICE(b->device);
    return process_host_impl(b, out, in, false, vad, n_frames);
}

int rnnoise_batch_process_pcm16_host(RNNoiseBatch* b, short* out, const short* in, float* vad, int n_frames) {
    if (!b || !out || !in) return fail("null argument");
    if (check_no_pending(b)) return -1;
    if (n_frames <= 0) return n_frames == 0 ? 0 : fail("negative n_frames");
    ON_DEVICE(b->device);
    return process_host_impl(b, out, in, true, vad, n_frames);
}

int rnnoise_batch_pitch_stats(RNNoiseBatch* b, unsigned long long out[3]) {
    if (!b || !out) return fail("null argument");
    ON_DEVICE(b->device);
    if (sync_all(b)) return -1;
    CK(cudaMemcpy(out, b->buf.pitch_stats, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return 0;
}

int rnnoise_batch_get_taps(RNNoiseBatch* b, int* pitch, int* silence, float* features, float* gains) {
    return read_taps(b, [&](const BatchBuffers& v, size_t B) {
        if (pitch) CK(cudaMemcpy(pitch, v.pitch, B * sizeof(int), cudaMemcpyDeviceToHost));
        if (silence) CK(cudaMemcpy(silence, v.silence, B * sizeof(int), cudaMemcpyDeviceToHost));
        if (features) CK(cudaMemcpy(features, v.features, B * NB_FEATURES * sizeof(float), cudaMemcpyDeviceToHost));
        if (gains) CK(cudaMemcpy(gains, v.lastg, B * NB_BANDS * sizeof(float), cudaMemcpyDeviceToHost));
        return 0;
    });
}

int rnnoise_batch_get_rnn_taps(RNNoiseBatch* b, float* gains, float* vad, float* gru_state) {
    return read_taps(b, [&](const BatchBuffers& v, size_t B) {
        if (gains) CK(cudaMemcpy(gains, v.gains, B * NB_BANDS * sizeof(float), cudaMemcpyDeviceToHost));
        if (vad) CK(cudaMemcpy(vad, v.vad, B * sizeof(float), cudaMemcpyDeviceToHost));
        if (gru_state) CK(cudaMemcpy(gru_state, v.gru_state, B * b->model.state_size() * sizeof(float), cudaMemcpyDeviceToHost));
        return 0;
    });
}

int rnnoise_batch_get_spectral_taps(RNNoiseBatch* b, float* X, float* P, float* ex, float* ep, float* exp) {
    return read_taps(b, [&](const BatchBuffers& v, size_t B) {
        if (X) CK(cudaMemcpy(X, v.X, B * FREQ_SIZE * sizeof(float2), cudaMemcpyDeviceToHost));
        if (P) CK(cudaMemcpy(P, v.P, B * NB_BINS_BANDED * sizeof(float2), cudaMemcpyDeviceToHost));
        if (ex) CK(cudaMemcpy(ex, v.ex, B * NB_BANDS * sizeof(float), cudaMemcpyDeviceToHost));
        if (ep) CK(cudaMemcpy(ep, v.ep, B * NB_BANDS * sizeof(float), cudaMemcpyDeviceToHost));
        if (exp) CK(cudaMemcpy(exp, v.exp, B * NB_BANDS * sizeof(float), cudaMemcpyDeviceToHost));
        return 0;
    });
}

}  // extern "C"

// ---- per-stream state records (layout: include/rnnoise.h; kernels: state.cu) ----------------------------------------
namespace {

size_t record_bytes(const RNNoiseBatch* b) { return state_record_bytes(b->model.state_size()); }

// the ring slot of the most recent frame: records are read from and written to the positions the next frame expects
int last_slot(const RNNoiseBatch* b) { return (int)((b->phase + HIST_SLOTS - 1) % HIST_SLOTS); }

// 1: device memory of the batch's device, 0: host memory, -1: error
int classify(const RNNoiseBatch* b, const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) return 0;
    if (a.type == cudaMemoryTypeDevice && a.device != b->device) {
        fail("record buffer is on device " + std::to_string(a.device) + ", the batch on device " + std::to_string(b->device));
        return -1;
    }
    if (reinterpret_cast<uintptr_t>(p) & 15) {
        fail("device record buffer must be 16-byte aligned");
        return -1;
    }
    return 1;
}

// Order st[0] after the caller's stream and after every frame issued so far; upload the stream indices (NULL: 0..n-1).
int state_call_begin(RNNoiseBatch* b, const int* streams, int n, cudaStream_t us, const int** d_idx) {
    cudaStream_t s = b->st[0];
    if (wait_for_caller(s, us, b->ev_call) || join_into(b, s)) return -1;
    *d_idx = nullptr;
    if (!streams) return 0;
    if (grow(b, &b->idx, (size_t)n * sizeof(int))) return -1;
    CK(cudaMemcpyAsync(b->idx.get(), streams, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    *d_idx = b->idx.get<int>();
    return 0;
}

// Route the rows of a frame, row i on model model_of[i]: one model, or (several) the rows grouped by model with a stable
// counting sort and cut into tiles of the GRU kernel's height that never span two models.  The tables are uploaded on
// st[0] behind every frame issued so far, so no frame in flight sees them change; later frames start on st[0].
int route_rows(RNNoiseBatch* b, ModelRoute* r, const std::vector<int>& model_of) {
    const size_t K = b->model_acts.size(), n = model_of.size();
    std::vector<int> start(K + 1, 0);
    for (int m : model_of) start[(size_t)m + 1]++;
    int used = 0, only = 0;
    for (size_t k = 0; k < K; k++)
        if (start[k + 1]) {
            used++;
            only = (int)k;
        }
    if (used <= 1) {
        r->uniform = only;
        return 0;
    }
    for (size_t k = 0; k < K; k++) start[k + 1] += start[k];
    std::vector<int> rows(n), next(start.begin(), start.end() - 1);
    for (size_t i = 0; i < n; i++) rows[(size_t)next[(size_t)model_of[i]]++] = (int)i;
    const int T = std::visit([](const auto& m0) { return tile_rows(m0); }, b->gru0);
    std::vector<ModelTile> tiles;
    for (size_t k = 0; k < K; k++)
        for (int f = start[k]; f < start[k + 1]; f += T) tiles.push_back({(int)k, f, std::min(T, start[k + 1] - f), b->model_acts[k]});
    if (join_into(b, b->st[0])) return -1;
    // frames issued earlier may still read the old tables: grow() waits for them
    const size_t cap = (size_t)b->n_streams / MMA_TILE_ROWS + 2 * K;  // >= n / T + K tiles for every n <= n_streams
    if (grow(b, &r->rows, (size_t)b->n_streams * sizeof(int)) ||
        (tiles.size() * sizeof(ModelTile) > r->tiles.bytes() && grow(b, &r->tiles, cap * sizeof(ModelTile)))) {
        r->uniform = 0;  // the old tables may be gone
        return -1;
    }
    CK(cudaMemcpyAsync(r->rows.get(), rows.data(), n * sizeof(int), cudaMemcpyHostToDevice, b->st[0]));
    CK(cudaMemcpyAsync(r->tiles.get(), tiles.data(), tiles.size() * sizeof(ModelTile), cudaMemcpyHostToDevice, b->st[0]));
    r->h_rows = std::move(rows);  // the copies' sources stay alive until the next upload
    r->h_tiles = std::move(tiles);
    r->uniform = -1;
    return 0;
}

// heads: n records `stride` bytes apart, the first being record number r0 of the call
int validate_records(const RNNoiseBatch* b, const unsigned char* heads, size_t stride, int n, int r0 = 0) {
    const int w[3] = {b->model.vad_gru.nn, b->model.noise_gru.nn, b->model.denoise_gru.nn};
    for (int r = 0; r < n; r++) {
        int32_t f[8];
        std::memcpy(f, heads + (size_t)r * stride, sizeof f);
        const bool ok = (uint32_t)f[0] == RNNOISE_STATE_MAGIC && f[1] == RNNOISE_STATE_VERSION && f[2] == w[0] && f[3] == w[1] &&
                        f[4] == w[2] && f[5] >= 0 && f[5] < CEPS_MEM && f[6] >= 0 && f[6] <= PITCH_MAX_PERIOD;
        if (ok) continue;
        const std::string at = "state record " + std::to_string(r0 + r) + ": ";
        if ((uint32_t)f[0] != RNNOISE_STATE_MAGIC) return fail(at + "bad magic");
        if (f[1] != RNNOISE_STATE_VERSION) return fail(at + "unsupported version " + std::to_string(f[1]));
        if (f[2] != w[0] || f[3] != w[1] || f[4] != w[2])
            return fail(at + "GRU widths " + std::to_string(f[2]) + "/" + std::to_string(f[3]) + "/" + std::to_string(f[4]) +
                        " differ from the model's " + std::to_string(w[0]) + "/" + std::to_string(w[1]) + "/" + std::to_string(w[2]));
        if (f[5] < 0 || f[5] >= CEPS_MEM) return fail(at + "mem_id " + std::to_string(f[5]) + " out of range 0..7");
        if (f[6] < 0 || f[6] > PITCH_MAX_PERIOD) return fail(at + "last_period " + std::to_string(f[6]) + " out of range 0..768");
    }
    return 0;
}

}  // namespace

extern "C" {

size_t rnnoise_batch_state_bytes(const RNNoiseBatch* b) { return b ? record_bytes(b) : 0; }

int rnnoise_batch_get_states(RNNoiseBatch* b, const int* streams, int n, void* dst, void* cuda_stream) {
    if (!b) return fail("null batch");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n == 0) return 0;
    if (!dst) return fail("null argument");
    ON_DEVICE(b->device);
    const int dev = classify(b, dst);
    if (dev < 0) return -1;
    cudaStream_t us = (cudaStream_t)cuda_stream, s = b->st[0];
    const size_t bytes = (size_t)n * record_bytes(b);
    if (!dev && grow(b, &b->rec_stage, bytes)) return -1;
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    const int widths[3] = {b->model.vad_gru.nn, b->model.noise_gru.nn, b->model.denoise_gru.nn};
    CK(launch_state_gather(b->buf, widths, d_idx, n, last_slot(b), dev ? dst : b->rec_stage.get(), s));
    if (!dev) CK(cudaMemcpyAsync(dst, b->rec_stage.get(), bytes, cudaMemcpyDeviceToHost, s));
    return resume_caller(s, dev ? us : nullptr, b->ev_state);
}

int rnnoise_batch_set_states(RNNoiseBatch* b, const int* streams, int n, const void* src, void* cuda_stream) {
    if (!b) return fail("null batch");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n == 0) return 0;
    if (!src) return fail("null argument");
    ON_DEVICE(b->device);
    const int dev = classify(b, src);
    if (dev < 0) return -1;
    cudaStream_t us = (cudaStream_t)cuda_stream, s = b->st[0];
    const size_t R = record_bytes(b), bytes = (size_t)n * R;
    if (dev) {  // device-resident records are checked on the device, after the caller's stream; the host reads one index
        cudaStream_t hs = us ? us : s;
        const int widths[3] = {b->model.vad_gru.nn, b->model.noise_gru.nn, b->model.denoise_gru.nn};
        int first_bad = n;
        CK(cudaMemcpyAsync(b->d_first_bad, &first_bad, sizeof(int), cudaMemcpyHostToDevice, hs));
        CK(launch_state_check(src, n, widths, b->d_first_bad, hs));
        CK(cudaMemcpyAsync(&first_bad, b->d_first_bad, sizeof(int), cudaMemcpyDeviceToHost, hs));
        CK(cudaStreamSynchronize(hs));
        if (first_bad < n) {  // the offending record's head, for the error text
            unsigned char head[32];
            CK(cudaMemcpy(head, static_cast<const unsigned char*>(src) + (size_t)first_bad * R, sizeof head, cudaMemcpyDeviceToHost));
            if (validate_records(b, head, sizeof head, 1, first_bad)) return -1;
            return fail("state record " + std::to_string(first_bad) + " rejected");
        }
    } else {
        if (validate_records(b, static_cast<const unsigned char*>(src), R, n)) return -1;
        if (grow(b, &b->rec_stage, bytes)) return -1;
    }
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    if (!dev) CK(cudaMemcpyAsync(b->rec_stage.get(), src, bytes, cudaMemcpyHostToDevice, s));
    CK(launch_state_scatter(b->buf, b->model.state_size(), d_idx, n, last_slot(b), dev ? src : b->rec_stage.get(), s));
    return resume_caller(s, dev ? us : nullptr, b->ev_state);
}

int rnnoise_batch_reset_streams(RNNoiseBatch* b, const int* streams, int n, void* cuda_stream) {
    if (!b) return fail("null batch");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n == 0) return 0;
    ON_DEVICE(b->device);
    cudaStream_t us = (cudaStream_t)cuda_stream, s = b->st[0];
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    CK(launch_state_scatter(b->buf, b->model.state_size(), d_idx, n, last_slot(b), nullptr, s));
    for (int r = 0; r < n; r++) reset_ctl_live(b, (size_t)stream_of(streams, r));
    return resume_caller(s, us, b->ev_state);
}

}  // extern "C"

// ---- model table: streams of one batch on different models of one geometry (DESIGN.md 7c) ---------------------------
namespace {

// The first of the six layers whose shape differs from the batch model's, or "".
std::string geometry_mismatch(const HostModel& a, const HostModel& m) {
    struct L { const char* name; int ni0, nn0, ni, nn; };
    const L layers[6] = {{"input_dense", a.input_dense.ni, a.input_dense.nn, m.input_dense.ni, m.input_dense.nn},
                         {"vad_gru", a.vad_gru.ni, a.vad_gru.nn, m.vad_gru.ni, m.vad_gru.nn},
                         {"noise_gru", a.noise_gru.ni, a.noise_gru.nn, m.noise_gru.ni, m.noise_gru.nn},
                         {"denoise_gru", a.denoise_gru.ni, a.denoise_gru.nn, m.denoise_gru.ni, m.denoise_gru.nn},
                         {"denoise_output", a.denoise_output.ni, a.denoise_output.nn, m.denoise_output.ni, m.denoise_output.nn},
                         {"vad_output", a.vad_output.ni, a.vad_output.nn, m.vad_output.ni, m.vad_output.nn}};
    for (const L& l : layers)
        if (l.ni != l.ni0 || l.nn != l.nn0)
            return std::string("model geometry differs from the batch's model in layer ") + l.name + ": " + std::to_string(l.ni) + " inputs x " +
                   std::to_string(l.nn) + " neurons, the batch's model has " + std::to_string(l.ni0) + " x " + std::to_string(l.nn0);
    return "";
}

}  // namespace

extern "C" {

int rnnoise_batch_add_model(RNNoiseBatch* b, const RNNModel* model) {
    if (!b) return fail("null batch");
    const HostModel& hm = model ? model->m : HostModel::builtin();
    const std::string bad = geometry_mismatch(b->model, hm);
    if (!bad.empty()) return fail(bad);
    ON_DEVICE(b->device);
    // The descriptor follows from the geometry alone, so it must equal model 0's byte for byte: checked as an invariant.
    std::vector<unsigned char> img;
    const bool same = std::visit(
        [&](const auto& m0) {
            std::decay_t<decltype(m0)> d;
            return pack_model(hm, &d, &img) && std::memcmp(&d, &m0, sizeof d) == 0;
        },
        b->gru0);
    if (!same || img.size() != b->mtab_bytes) return fail("packed layout of the model differs from the batch model's (internal error)");
    // image K goes to the first free entry; a full table moves to an allocation of twice the capacity, the old images
    // first.  Frames in flight may read the table.
    const size_t K = b->model_acts.size(), stride = b->mtab_stride;
    if (sync_all(b)) return -1;
    DeviceMem grown;
    cudaError_t e = cudaSuccess;
    if (K * stride == b->mtab.bytes()) {
        CK(grown.alloc(stride * 2 * K));
        e = cudaMemcpyAsync(grown.get(), b->mtab.get(), stride * K, cudaMemcpyDeviceToDevice, b->st[0]);
    }
    unsigned char* d = (grown.bytes() ? grown : b->mtab).get<unsigned char>();
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + stride * K, img.data(), img.size(), cudaMemcpyHostToDevice, b->st[0]);
    if (e == cudaSuccess) e = cudaStreamSynchronize(b->st[0]);
    if (e != cudaSuccess) return fail("model table upload", e);
    if (grown.bytes()) b->mtab = std::move(grown);
    b->model_acts.push_back(model_acts(hm));
    return (int)K;
}

int rnnoise_batch_set_stream_models(RNNoiseBatch* b, const int* streams, int n, const int* model_ids) {
    if (!b) return fail("null batch");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n == 0) return 0;
    if (!model_ids) return fail("null argument");
    const int K = (int)b->model_acts.size();
    for (int r = 0; r < n; r++)
        if (model_ids[r] < 0 || model_ids[r] >= K)
            return fail("model id " + std::to_string(model_ids[r]) + " of stream " + std::to_string(stream_of(streams, r)) + " out of range 0.." +
                        std::to_string(K - 1));
    ON_DEVICE(b->device);
    std::vector<int> next(b->stream_model);
    for (int r = 0; r < n; r++) next[(size_t)stream_of(streams, r)] = model_ids[r];
    if (route_rows(b, &b->route, next)) return -1;
    b->stream_model = std::move(next);
    return 0;
}

int rnnoise_batch_get_stream_models(const RNNoiseBatch* b, const int* streams, int n, int* model_ids) {
    if (!b) return fail("null batch");
    if (check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n == 0) return 0;
    if (!model_ids) return fail("null argument");
    for (int r = 0; r < n; r++) model_ids[r] = b->stream_model[(size_t)stream_of(streams, r)];
    return 0;
}

}  // extern "C"

// ---- stream controls: attenuation limit and voice-activity gate (DESIGN.md 7m) ---------------------------------------
static_assert(sizeof(RNNoiseStreamControls) == 24, "RNNoiseStreamControls is ABI");

namespace {

// "" if a controls record passes the checks of rnnoise_batch_set_stream_controls, else what fails
std::string controls_error(const RNNoiseStreamControls& c) {
    auto unit = [](float v) { return v >= 0.0f && v <= 1.0f; };  // false for NaN
    if (std::isnan(c.atten_lim_db) || c.atten_lim_db < 0.0f) return "atten_lim_db must be >= 0 (+INFINITY: no limit)";
    if (!unit(c.gate_threshold)) return "gate_threshold must be in 0..1";
    if (!unit(c.gate_closed_gain)) return "gate_closed_gain must be in 0..1";
    if (c.gate_hold_frames < 0 || c.gate_hold_frames > RNNOISE_GATE_MAX_HOLD_FRAMES)
        return "gate_hold_frames must be in 0.." + std::to_string(RNNOISE_GATE_MAX_HOLD_FRAMES);
    if (c.gate_hold_left < 0 || c.gate_hold_left > c.gate_hold_frames) return "gate_hold_left must be in 0..gate_hold_frames";
    if (c.gate_closed != 0 && c.gate_closed != 1) return "gate_closed must be 0 or 1";
    return "";
}

}  // namespace

extern "C" {

int rnnoise_batch_set_stream_controls(RNNoiseBatch* b, const int* streams, int n, const RNNoiseStreamControls* c) {
    if (!b) return fail("null batch");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n == 0) return 0;
    if (!c) return fail("null argument");
    std::vector<StreamCtl> ctl((size_t)n);
    std::vector<int2> gate((size_t)n);
    for (int r = 0; r < n; r++) {
        const std::string bad = controls_error(c[r]);
        if (!bad.empty())
            return fail("stream controls record " + std::to_string(r) + " (stream " + std::to_string(stream_of(streams, r)) + "): " + bad);
        const float a = c[r].atten_lim_db;
        ctl[(size_t)r] = {std::isinf(a) ? 0.0f : (float)std::pow(10.0, -(double)a / 20.0), c[r].gate_threshold, c[r].gate_closed_gain,
                          c[r].gate_hold_frames};
        gate[(size_t)r] = make_int2(c[r].gate_hold_left, c[r].gate_closed);
    }
    ON_DEVICE(b->device);
    const size_t cb = (size_t)n * sizeof(StreamCtl), bytes = cb + (size_t)n * sizeof(int2);
    if (grow(b, &b->rec_stage, bytes)) return -1;
    const int* d_idx;
    if (state_call_begin(b, streams, n, nullptr, &d_idx)) return -1;
    cudaStream_t s = b->st[0];
    unsigned char* stage = b->rec_stage.get<unsigned char>();
    CK(cudaMemcpyAsync(stage, ctl.data(), cb, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(stage + cb, gate.data(), bytes - cb, cudaMemcpyHostToDevice, s));
    CK(launch_controls_scatter(b->buf, d_idx, n, reinterpret_cast<const StreamCtl*>(stage), reinterpret_cast<const int2*>(stage + cb), s));
    CK(cudaStreamSynchronize(s));
    for (int r = 0; r < n; r++) {
        b->stream_ctl[(size_t)stream_of(streams, r)] = c[r];
        set_ctl_live(b, (size_t)stream_of(streams, r), !default_controls(c[r]));
    }
    return 0;
}

int rnnoise_batch_get_stream_controls(RNNoiseBatch* b, const int* streams, int n, RNNoiseStreamControls* c) {
    if (!b) return fail("null batch");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n == 0) return 0;
    if (!c) return fail("null argument");
    ON_DEVICE(b->device);
    const size_t bytes = (size_t)n * sizeof(int2);
    if (grow(b, &b->rec_stage, bytes)) return -1;
    const int* d_idx;
    if (state_call_begin(b, streams, n, nullptr, &d_idx)) return -1;
    cudaStream_t s = b->st[0];
    std::vector<int2> gate((size_t)n);
    CK(launch_controls_gather(b->buf, d_idx, n, b->rec_stage.get<int2>(), s));
    CK(cudaMemcpyAsync(gate.data(), b->rec_stage.get(), bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int r = 0; r < n; r++) {
        c[r] = b->stream_ctl[(size_t)stream_of(streams, r)];
        c[r].gate_hold_left = gate[(size_t)r].x;
        c[r].gate_closed = gate[(size_t)r].y;
    }
    return 0;
}

}  // extern "C"

// ---- stream links: one gain curve for several streams (DESIGN.md 7n) -------------------------------------------------
static_assert(RNNOISE_LINK_MAX == LINK_MODE_MAX && RNNOISE_LINK_MEAN == LINK_MODE_MEAN, "link modes");

namespace {

// The LinkTable (common.cuh) of the rows streams[0..n) (NULL: 0..n-1), every group of a listed stream listed whole, in
// *img; false when no row is linked.
bool link_table(const RNNoiseBatch* b, const int* streams, int n, std::vector<int>* img) {
    std::vector<int> row_of, first((size_t)b->n_streams, -1);  // first[g]: offset of group g's members in the list
    if (streams) {
        row_of.assign((size_t)b->n_streams, -1);
        for (int r = 0; r < n; r++) row_of[(size_t)streams[r]] = r;
    }
    img->assign((size_t)n * 5, 0);
    int next = 0;
    bool any = false;
    for (int r = 0; r < n; r++) {
        const size_t s = (size_t)stream_of(streams, r);
        if (!b->link_mode[s]) continue;
        const int gid = b->link_group[s];
        const LinkGroup& g = b->groups.at(gid);
        if (first[(size_t)gid] < 0) {
            first[(size_t)gid] = next;
            for (int m : g.members) (*img)[(size_t)n * 4 + (size_t)next++] = streams ? row_of[(size_t)m] : m;
        }
        int* rec = img->data() + (size_t)r * 4;
        rec[0] = first[(size_t)gid];
        rec[1] = (int)g.members.size();
        rec[2] = g.mode;
        any = true;
    }
    return any;
}

// Stream s leaves its group (if any); a group left with one member dissolves, and one that lost its lowest member is
// filed under the next.
void leave_group(RNNoiseBatch* b, int s) {
    if (!b->link_mode[(size_t)s]) return;
    const auto it = b->groups.find(b->link_group[(size_t)s]);
    LinkGroup g = std::move(it->second);
    b->groups.erase(it);
    g.members.erase(std::find(g.members.begin(), g.members.end(), s));
    b->link_group[(size_t)s] = s;
    b->link_mode[(size_t)s] = 0;
    if (g.members.size() < 2) {
        for (int m : g.members) {
            b->link_group[(size_t)m] = m;
            b->link_mode[(size_t)m] = 0;
        }
        return;
    }
    for (int m : g.members) b->link_group[(size_t)m] = g.members[0];
    const int lead = g.members[0];
    b->groups.emplace(lead, std::move(g));
}

}  // namespace

// Every group of a listed stream must be listed whole (streams NULL: 0..n-1).
int check_whole_groups(const RNNoiseBatch* b, const int* streams, int n) {
    if (b->groups.empty() || (!streams && n == b->n_streams)) return 0;
    std::vector<char> listed((size_t)b->n_streams, 0);
    for (int r = 0; r < n; r++) listed[(size_t)stream_of(streams, r)] = 1;
    for (int r = 0; r < n; r++) {
        const size_t s = (size_t)stream_of(streams, r);
        if (!b->link_mode[s]) continue;
        for (int m : b->groups.at(b->link_group[s]).members)
            if (!listed[(size_t)m])
                return fail("stream " + std::to_string(s) + " is linked with stream " + std::to_string(m) +
                            ", which is not listed: a subset call lists every group of its streams whole");
    }
    return 0;
}

int nnb::batch_check_whole_groups(const RNNoiseBatch* b, const int* streams, int n) { return check_whole_groups(b, streams, n); }

// Before a full-batch fused frame: after a link change, the batch's LinkTable is rebuilt and uploaded on st[0] behind
// every frame issued so far, so frames in flight keep reading the old one and the frames issued next read the new one.
int refresh_links(RNNoiseBatch* b) {
    if (!b->links_stale) return 0;
    if (!b->groups.empty()) {
        std::vector<int> img;
        link_table(b, nullptr, b->n_streams, &img);
        if (grow(b, &b->link_tab, img.size() * sizeof(int)) || join_into(b, b->st[0])) return -1;
        CK(cudaMemcpyAsync(b->link_tab.get(), img.data(), img.size() * sizeof(int), cudaMemcpyHostToDevice, b->st[0]));
        b->h_link = std::move(img);
    }
    b->links_stale = false;
    return 0;
}

extern "C" {

int rnnoise_batch_link_streams(RNNoiseBatch* b, const int* streams, int n, int mode) {
    if (!b) return fail("null batch");
    if (!streams) return fail("null argument");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    if (n < 2 || n > RNNOISE_LINK_MAX_MEMBERS)
        return fail("a group links 2.." + std::to_string(RNNOISE_LINK_MAX_MEMBERS) + " streams, not " + std::to_string(n));
    if (mode != RNNOISE_LINK_MAX && mode != RNNOISE_LINK_MEAN)
        return fail("link mode " + std::to_string(mode) + " is neither RNNOISE_LINK_MAX (1) nor RNNOISE_LINK_MEAN (2)");
    LinkGroup g{mode, std::vector<int>(streams, streams + n)};
    std::sort(g.members.begin(), g.members.end());
    for (int s : g.members) leave_group(b, s);
    for (int s : g.members) {
        b->link_group[(size_t)s] = g.members[0];
        b->link_mode[(size_t)s] = mode;
    }
    const int lead = g.members[0];
    b->groups.emplace(lead, std::move(g));
    b->links_stale = true;
    return 0;
}

int rnnoise_batch_unlink_streams(RNNoiseBatch* b, const int* streams, int n) {
    if (!b) return fail("null batch");
    if (!streams) n = b->n_streams;
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch")) return -1;
    for (int r = 0; r < n; r++) leave_group(b, stream_of(streams, r));
    b->links_stale = true;
    return 0;
}

int rnnoise_batch_get_stream_links(RNNoiseBatch* b, const int* streams, int n, int* group, int* mode) {
    if (!b) return fail("null batch");
    if (check_streams(b->n_streams, streams, n, "batch")) return -1;
    for (int r = 0; r < n; r++) {
        const size_t s = (size_t)stream_of(streams, r);
        if (group) group[r] = b->link_group[s];
        if (mode) mode[r] = b->link_mode[s];
    }
    return 0;
}

}  // extern "C"

// ---- subset calls: advance only the listed streams (rnnoise_batch_process_streams_*; DESIGN.md 7b) ------------------
namespace {

// Checks every argument of a subset call; 1: nothing to do, 0: go ahead, -1: error (nothing has run).
int subset_check(RNNoiseBatch* b, const int* streams, int n, const void* out, const void* in, int n_frames) {
    if (!b) return fail("null batch");
    if (check_no_pending(b) || check_streams(b->n_streams, streams, n, "batch") || check_whole_groups(b, streams, n)) return -1;
    if (n_frames < 0) return fail("negative n_frames");
    if (n == 0 || n_frames == 0) return 1;
    if (!out || !in) return fail("null argument");
    return 0;
}

// After every frame and state call issued so far (and the caller's stream): gather the listed streams into the work rows.
int subset_begin(RNNoiseBatch* b, const int* streams, int n, cudaStream_t us) {
    if (grow_state(b, &b->work, &b->work_mem, (size_t)n)) return fail("work state of " + std::to_string(n) + " streams: " + g_err);
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    b->work.n_streams = n;
    b->work_frames = 0;
    b->work_route.uniform = 0;
    if (b->model_acts.size() > 1) {  // the work rows' models
        std::vector<int> model_of((size_t)n);
        for (int r = 0; r < n; r++) model_of[(size_t)r] = b->stream_model[(size_t)stream_of(streams, r)];
        if (route_rows(b, &b->work_route, model_of)) return -1;
    }
    b->work_linked = false;
    if (!b->groups.empty()) {  // the work rows' link table, uploaded with the gather
        std::vector<int> img;
        if (link_table(b, streams, n, &img)) {
            if (grow(b, &b->work_link, img.size() * sizeof(int))) return -1;
            CK(cudaMemcpyAsync(b->work_link.get(), img.data(), img.size() * sizeof(int), cudaMemcpyHostToDevice, b->st[0]));
            b->h_work_link = std::move(img);
            b->work_linked = true;
        }
    }
    CK(launch_subset_gather(b->buf, b->work, b->model.state_size(), d_idx, n, (int)(b->phase % HIST_SLOTS), b->st[0]));
    return 0;
}

// After the call's last frame: scatter the work rows back, rotated from the work ring's phase to the batch's.  Later
// frames and state calls start on st[0], behind the scatter.
int subset_end(RNNoiseBatch* b, const int* streams, int n) {
    cudaStream_t s = b->st[0];
    if (join_into(b, s)) return -1;
    const int work_slot = (int)((b->phase + b->work_frames + HIST_SLOTS - 1) % HIST_SLOTS);
    CK(launch_subset_scatter(b->buf, b->work, b->model.state_size(), streams ? b->idx.get<int>() : nullptr, n, work_slot, last_slot(b), s));
    return 0;
}

}  // namespace

extern "C" {

int rnnoise_batch_process_streams_device(RNNoiseBatch* b, const int* streams, int n, void* out, const void* in, int pcm16, float* vad,
                                         int n_frames, long stream_stride, long sample_stride, long frame_stride, void* cuda_stream) {
    const int rc = subset_check(b, streams, n, out, in, n_frames);
    if (rc) return rc < 0 ? -1 : 0;
    if (pcm16 < 0 || pcm16 > 3) return fail("pcm16 must be 0..3");
    if (sample_stride < 1) return fail("sample_stride must be >= 1");
    ON_DEVICE(b->device);
    const FrameIO io{out, in, pcm16_fmt(pcm16), vad, stream_stride, sample_stride};
    return device_call(
        b, (cudaStream_t)cuda_stream, n_frames,
        [&](int t, cudaEvent_t ready) { return issue_frame(b, DenoiseStages{b, io.at(t, frame_stride, n), true}, true, ready); }, true, streams,
        n);
}

int rnnoise_batch_process_streams_host(RNNoiseBatch* b, const int* streams, int n, float* out, const float* in, float* vad, int n_frames) {
    const int rc = subset_check(b, streams, n, out, in, n_frames);
    if (rc) return rc < 0 ? -1 : 0;
    ON_DEVICE(b->device);
    if (ensure_stage(b, false)) return -1;
    if (subset_begin(b, streams, n, nullptr)) return -1;
    if (process_host_impl(b, out, in, false, vad, n_frames, true)) return -1;
    if (subset_end(b, streams, n)) return -1;
    return resume_caller(b->st[0], nullptr, b->ev_state);
}

}  // extern "C"

// ---- training-data rows (src/training.rs): 3 feature extractors per lane on the denoise path's kernels ----------
static_assert(sizeof(RNNoiseSimParams) == sizeof(TrainLaneParams), "C ABI struct and device struct must match");
constexpr int kTrainStages = 4;  // front, pitch, analysis, rows
constexpr size_t kTrainStageBytes = size_t(256) << 20;  // bound of each device staging buffer of the host-buffer calls

constexpr int kWaveSlots = 4;  // offset staging slots of the waveform calls: up to 4 calls in flight before the host waits

// A trainer makes rows or waveforms, never both, until rnnoise_train_reset: waveform calls leave the 3L feature
// extractors' pitch and analysis state behind, so rows after them would be wrong.
enum class TrainMode { kNone, kRows, kWaves };

struct RNNoiseTrainer {
    TrainBuffers tb{};
    std::vector<DeviceMem> lanes;  // owners of tb's buffers
    DeviceMem stage_sig, stage_noise, stage_rows, stage_pool, stage_at;
    TrainMode mode = TrainMode::kNone;
    // waveform calls: the resident int16 sample pool, and per call slot the staged offsets [2][n_frames][L] (pinned host
    // and device) and the event after the kernel that reads them
    DeviceMem pool;
    long long pool_len = 0;
    PinnedMem wave_host[kWaveSlots];
    size_t wave_host_bytes[kWaveSlots] = {};
    DeviceMem wave_at[kWaveSlots];
    Event wave_done[kWaveSlots], wave_caller;
    unsigned long long wave_calls = 0;
    // 3 * n_lanes streams: [0, L) clean, [L, 2L) noise, [2L, 3L) combined.  Declared last, so destroyed first: its
    // release waits for the frames that use the buffers above.
    BatchPtr batch;
};

namespace {

// Frees the batch once its frames have finished, then the trainer's buffers.  Reports no error.
struct TrainerRelease {
    void operator()(RNNoiseTrainer* t) const {
        DeviceGuard guard(t->batch ? t->batch->device : 0);
        delete t;
    }
};

// Every lane as NoiseSimulator::new leaves it (src/training.rs:319-340): default parameters, filter memories and VAD
// counter zeroed.  Called with the trainer's device selected and nothing in flight.
int trainer_defaults(RNNoiseTrainer* t) {
    const TrainBuffers& tb = t->tb;
    const size_t L = (size_t)tb.n_lanes;
    CK(cudaMemset(tb.resp_mem, 0, L * 4 * sizeof(float)));
    CK(cudaMemset(tb.vad_count, 0, L * sizeof(int32_t)));
    TrainLaneParams d{};
    d.signal_gain = 1.0f;
    d.noise_gain = 1.0f;
    d.band_lp = NB_BANDS - 1;
    std::vector<TrainLaneParams> init(L, d);
    CK(cudaMemcpy(tb.params, init.data(), L * sizeof(TrainLaneParams), cudaMemcpyHostToDevice));
    return 0;
}

// The mode check of every frame call: a trainer in the other mode refuses it.
int trainer_mode(const RNNoiseTrainer* t, TrainMode want) {
    if (t->mode == TrainMode::kNone || t->mode == want) return 0;
    return fail(want == TrainMode::kRows ? "this trainer has made waveform frames: rows need rnnoise_train_reset first"
                                         : "this trainer has made rows: waveform frames need rnnoise_train_reset first");
}

// The trainer's own buffers, on the batch's device.
int trainer_init(RNNoiseTrainer* t, int n_lanes) {
    ON_DEVICE(t->batch->device);
    const size_t L = (size_t)n_lanes;
    TrainBuffers& tb = t->tb;
    tb.n_lanes = n_lanes;
    CK(dalloc(&t->lanes, &tb.params, L));
    CK(dalloc(&t->lanes, &tb.resp_mem, L * 4));
    CK(dalloc(&t->lanes, &tb.vad_count, L));
    CK(dalloc(&t->lanes, &tb.vad, PIPE_DEPTH * L));
    CK(dalloc(&t->lanes, &tb.cutoff, PIPE_DEPTH * L));
    for (int k = 0; k < kWaveSlots; k++) CK(cudaEventCreateWithFlags(t->wave_done[k].put(), cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(t->wave_caller.put(), cudaEventDisableTiming));
    return trainer_defaults(t);
}

// The four stages of a training frame of every lane: front -> pitch -> analysis -> rows; `set` is the frame's
// intermediate set.
struct TrainStages {
    const RNNoiseTrainer* t;
    int set;
    float* rows;
    long row_lane_stride;
    const float* sig;
    const float* noise;
    long stream_stride;
    const short* pool = nullptr;  // non-NULL: the frame's samples come from this int16 pool, at the lane offsets below
    const long long* sig_at = nullptr;
    const long long* noise_at = nullptr;

    int operator()(int i, const BatchBuffers& v, int slot, cudaStream_t s) const {
        const RNNoiseBatch* b = t->batch.get();
        switch (i) {
            case 0:
                if (pool) CK(launch_train_front_pool(v, t->tb, set, pool, sig_at, noise_at, slot, s));
                else CK(launch_train_front(v, t->tb, set, sig, noise, stream_stride, slot, s));
                break;
            case 1: CK(launch_pitch(v, slot, b->pitch_exact, s)); break;
            case 2: CK(launch_analysis_warp(v, b->d_tab, slot, s)); break;
            default: CK(launch_train_rows(v, t->tb, set, rows, row_lane_stride, s)); break;
        }
        return 0;
    }
};

}  // namespace

extern "C" {

RNNoiseTrainer* rnnoise_train_create(int n_lanes, int device) {
    if (n_lanes <= 0 || n_lanes > (1 << 29) / 3) {
        fail("n_lanes out of range");
        return nullptr;
    }
    std::unique_ptr<RNNoiseTrainer, TrainerRelease> t(new (std::nothrow) RNNoiseTrainer());
    if (!t) return nullptr;
    t->batch = create_batch(HostModel::builtin(), 3 * n_lanes, device);
    if (!t->batch) return nullptr;
    t->batch->n_stages = kTrainStages;
    return trainer_init(t.get(), n_lanes) ? nullptr : t.release();
}

void rnnoise_train_destroy(RNNoiseTrainer* t) {
    if (t) TrainerRelease()(t);
}
int rnnoise_train_lanes(const RNNoiseTrainer* t) { return t ? t->tb.n_lanes : 0; }
RNNoiseBatch* rnnoise_train_feature_batch(RNNoiseTrainer* t) { return t ? t->batch.get() : nullptr; }

int rnnoise_train_band_lp(int lowpass) {
    static const int eband[NB_BANDS] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 34, 40, 48, 60, 78, 100};  // src/lib.rs:55-58
    for (int i = 0; i < NB_BANDS; i++)
        if ((eband[i] << 2) > lowpass) return i;
    return NB_BANDS - 1;
}

int rnnoise_train_set_params(RNNoiseTrainer* t, int first_lane, int n, const RNNoiseSimParams* params) {
    if (!t || !params) return fail("null argument");
    if (first_lane < 0 || n < 0 || first_lane + n > t->tb.n_lanes) return fail("lane range out of bounds");
    for (int i = 0; i < n; i++)
        if (params[i].band_lp < 0 || params[i].band_lp >= NB_BANDS) return fail("band_lp must be in [0, 21]");
    ON_DEVICE(t->batch->device);
    if (sync_all(t->batch.get())) return -1;  // frames in flight still read the old parameters
    CK(cudaMemcpy(t->tb.params + first_lane, params, (size_t)n * sizeof(TrainLaneParams), cudaMemcpyHostToDevice));
    return 0;
}

int rnnoise_train_process_device(RNNoiseTrainer* t, float* rows, const float* signal, const float* noise, int n_frames, long stream_stride,
                                 long frame_stride, long row_lane_stride, long row_frame_stride, void* cuda_stream) {
    if (!t || !rows || !signal || !noise) return fail("null argument");
    if (n_frames < 0) return fail("negative n_frames");
    if (trainer_mode(t, TrainMode::kRows)) return -1;
    if (n_frames == 0) return 0;
    RNNoiseBatch* b = t->batch.get();
    ON_DEVICE(b->device);
    t->mode = TrainMode::kRows;
    return device_call(b, (cudaStream_t)cuda_stream, n_frames, [&](int f, cudaEvent_t ready) {
        const TrainStages stages{t, (int)(b->seq % PIPE_DEPTH), rows + (size_t)f * row_frame_stride, row_lane_stride,
                                 signal + (size_t)f * frame_stride, noise + (size_t)f * frame_stride, stream_stride};
        return issue_frame(b, stages, false, ready);
    });
}

int rnnoise_train_process_host(RNNoiseTrainer* t, float* rows, const float* signal, const float* noise, int n_frames) {
    if (!t || !rows || !signal || !noise) return fail("null argument");
    if (n_frames < 0) return fail("negative n_frames");
    if (trainer_mode(t, TrainMode::kRows)) return -1;
    if (n_frames == 0) return 0;
    RNNoiseBatch* b = t->batch.get();
    ON_DEVICE(b->device);
    const size_t L = (size_t)t->tb.n_lanes;
    // staging is bounded (<= 256 MiB per input buffer): long runs go through in chunks of frames
    const int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_frames, kTrainStageBytes / (L * FRAME_SIZE * sizeof(float))));
    const size_t in_bytes = (size_t)chunk * L * FRAME_SIZE * sizeof(float);
    if (grow(b, &t->stage_sig, in_bytes) || grow(b, &t->stage_noise, in_bytes) ||
        grow(b, &t->stage_rows, (size_t)chunk * L * TRAIN_ROW * sizeof(float)))
        return -1;
    float* sig = t->stage_sig.get<float>();
    float* noi = t->stage_noise.get<float>();
    float* out = t->stage_rows.get<float>();
    for (int f0 = 0; f0 < n_frames; f0 += chunk) {
        const int nf = std::min(chunk, n_frames - f0);
        const size_t off = (size_t)f0 * L;
        CK(cudaMemcpyAsync(sig, signal + off * FRAME_SIZE, (size_t)nf * L * FRAME_SIZE * sizeof(float), cudaMemcpyHostToDevice, b->c_in));
        CK(cudaMemcpyAsync(noi, noise + off * FRAME_SIZE, (size_t)nf * L * FRAME_SIZE * sizeof(float), cudaMemcpyHostToDevice, b->c_in));
        if (rnnoise_train_process_device(t, out, sig, noi, nf, FRAME_SIZE, (long)(L * FRAME_SIZE), TRAIN_ROW,
                                         (long)(L * TRAIN_ROW), b->c_in))
            return -1;
        CK(cudaMemcpyAsync(rows + off * TRAIN_ROW, out, (size_t)nf * L * TRAIN_ROW * sizeof(float), cudaMemcpyDeviceToHost, b->c_in));
        CK(cudaStreamSynchronize(b->c_in));
    }
    return 0;
}

int rnnoise_train_process_pool_host(RNNoiseTrainer* t, float* rows, const short* pool, long pool_len, const long long* sig_at,
                                    const long long* noise_at, int n_frames) {
    if (!t || !rows || !pool || !sig_at || !noise_at) return fail("null argument");
    if (n_frames < 0) return fail("negative n_frames");
    if (trainer_mode(t, TrainMode::kRows)) return -1;
    if (pool_len < 0 || (size_t)pool_len * sizeof(short) > kTrainStageBytes)
        return fail("pool_len " + std::to_string(pool_len) + " out of range [0, " + std::to_string(kTrainStageBytes / sizeof(short)) + "]");
    const size_t L = (size_t)t->tb.n_lanes;
    // the offsets come from outside the library: every one is checked before anything is uploaded or run
    const long long last = (long long)pool_len - FRAME_SIZE;
    for (int k = 0; k < 2; k++) {
        const long long* at = k ? noise_at : sig_at;
        for (size_t i = 0; i < (size_t)n_frames * L; i++)
            if (at[i] != -1 && (at[i] < 0 || at[i] > last))
                return fail(std::string(k ? "noise_at" : "sig_at") + " = " + std::to_string(at[i]) + " at frame " + std::to_string(i / L) +
                            ", lane " + std::to_string(i % L) + ": must be -1 or in [0, pool_len - 480 = " + std::to_string(last) + "]");
    }
    if (n_frames == 0) return 0;
    RNNoiseBatch* b = t->batch.get();
    ON_DEVICE(b->device);
    // the pool goes up whole, once; offsets and rows go through in chunks of frames of at most 256 MiB of rows
    const int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_frames, kTrainStageBytes / (L * TRAIN_ROW * sizeof(float))));
    const size_t at_count = (size_t)chunk * L;
    if (grow(b, &t->stage_pool, std::max<size_t>(1, (size_t)pool_len) * sizeof(short)) ||
        grow(b, &t->stage_at, 2 * at_count * sizeof(long long)) || grow(b, &t->stage_rows, at_count * TRAIN_ROW * sizeof(float)))
        return -1;
    short* dpool = t->stage_pool.get<short>();
    long long* dsig = t->stage_at.get<long long>();
    long long* dnoi = dsig + at_count;
    float* out = t->stage_rows.get<float>();
    CK(cudaMemcpyAsync(dpool, pool, (size_t)pool_len * sizeof(short), cudaMemcpyHostToDevice, b->c_in));
    t->mode = TrainMode::kRows;
    for (int f0 = 0; f0 < n_frames; f0 += chunk) {
        const int nf = std::min(chunk, n_frames - f0);
        const size_t off = (size_t)f0 * L;
        CK(cudaMemcpyAsync(dsig, sig_at + off, (size_t)nf * L * sizeof(long long), cudaMemcpyHostToDevice, b->c_in));
        CK(cudaMemcpyAsync(dnoi, noise_at + off, (size_t)nf * L * sizeof(long long), cudaMemcpyHostToDevice, b->c_in));
        const int rc = device_call(b, b->c_in, nf, [&](int f, cudaEvent_t ready) {
            TrainStages stages{t, (int)(b->seq % PIPE_DEPTH), out + (size_t)f * L * TRAIN_ROW, TRAIN_ROW, nullptr, nullptr, 0};
            stages.pool = dpool;
            stages.sig_at = dsig + (size_t)f * L;
            stages.noise_at = dnoi + (size_t)f * L;
            return issue_frame(b, stages, false, ready);
        });
        if (rc) return -1;
        CK(cudaMemcpyAsync(rows + off * TRAIN_ROW, out, (size_t)nf * L * TRAIN_ROW * sizeof(float), cudaMemcpyDeviceToHost, b->c_in));
        CK(cudaStreamSynchronize(b->c_in));
    }
    return 0;
}

// ---- waveform windows (DESIGN.md §7k) -------------------------------------------------------------------------------
int rnnoise_train_reset(RNNoiseTrainer* t) {
    if (!t) return fail("null trainer");
    RNNoiseBatch* b = t->batch.get();
    ON_DEVICE(b->device);
    if (zero_state(b)) return -1;  // waits for every frame in flight; the 3L streams' history and high-pass memories
    if (trainer_defaults(t)) return -1;
    t->mode = TrainMode::kNone;
    return 0;
}

int rnnoise_train_pool_reserve(RNNoiseTrainer* t, long long n_samples) {
    if (!t) return fail("null trainer");
    if (n_samples < 0) return fail("negative pool size");
    RNNoiseBatch* b = t->batch.get();
    ON_DEVICE(b->device);
    const size_t bytes = (size_t)n_samples * sizeof(short);
    size_t room = 0, total_b = 0;
    if (rnnoise_train_pool_room(t, &room, &total_b)) return -1;
    if (bytes > room)
        return fail("a pool of " + std::to_string(n_samples) + " samples (" + std::to_string(bytes) + " bytes) does not fit on device " +
                    std::to_string(b->device) + ": " + std::to_string(room) + " bytes free of " + std::to_string(total_b));
    if (sync_all(b)) return -1;  // waveform frames in flight read the old pool
    t->pool.reset();
    t->pool_len = 0;
    if (n_samples == 0) return 0;
    const cudaError_t e = t->pool.alloc(bytes);
    if (e != cudaSuccess) return fail("a pool of " + std::to_string(bytes) + " bytes", e);
    CK(cudaMemset(t->pool.get(), 0, bytes));
    t->pool_len = n_samples;
    return 0;
}

int rnnoise_train_pool_write(RNNoiseTrainer* t, long long at, const short* src, long long n) {
    if (!t || (!src && n > 0)) return fail("null argument");
    if (at < 0 || n < 0 || at > t->pool_len || n > t->pool_len - at)
        return fail("pool write of " + std::to_string(n) + " samples at " + std::to_string(at) + " runs outside the pool of " +
                    std::to_string(t->pool_len) + " samples");
    if (n == 0) return 0;
    RNNoiseBatch* b = t->batch.get();
    ON_DEVICE(b->device);
    if (sync_all(b)) return -1;  // waveform frames in flight may read these samples
    CK(cudaMemcpy(t->pool.get<short>() + at, src, (size_t)n * sizeof(short), cudaMemcpyHostToDevice));
    return 0;
}

long long rnnoise_train_pool_samples(const RNNoiseTrainer* t) { return t ? t->pool_len : 0; }

int rnnoise_train_pool_room(const RNNoiseTrainer* t, size_t* room_bytes, size_t* total_bytes) {
    if (!t || !room_bytes || !total_bytes) return fail("null argument");
    ON_DEVICE(t->batch->device);
    CK(cudaMemGetInfo(room_bytes, total_bytes));
    *room_bytes += t->pool.bytes();
    return 0;
}

int rnnoise_train_waves_device(RNNoiseTrainer* t, const long long* sig_at, const long long* noise_at, int n_frames, float* noisy,
                               float* clean, float* noise, float* vad, long stream_stride, long frame_stride, long vad_stream_stride,
                               long vad_frame_stride, void* cuda_stream) {
    if (!t) return fail("null trainer");
    if (!sig_at || !noise_at || !noisy || !clean) return fail("null argument");
    if (n_frames < 0) return fail("negative n_frames");
    if (trainer_mode(t, TrainMode::kWaves)) return -1;
    if (t->pool_len == 0) return fail("no sample pool: rnnoise_train_pool_reserve and rnnoise_train_pool_write fill it first");
    const int L = t->tb.n_lanes;
    if (!rows_disjoint(L, n_frames, stream_stride, frame_stride, FRAME_SIZE)) return fail("sample strides overlap frames");
    if (vad && !rows_disjoint(L, n_frames, vad_stream_stride, vad_frame_stride, 1)) return fail("vad strides overlap");
    // the offsets come from outside the library: every one is checked before anything is uploaded or run
    const long long last = t->pool_len - FRAME_SIZE;
    for (int k = 0; k < 2; k++) {
        const long long* at = k ? noise_at : sig_at;
        for (size_t i = 0; i < (size_t)n_frames * L; i++)
            if (at[i] != -1 && (at[i] < 0 || at[i] > last))
                return fail(std::string(k ? "noise_at" : "sig_at") + " = " + std::to_string(at[i]) + " at frame " + std::to_string(i / L) +
                            ", lane " + std::to_string(i % L) + ": must be -1 or in [0, pool_len - 480 = " + std::to_string(last) + "]");
    }
    if (n_frames == 0) return 0;
    RNNoiseBatch* b = t->batch.get();
    ON_DEVICE(b->device);
    // slot k's offsets were last read by the call kWaveSlots calls ago: wait for it before overwriting them
    const int k = (int)(t->wave_calls % kWaveSlots);
    CK(cudaEventSynchronize(t->wave_done[k]));
    const size_t n_at = (size_t)n_frames * L, bytes = 2 * n_at * sizeof(long long);
    if (t->wave_host_bytes[k] < bytes) {
        t->wave_host[k].reset();
        t->wave_host_bytes[k] = 0;
        CK(cudaHostAlloc(t->wave_host[k].put(), bytes, cudaHostAllocDefault));
        t->wave_host_bytes[k] = bytes;
    }
    if (t->wave_at[k].bytes() < bytes) CK(t->wave_at[k].alloc(bytes));
    long long* h = static_cast<long long*>(static_cast<void*>(t->wave_host[k]));
    std::memcpy(h, sig_at, n_at * sizeof(long long));
    std::memcpy(h + n_at, noise_at, n_at * sizeof(long long));
    long long* d = t->wave_at[k].get<long long>();
    cudaStream_t s = b->st[0], us = (cudaStream_t)cuda_stream;
    if (wait_for_caller(s, us, t->wave_caller)) return -1;
    CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s));
    CK(launch_train_waves(b->buf, t->tb, t->pool.get<short>(), d, d + n_at, n_frames, noisy, clean, noise, vad, stream_stride, frame_stride,
                          vad_stream_stride, vad_frame_stride, s));
    count_launches(1);
    CK(cudaEventRecord(t->wave_done[k], s));
    t->wave_calls++;
    t->mode = TrainMode::kWaves;
    return resume_caller(s, us, t->wave_done[k]);
}

}  // extern "C"

extern "C" {

// ---- legacy single-stream API (src/capi.rs) = a batch of one ------------------------------------------
struct DenoiseState {
    RNNoiseBatch* batch;
};

int rnnoise_get_frame_size(void) { return FRAME_SIZE; }
int rnnoise_get_size(void) { return (int)sizeof(DenoiseState); }

int rnnoise_init(DenoiseState* st, RNNModel* model) {
    if (!st) return fail("null state");
    st->batch = rnnoise_batch_create(model, 1, -1);
    return st->batch ? 0 : -1;
}

DenoiseState* rnnoise_create(RNNModel* model) {
    std::unique_ptr<DenoiseState> st(new (std::nothrow) DenoiseState());
    if (!st || rnnoise_init(st.get(), model) != 0) return nullptr;
    return st.release();
}

void rnnoise_destroy(DenoiseState* st) {
    if (!st) return;
    rnnoise_batch_destroy(st->batch);
    delete st;
}

// A new batch of one with the original's model and device, given the original's state record.
DenoiseState* rnnoise_clone(const DenoiseState* st) {
    if (!st || !st->batch) {
        fail("null state");
        return nullptr;
    }
    RNNoiseBatch* src = st->batch;
    std::unique_ptr<DenoiseState> c(new (std::nothrow) DenoiseState());
    if (!c) {
        fail("out of memory");
        return nullptr;
    }
    BatchPtr b = create_batch(src->model, 1, src->device);
    if (!b) return nullptr;
    std::vector<unsigned char> rec(record_bytes(src));
    if (rnnoise_batch_get_states(src, nullptr, 1, rec.data(), nullptr) || rnnoise_batch_set_states(b.get(), nullptr, 1, rec.data(), nullptr))
        return nullptr;
    c->batch = b.release();
    return c.release();
}

float rnnoise_process_frame(DenoiseState* st, float* out, float* in) {
    if (!st || !st->batch) {
        fprintf(stderr, "rnnoise_process_frame: Invalid pointer\n");  // the reference panics (src/capi.rs:80)
        abort();
    }
    float vad = 0.0f;
    if (rnnoise_batch_process_host(st->batch, out, in, &vad, 1) != 0) {
        fprintf(stderr, "rnnoise_process_frame: %s\n", g_err.c_str());
        abort();  // no CPU fallback: a CUDA failure is fatal, like a panic across the FFI
    }
    return vad;
}

}  // extern "C"
