// host.cu -- host side of the C ABI declared in include/rnnoise.h: table construction, model upload,
// the batch handle that owns the per-stream device state, and the per-frame launch sequence
//   hp_filter -> pitch -> analysis -> rnn -> synthesis
// which together are DenoiseState::process_frame (src/denoise.rs:95-116) for n_streams streams.
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <algorithm>
#include <type_traits>
#include <utility>
#include <vector>

#include <cuda_fp16.h>

#include "../../include/rnnoise.h"
#include "common.cuh"
#include "model.hpp"

using namespace nnb;

struct RNNModel {
    HostModel m;
};

namespace {

thread_local std::string g_err;
std::atomic<unsigned long long> g_launches{0};

int fail(const std::string& what, cudaError_t e = cudaSuccess) {
    g_err = what;
    if (e != cudaSuccess) {
        g_err += ": ";
        g_err += cudaGetErrorString(e);
    }
    return -1;
}

}  // namespace

// used by frontend.cu
namespace nnb {
int set_error(const std::string& what) { return fail(what); }
void count_launches(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
}  // namespace nnb

namespace {

#define ON_DEVICE(dev)                                                   \
    DeviceGuard guard__(dev);                                            \
    if (guard__.err != cudaSuccess) return fail("cudaSetDevice", guard__.err)

#define CK(call)                                         \
    do {                                                 \
        cudaError_t e__ = (call);                        \
        if (e__ != cudaSuccess) return fail(#call, e__); \
    } while (0)

// ---- tables (src/lib.rs:99-136, src/util.rs:3-27) -------------------------------------------------
}  // namespace
namespace nnb {
extern const float kTansigTable[201] = {
    0.000000f, 0.039979f, 0.079830f, 0.119427f, 0.158649f, 0.197375f, 0.235496f, 0.272905f, 0.309507f, 0.345214f, 0.379949f,
    0.413644f, 0.446244f, 0.477700f, 0.507977f, 0.537050f, 0.564900f, 0.591519f, 0.616909f, 0.641077f, 0.664037f, 0.685809f,
    0.706419f, 0.725897f, 0.744277f, 0.761594f, 0.777888f, 0.793199f, 0.807569f, 0.821040f, 0.833655f, 0.845456f, 0.856485f,
    0.866784f, 0.876393f, 0.885352f, 0.893698f, 0.901468f, 0.908698f, 0.915420f, 0.921669f, 0.927473f, 0.932862f, 0.937863f,
    0.942503f, 0.946806f, 0.950795f, 0.954492f, 0.957917f, 0.961090f, 0.964028f, 0.966747f, 0.969265f, 0.971594f, 0.973749f,
    0.975743f, 0.977587f, 0.979293f, 0.980869f, 0.982327f, 0.983675f, 0.984921f, 0.986072f, 0.987136f, 0.988119f, 0.989027f,
    0.989867f, 0.990642f, 0.991359f, 0.992020f, 0.992631f, 0.993196f, 0.993718f, 0.994199f, 0.994644f, 0.995055f, 0.995434f,
    0.995784f, 0.996108f, 0.996407f, 0.996682f, 0.996937f, 0.997172f, 0.997389f, 0.997590f, 0.997775f, 0.997946f, 0.998104f,
    0.998249f, 0.998384f, 0.998508f, 0.998623f, 0.998728f, 0.998826f, 0.998916f, 0.999000f, 0.999076f, 0.999147f, 0.999213f,
    0.999273f, 0.999329f, 0.999381f, 0.999428f, 0.999472f, 0.999513f, 0.999550f, 0.999585f, 0.999617f, 0.999646f, 0.999673f,
    0.999699f, 0.999722f, 0.999743f, 0.999763f, 0.999781f, 0.999798f, 0.999813f, 0.999828f, 0.999841f, 0.999853f, 0.999865f,
    0.999875f, 0.999885f, 0.999893f, 0.999902f, 0.999909f, 0.999916f, 0.999923f, 0.999929f, 0.999934f, 0.999939f, 0.999944f,
    0.999948f, 0.999952f, 0.999956f, 0.999959f, 0.999962f, 0.999965f, 0.999968f, 0.999970f, 0.999973f, 0.999975f, 0.999977f,
    0.999978f, 0.999980f, 0.999982f, 0.999983f, 0.999984f, 0.999986f, 0.999987f, 0.999988f, 0.999989f, 0.999990f, 0.999990f,
    0.999991f, 0.999992f, 0.999992f, 0.999993f, 0.999994f, 0.999994f, 0.999994f, 0.999995f, 0.999995f, 0.999996f, 0.999996f,
    0.999996f, 0.999997f, 0.999997f, 0.999997f, 0.999997f, 0.999997f, 0.999998f, 0.999998f, 0.999998f, 0.999998f, 0.999998f,
    0.999998f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f, 0.999999f,
    0.999999f, 0.999999f, 0.999999f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f, 1.000000f,
    1.000000f, 1.000000f, 1.000000f,
};
}  // namespace nnb
namespace {
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
    volatile float acc = 0.0f;  // f32 sequential sum (src/lib.rs:116)
    for (int i = 0; i < WINDOW_SIZE; i++) acc = acc + t->window[i] * t->window[i];
    t->wnorm = 1.0f / acc;
    for (int i = 0; i < NB_BANDS; i++)
        for (int j = 0; j < NB_BANDS; j++) {
            float v = (float)std::cos(((double)i + 0.5) * (double)j * pi / (double)NB_BANDS);
            if (j == 0) v *= std::sqrt(0.5f);
            t->dct[i * NB_BANDS + j] = v;
        }
    for (int i = 0; i < 201; i++) t->tansig[i] = kTansigTable[i];
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

// ---- tensor-core formulation: weights packed in mma.sync m16n8k16 B-fragment order (see common.cuh MmaPhase) ----
struct Seg {
    int acol, len, recurrent, src_off;  // A column, valid rows, 0 = input matrix / 1 = recurrent matrix, first source row
};

inline int pad16(int n) { return (n + 15) & ~15; }
inline uint32_t pack_h2(int a, int b) {
    return (uint32_t)__half_as_ushort(__float2half((float)a)) | ((uint32_t)__half_as_ushort(__float2half((float)b)) << 16);
}

struct PhaseBuilder {
    std::vector<unsigned char> blob;  // host image of the device blob
    std::vector<std::pair<MmaPhase*, std::pair<size_t, size_t>>> fixups;  // phase, (wfrag offset, bias offset)

    // weight(i_seg_row, out_col) -> int8 value; nout valid outputs per gate; ngates gates laid out as consecutive tile groups
    template <typename WF, typename BF>
    void add(MmaPhase* ph, const std::vector<Seg>& segs, int nout, int ngates, WF weight, BF bias) {
        const int ot = (nout + 7) / 8;
        ph->ntiles = ngates * ot;
        ph->nchunks = 0;
        std::vector<std::pair<int, int>> chunks;  // (segment index, first row in segment)
        for (size_t si = 0; si < segs.size(); si++)
            for (int c = 0; c < pad16(segs[si].len); c += 16) {
                if (ph->nchunks >= MMA_MAX_CHUNKS) abort();
                ph->col[ph->nchunks++] = (short)(segs[si].acol + c);
                chunks.push_back({(int)si, c});
            }
        while (blob.size() % 16) blob.push_back(0);
        const size_t woff = blob.size();
        blob.resize(woff + (size_t)ph->nchunks * ph->ntiles * 32 * sizeof(uint2));
        uint2* wf = reinterpret_cast<uint2*>(blob.data() + woff);
        for (int kc = 0; kc < ph->nchunks; kc++) {
            const Seg& sg = segs[chunks[kc].first];
            const int r0 = chunks[kc].second;
            for (int nt = 0; nt < ph->ntiles; nt++) {
                const int gate = nt / ot, o0 = (nt % ot) * 8;
                for (int lane = 0; lane < 32; lane++) {
                    const int g = lane >> 2, t = lane & 3, n = o0 + g;
                    auto w = [&](int kr) -> int {
                        const int i = r0 + kr;
                        if (i >= sg.len || n >= nout) return 0;
                        return weight(sg, i, gate, n);
                    };
                    wf[((size_t)kc * ph->ntiles + nt) * 32 + lane] =
                        make_uint2(pack_h2(w(2 * t), w(2 * t + 1)), pack_h2(w(2 * t + 8), w(2 * t + 9)));
                }
            }
        }
        const size_t boff = blob.size();
        blob.resize(boff + (size_t)ph->ntiles * 8 * sizeof(float));
        float* bf = reinterpret_cast<float*>(blob.data() + boff);
        for (int nt = 0; nt < ph->ntiles; nt++)
            for (int j = 0; j < 8; j++) {
                const int gate = nt / ot, o = (nt % ot) * 8 + j;
                bf[nt * 8 + j] = o < nout ? (float)bias(gate, o) : 0.0f;
            }
        fixups.push_back({ph, {woff, boff}});
    }
};

// the nine phases of an mma.sync model
std::vector<MmaPhase*> mma_phases(DeviceModelMma* d) {
    return {&d->dense, &d->vad_zr, &d->vad_h, &d->vad_out, &d->noise_zr, &d->noise_h, &d->den_zr, &d->den_h, &d->out};
}

// The host image of the mma.sync model: until relocate_mma, d's fragment and bias pointers hold byte offsets into blob.
// *dp is zeroed first, so two descriptors of one layout are equal byte for byte.
void pack_model_mma(const HostModel& m, DeviceModelMma* dp, std::vector<unsigned char>* blob) {
    std::memset(dp, 0, sizeof *dp);
    DeviceModelMma& d = *dp;
    const int nd = m.input_dense.nn, nv = m.vad_gru.nn, nn = m.noise_gru.nn, ndn = m.denoise_gru.nn;
    d.nd = nd; d.nv = nv; d.nn = nn; d.ndn = ndn;
    d.act_dense = m.input_dense.act; d.act_vad = m.vad_gru.act; d.act_noise = m.noise_gru.act; d.act_den = m.denoise_gru.act;
    d.act_out = m.denoise_output.act; d.act_vadout = m.vad_output.act;
    d.c_feat = 0;
    d.c_dense = pad16(NB_FEATURES);
    d.c_vad = d.c_dense + pad16(nd);
    d.c_noise = d.c_vad + pad16(nv);
    d.c_den = d.c_noise + pad16(nn);
    d.c_rh = d.c_den + pad16(ndn);
    int cols = d.c_rh + pad16(std::max(nv, std::max(nn, ndn)));
    int kp = cols;
    while ((kp / 2) % 8 != 4) kp += 2;
    d.kp = kp;
    int hs = ((nv + 7) & ~7) + ((nn + 7) & ~7) + ((ndn + 7) & ~7);
    while (hs % 32 != 8) hs++;
    d.hs = hs;
    d.state_size = nv + nn + ndn;

    const int8_t* B = m.bytes.data();
    PhaseBuilder pb;
    auto dense_w = [&](const HostDense& L) {
        return [&, B](const Seg& sg, int i, int, int n) -> int { return B[L.w_off + (size_t)(sg.src_off + i) * L.nn + n]; };
    };
    auto dense_b = [&](const HostDense& L) { return [&, B](int, int o) -> int { return B[L.b_off + o]; }; };
    auto gru_w = [&](const HostGru& L, int gate0) {
        return [&, B, gate0](const Seg& sg, int i, int gate, int n) -> int {
            const size_t st3 = (size_t)3 * L.nn;
            const size_t base = sg.recurrent ? L.r_off : L.w_off;
            return B[base + (size_t)(sg.src_off + i) * st3 + (size_t)(gate0 + gate) * L.nn + n];
        };
    };
    auto gru_b = [&](const HostGru& L, int gate0) { return [&, B, gate0](int gate, int o) -> int { return B[L.b_off + (size_t)(gate0 + gate) * L.nn + o]; }; };

    pb.add(&d.dense, {{d.c_feat, NB_FEATURES, 0, 0}}, nd, 1, dense_w(m.input_dense), dense_b(m.input_dense));
    pb.add(&d.vad_zr, {{d.c_dense, nd, 0, 0}, {d.c_vad, nv, 1, 0}}, nv, 2, gru_w(m.vad_gru, 0), gru_b(m.vad_gru, 0));
    pb.add(&d.vad_h, {{d.c_dense, nd, 0, 0}, {d.c_rh, nv, 1, 0}}, nv, 1, gru_w(m.vad_gru, 2), gru_b(m.vad_gru, 2));
    pb.add(&d.vad_out, {{d.c_vad, nv, 0, 0}}, 1, 1, dense_w(m.vad_output), dense_b(m.vad_output));
    pb.add(&d.noise_zr, {{d.c_dense, nd, 0, 0}, {d.c_vad, nv, 0, nd}, {d.c_feat, NB_FEATURES, 0, nd + nv}, {d.c_noise, nn, 1, 0}}, nn, 2,
           gru_w(m.noise_gru, 0), gru_b(m.noise_gru, 0));
    pb.add(&d.noise_h, {{d.c_dense, nd, 0, 0}, {d.c_vad, nv, 0, nd}, {d.c_feat, NB_FEATURES, 0, nd + nv}, {d.c_rh, nn, 1, 0}}, nn, 1,
           gru_w(m.noise_gru, 2), gru_b(m.noise_gru, 2));
    pb.add(&d.den_zr, {{d.c_vad, nv, 0, 0}, {d.c_noise, nn, 0, nv}, {d.c_feat, NB_FEATURES, 0, nv + nn}, {d.c_den, ndn, 1, 0}}, ndn, 2,
           gru_w(m.denoise_gru, 0), gru_b(m.denoise_gru, 0));
    pb.add(&d.den_h, {{d.c_vad, nv, 0, 0}, {d.c_noise, nn, 0, nv}, {d.c_feat, NB_FEATURES, 0, nv + nn}, {d.c_rh, ndn, 1, 0}}, ndn, 1,
           gru_w(m.denoise_gru, 2), gru_b(m.denoise_gru, 2));
    pb.add(&d.out, {{d.c_den, ndn, 0, 0}}, NB_BANDS, 1, dense_w(m.denoise_output), dense_b(m.denoise_output));
    for (auto& f : pb.fixups) {
        f.first->wfrag = reinterpret_cast<const uint2*>(f.second.first);
        f.first->bias = reinterpret_cast<const float*>(f.second.second);
    }
    *blob = std::move(pb.blob);
}

// the packed model's offsets -> pointers into its image at `base`
void relocate_mma(DeviceModelMma* d, const unsigned char* base) {
    for (MmaPhase* ph : mma_phases(d)) {
        ph->wfrag = reinterpret_cast<const uint2*>(base + reinterpret_cast<uintptr_t>(ph->wfrag));
        ph->bias = reinterpret_cast<const float*>(base + reinterpret_cast<uintptr_t>(ph->bias));
    }
}

}  // namespace

// ---- the batch handle -----------------------------------------------------------------------------------
constexpr int kNumKernels = 5;
const char* const kKernelNames[kNumKernels] = {"hp_filter", "pitch", "analysis", "rnn", "synthesis"};
constexpr int kEvRing = 16;  // events are recycled after 16 frames (PIPE_DEPTH << 16)

// Which model each row of a frame runs on (DESIGN.md 7c): one model for all rows, or rows grouped by model into tiles.
struct ModelRoute {
    int uniform = 0;                  // the model of every row, or -1: several models, see the tile table
    std::vector<int> h_rows;          // host images of the two tables
    std::vector<ModelTile> h_tiles;
    int* d_rows = nullptr;            // device tables (ModelTiles)
    ModelTile* d_tiles = nullptr;
    size_t rows_cap = 0, tiles_cap = 0;
};

struct RNNoiseBatch {
    int device = 0;
    int n_streams = 0;
    // Frame pipeline: stage i of every frame runs on st[i], so K_i(f) -> K_i(f+1) is stream order; K_{i-1}(f) ->
    // K_i(f) and the back-pressure K_4(f - PIPE_DEPTH) -> K_0(f) are events.  At small batches one kernel cannot
    // fill 132 SMs; overlapping the five stages of up to four consecutive frames does.
    cudaStream_t st[kNumKernels] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    int n_stages = kNumKernels;  // stages per frame: the denoise path's five, or a trainer's four (its last stage ends a frame)
    cudaStream_t c_in = nullptr, c_out = nullptr;  // host-API copy streams
    cudaEvent_t ev[kNumKernels][kEvRing];
    cudaEvent_t ev_in[kEvRing], ev_call = nullptr;
    bool events_ok = false;
    BatchBuffers buf{};  // persistent state + set 0 of the intermediates
    std::vector<void*> allocs;
    DeviceTables* d_tab = nullptr;
    // The GRU kernel, chosen at creation: wgmma when model 0 fits its budget, else (or with NNB_RNN_MMA=1) mma.sync
    bool gru_tc = false;
    int pitch_exact = 0;  // NNB_PITCH_EXACT=1: every stream takes the pitch kernel's order-exact recomputation paths (2: coarse only, 3: ladder only)
    // Two frame counters; without subset calls they are equal.
    unsigned long long seq = 0;    // frames issued, full-batch or subset: intermediate set seq % PIPE_DEPTH, event ring, back-pressure
    unsigned long long phase = 0;  // full-batch frames: ring slot phase % HIST_SLOTS of the batch's own streams
    bool taps_subset = false;      // the most recent frame was a subset frame: its intermediates do not describe the batch's rows
    // host-call staging: kStageSlots frames of device memory, recycled while a call of any length streams through
    // (sized for the sample type in use only: float or int16)
    char* stage_in = nullptr;
    char* stage_out = nullptr;
    float* stage_vad = nullptr;
    size_t stage_bytes = 0;  // per buffer
    cudaEvent_t ev_out[8];   // D2H copy of the frame that last used staging slot k
    int slot_ev[8];          // event-ring index of the frame that last used staging slot k
    // per-stream state records (state.cu): the gather / scatter kernels run on st[0], ahead of the next frame's stage 0
    HostModel model;                        // the batch's model, for rnnoise_clone; its GRU widths fix the record format
    int* d_idx = nullptr;                   // stream indices of the most recent state call
    int idx_cap = 0;
    unsigned char* rec_stage = nullptr;     // records of host-memory calls
    size_t rec_stage_bytes = 0;
    int* d_first_bad = nullptr;             // validation of device-resident records
    cudaEvent_t ev_state = nullptr;         // end of the most recent state call on st[0]
    // subset calls (rnnoise_batch_process_streams_*): the listed streams' persistent state is gathered into rows 0..n-1 of
    // the work state, advanced there by the unchanged frame kernels, and scattered back
    BatchBuffers work{};                    // persistent buffers only (intermediates: the batch's own sets); n_streams = rows in use
    int work_cap = 0;                       // rows allocated (high-water n)
    unsigned long long work_frames = 0;     // frames of the current subset call issued so far: work ring slot (phase + work_frames) % 8
    // model table (rnnoise_batch_add_model; DESIGN.md 7c): models of the batch model's geometry, model 0 = `model`.  Their
    // images for the batch's GRU kernel lie `mtab_stride` bytes apart in d_mtab.  Every model's descriptor is model 0's
    // with its own activation codes and image (launch_rnn).
    std::vector<int> model_acts;            // activation codes of each model, packed as ModelTile::acts
    unsigned char* d_mtab = nullptr;
    size_t mtab_bytes = 0;                  // bytes of each image
    size_t mtab_stride = 0;                 // mtab_bytes rounded up to 256
    size_t mtab_cap = 0;                    // models d_mtab has room for
    union {                                 // model 0's descriptor for the batch's kernel, in offset form
        DeviceModelTc tc0;                  // gru_tc: blob unset
        DeviceModelMma mma0;                // !gru_tc: fragment and bias pointers hold offsets into the image
    };
    std::vector<int> stream_model;          // host mirror: the model of every stream
    ModelRoute route;                       // full-batch frames
    ModelRoute work_route;                  // frames of the current subset call (rows = work rows)
};
constexpr int kStageSlots = 8;  // >= PIPE_DEPTH frames in the kernels + frames in the two copy engines

namespace {

template <typename T>
int dalloc(RNNoiseBatch* b, T** p, size_t count) {
    void* q = nullptr;
    CK(cudaMalloc(&q, count * sizeof(T)));
    b->allocs.push_back(q);
    *p = reinterpret_cast<T*>(q);
    return 0;
}

int model_acts(const HostModel& m) {
    const int a[6] = {m.input_dense.act, m.vad_gru.act, m.noise_gru.act, m.denoise_gru.act, m.denoise_output.act, m.vad_output.act};
    int acts = 0;
    for (int i = 0; i < 6; i++) acts |= a[i] << (4 * i);
    return acts;
}

// intermediates of frame f live in set f % PIPE_DEPTH
BatchBuffers view(const RNNoiseBatch* b, unsigned long long f) {
    BatchBuffers v = b->buf;
    const size_t k = (size_t)(f % PIPE_DEPTH), B = (size_t)b->n_streams;
    v.X += k * B * FREQ_SIZE;
    v.P += k * B * NB_BINS_BANDED;
    v.ex += k * B * NB_BANDS;
    v.ep += k * B * NB_BANDS;
    v.exp += k * B * NB_BANDS;
    v.features += k * B * NB_FEATURES;
    v.silence += k * B;
    v.pitch += k * B;
    v.gains += k * B * NB_BANDS;
    v.vad += k * B;
    return v;
}

// a frame of a subset call: intermediates of set f % PIPE_DEPTH (rows 0..n-1), persistent state of the work rows
BatchBuffers work_view(const RNNoiseBatch* b, unsigned long long f) {
    BatchBuffers v = view(b, f);
    const BatchBuffers& w = b->work;
    v.n_streams = w.n_streams;
    v.hist = w.hist;
    v.hp_mem = w.hp_mem;
    v.synth_mem = w.synth_mem;
    v.ceps_mem = w.ceps_mem;
    v.ceps_id = w.ceps_id;
    v.last_period = w.last_period;
    v.last_gain = w.last_gain;
    v.gru_state = w.gru_state;
    v.lastg = w.lastg;
    return v;
}

int sync_all(RNNoiseBatch* b) {
    for (int i = 0; i < kNumKernels; i++) CK(cudaStreamSynchronize(b->st[i]));
    CK(cudaStreamSynchronize(b->c_in));
    CK(cudaStreamSynchronize(b->c_out));
    return 0;
}

int zero_state(RNNoiseBatch* b) {
    const size_t B = (size_t)b->n_streams, D = PIPE_DEPTH;
    BatchBuffers& u = b->buf;
    const int SS = b->model.state_size();
    if (sync_all(b)) return -1;
    cudaStream_t s = b->st[0];
    CK(cudaMemsetAsync(u.hist, 0, B * HIST_CAP * sizeof(float), s));
    CK(cudaMemsetAsync(u.hp_mem, 0, B * 2 * sizeof(float), s));
    CK(cudaMemsetAsync(u.synth_mem, 0, B * FRAME_SIZE * sizeof(float), s));
    CK(cudaMemsetAsync(u.ceps_mem, 0, B * CEPS_MEM * NB_BANDS * sizeof(float), s));
    CK(cudaMemsetAsync(u.ceps_id, 0, B * sizeof(int32_t), s));
    CK(cudaMemsetAsync(u.last_period, 0, B * sizeof(int32_t), s));
    CK(cudaMemsetAsync(u.last_gain, 0, B * sizeof(float), s));
    CK(cudaMemsetAsync(u.gru_state, 0, B * SS * sizeof(float), s));
    CK(cudaMemsetAsync(u.lastg, 0, B * NB_BANDS * sizeof(float), s));
    CK(cudaMemsetAsync(u.gains, 0, D * B * NB_BANDS * sizeof(float), s));
    CK(cudaMemsetAsync(u.vad, 0, D * B * sizeof(float), s));
    CK(cudaMemsetAsync(u.silence, 0, D * B * sizeof(int32_t), s));
    CK(cudaMemsetAsync(u.pitch, 0, D * B * sizeof(int32_t), s));
    CK(cudaMemsetAsync(u.features, 0, D * B * NB_FEATURES * sizeof(float), s));
    b->seq = b->phase = 0;
    b->taps_subset = false;
    CK(cudaStreamSynchronize(s));
    return 0;
}

// Picks the batch's GRU kernel and uploads model 0, packed for that kernel only, as entry 0 of the model table.  The
// table has room for one more model; its capacity doubles whenever rnnoise_batch_add_model finds it full.
int init_model_table(RNNoiseBatch* b, const HostModel& hm) {
    const char* e = getenv("NNB_RNN_MMA");
    std::vector<unsigned char> img;
    b->gru_tc = !(e && e[0] == '1') && pack_model_tc(hm, &b->tc0, &img);
    if (!b->gru_tc) pack_model_mma(hm, &b->mma0, &img);
    b->mtab_bytes = img.size();
    b->mtab_stride = (img.size() + 255) & ~(size_t)255;
    b->mtab_cap = 2;
    CK(cudaMalloc(&b->d_mtab, b->mtab_stride * b->mtab_cap));
    CK(cudaMemcpyAsync(b->d_mtab, img.data(), img.size(), cudaMemcpyHostToDevice, b->st[0]));
    CK(cudaStreamSynchronize(b->st[0]));
    return 0;
}

int batch_init(RNNoiseBatch* b, const HostModel& hm, int n_streams, int device) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return fail("no CUDA device available (this library has no CPU fallback)", e);
    if (device < 0) CK(cudaGetDevice(&device));
    if (device >= ndev) return fail("device index out of range");
    if (n_streams <= 0) return fail("n_streams must be positive");
    CK(cudaSetDevice(device));
    b->device = device;
    b->n_streams = n_streams;
    for (int i = 0; i < kNumKernels; i++) CK(cudaStreamCreateWithFlags(&b->st[i], cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&b->c_in, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&b->c_out, cudaStreamNonBlocking));
    for (int i = 0; i < kNumKernels; i++)
        for (int k = 0; k < kEvRing; k++) CK(cudaEventCreateWithFlags(&b->ev[i][k], cudaEventDisableTiming));
    for (int k = 0; k < kEvRing; k++) CK(cudaEventCreateWithFlags(&b->ev_in[k], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&b->ev_call, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&b->ev_state, cudaEventDisableTiming));
    for (int k = 0; k < kStageSlots; k++) CK(cudaEventCreateWithFlags(&b->ev_out[k], cudaEventDisableTiming));
    b->events_ok = true;
    b->model = hm;
    b->model_acts.assign(1, model_acts(hm));
    b->stream_model.assign((size_t)n_streams, 0);
    const size_t B = (size_t)n_streams, D = PIPE_DEPTH;
    BatchBuffers& u = b->buf;
    u.n_streams = n_streams;
    if (init_model_table(b, hm)) return -1;
    {
        const char* e3 = getenv("NNB_PITCH_EXACT");
        b->pitch_exact = !e3 ? 0 : (e3[0] == '1' ? 3 : (e3[0] == '2' ? 1 : (e3[0] == '3' ? 2 : 0)));
    }
    const int SS = b->model.state_size();
    if (dalloc(b, &u.hist, B * HIST_CAP) || dalloc(b, &u.hp_mem, B * 2) || dalloc(b, &u.synth_mem, B * FRAME_SIZE) ||
        dalloc(b, &u.ceps_mem, B * CEPS_MEM * NB_BANDS) || dalloc(b, &u.ceps_id, B) || dalloc(b, &u.last_period, B) ||
        dalloc(b, &u.last_gain, B) || dalloc(b, &u.gru_state, B * SS) || dalloc(b, &u.lastg, B * NB_BANDS) ||
        dalloc(b, &u.X, D * B * FREQ_SIZE) || dalloc(b, &u.P, D * B * NB_BINS_BANDED) || dalloc(b, &u.ex, D * B * NB_BANDS) ||
        dalloc(b, &u.ep, D * B * NB_BANDS) || dalloc(b, &u.exp, D * B * NB_BANDS) || dalloc(b, &u.features, D * B * NB_FEATURES) ||
        dalloc(b, &u.silence, D * B) || dalloc(b, &u.pitch, D * B) || dalloc(b, &u.gains, D * B * NB_BANDS) ||
        dalloc(b, &u.vad, D * B) || dalloc(b, &b->d_tab, 1) || dalloc(b, &u.pitch_stats, 3) || dalloc(b, &b->d_first_bad, 1))
        return -1;
    CK(cudaMemsetAsync(u.pitch_stats, 0, 3 * sizeof(unsigned long long), b->st[0]));
    DeviceTables* ht = new DeviceTables();
    build_tables(ht);
    cudaError_t ce = cudaMemcpyAsync(b->d_tab, ht, sizeof(DeviceTables), cudaMemcpyHostToDevice, b->st[0]);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(b->st[0]);
    delete ht;
    if (ce != cudaSuccess) return fail("table upload", ce);
    return zero_state(b);
}

void free_stage(RNNoiseBatch* b) {
    if (b->stage_in) cudaFree(b->stage_in);
    if (b->stage_out) cudaFree(b->stage_out);
    if (b->stage_vad) cudaFree(b->stage_vad);
    b->stage_in = b->stage_out = nullptr;
    b->stage_vad = nullptr;
    b->stage_bytes = 0;
}

void free_work(RNNoiseBatch* b) {
    BatchBuffers& w = b->work;
    for (void* p : {(void*)w.hist, (void*)w.hp_mem, (void*)w.synth_mem, (void*)w.ceps_mem, (void*)w.ceps_id, (void*)w.last_period,
                    (void*)w.last_gain, (void*)w.gru_state, (void*)w.lastg})
        if (p) cudaFree(p);
    w = BatchBuffers{};
    b->work_cap = 0;
}

// The work state of subset calls, grown to n rows.  Zeroed once when allocated: rows and ring positions a call does not
// gather are never read by the frame kernels, but they are then defined.
int ensure_work(RNNoiseBatch* b, int n) {
    if (n <= b->work_cap) return 0;
    if (sync_all(b)) return -1;
    free_work(b);
    const size_t N = (size_t)n, SS = (size_t)b->model.state_size();
    BatchBuffers& w = b->work;
    cudaStream_t s = b->st[0];
    auto get = [&](auto** p, size_t count) {
        void* q = nullptr;
        cudaError_t e = cudaMalloc(&q, count * sizeof(**p));
        if (e == cudaSuccess) e = cudaMemsetAsync(q, 0, count * sizeof(**p), s);
        *p = reinterpret_cast<std::remove_reference_t<decltype(*p)>>(q);
        return e;
    };
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess) e = get(&w.hist, N * HIST_CAP);
    if (e == cudaSuccess) e = get(&w.hp_mem, N * 2);
    if (e == cudaSuccess) e = get(&w.synth_mem, N * FRAME_SIZE);
    if (e == cudaSuccess) e = get(&w.ceps_mem, N * CEPS_MEM * NB_BANDS);
    if (e == cudaSuccess) e = get(&w.ceps_id, N);
    if (e == cudaSuccess) e = get(&w.last_period, N);
    if (e == cudaSuccess) e = get(&w.last_gain, N);
    if (e == cudaSuccess) e = get(&w.gru_state, N * std::max<size_t>(SS, 1));
    if (e == cudaSuccess) e = get(&w.lastg, N * NB_BANDS);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        free_work(b);
        return fail("work state of " + std::to_string(n) + " streams", e);
    }
    b->work_cap = n;
    return 0;
}

void batch_release(RNNoiseBatch* b) {
    if (!b) return;
    DeviceGuard guard(b->device);
    for (int i = 0; i < kNumKernels; i++)
        if (b->st[i]) cudaStreamSynchronize(b->st[i]);
    if (b->c_in) cudaStreamSynchronize(b->c_in);
    if (b->c_out) cudaStreamSynchronize(b->c_out);
    for (void* p : b->allocs) cudaFree(p);
    b->allocs.clear();
    free_stage(b);
    free_work(b);
    if (b->d_idx) cudaFree(b->d_idx);
    if (b->rec_stage) cudaFree(b->rec_stage);
    if (b->d_mtab) cudaFree(b->d_mtab);
    b->d_mtab = nullptr;
    for (ModelRoute* r : {&b->route, &b->work_route}) {
        if (r->d_rows) cudaFree(r->d_rows);
        if (r->d_tiles) cudaFree(r->d_tiles);
        r->d_rows = nullptr;
        r->d_tiles = nullptr;
    }
    b->d_idx = nullptr;
    b->rec_stage = nullptr;
    if (b->events_ok) {
        for (int i = 0; i < kNumKernels; i++)
            for (int k = 0; k < kEvRing; k++) cudaEventDestroy(b->ev[i][k]);
        for (int k = 0; k < kEvRing; k++) cudaEventDestroy(b->ev_in[k]);
        for (int k = 0; k < kStageSlots; k++) cudaEventDestroy(b->ev_out[k]);
        cudaEventDestroy(b->ev_call);
        cudaEventDestroy(b->ev_state);
        b->events_ok = false;
    }
    for (int i = 0; i < kNumKernels; i++)
        if (b->st[i]) {
            cudaStreamDestroy(b->st[i]);
            b->st[i] = nullptr;
        }
    if (b->c_in) cudaStreamDestroy(b->c_in);
    if (b->c_out) cudaStreamDestroy(b->c_out);
    b->c_in = b->c_out = nullptr;
}

int ensure_stage(RNNoiseBatch* b, bool pcm) {
    const size_t need = (size_t)kStageSlots * b->n_streams * FRAME_SIZE * (pcm ? sizeof(short) : sizeof(float));
    if (need > b->stage_bytes) {
        if (sync_all(b)) return -1;
        free_stage(b);
        CK(cudaMalloc(&b->stage_in, need));
        CK(cudaMalloc(&b->stage_out, need));
        CK(cudaMalloc(&b->stage_vad, (size_t)kStageSlots * b->n_streams * sizeof(float)));
        b->stage_bytes = need;
    }
    return 0;
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

// A descriptor's six activation codes, given packed as ModelTile::acts.
template <typename DeviceModel>
void set_acts(DeviceModel* d, int acts) {
    d->act_dense = tile_act(acts, 0);
    d->act_vad = tile_act(acts, 1);
    d->act_noise = tile_act(acts, 2);
    d->act_den = tile_act(acts, 3);
    d->act_out = tile_act(acts, 4);
    d->act_vadout = tile_act(acts, 5);
}

// The five stages of a denoise frame: hp_filter -> pitch -> analysis -> rnn -> synthesis.
// The GRU stage of a frame: the one-model kernel with the model of every row, or the tiled kernel with model 0's
// descriptor over the route's table.  Model k's descriptor is model 0's with model k's activation codes, pointed at
// image k of the table.
int launch_rnn(const RNNoiseBatch* b, const BatchBuffers& v, const ModelRoute& r, cudaStream_t s) {
    const size_t k = (size_t)std::max(r.uniform, 0);
    const unsigned char* img = b->d_mtab + k * b->mtab_stride;
    const ModelTiles mt{r.d_tiles, r.d_rows, (int)r.h_tiles.size(), (uint32_t)b->mtab_stride};
    if (b->gru_tc) {
        DeviceModelTc m = b->tc0;
        set_acts(&m, b->model_acts[k]);
        m.blob = img;
        if (r.uniform >= 0) CK(launch_rnn_tc(v, m, s));
        else CK(launch_rnn_tc_multi(v, m, mt, s));
    } else {
        DeviceModelMma m = b->mma0;
        set_acts(&m, b->model_acts[k]);
        relocate_mma(&m, img);
        if (r.uniform >= 0) CK(launch_rnn_mma(v, m, b->d_tab, s));
        else CK(launch_rnn_mma_multi(v, m, b->d_tab, mt, s));
    }
    return 0;
}

struct DenoiseStages {
    const RNNoiseBatch* b;
    FrameIO io;
    bool work = false;  // the frame advances a subset call's work rows

    int operator()(int i, const BatchBuffers& v, int slot, cudaStream_t s) const {
        switch (i) {
            case 0: CK(launch_hp_filter(v, io.in, (io.fmt & kFmtPcmIn) != 0, io.stream_stride, io.sample_stride, slot, s)); break;
            case 1: CK(launch_pitch(v, slot, b->pitch_exact, s)); break;
            case 2: CK(launch_analysis_warp(v, b->d_tab, slot, s)); break;
            case 3:
                if (launch_rnn(b, v, work ? b->work_route : b->route, s)) return -1;
                break;
            default:
                CK(launch_synthesis_warp(v, b->d_tab, io.out, (io.fmt & kFmtPcmOut) != 0, io.stream_stride, io.sample_stride, io.vad, s));
                break;
        }
        return 0;
    }
};

// Issues one frame: launch(i, v, slot, s) launches stage i of the batch's n_stages on stream s, for the frame's buffers v
// and history ring slot.  Stage i runs on st[i], after stage i-1 of the frame (event ev[i-1][seq % kEvRing]); stage 0
// runs after in_ready (optional) and after the last stage of frame seq - PIPE_DEPTH, whose intermediate set it reuses.
// work_rows: the frame advances the work rows of a subset call, whose ring continues the batch's phase.
// one (optional): every stage runs on this stream instead.  The caller orders it after the batch's earlier work and later
// work after it; the ring events are recorded all the same.  tev (optional): n_stages + 1 timing events around the stages.
template <typename Launch>
int issue_frame(RNNoiseBatch* b, const Launch& launch, bool work_rows, cudaEvent_t in_ready, cudaStream_t one = nullptr,
                cudaEvent_t* tev = nullptr) {
    const unsigned long long f = b->seq;
    const int n = b->n_stages, e = (int)(f % kEvRing);
    const int slot = (int)((work_rows ? b->phase + b->work_frames : b->phase) % HIST_SLOTS);
    const BatchBuffers v = work_rows ? work_view(b, f) : view(b, f);
    auto S = [&](int i) { return one ? one : b->st[i]; };
    if (in_ready) CK(cudaStreamWaitEvent(S(0), in_ready, 0));
    if (f >= (unsigned long long)PIPE_DEPTH) CK(cudaStreamWaitEvent(S(0), b->ev[n - 1][(int)((f - PIPE_DEPTH) % kEvRing)], 0));
    for (int i = 0; i < n; i++) {
        if (!one && i > 0) CK(cudaStreamWaitEvent(S(i), b->ev[i - 1][e], 0));
        if (tev) CK(cudaEventRecord(tev[i], S(i)));
        if (launch(i, v, slot, S(i))) return -1;
        CK(cudaEventRecord(b->ev[i][e], S(i)));
    }
    if (tev) CK(cudaEventRecord(tev[n], S(n - 1)));
    g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed);
    b->seq++;
    if (work_rows) b->work_frames++;
    else b->phase++;
    b->taps_subset = work_rows;
    return 0;
}

// Join: make `s` wait for everything issued so far on the stage streams.
int join_into(RNNoiseBatch* b, cudaStream_t s) {
    if (b->seq == 0) return 0;
    // the last stage follows every earlier kernel of its frame; earlier frames precede it in stream order per stage
    CK(cudaStreamWaitEvent(s, b->ev[b->n_stages - 1][(int)((b->seq - 1) % kEvRing)], 0));
    return 0;
}

int subset_begin(RNNoiseBatch* b, const int* streams, int n, cudaStream_t us);
int subset_end(RNNoiseBatch* b, const int* streams, int n);
int state_call_end(RNNoiseBatch* b, cudaStream_t us);

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
    if (subset) return subset_end(b, streams, n) ? -1 : state_call_end(b, us);
    if (us) return join_into(b, us);
    CK(cudaStreamSynchronize(b->st[b->n_stages - 1]));
    return 0;
}

// copy(v, B) reads the intermediates v of the most recent full-batch frame of the batch's B streams, after every frame
// issued so far has finished.
template <typename Copy>
int read_taps(RNNoiseBatch* b, const Copy& copy) {
    if (!b) return fail("null batch");
    ON_DEVICE(b->device);
    if (b->taps_subset) return fail("the most recent frame was a subset frame: taps describe full-batch frames only");
    if (sync_all(b)) return -1;
    return copy(view(b, b->seq ? b->seq - 1 : 0), (size_t)b->n_streams);
}

}  // namespace

// ============================================================================================== C ABI
extern "C" {

const char* rnnoise_last_error(void) { return g_err.c_str(); }
unsigned long long rnnoise_kernel_launches(void) { return g_launches.load(); }

RNNModel* rnnoise_model_from_bytes(const unsigned char* bytes, size_t len) {
    RNNModel* m = new (std::nothrow) RNNModel();
    if (!m) return nullptr;
    if (!bytes || !HostModel::parse(bytes, len, &m->m)) {
        delete m;
        fail("model bytes rejected (src/rnn.rs:116-232 validation)");
        return nullptr;
    }
    return m;
}

RNNModel* rnnoise_model_from_text(const char* text, size_t len) {
    RNNModel* m = new (std::nothrow) RNNModel();
    if (!m) return nullptr;
    if (!text || !HostModel::parse_text(text, len, &m->m)) {
        delete m;
        fail("text model rejected");
        return nullptr;
    }
    return m;
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
    RNNoiseBatch* b = new (std::nothrow) RNNoiseBatch();
    if (!b) return nullptr;
    const HostModel& hm = model ? model->m : HostModel::builtin();
    int prev_dev = -1;
    cudaGetDevice(&prev_dev);  // batch_init selects the batch's device; the caller's current device is restored below
    const int rc = batch_init(b, hm, n_streams, device);
    if (prev_dev >= 0) cudaSetDevice(prev_dev);
    if (rc != 0) {
        std::string keep = g_err;
        batch_release(b);
        delete b;
        g_err = keep;
        return nullptr;
    }
    return b;
}

void rnnoise_batch_destroy(RNNoiseBatch* b) {
    if (!b) return;
    batch_release(b);
    delete b;
}

int rnnoise_batch_streams(const RNNoiseBatch* b) { return b ? b->n_streams : 0; }

int rnnoise_batch_reset(RNNoiseBatch* b) {
    if (!b) return fail("null batch");
    ON_DEVICE(b->device);
    return zero_state(b);
}

static int process_device_impl(RNNoiseBatch* b, const FrameIO& io, int n_frames, long frame_stride, void* cuda_stream) {
    if (!b || !io.out || !io.in) return fail("null argument");
    if (io.sample_stride < 1) return fail("sample_stride must be >= 1");
    if (n_frames < 0) return fail("negative n_frames");
    if (n_frames == 0) return 0;
    ON_DEVICE(b->device);
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

const char* rnnoise_kernel_name(int i) { return (i >= 0 && i < kNumKernels) ? kKernelNames[i] : nullptr; }

int rnnoise_batch_profile_step(RNNoiseBatch* b, float* out, const float* in, float* vad, long stream_stride, void* cuda_stream,
                               float* ms, int cap) {
    if (!b || !out || !in || !ms) return fail("null argument");
    if (cap < kNumKernels) return fail("ms[] too small");
    ON_DEVICE(b->device);
    if (sync_all(b)) return -1;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : b->st[0];
    cudaEvent_t ev[kNumKernels + 1];
    for (int i = 0; i <= kNumKernels; i++) CK(cudaEventCreate(&ev[i]));
    int rc = issue_frame(b, DenoiseStages{b, {out, in, kFmtF32, vad, stream_stride, 1}}, false, nullptr, st, ev);
    if (rc == 0) {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) rc = fail("profile_step sync", e);
    }
    if (rc == 0)
        for (int i = 0; i < kNumKernels; i++) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
    for (int i = 0; i <= kNumKernels; i++) cudaEventDestroy(ev[i]);
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
    if (ensure_stage(b, pcm)) return -1;
    const size_t B = (size_t)(subset ? b->work.n_streams : b->n_streams), fs = B * FRAME_SIZE;
    const size_t esz = pcm ? sizeof(short) : sizeof(float);
    char* din = b->stage_in;
    char* dout = b->stage_out;
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
        const FrameIO io{dout + k * fs * esz, din + k * fs * esz, pcm ? kFmtPcm : kFmtF32, b->stage_vad + (size_t)k * B, FRAME_SIZE, 1};
        if (issue_frame(b, DenoiseStages{b, io, subset}, subset, b->ev_in[e])) return -1;
        CK(cudaStreamWaitEvent(b->c_out, b->ev[last][e], 0));
        CK(cudaMemcpyAsync((char*)out + (size_t)t * fs * esz, dout + k * fs * esz, fs * esz, cudaMemcpyDeviceToHost, b->c_out));
        if (vad) CK(cudaMemcpyAsync(vad + (size_t)t * B, b->stage_vad + (size_t)k * B, B * sizeof(float), cudaMemcpyDeviceToHost, b->c_out));
        CK(cudaEventRecord(b->ev_out[k], b->c_out));
        b->slot_ev[k] = e;
    }
    CK(cudaStreamSynchronize(b->c_out));
    CK(cudaStreamSynchronize(b->c_in));
    return 0;
}

int rnnoise_batch_process_host(RNNoiseBatch* b, float* out, const float* in, float* vad, int n_frames) {
    if (!b || !out || !in) return fail("null argument");
    if (n_frames <= 0) return n_frames == 0 ? 0 : fail("negative n_frames");
    ON_DEVICE(b->device);
    return process_host_impl(b, out, in, false, vad, n_frames);
}

int rnnoise_batch_process_pcm16_host(RNNoiseBatch* b, short* out, const short* in, float* vad, int n_frames) {
    if (!b || !out || !in) return fail("null argument");
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

int check_streams(const RNNoiseBatch* b, const int* streams, int n) {
    if (n < 0) return fail("negative number of streams");
    if (!streams) return n <= b->n_streams ? 0 : fail("more streams than the batch holds");
    std::vector<char> seen((size_t)b->n_streams, 0);
    for (int i = 0; i < n; i++) {
        const int s = streams[i];
        if (s < 0 || s >= b->n_streams) return fail("stream index " + std::to_string(s) + " out of range");
        if (seen[(size_t)s]) return fail("stream index " + std::to_string(s) + " given twice");
        seen[(size_t)s] = 1;
    }
    return 0;
}

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
    if (us) {
        CK(cudaEventRecord(b->ev_call, us));
        CK(cudaStreamWaitEvent(s, b->ev_call, 0));
    }
    if (join_into(b, s)) return -1;
    *d_idx = nullptr;
    if (!streams) return 0;
    if (n > b->idx_cap) {  // every user of d_idx runs on st[0]
        CK(cudaStreamSynchronize(s));
        if (b->d_idx) cudaFree(b->d_idx);
        b->d_idx = nullptr;
        b->idx_cap = 0;
        CK(cudaMalloc(&b->d_idx, (size_t)n * sizeof(int)));
        b->idx_cap = n;
    }
    CK(cudaMemcpyAsync(b->d_idx, streams, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    *d_idx = b->d_idx;
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
    const int T = b->gru_tc ? TC_TILE_ROWS : MMA_TILE_ROWS;
    std::vector<ModelTile> tiles;
    for (size_t k = 0; k < K; k++)
        for (int f = start[k]; f < start[k + 1]; f += T) tiles.push_back({(int)k, f, std::min(T, start[k + 1] - f), b->model_acts[k]});
    if (join_into(b, b->st[0])) return -1;
    if (n > r->rows_cap || tiles.size() > r->tiles_cap) {  // frames issued earlier may still read the old tables
        if (sync_all(b)) return -1;
        if (r->d_rows) cudaFree(r->d_rows);
        if (r->d_tiles) cudaFree(r->d_tiles);
        r->d_rows = nullptr;
        r->d_tiles = nullptr;
        r->rows_cap = r->tiles_cap = 0;
        r->uniform = 0;
        const size_t cap = (size_t)b->n_streams / MMA_TILE_ROWS + 2 * K;  // >= n / T + K tiles for every n <= n_streams
        CK(cudaMalloc(&r->d_rows, (size_t)b->n_streams * sizeof(int)));
        CK(cudaMalloc(&r->d_tiles, cap * sizeof(ModelTile)));
        r->rows_cap = (size_t)b->n_streams;
        r->tiles_cap = cap;
    }
    CK(cudaMemcpyAsync(r->d_rows, rows.data(), n * sizeof(int), cudaMemcpyHostToDevice, b->st[0]));
    CK(cudaMemcpyAsync(r->d_tiles, tiles.data(), tiles.size() * sizeof(ModelTile), cudaMemcpyHostToDevice, b->st[0]));
    r->h_rows = std::move(rows);  // the copies' sources stay alive until the next upload
    r->h_tiles = std::move(tiles);
    r->uniform = -1;
    return 0;
}

// The caller's stream continues after the state call; without one the call synchronises.
int state_call_end(RNNoiseBatch* b, cudaStream_t us) {
    cudaStream_t s = b->st[0];
    if (us) {
        CK(cudaEventRecord(b->ev_state, s));
        CK(cudaStreamWaitEvent(us, b->ev_state, 0));
        return 0;
    }
    CK(cudaStreamSynchronize(s));
    return 0;
}

int ensure_rec_stage(RNNoiseBatch* b, size_t bytes) {
    if (bytes <= b->rec_stage_bytes) return 0;
    CK(cudaStreamSynchronize(b->st[0]));
    if (b->rec_stage) cudaFree(b->rec_stage);
    b->rec_stage = nullptr;
    b->rec_stage_bytes = 0;
    CK(cudaMalloc(&b->rec_stage, bytes));
    b->rec_stage_bytes = bytes;
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
    if (check_streams(b, streams, n)) return -1;
    if (n == 0) return 0;
    if (!dst) return fail("null argument");
    ON_DEVICE(b->device);
    const int dev = classify(b, dst);
    if (dev < 0) return -1;
    cudaStream_t us = (cudaStream_t)cuda_stream, s = b->st[0];
    const size_t bytes = (size_t)n * record_bytes(b);
    if (!dev && ensure_rec_stage(b, bytes)) return -1;
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    const int widths[3] = {b->model.vad_gru.nn, b->model.noise_gru.nn, b->model.denoise_gru.nn};
    CK(launch_state_gather(b->buf, widths, d_idx, n, last_slot(b), dev ? dst : b->rec_stage, s));
    if (!dev) {
        CK(cudaMemcpyAsync(dst, b->rec_stage, bytes, cudaMemcpyDeviceToHost, s));
        return state_call_end(b, nullptr);
    }
    return state_call_end(b, us);
}

int rnnoise_batch_set_states(RNNoiseBatch* b, const int* streams, int n, const void* src, void* cuda_stream) {
    if (!b) return fail("null batch");
    if (check_streams(b, streams, n)) return -1;
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
        if (ensure_rec_stage(b, bytes)) return -1;
    }
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    if (!dev) CK(cudaMemcpyAsync(b->rec_stage, src, bytes, cudaMemcpyHostToDevice, s));
    CK(launch_state_scatter(b->buf, b->model.state_size(), d_idx, n, last_slot(b), dev ? src : b->rec_stage, s));
    return state_call_end(b, dev ? us : nullptr);
}

int rnnoise_batch_reset_streams(RNNoiseBatch* b, const int* streams, int n, void* cuda_stream) {
    if (!b) return fail("null batch");
    if (check_streams(b, streams, n)) return -1;
    if (n == 0) return 0;
    ON_DEVICE(b->device);
    cudaStream_t us = (cudaStream_t)cuda_stream;
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    CK(launch_state_scatter(b->buf, b->model.state_size(), d_idx, n, last_slot(b), nullptr, b->st[0]));
    return state_call_end(b, us);
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

// The packed layout of a model of the batch's geometry equals model 0's in everything but the image bytes and the
// activation codes.  It follows from the geometry alone; checked as an invariant on descriptors in offset form.
template <typename DeviceModel>
bool same_layout(const DeviceModel& a, const DeviceModel& b) {
    DeviceModel x, y;
    std::memcpy(&x, &a, sizeof x);
    std::memcpy(&y, &b, sizeof y);
    set_acts(&x, 0);
    set_acts(&y, 0);
    return std::memcmp(&x, &y, sizeof x) == 0;
}

}  // namespace

extern "C" {

int rnnoise_batch_add_model(RNNoiseBatch* b, const RNNModel* model) {
    if (!b) return fail("null batch");
    const HostModel& hm = model ? model->m : HostModel::builtin();
    const std::string bad = geometry_mismatch(b->model, hm);
    if (!bad.empty()) return fail(bad);
    ON_DEVICE(b->device);
    std::vector<unsigned char> img;
    bool same;
    if (b->gru_tc) {
        DeviceModelTc d;
        same = pack_model_tc(hm, &d, &img) && same_layout(d, b->tc0);
    } else {
        DeviceModelMma d;
        pack_model_mma(hm, &d, &img);
        same = same_layout(d, b->mma0);
    }
    if (!same || img.size() != b->mtab_bytes) return fail("packed layout of the model differs from the batch model's (internal error)");
    // image K goes to the first free entry; a full table moves to an allocation of twice the capacity, the old images
    // first.  Frames in flight may read the table.
    const size_t K = b->model_acts.size(), stride = b->mtab_stride;
    if (sync_all(b)) return -1;
    unsigned char* d = b->d_mtab;
    cudaError_t e = cudaSuccess;
    if (K == b->mtab_cap) {
        CK(cudaMalloc(&d, stride * 2 * K));
        e = cudaMemcpyAsync(d, b->d_mtab, stride * K, cudaMemcpyDeviceToDevice, b->st[0]);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(d + stride * K, img.data(), img.size(), cudaMemcpyHostToDevice, b->st[0]);
    if (e == cudaSuccess) e = cudaStreamSynchronize(b->st[0]);
    if (e != cudaSuccess) {
        if (d != b->d_mtab) cudaFree(d);
        return fail("model table upload", e);
    }
    if (d != b->d_mtab) {
        cudaFree(b->d_mtab);
        b->d_mtab = d;
        b->mtab_cap = 2 * K;
    }
    b->model_acts.push_back(model_acts(hm));
    return (int)K;
}

int rnnoise_batch_set_stream_models(RNNoiseBatch* b, const int* streams, int n, const int* model_ids) {
    if (!b) return fail("null batch");
    if (check_streams(b, streams, n)) return -1;
    if (n == 0) return 0;
    if (!model_ids) return fail("null argument");
    const int K = (int)b->model_acts.size();
    for (int r = 0; r < n; r++)
        if (model_ids[r] < 0 || model_ids[r] >= K)
            return fail("model id " + std::to_string(model_ids[r]) + " of stream " + std::to_string(streams ? streams[r] : r) + " out of range 0.." +
                        std::to_string(K - 1));
    ON_DEVICE(b->device);
    std::vector<int> next(b->stream_model);
    for (int r = 0; r < n; r++) next[(size_t)(streams ? streams[r] : r)] = model_ids[r];
    if (route_rows(b, &b->route, next)) return -1;
    b->stream_model = std::move(next);
    return 0;
}

int rnnoise_batch_get_stream_models(const RNNoiseBatch* b, const int* streams, int n, int* model_ids) {
    if (!b) return fail("null batch");
    if (check_streams(b, streams, n)) return -1;
    if (n == 0) return 0;
    if (!model_ids) return fail("null argument");
    for (int r = 0; r < n; r++) model_ids[r] = b->stream_model[(size_t)(streams ? streams[r] : r)];
    return 0;
}

}  // extern "C"

// ---- subset calls: advance only the listed streams (rnnoise_batch_process_streams_*; DESIGN.md 7b) ------------------
namespace {

// Checks every argument of a subset call; 1: nothing to do, 0: go ahead, -1: error (nothing has run).
int subset_check(RNNoiseBatch* b, const int* streams, int n, const void* out, const void* in, int n_frames) {
    if (!b) return fail("null batch");
    if (check_streams(b, streams, n)) return -1;
    if (n_frames < 0) return fail("negative n_frames");
    if (n == 0 || n_frames == 0) return 1;
    if (!out || !in) return fail("null argument");
    return 0;
}

// After every frame and state call issued so far (and the caller's stream): gather the listed streams into the work rows.
int subset_begin(RNNoiseBatch* b, const int* streams, int n, cudaStream_t us) {
    if (ensure_work(b, n)) return -1;
    const int* d_idx;
    if (state_call_begin(b, streams, n, us, &d_idx)) return -1;
    b->work.n_streams = n;
    b->work_frames = 0;
    b->work_route.uniform = 0;
    if (b->model_acts.size() > 1) {  // the work rows' models
        std::vector<int> model_of((size_t)n);
        for (int r = 0; r < n; r++) model_of[(size_t)r] = b->stream_model[(size_t)(streams ? streams[r] : r)];
        if (route_rows(b, &b->work_route, model_of)) return -1;
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
    CK(launch_subset_scatter(b->buf, b->work, b->model.state_size(), streams ? b->d_idx : nullptr, n, work_slot, last_slot(b), s));
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
    return state_call_end(b, nullptr);
}

}  // extern "C"

// ---- training-data rows (src/training.rs): 3 feature extractors per lane on the denoise path's kernels ----------
static_assert(sizeof(RNNoiseSimParams) == sizeof(TrainLaneParams), "C ABI struct and device struct must match");
constexpr int kTrainStages = 4;  // front, pitch, analysis, rows

struct RNNoiseTrainer {
    RNNoiseBatch* batch = nullptr;  // 3 * n_lanes streams: [0, L) clean, [L, 2L) noise, [2L, 3L) combined
    TrainBuffers tb{};
    float* stage_sig = nullptr;
    float* stage_noise = nullptr;
    float* stage_rows = nullptr;
    int stage_frames = 0;
};

namespace {

void trainer_release(RNNoiseTrainer* t) {
    if (!t) return;
    DeviceGuard guard(t->batch ? t->batch->device : 0);
    if (t->batch) sync_all(t->batch);
    cudaFree(t->tb.params);
    cudaFree(t->tb.resp_mem);
    cudaFree(t->tb.vad_count);
    cudaFree(t->tb.vad);
    cudaFree(t->tb.cutoff);
    cudaFree(t->stage_sig);
    cudaFree(t->stage_noise);
    cudaFree(t->stage_rows);
    if (t->batch) rnnoise_batch_destroy(t->batch);
    delete t;
}

int trainer_init(RNNoiseTrainer* t, int n_lanes) {
    const size_t L = (size_t)n_lanes;
    TrainBuffers& tb = t->tb;
    tb.n_lanes = n_lanes;
    CK(cudaMalloc(&tb.params, L * sizeof(TrainLaneParams)));
    CK(cudaMalloc(&tb.resp_mem, L * 4 * sizeof(float)));
    CK(cudaMalloc(&tb.vad_count, L * sizeof(int32_t)));
    CK(cudaMalloc(&tb.vad, PIPE_DEPTH * L * sizeof(float)));
    CK(cudaMalloc(&tb.cutoff, PIPE_DEPTH * L * sizeof(int32_t)));
    CK(cudaMemset(tb.resp_mem, 0, L * 4 * sizeof(float)));
    CK(cudaMemset(tb.vad_count, 0, L * sizeof(int32_t)));
    TrainLaneParams d{};  // NoiseSimulator::new, src/training.rs:319-340
    d.signal_gain = 1.0f;
    d.noise_gain = 1.0f;
    d.band_lp = NB_BANDS - 1;
    std::vector<TrainLaneParams> init(L, d);
    CK(cudaMemcpy(tb.params, init.data(), L * sizeof(TrainLaneParams), cudaMemcpyHostToDevice));
    return 0;
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

    int operator()(int i, const BatchBuffers& v, int slot, cudaStream_t s) const {
        const RNNoiseBatch* b = t->batch;
        switch (i) {
            case 0: CK(launch_train_front(v, t->tb, set, sig, noise, stream_stride, slot, s)); break;
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
    RNNoiseTrainer* t = new (std::nothrow) RNNoiseTrainer();
    if (!t) return nullptr;
    t->batch = rnnoise_batch_create(nullptr, 3 * n_lanes, device);
    int trc = -1;
    if (t->batch) {
        t->batch->n_stages = kTrainStages;
        DeviceGuard guard(t->batch->device);  // the trainer's own buffers live on the batch's device
        trc = guard.err == cudaSuccess ? trainer_init(t, n_lanes) : fail("cudaSetDevice", guard.err);
    }
    if (!t->batch || trc != 0) {
        std::string keep = g_err;
        trainer_release(t);
        g_err = keep;
        return nullptr;
    }
    return t;
}

void rnnoise_train_destroy(RNNoiseTrainer* t) { trainer_release(t); }
int rnnoise_train_lanes(const RNNoiseTrainer* t) { return t ? t->tb.n_lanes : 0; }
RNNoiseBatch* rnnoise_train_feature_batch(RNNoiseTrainer* t) { return t ? t->batch : nullptr; }

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
    if (sync_all(t->batch)) return -1;  // frames in flight still read the old parameters
    CK(cudaMemcpy(t->tb.params + first_lane, params, (size_t)n * sizeof(TrainLaneParams), cudaMemcpyHostToDevice));
    return 0;
}

int rnnoise_train_process_device(RNNoiseTrainer* t, float* rows, const float* signal, const float* noise, int n_frames, long stream_stride,
                                 long frame_stride, long row_lane_stride, long row_frame_stride, void* cuda_stream) {
    if (!t || !rows || !signal || !noise) return fail("null argument");
    if (n_frames < 0) return fail("negative n_frames");
    if (n_frames == 0) return 0;
    RNNoiseBatch* b = t->batch;
    ON_DEVICE(b->device);
    return device_call(b, (cudaStream_t)cuda_stream, n_frames, [&](int f, cudaEvent_t ready) {
        const TrainStages stages{t, (int)(b->seq % PIPE_DEPTH), rows + (size_t)f * row_frame_stride, row_lane_stride,
                                 signal + (size_t)f * frame_stride, noise + (size_t)f * frame_stride, stream_stride};
        return issue_frame(b, stages, false, ready);
    });
}

int rnnoise_train_process_host(RNNoiseTrainer* t, float* rows, const float* signal, const float* noise, int n_frames) {
    if (!t || !rows || !signal || !noise) return fail("null argument");
    if (n_frames < 0) return fail("negative n_frames");
    if (n_frames == 0) return 0;
    RNNoiseBatch* b = t->batch;
    ON_DEVICE(b->device);
    const size_t L = (size_t)t->tb.n_lanes;
    // staging is bounded (<= 256 MiB per input buffer): long runs go through in chunks of frames
    const int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_frames, (size_t(256) << 20) / (L * FRAME_SIZE * sizeof(float))));
    if (chunk > t->stage_frames) {
        if (sync_all(b)) return -1;
        cudaFree(t->stage_sig);
        cudaFree(t->stage_noise);
        cudaFree(t->stage_rows);
        t->stage_sig = t->stage_noise = t->stage_rows = nullptr;
        t->stage_frames = 0;
        CK(cudaMalloc(&t->stage_sig, (size_t)chunk * L * FRAME_SIZE * sizeof(float)));
        CK(cudaMalloc(&t->stage_noise, (size_t)chunk * L * FRAME_SIZE * sizeof(float)));
        CK(cudaMalloc(&t->stage_rows, (size_t)chunk * L * TRAIN_ROW * sizeof(float)));
        t->stage_frames = chunk;
    }
    for (int f0 = 0; f0 < n_frames; f0 += chunk) {
        const int nf = std::min(chunk, n_frames - f0);
        const size_t off = (size_t)f0 * L;
        CK(cudaMemcpyAsync(t->stage_sig, signal + off * FRAME_SIZE, (size_t)nf * L * FRAME_SIZE * sizeof(float), cudaMemcpyHostToDevice, b->c_in));
        CK(cudaMemcpyAsync(t->stage_noise, noise + off * FRAME_SIZE, (size_t)nf * L * FRAME_SIZE * sizeof(float), cudaMemcpyHostToDevice, b->c_in));
        if (rnnoise_train_process_device(t, t->stage_rows, t->stage_sig, t->stage_noise, nf, FRAME_SIZE, (long)(L * FRAME_SIZE), TRAIN_ROW,
                                         (long)(L * TRAIN_ROW), b->c_in))
            return -1;
        CK(cudaMemcpyAsync(rows + off * TRAIN_ROW, t->stage_rows, (size_t)nf * L * TRAIN_ROW * sizeof(float), cudaMemcpyDeviceToHost, b->c_in));
        CK(cudaStreamSynchronize(b->c_in));
    }
    return 0;
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
    DenoiseState* st = new (std::nothrow) DenoiseState();
    if (!st) return nullptr;
    if (rnnoise_init(st, model) != 0) {
        delete st;
        return nullptr;
    }
    return st;
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
    RNNoiseBatch* b = new (std::nothrow) RNNoiseBatch();
    DenoiseState* c = new (std::nothrow) DenoiseState();
    if (!b || !c) {
        delete b;
        delete c;
        fail("out of memory");
        return nullptr;
    }
    c->batch = b;
    int prev_dev = -1;
    cudaGetDevice(&prev_dev);
    int rc = batch_init(b, src->model, 1, src->device);
    if (prev_dev >= 0) cudaSetDevice(prev_dev);
    std::vector<unsigned char> rec(record_bytes(src));
    if (rc == 0) rc = rnnoise_batch_get_states(src, nullptr, 1, rec.data(), nullptr);
    if (rc == 0) rc = rnnoise_batch_set_states(b, nullptr, 1, rec.data(), nullptr);
    if (rc != 0) {
        std::string keep = g_err;
        rnnoise_destroy(c);
        g_err = keep;
        return nullptr;
    }
    return c;
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
