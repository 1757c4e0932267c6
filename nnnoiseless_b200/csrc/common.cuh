// common.cuh -- shared constants, device tables and per-batch state layout for the
// H100 (sm_90a) implementation of nnnoiseless' DenoiseState::process_frame.
//
// Reference constants: src/lib.rs:36-58 (jneem/nnnoiseless @ 7b47c9b).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace nnb {

constexpr int FRAME_SIZE = 480;
constexpr int WINDOW_SIZE = 960;
constexpr int FREQ_SIZE = 481;
constexpr int PITCH_MIN_PERIOD = 60;
constexpr int PITCH_MAX_PERIOD = 768;
constexpr int PITCH_FRAME_SIZE = 960;
constexpr int PITCH_BUF_SIZE = PITCH_MAX_PERIOD + PITCH_FRAME_SIZE;  // 1728
constexpr int NB_BANDS = 22;
constexpr int CEPS_MEM = 8;
constexpr int NB_DELTA_CEPS = 6;
constexpr int NB_FEATURES = 42;
constexpr int MAX_NEURONS = 128;
constexpr int NB_BINS_BANDED = 400;  // bins covered by the 21 band segments (EBAND_5MS[21] << 2)

// History ring: 8 slots of one frame each.  After frame f is written to slot f % 8 the most
// recent PITCH_BUF_SIZE samples (the reference's input_mem, src/features.rs:21,97-104) are the
// ring positions (base + i) mod HIST_CAP, i = 0..1727, base = (slot*480 + HIST_CAP - 1248) mod HIST_CAP.
// (3.6 frames are live; 8 slots let the high-pass kernel of frame f+4 run while frame f is still analysed.)
constexpr int HIST_SLOTS = 8;
constexpr int HIST_CAP = HIST_SLOTS * FRAME_SIZE;  // 3840
// Up to PIPE_DEPTH consecutive frames are in flight at once (each stage on its own CUDA stream); the per-frame
// intermediates (X, P, band energies, features, pitch, gains, vad) therefore exist in PIPE_DEPTH copies.
constexpr int PIPE_DEPTH = 4;

__host__ __device__ inline int hist_base(int slot) { return (slot * FRAME_SIZE + (HIST_CAP - (PITCH_BUF_SIZE - FRAME_SIZE))) % HIST_CAP; }

// Read-only tables shared by all kernels (built on the host in f64 exactly as src/lib.rs:107-127).
struct DeviceTables {
    float window[WINDOW_SIZE];
    float ramp[FRAME_SIZE];          // (float)(i + 1) / 480.0f: the voice-activity gate's cross-fade weights
    float dct[NB_BANDS * NB_BANDS];  // [i][j] = cos((i+.5) j pi/22), column 0 scaled by sqrt(.5)
    float wnorm;                     // 1 / sum(window^2)
    float2 tw960[FREQ_SIZE + 3];     // exp(-2 pi i k/960), k = 0..480
    // band interpolation tables for bins 0..399 (src/lib.rs:65-97): bin idx belongs to band
    // segment band_of[idx] with frac band_frac[idx] = j / band_size (f32 division)
    float band_frac[NB_BINS_BANDED];
    int32_t band_of[NB_BINS_BANDED];
    int32_t band_start[NB_BANDS];  // EBAND_5MS[i] << 2
    // ---- warp-per-stream spectral kernels (spectral_warp.cu) ----
    float2 twl[15][32];              // exp(-2 pi i b k1 / 480), lane-major: step-2 twiddles of the 32 x 15 FFT
    // band sums with one warp per stream: the 21 band segments (bins 0..399) are dealt to the 32 lanes, every lane stays
    // inside ONE segment (segments of <= 16 bins: one lane; 24, 32: two; 48: three; 72, 88: four -- 32 lanes in all)
    int16_t bp_seg[32];              // segment of lane l (lanes of a segment are contiguous)
    int16_t bp_b0[32];               // its first bin
    int16_t bp_n[32];                // its number of bins (<= 22)
    int16_t bp_rot[32];              // rotation of its walk (lane visits bin b0 + (t + rot) mod n): spreads the lanes over the banks
    int16_t bp_off[32];              // b0 - first bin of the segment
    float bp_inv[32];                // 1 / (bins of the segment): frac = (off + i) * inv
};
constexpr int BP_MAXBINS = 22;
// The tables' values (host.cu), built on the host for a copy to the device.
void build_tables(DeviceTables* t);

// Stream links (rnnoise_batch_link_streams) as the synthesis kernel reads them: one int4 {first, count, mode, 0} per row
// (count 0: not linked), then one int per row, the members of every group as rows, each group's ascending by batch
// stream index.  mode is RNNOISE_LINK_MAX or RNNOISE_LINK_MEAN.
constexpr int LINK_MODE_MAX = 1, LINK_MODE_MEAN = 2;

// A stream's controls (rnnoise_batch_set_stream_controls) as the synthesis kernel reads them.  All zero: no limit and
// the gate always open, what a stream that never had controls set gives.
struct __align__(16) StreamCtl {
    float g_min;        // raw gains are raised to g_min when g_min > 0
    float threshold;    // gate threshold; 0: always open
    float closed_gain;
    int32_t hold;       // frames the gate stays open after the vad falls below the threshold
};

// Per-batch persistent state + per-step intermediates, all [n_streams][...] row-major in HBM.
struct BatchBuffers {
    int n_streams;
    // persistent (src/features.rs:18-46, src/pitch.rs:4-17, src/rnn.rs:65-70, src/denoise.rs:39)
    float* hist;         // [B][HIST_CAP] ring of high-passed input
    float* hp_mem;       // [B][2]
    float* synth_mem;    // [B][480]
    float* ceps_mem;     // [B][8][22]
    int32_t* ceps_id;    // [B]
    int32_t* last_period;  // [B]
    float* last_gain;    // [B]
    float* gru_state;    // [B][state_size]  (vad | noise | denoise)
    float* lastg;        // [B][22]
    StreamCtl* ctl;      // [B]  stream controls' parameters (kept by a reset)
    int2* gate;          // [B]  gate state: hold_left, closed (0 after a reset)
    // per-step intermediates
    float2* X;           // [B][481]
    float2* P;           // [B][400]
    float* ex;           // [B][22]
    float* ep;           // [B][22]
    float* exp;          // [B][22]
    float* features;     // [B][42]
    int32_t* silence;    // [B]
    int32_t* pitch;      // [B]
    float* gains;        // [B][22]  raw RNN gains
    float* vad;          // [B]
    // pitch_kernel statistics: [0] streams whose coarse search was recomputed exactly, [1] streams whose sub-harmonic
    // ladder was, [2] stream-frames processed (cumulative since the handle was created)
    unsigned long long* pitch_stats;
};

// ---- training-data rows (src/training.rs): per-lane simulator parameters and state --------------------
constexpr int TRAIN_ROW = NB_FEATURES + 2 * NB_BANDS + 1;  // 87, src/training.rs:90
struct TrainLaneParams {  // == RNNoiseSimParams (include/rnnoise.h)
    float signal_gain, noise_gain;
    float sig_a[2], sig_b[2], noise_a[2], noise_b[2];
    int32_t band_lp;
};
struct TrainBuffers {
    int n_lanes;
    TrainLaneParams* params;  // [L]
    float* resp_mem;          // [L][4]  signal_resp_mem | noise_resp_mem
    int32_t* vad_count;       // [L]
    float* vad;               // [PIPE_DEPTH][L]
    int32_t* cutoff;          // [PIPE_DEPTH][L]  band_gain_cutoff before the silence override
};

// float sample -> int16: clamp to the int16 range then round half away from zero (what both reference front-ends do:
// src/nnnoiseless.rs:152 `clamp().round() as i16`, test_data/rnnoise_demo.c:53 roundf).  The synthesis kernel's and the
// down resampler's int16 output.
__device__ __forceinline__ short to_pcm16w(float v) { return (short)roundf(fminf(fmaxf(v, -32768.0f), 32767.0f)); }

// ---- launchers (one per translation unit) ------------------------------------------------------
// exact.cu (compiled with -fmad=false: bit-exact pitch path)
cudaError_t launch_hp_filter(const BatchBuffers& b, const void* in, bool pcm16, long stream_stride, long sample_stride, int slot,
                             cudaStream_t st);
// force_exact bit 0: every stream recomputes its coarse search order-exact, bit 1: its sub-harmonic ladder
// (NNB_PITCH_EXACT=1 sets both: the test reference; 2 / 3 select one of them)
cudaError_t launch_pitch(const BatchBuffers& b, int slot, int force_exact, cudaStream_t st);
// spectral_warp.cu (warp-per-stream)
// A split frame (rnnoise_batch_analyze_device / _synthesize_device) passes the caller's buffers: analysis writes stream s's
// features to features[s * feature_stride ..] (and its silence flag to silence[s], if not NULL) instead of the frame's set;
// synthesis reads its raw gains from gains[s * gain_stride ..] and writes no vad.  A window frame (_analyze_window_device /
// _synthesize_window_device) also passes ctx: the spectra and silence flag go through stream s's context record at
// ctx + s * ctx_stride records (layout below) instead of the set, and synthesis adds lastg and the gains to it.
cudaError_t launch_analysis_warp(const BatchBuffers& b, const DeviceTables* tab, int slot, cudaStream_t st, float* features = nullptr,
                                 long feature_stride = 0, int* silence = nullptr, void* ctx = nullptr, long ctx_stride = 0);
// controls (fused frames): apply the streams' controls (ctl, gate); false: every stream is on default controls.
// link (fused frames; implies controls): the rows' link table, n_streams records then the member list (LinkTable).
cudaError_t launch_synthesis_warp(const BatchBuffers& b, const DeviceTables* tab, void* out, bool pcm16, long stream_stride,
                                  long sample_stride, float* vad_out, cudaStream_t st, const float* gains = nullptr, long gain_stride = 0,
                                  void* ctx = nullptr, long ctx_stride = 0, bool controls = false, const int4* link = nullptr);
// synth_grad.cu: a saving split frame's context records (include/rnnoise.h), stream s's at ctx + s * ctx_stride records,
// from what synthesis of the frame in b is about to read; launched on synthesis' stream just before it.
cudaError_t launch_synth_context(const BatchBuffers& b, const float* gains, long gain_stride, void* ctx, long ctx_stride, cudaStream_t st);
// Synthesis context record (include/rnnoise.h, RNNOISE_SYNTH_CONTEXT_BYTES): float offsets of its sections.  Written by
// the saving split frame's copy kernel (synth_grad.cu) or by a window frame's analysis and synthesis (spectral_warp.cu),
// read by a window frame's synthesis and the synthesis backward.  Every band section is 24 floats, the last two zero.
constexpr int CX_X = 0, CX_P = 964, CX_EX = 1764, CX_EP = 1788, CX_EXP = 1812, CX_LASTG = 1836, CX_G = 1860, CX_SIL = 1884;
constexpr int CX_BAND_SECTION = 24;
constexpr int CX_FLOATS = CX_SIL + 4;  // the silence flag and three zero words
static_assert(CX_P == 2 * (FREQ_SIZE + 1) && CX_EX == CX_P + 2 * NB_BINS_BANDED, "record layout");
// Rows of `len` elements at s * ss + t * ts (s < ns, t < nt) overlap nowhere and have positive strides.
bool rows_disjoint(int ns, int nt, long ss, long ts, long len);
// ---- model tables (DESIGN.md 7c): models of one geometry side by side in one allocation, `stride` bytes apart ----
// Model 0, the batch's own model, is entry 0 from the batch's creation.  A frame whose rows run on several models is
// cut into tiles that never span two models: tile i covers the frame rows rows[first .. first + count), all on model
// `model`, whose six activation codes are packed 4 bits each in `acts` (bits 0-3 dense, 4-7 vad, 8-11 noise, 12-15
// denoise, 16-19 output, 20-23 vad output).
constexpr int TC_TILE_ROWS = 64, MMA_TILE_ROWS = 32;  // rows per tile of the wgmma and the mma.sync kernel
struct ModelTile {
    int model, first, count, acts;
};
struct ModelTiles {
    const ModelTile* tile;  // [n_tiles], device memory
    const int* rows;        // frame rows grouped by model, ascending within a model, device memory
    int n_tiles;
    uint32_t stride;        // bytes between two models' images
};
__host__ __device__ inline int tile_act(int acts, int layer) { return (acts >> (4 * layer)) & 15; }

// ---- the two GRU kernels (rnn_tc.cu, rnn_mma.cu) and their packed models -------------------------------------------
// A model packed for a GRU kernel is three things:
//   * an image: the bytes of one entry of the model table, holding everything the kernel reads of the model (weights,
//     biases, the tanh table of src/util.rs:3-27);
//   * a descriptor in offset form: byte offsets into the image and the layout of the kernel's operands.  It depends on
//     the model's geometry only, so the models of one table share model 0's descriptor byte for byte;
//   * its activation codes, packed as ModelTile::acts and given at launch.
// pack_model fills the descriptor (zeroed first, padding included) and the image; false if the model does not fit the
// kernel.  launch_gru runs one frame: tiles == nullptr runs every row on the model at `image` with codes `acts`; else
// `image` is the table's model 0 and each tile brings its model and codes.  tile_rows is the kernel's tile height.

// rnn_mma.cu: mma.sync m16n8k16 (f16 x f16 -> f32) formulation.
// The activations of TS streams live in one shared-memory matrix A[stream][column] (f16 "hi" + f16 "lo" copies:
// x = hi + lo to ~22 bits); every layer is a product of a column-subset of A with int8 weights (exact in f16),
// accumulated in f32.  A phase is a list of 16-column chunks of A and the weights pre-packed on the host in
// mma B-fragment order: wfrag[(chunk * ntiles + tile) * 32 + lane] = {b0, b1} (src/rnn.rs:251-327 semantics).
constexpr int MMA_MAX_CHUNKS = 28;
struct MmaPhase {
    int nchunks;          // K / 16
    int ntiles;           // output tiles of 8 columns (GRU z|r phase: z tiles then r tiles)
    uint32_t w_off;       // byte offset of the uint2 fragments wfrag[nchunks][ntiles][32] in the image
    uint32_t b_off;       // byte offset of the [ntiles * 8] f32 biases, zero padded
    short col[MMA_MAX_CHUNKS];  // first A column of each chunk
};
struct DeviceModelMma {
    MmaPhase dense, vad_zr, vad_h, vad_out, noise_zr, noise_h, den_zr, den_h, out;
    int nd, nv, nn, ndn;                                   // neurons of dense / vad / noise / denoise
    int c_feat, c_dense, c_vad, c_noise, c_den, c_rh;      // A column offsets (all multiples of 16)
    int kp;                                                // A row stride in halves; kp/2 = 4 (mod 8): conflict-free fragment loads
    int hs;                                                // f32 state row stride (floats)
    int state_size;
    uint32_t table_off;                                    // byte offset of the tanh table in the image
};

// rnn_tc.cu: wgmma formulation (Hopper warpgroup MMA, weights streamed by TMA bulk copies)
// ---- model image for this kernel (built on the host; each CTA streams it through shared memory in slabs) ----
constexpr int TC_PHASES = 9;
enum { PH_DENSE = 0, PH_VAD_ZR, PH_VAD_H, PH_VAD_OUT, PH_NOISE_ZR, PH_NOISE_H, PH_DEN_ZR, PH_DEN_H, PH_OUT };
struct TcPhase {
    int n;            // MMA N (multiple of 16); GRU z | r phases interleave the gates in blocks of 8 columns
    int nk;           // K chunks of 16 activations
    uint32_t w_off;   // byte offset of the [16 nk][n] weight operand in the image (K chunk kc at w_off + kc * n * 32)
    uint32_t b_off;   // byte offset of the n f32 biases
    short chunk[16];  // >= 0: shared-memory activation chunk (16 halves); < 0: feature chunk -(f + 1)
};
// One bulk copy of weights (one stage of the kernel's ring): K chunks [kc0, kc1) of phase `phase`, `bytes` bytes from
// image offset `off`.  The built-in model takes 33 slabs of at most 8 KB; 64 keeps the kernel parameters under 2 KB.
constexpr int TC_MAX_SLABS = 64;
struct TcSlab {
    uint32_t off, bytes;
    short phase, kc0, kc1;
};
struct DeviceModelTc {
    TcPhase ph[TC_PHASES];
    int nd, nv, nn, ndn;                                   // neurons of dense / vad / noise / denoise
    int p_d, p_v, p_n, p_dn;                               // the same padded to multiples of 8
    int o_dense, o_vad, o_noise, o_den, o_rh;              // activation offsets in halves (multiples of 8)
    int state_size;
    uint32_t table_off;                                    // byte offset of the tanh table in the image
    int n_slabs;
    short slab0[TC_PHASES + 1];                            // slabs of phase p: [slab0[p], slab0[p + 1])
    TcSlab slab[TC_MAX_SLABS];
};

struct HostModel;
// false if the model's layers do not fit the wgmma kernel's register / shared-memory budget, or one has 0 neurons
bool pack_model(const HostModel& hm, DeviceModelTc* d, std::vector<unsigned char>* image);
// every model fits the mma.sync kernel: always true
bool pack_model(const HostModel& hm, DeviceModelMma* d, std::vector<unsigned char>* image);
cudaError_t launch_gru(const BatchBuffers& b, const DeviceModelTc& m, const unsigned char* image, int acts, const ModelTiles* tiles,
                       cudaStream_t st);
cudaError_t launch_gru(const BatchBuffers& b, const DeviceModelMma& m, const unsigned char* image, int acts, const ModelTiles* tiles,
                       cudaStream_t st);
inline int tile_rows(const DeviceModelTc&) { return TC_TILE_ROWS; }
inline int tile_rows(const DeviceModelMma&) { return MMA_TILE_ROWS; }

// state.cu: per-stream state records (layout: rnnoise_batch_get_states in include/rnnoise.h).  Byte offsets of the
// sections; the 128-byte head holds magic, version, the three GRU widths, mem_id, last_period, last_gain, mem_hp_x, lastg.
constexpr int STATE_OFF_INPUT = 128, STATE_OFF_CEPS = 7040, STATE_OFF_SYNTH = 7744, STATE_OFF_GRU = 9664;
__host__ __device__ inline size_t state_record_bytes(int state_size) { return ((size_t)STATE_OFF_GRU + 4 * (size_t)state_size + 15) & ~(size_t)15; }
// slot: ring slot of the batch's most recent frame ((frame - 1) mod HIST_SLOTS).  idx: device array of n stream indices
// (NULL: streams 0..n-1).  Records are state_record_bytes apart and 16-byte aligned.
cudaError_t launch_state_gather(const BatchBuffers& b, const int widths[3], const int* idx, int n, int slot, void* dst, cudaStream_t st);
// device-resident records: *first_bad = min(*first_bad, index of each record whose head fails the import checks)
cudaError_t launch_state_check(const void* src, int n, const int widths[3], int* first_bad, cudaStream_t st);
// src NULL: reset the streams to the freshly created state, gate state included (records leave the controls alone)
cudaError_t launch_state_scatter(const BatchBuffers& b, int state_size, const int* idx, int n, int slot, const void* src, cudaStream_t st);
// Subset calls: the persistent state of batch stream idx[r] <-> row r of the work state `work` (same buffer layout, n rows).
// Gather copies what the next frame reads: the 1248 ring samples before slot `slot` (the batch's next slot; the same ring
// positions on both sides), mem_hp_x, synthesis_mem, the cepstral ring and mem_id, last_period / last_gain, the GRU
// states, lastg and the stream's controls and gate state (8,420 bytes for the built-in model).  Scatter copies the same fields back, with the full 1728-sample
// window of the work state's most recent slot `work_slot` rotated to the batch's most recent slot `batch_slot`, so that
// a state record taken afterwards is the one the same frames would have left (10,340 bytes for the built-in model).
cudaError_t launch_subset_gather(const BatchBuffers& batch, const BatchBuffers& work, int state_size, const int* idx, int n, int slot,
                                 cudaStream_t st);
cudaError_t launch_subset_scatter(const BatchBuffers& batch, const BatchBuffers& work, int state_size, const int* idx, int n, int work_slot,
                                  int batch_slot, cudaStream_t st);
// Stream controls: stream idx[r] (idx NULL: stream r) takes ctl[r] and gate[r] (device arrays), or gives its gate state.
cudaError_t launch_controls_scatter(const BatchBuffers& b, const int* idx, int n, const StreamCtl* ctl, const int2* gate, cudaStream_t st);
cudaError_t launch_controls_gather(const BatchBuffers& b, const int* idx, int n, int2* gate, cudaStream_t st);

// train.cu (-fmad=false)
cudaError_t launch_train_front(const BatchBuffers& b, const TrainBuffers& tb, int set, const float* signal, const float* noise,
                               long stream_stride, int slot, cudaStream_t st);
// The same from a device pool of int16 samples: lane l's frame at pool[sig_at[l] ..) / pool[noise_at[l] ..), -1 = zeros.
cudaError_t launch_train_front_pool(const BatchBuffers& b, const TrainBuffers& tb, int set, const short* pool, const long long* sig_at,
                                    const long long* noise_at, int slot, cudaStream_t st);
cudaError_t launch_train_rows(const BatchBuffers& b, const TrainBuffers& tb, int set, float* rows, long lane_stride, cudaStream_t st);
// n_frames frames of every lane from the int16 pool at sig_at / noise_at [n_frames][L] (-1: zeros): noisy, clean and (if
// not NULL) noise sample (l, t, i) at ptr[l * stream_stride + t * frame_stride + i], vad (if not NULL) at
// vad[l * vad_stream_stride + t * vad_frame_stride].  Carries resp_mem, vad_count and b.hp_mem of streams l and L + l.
cudaError_t launch_train_waves(const BatchBuffers& b, const TrainBuffers& tb, const short* pool, const long long* sig_at,
                               const long long* noise_at, int n_frames, float* noisy, float* clean, float* noise, float* vad,
                               long stream_stride, long frame_stride, long vad_stream_stride, long vad_frame_stride, cudaStream_t st);

}  // namespace nnb
