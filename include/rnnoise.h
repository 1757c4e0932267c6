/* SPDX-License-Identifier: BSD-3-Clause */
/*
 * rnnoise.h -- C ABI of nnnoiseless-b200.
 *
 * Part 1 is the drop-in boundary: the eight rnnoise_* functions the reference exports from
 * src/capi.rs (jneem/nnnoiseless @ 7b47c9b; header generated there by cbindgen per cbindgen.toml:
 * guard RNNOISE_H, <stdio.h>, C++ compatible).  Same names, argument meaning, ownership and error
 * behaviour -- test_data/rnnoise_demo.c compiles against this header unchanged.
 *
 * Part 2 is additive: a batched entry point (one call advances N independent streams), because a
 * one-frame-one-stream call cannot feed a GPU.  The legacy functions are N = 1 wrappers over the
 * same kernels.
 *
 * All computation runs in hand-written sm_90a CUDA kernels; there is no CPU fallback: without a
 * usable CUDA device rnnoise_create / rnnoise_batch_create return NULL and rnnoise_last_error()
 * says why.
 */
#ifndef RNNOISE_H
#define RNNOISE_H

#include <stdio.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct DenoiseState DenoiseState; /* src/capi.rs:9  */
typedef struct RNNModel RNNModel;         /* src/capi.rs:11 */

/* ------------------------------------------------------------------ Part 1: reference ABI ---- */

/* Number of samples processed per call: 480.  Replaces src/capi.rs:17-19. */
int rnnoise_get_frame_size(void);

/* Size of DenoiseState in bytes (for rnnoise_init on caller memory).  Replaces src/capi.rs:25-27. */
int rnnoise_get_size(void);

/* Initialise a caller-allocated DenoiseState of rnnoise_get_size() bytes; model NULL = built-in.
 * Returns 0 on success (the reference always returns 0; we return -1 if no CUDA device/stream could
 * be set up -- see rnnoise_last_error).  Replaces src/capi.rs:29-43. */
int rnnoise_init(DenoiseState *st, RNNModel *model);

/* Allocate + initialise a state; model NULL = built-in weights.  A non-NULL model is BORROWED and
 * must outlive the state (Cow::Borrowed, src/capi.rs:53).  Replaces src/capi.rs:49-57. */
DenoiseState *rnnoise_create(RNNModel *model);

/* Free a state returned by rnnoise_create.  Replaces src/capi.rs:63-65. */
void rnnoise_destroy(DenoiseState *st);

/* Denoise one frame of 480 samples (floats in the int16 range); out may alias in.  Returns the
 * voice-activity probability.  A NULL state aborts, as the reference's `expect` does.
 * Replaces src/capi.rs:75-85. */
float rnnoise_process_frame(DenoiseState *st, float *out, float *in);

/* Load a model in the nnnoiseless binary format.  Takes over the FILE: it is read to EOF and
 * fclose()d.  NULL on read error or malformed model.  Replaces src/capi.rs:89-105. */
RNNModel *rnnoise_model_from_file(FILE *file);

/* Free a model returned by rnnoise_model_from_file / _from_bytes.  Replaces src/capi.rs:111-113. */
void rnnoise_model_free(RNNModel *model);

/* ------------------------------------------------------------------ Part 2: additive ---------- */

/* RnnModel::from_bytes (src/rnn.rs:75): parse a model from memory (bytes are copied).  NULL if the
 * bytes are not a valid model (same validation as src/rnn.rs:189-222). */
RNNModel *rnnoise_model_from_bytes(const unsigned char *bytes, size_t len);

/* RNNoise text format ("rnnoise-nu model file version 1", e.g. test_data/sh.rnnn) -> model, i.e.
 * train/convert_rnnoise.py:18-29 followed by from_bytes. */
RNNModel *rnnoise_model_from_text(const char *text, size_t len);

/* Copy the model's binary image (the exact bytes from_bytes accepted) into buf; returns its size.
 * With buf NULL only the size is returned.  Used to broadcast a model between ranks. */
size_t rnnoise_model_bytes(const RNNModel *model, unsigned char *buf, size_t cap);

typedef struct RNNoiseBatch RNNoiseBatch;

/* A batch of n_streams independent DenoiseStates living on CUDA device `device` (-1: current).
 * model NULL = built-in; the model's weights are copied to the device (the model may be freed). */
RNNoiseBatch *rnnoise_batch_create(const RNNModel *model, int n_streams, int device);
void rnnoise_batch_destroy(RNNoiseBatch *b);
int rnnoise_batch_streams(const RNNoiseBatch *b);
/* Zero every stream's state (== freshly created). */
int rnnoise_batch_reset(RNNoiseBatch *b);

/* Advance every stream by n_frames frames.  DEVICE pointers.
 *   in, out : sample (s, t, i) at  ptr[s * stream_stride + t * frame_stride + i],  i < 480
 *             (floats; strides in floats; out may alias in)
 *   vad     : [n_frames][n_streams] voice-activity probabilities, or NULL
 *   cuda_stream : a cudaStream_t (NULL = the batch's own stream); the call is asynchronous
 *             with respect to the host when a stream is given.
 * Returns 0, or a negative error code (rnnoise_last_error() has the text). */
int rnnoise_batch_process_device(RNNoiseBatch *b, float *out, const float *in, float *vad, int n_frames,
                                 long stream_stride, long frame_stride, void *cuda_stream);

/* The same with 16-bit PCM device buffers (strides in samples): the int16 -> float widening and the
 * clamp + round-to-nearest back to int16 (src/nnnoiseless.rs:147-177, test_data/rnnoise_demo.c:51-55) happen
 * inside the first and last kernel of the path. */
int rnnoise_batch_process_device_pcm16(RNNoiseBatch *b, short *out, const short *in, float *vad, int n_frames,
                                       long stream_stride, long frame_stride, void *cuda_stream);

/* General layout: sample (s, t, i) at ptr[s*stream_stride + t*frame_stride + i*sample_stride] (element strides;
 * pcm16 = 0: float samples in and out; 1: int16 in and out; 2: float in, int16 out (clamp + round); 3: int16 in,
 * float out).  Interleaved multi-channel audio, where every channel is its own stream
 * (src/signal.rs:90-107, src/nnnoiseless.rs:301-330), is stream_stride = 1, sample_stride = n_channels,
 * frame_stride = 480 * n_channels. */
int rnnoise_batch_process_device_strided(RNNoiseBatch *b, void *out, const void *in, int pcm16, float *vad, int n_frames,
                                         long stream_stride, long sample_stride, long frame_stride, void *cuda_stream);

/* Same through HOST buffers: copies in -> device, runs, copies out/vad back, synchronises.
 * Layout [n_frames][n_streams][480] (frame-major), vad [n_frames][n_streams]. */
int rnnoise_batch_process_host(RNNoiseBatch *b, float *out, const float *in, float *vad, int n_frames);

/* PCM front-end (what both reference front-ends do around the path: src/nnnoiseless.rs:147-177,
 * test_data/rnnoise_demo.c:51-55): int16 samples in, process, round-to-nearest + clamp to int16
 * out.  HOST buffers, layout [n_frames][n_streams][480]. */
int rnnoise_batch_process_pcm16_host(RNNoiseBatch *b, short *out, const short *in, float *vad, int n_frames);

/* Debug taps of the most recent frame (DEVICE -> host copies; any pointer may be NULL):
 *   pitch [n_streams] int, silence [n_streams] int, features [n_streams][42], gains [n_streams][22]
 *   (gains after the 0.6*lastg floor). */
int rnnoise_batch_get_taps(RNNoiseBatch *b, int *pitch, int *silence, float *features, float *gains);

/* Debug taps of the GRU network alone (DEVICE -> host copies; any pointer may be NULL): the raw outputs of the most
 * recent frame, gains [n_streams][22] (before the gain floor) and vad [n_streams], and the persistent GRU state after
 * it, gru_state [n_streams][vad_gru + noise_gru + denoise_gru neurons] (the three states back to back).  The network
 * writes nothing for a stream whose frame was silent: its state is the previous frame's, and its gains and vad entries
 * are stale (the vad the process calls return for it is 0). */
int rnnoise_batch_get_rnn_taps(RNNoiseBatch *b, float *gains, float *vad, float *gru_state);

/* Debug taps of the frequency-domain intermediates that analysis hands to synthesis (DEVICE -> host copies; any pointer
 * may be NULL), for the most recent frame: the spectra X [n_streams][481][2] of the current window and P [n_streams][400][2]
 * of the pitch-lagged window (re, im; wnorm applied; P holds only the 400 bins the 21 band segments cover, the reference
 * never reads the others), the band energies ex and ep [n_streams][22] and the normalised band correlation
 * exp [n_streams][22] = corr / sqrt(0.001 + ex * ep) (src/features.rs:115-138).  They are written on silent frames too
 * (synthesis reads X to produce the output). */
int rnnoise_batch_get_spectral_taps(RNNoiseBatch *b, float *X, float *P, float *ex, float *ep, float *exp);

/* ---- per-stream state: save, restore, move, clone and reset single streams ---------------------------------------
 * A state record holds the persistent fields of one stream's DenoiseState (src/denoise.rs:37-42) in the reference's own
 * order and indexing, so a record does not depend on where it came from: not on the batch size, the slot, the frame
 * counter, the device or the GRU kernel that ran.  Version 1, little-endian 4-byte fields:
 *   offset  field
 *        0  u32 magic RNNOISE_STATE_MAGIC ("RNST"), i32 version = 1
 *        8  i32 nv, nn, nd: neurons of the vad, noise and denoise GRUs of the model  (src/rnn.rs:65-70)
 *       20  i32 mem_id, 0..7: next row of cepstral_mem                                (src/features.rs:26)
 *       24  i32 last_period, 0..768; f32 last_gain                                    (src/pitch.rs, PitchFinder)
 *       32  f32 mem_hp_x[2]: high-pass filter memory                                  (src/features.rs:27)
 *       40  f32 lastg[22]: most recent gains applied                                  (src/denoise.rs:39)
 *      128  f32 input_mem[1728], oldest sample first                                  (src/features.rs:21)
 *     7040  f32 cepstral_mem[8][22], row k = ring slot k                              (src/features.rs:23)
 *     7744  f32 synthesis_mem[480]                                                    (src/features.rs:28)
 *     9664  f32 GRU state: vad[nv], then noise[nn], then denoise[nd]                  (src/rnn.rs:65-70)
 *   then zero padding up to rnnoise_batch_state_bytes() = 9664 + 4 (nv + nn + nd) rounded up to a multiple of 16
 *   (10,336 bytes for the built-in model).  Records of n streams are packed back to back.
 * A record restores a stream bit for bit on any batch whose model has the same GRU widths.  Only the widths are checked:
 * a record taken under another model of the same geometry is accepted, and the stream continues with the receiving
 * batch's weights.
 *
 * streams: HOST array of n distinct stream indices (NULL: streams 0..n-1).  dst / src: n records, in host memory or in
 * device memory of the batch's device (16-byte aligned), told apart with cudaPointerGetAttributes.  With device memory
 * and a cuda_stream the call is asynchronous with respect to the host, ordered after the work already queued on
 * cuda_stream, and later work on cuda_stream sees its effect; otherwise it synchronises before returning.  The calls are
 * ordered with the batch's frames: a get sees every frame issued before it, a set or reset takes effect before the next
 * frame.  Other streams are not touched. */
#define RNNOISE_STATE_MAGIC 0x54534E52u
#define RNNOISE_STATE_VERSION 1
/* Size in bytes of one state record of this batch. */
size_t rnnoise_batch_state_bytes(const RNNoiseBatch *b);
/* Export the state of the given streams into dst[n][rnnoise_batch_state_bytes(b)]. */
int rnnoise_batch_get_states(RNNoiseBatch *b, const int *streams, int n, void *dst, void *cuda_stream);
/* Import src[n][rnnoise_batch_state_bytes(b)] into the given streams.  Every record and index is validated before
 * anything is written (magic, version, GRU widths equal to the batch model's, mem_id in 0..7, last_period in 0..768;
 * indices in range and distinct); if one check fails the call returns an error, rnnoise_last_error() says which, and no
 * stream changes.  Validating device-resident records synchronises with cuda_stream. */
int rnnoise_batch_set_states(RNNoiseBatch *b, const int *streams, int n, const void *src, void *cuda_stream);
/* Reset the given streams to the state of a freshly created stream; other streams are not touched. */
int rnnoise_batch_reset_streams(RNNoiseBatch *b, const int *streams, int n, void *cuda_stream);

/* ---- subset calls: advance only some streams of a batch ----------------------------------------------------------
 * Advance only streams[0..n) by n_frames frames; every other stream is left exactly as it was (its state record is
 * byte-identical before and after).  Row r of in / out / vad belongs to stream streams[r]:
 *   sample (r, t, i) at ptr[r*stream_stride + t*frame_stride + i*sample_stride], pcm16 as in
 *   rnnoise_batch_process_device_strided; vad [n_frames][n] (row-major, may be NULL).  DEVICE pointers.
 * streams: HOST array of n distinct indices in 0..n_streams-1, in any order (NULL: streams 0..n-1).  n == 0 or
 * n_frames == 0 is a no-op that returns 0.  Every argument is checked before anything runs; on an error the call returns
 * a negative code, rnnoise_last_error() says which check failed, and no stream changes.
 * A listed stream gets bit for bit the output, vad and state it would get from the same frames in a full-batch call.
 * Ordering is that of the state calls: the call sees every frame and state call issued before it, and later frames,
 * subset calls and state calls see its effect.  With a cuda_stream the call is asynchronous and ordered on that stream;
 * without one it synchronises.  The cost grows with n: the listed streams' live state (8,420 bytes per stream for the
 * built-in model, controls included) is gathered into a compact work state, advanced there by the frame kernels, and scattered back
 * (10,340 bytes: the full 1728-sample input_mem of the record).
 * Device memory: the work state is allocated on first use and grows to the largest n used so far, about
 * 4 * (4529 + nv + nn + nd) bytes per row (18,788 bytes for the built-in model: 1.23 GB at n = 65,536); it is freed by
 * rnnoise_batch_destroy.  The frames' intermediates reuse the batch's own buffers.
 * rnnoise_batch_get_taps / get_rnn_taps / get_spectral_taps describe full-batch frames: after a subset call they return an error until the
 * next full-batch frame. */
int rnnoise_batch_process_streams_device(RNNoiseBatch *b, const int *streams, int n, void *out, const void *in, int pcm16, float *vad,
                                         int n_frames, long stream_stride, long sample_stride, long frame_stride, void *cuda_stream);
/* Same through HOST buffers, float samples, compact layout in/out [n_frames][n][480], vad [n_frames][n] (may be NULL).
 * Frames stream through the batch's staging ring: the device memory does not grow with n_frames. */
int rnnoise_batch_process_streams_host(RNNoiseBatch *b, const int *streams, int n, float *out, const float *in, float *vad,
                                       int n_frames);

/* ---- per-stream models: the streams of one batch on different models of one geometry -------------------------------
 * A batch holds a table of models that share the geometry of the model it was created with (model 0).  Each stream runs
 * on one model of the table; every stream starts on model 0, so a batch that never calls these functions behaves as
 * before.  A stream on model k gives bit for bit what it gives in a batch created with model k.
 *   - rnnoise_batch_reset and rnnoise_batch_reset_streams reset state only: the model table and the assignments stay.
 *   - State records do not carry a model (their format stays version 1): a record restores the state, and the stream
 *     continues on the model it is assigned to in the receiving batch.
 *   - Taps keep their meaning: row i is batch stream i, whatever model it ran.
 * Frames whose streams all run on one model take the one-model kernels; frames that mix models group their rows by
 * model (DESIGN.md section 7c). */
/* Add a model to the batch's model table; returns its index (1, 2, ...; index 0 is the model given to
 * rnnoise_batch_create), or a negative code.  model NULL: the built-in model.  The weights are copied to the device (the
 * model may be freed).
 * The model must have the batch's geometry: the same inputs and neurons in all six layers (src/rnn.rs:55-62).
 * Activations and weights may differ.  A model of another geometry is rejected; rnnoise_last_error() names the
 * first layer that differs.  Waits for the frames in flight. */
int rnnoise_batch_add_model(RNNoiseBatch *b, const RNNModel *model);
/* Stream streams[r] runs on model model_ids[r] from the next frame on (streams NULL: 0..n-1; HOST arrays).
 * Streams keep their state: the stream continues with the other weights, like a state record moved to a batch of
 * another model.  Ordered like the state calls: frames issued before the call use the old assignment, frames
 * issued after it use the new one, for full-batch and subset calls alike.  Every index and id is checked first;
 * on an error nothing changes. */
int rnnoise_batch_set_stream_models(RNNoiseBatch *b, const int *streams, int n, const int *model_ids);
/* Current model of each listed stream (host call, no GPU work). */
int rnnoise_batch_get_stream_models(const RNNoiseBatch *b, const int *streams, int n, int *model_ids);

/* ---- per-stream controls: an attenuation limit and a voice-activity gate (DESIGN.md section 7m) -------------------
 * Each stream of a batch has a controls record.  Every stream starts on the defaults {INFINITY, 0, 0, 0, 0, 0}, which
 * give bit for bit the output of a batch that never calls these functions.
 *
 * Limit.  Let g_min = (float)pow(10.0, -atten_lim_db / 20.0), and 0 for +INFINITY.  On a fused, non-silent frame every
 * raw network gain becomes g' = fmaxf(g, g_min) when g_min > 0.  From there on the frame is the reference's: the pitch
 * filter's r from g', the floor max(g', 0.6 lastg), and lastg stores that floored value.  So a limited stream is bit
 * for bit a split frame fed max(g, g_min).  The raw gains do not depend on the output: rnnoise_batch_get_rnn_taps keeps
 * reporting the network's own gains.  Silent frames are untouched, as in the reference.
 *
 * Gate.  The gate acts on the output samples only, after overlap-add: neither synthesis_mem nor any other state field
 * sees it, so a gated stream's state record and vad are byte-identical to an ungated twin's.  On each fused frame, with
 * v the frame's reported vad (0 on silent frames):
 *   - if v >= gate_threshold, or gate_threshold is 0: hold_left = gate_hold_frames; the gate is open;
 *   - else if hold_left > 0: hold_left is decremented; the gate is open;
 *   - otherwise the gate is closed.
 * The gains, in float32, each operation rounded, with no contraction:
 *   tau = open ? 1 : gate_closed_gain
 *   l   = gate_closed ? gate_closed_gain : 1          (the previous frame's decision)
 *   w_i = (float)(i + 1) / 480.0f
 *   a_i = l + (tau - l) * w_i
 *   output sample i is y_i * a_i, then the int16 conversion when the output is int16.
 * After the frame, gate_closed = !open.  With the defaults every a_i is exactly 1 and g_min is 0.
 *
 * Where the controls apply.  Every fused frame: full-batch, subset (rnnoise_batch_process_streams_*) and native-rate
 * (rnnoise_batch_process_native_*; at 48 kHz, before the down-resampler).  Split and window frames (DESIGN.md sections
 * 7h, 7j) ignore the controls and leave the gate state as it was: the caller owns their gains, and they have no vad.
 * The legacy one-stream ABI is unchanged.
 *
 * Interactions.  rnnoise_batch_reset and rnnoise_batch_reset_streams give the gate fresh state (hold_left 0, open) and
 * keep the parameters, as they keep the model assignment.  State records stay version 1 and do not carry controls, and
 * rnnoise_batch_set_states leaves the controls alone: moving a stream means moving both records. */
typedef struct {
    float atten_lim_db;     /* >= 0; +INFINITY = no limit (default).  0 dB = gains of 1, no suppression */
    float gate_threshold;   /* 0..1; 0 = gate always open (default) */
    float gate_closed_gain; /* 0..1, the output's gain while the gate is closed (0 = mute) */
    int gate_hold_frames;   /* 0..6000 frames of 10 ms kept open after the last frame at or above the threshold */
    int gate_hold_left;     /* state: 0..gate_hold_frames */
    int gate_closed;        /* state: 0 or 1, the gate's decision on the stream's previous fused frame */
} RNNoiseStreamControls;    /* 24 bytes; defaults {INFINITY, 0, 0, 0, 0, 0} */
#define RNNOISE_GATE_MAX_HOLD_FRAMES 6000
/* Set the controls records of streams[0..n) (NULL: 0..n-1; HOST arrays), state fields included.  Every field of every
 * record is checked before anything is written: no NaN, each field within the ranges above, gate_hold_left <=
 * gate_hold_frames.  A refused call returns a negative code, rnnoise_last_error() names the record and field, and
 * nothing changes.  Ordered like rnnoise_batch_set_stream_models: frames issued before the call use the old controls,
 * frames issued after it the new ones.  Refused while split or window frames are pending.  Synchronises. */
int rnnoise_batch_set_stream_controls(RNNoiseBatch *b, const int *streams, int n, const RNNoiseStreamControls *c);
/* The controls records of the listed streams, after every frame issued before the call (host call; synchronises).
 * Refused while split or window frames are pending. */
int rnnoise_batch_get_stream_controls(RNNoiseBatch *b, const int *streams, int n, RNNoiseStreamControls *c);

/* ---- stream links: one gain curve for several streams of a batch (DESIGN.md section 7n) ----------------------------
 * A group is a set of 2 to RNNOISE_LINK_MAX_MEMBERS distinct streams of one batch with a mode; a stream is in at most one
 * group.  Unlinked streams (every stream of a new batch) behave exactly as without links.
 *
 * On a fused frame, a linked stream's raw band gains are replaced by its group's gains.  For band i the group's gain is
 * a reduction of the raw gains g_m[i] of the group's members m that are not silent on that frame (a silent frame's gains
 * and vad are stale, and the reference passes a silent frame through ungained):
 *   RNNOISE_LINK_MAX:  fmaxf over those members;
 *   RNNOISE_LINK_MEAN: their float32 sum in ascending stream index, starting from the first such member's gain, each
 *                      addition rounded, then divided by (float)n, n the number of such members.
 * A silent member's own frame is unchanged (the reference's silent frame), and if every member is silent nothing changes.
 * From there on the frame is the reference's for that stream, with its own state: its attenuation limit (section 7m) is
 * applied to the linked gain, then the pitch filter's r and the floor max(g', 0.6 lastg) with its own lastg.  So a linked
 * stream is bit for bit a split frame fed the linked gains.  Members may run different models and controls: each member
 * contributes its own model's raw gains.
 * A linked stream's gate (section 7m) decides on the group's vad: the largest vad of the non-silent members, or 0 when
 * every member is silent.  The vad the process calls report, rnnoise_batch_get_rnn_taps and the GRU states stay each
 * stream's own.
 *
 * Where links apply.  Every fused frame: full-batch, subset and native-rate calls (at 48 kHz).  A subset call must list
 * every group of a listed stream whole; otherwise it is refused, rnnoise_last_error() names the stream and a missing
 * member, and nothing changes.  Split and window frames ignore links: their gains are the caller's.  State records stay
 * version 1 and carry no link; rnnoise_batch_reset and rnnoise_batch_reset_streams keep the links. */
#define RNNOISE_LINK_MAX 1
#define RNNOISE_LINK_MEAN 2
#define RNNOISE_LINK_MAX_MEMBERS 64
/* Make streams[0..n) (HOST array) one group of the given mode.  A listed stream that was in another group leaves it
 * first; a group left with one member dissolves.  Checked before anything changes: a non-NULL batch and streams, 2 <= n
 * <= 64, indices in range and distinct, a known mode.  A host call: frames issued before it keep the old links, frames
 * issued after it use the new ones (the batch's link table is uploaded behind every frame in flight, before the next
 * fused frame).  Refused while split or window frames are pending. */
int rnnoise_batch_link_streams(RNNoiseBatch *b, const int *streams, int n, int mode);
/* Take streams[0..n) (NULL: every stream) out of their groups; a group left with one member dissolves.  Unlinked
 * streams are accepted.  Checks and ordering as rnnoise_batch_link_streams. */
int rnnoise_batch_unlink_streams(RNNoiseBatch *b, const int *streams, int n);
/* For each listed stream (NULL: 0..n-1): group[r] = the lowest stream index of its group (the stream itself when
 * unlinked) and mode[r] = the group's mode (0 when unlinked).  Either output may be NULL.  Host call, no GPU work. */
int rnnoise_batch_get_stream_links(RNNoiseBatch *b, const int *streams, int n, int *group, int *mode);

/* ---- split frames: the caller's own network between analysis and synthesis (DESIGN.md section 7h) -----------------
 * A fused frame is hp_filter -> pitch -> analysis -> GRU network -> synthesis.  A split frame stops after analysis,
 * hands the caller the 42 features of every stream, and resumes at synthesis with the caller's raw band gains: the
 * reference's DenoiseState::process_frame (src/denoise.rs:100-115) with rnn.compute replaced by the caller's network.
 *   - The gains are used exactly as given (no clamping, no check); the floor g = max(g, 0.6 lastg) and lastg stay the
 *     library's.
 *   - On a silent frame the features are zeros, the caller's gains are ignored, the spectrum passes through unchanged
 *     and lastg is not touched.
 *   - Split frames do not run the batch's GRUs: the streams' GRU state stays as it was, and a stream that goes back to
 *     fused calls resumes the batch's network from that state.  Everything else in the state record advances as in a
 *     fused frame.
 * Up to RNNOISE_MAX_PENDING_FRAMES frames may be analyzed and not yet synthesized (up to 3 frames of lookahead for the
 * caller's network, or chunks of 4 frames); synthesize finishes the oldest pending frames first.  While frames are
 * pending, every process call, the state calls (get_states, set_states, reset_streams), set_stream_models,
 * profile_step and the taps are refused with an error and no effect; rnnoise_batch_reset drops the pending frames.
 * After a split frame the taps return an error until the next fused full-batch frame.
 * Ordering as rnnoise_batch_process_device: each call runs after the work already queued on cuda_stream, and later work
 * on cuda_stream sees the features and silence flags (analyze) or the output (synthesize); without a stream the call
 * synchronises before it returns.  Every argument is checked before anything runs; on an error the call returns a
 * negative code, rnnoise_last_error() says which check failed, and nothing changes.  n_frames == 0 is a no-op.
 * Split frames advance every stream of the batch; the batch's models play no part in them. */
#define RNNOISE_MAX_PENDING_FRAMES 4
/* Frames analyzed and not yet synthesized (0 .. RNNOISE_MAX_PENDING_FRAMES). */
int rnnoise_batch_pending_frames(const RNNoiseBatch *b);
/* Analyze the next n_frames frames of every stream.  DEVICE pointers.
 *   in: sample (s, t, i) at in[s*stream_stride + t*frame_stride + i*sample_stride]; pcm16 0 = float, 1 = int16
 *   features: feature j of (s, t) at features[s*feature_stream_stride + t*feature_frame_stride + j], j < 42 (float)
 *   silence: [n_frames][n_streams] int, 1 = silent frame (gains ignored), or NULL
 * Refused if it would take the pending frames above RNNOISE_MAX_PENDING_FRAMES. */
int rnnoise_batch_analyze_device(RNNoiseBatch *b, const void *in, int pcm16, float *features, int *silence, int n_frames,
                                 long stream_stride, long sample_stride, long frame_stride,
                                 long feature_stream_stride, long feature_frame_stride, void *cuda_stream);
/* Synthesize the n_frames oldest pending frames from the caller's raw band gains.  DEVICE pointers.
 *   gains: gain k of (s, t) at gains[s*gain_stream_stride + t*gain_frame_stride + k], k < 22 (float)
 *   out: as `in` above; pcm16 0 = float, 1 = int16 (clamp + round half away, as every int16 output)
 * Refused if fewer than n_frames frames are pending. */
int rnnoise_batch_synthesize_device(RNNoiseBatch *b, void *out, int pcm16, const float *gains, int n_frames,
                                    long stream_stride, long sample_stride, long frame_stride,
                                    long gain_stream_stride, long gain_frame_stride, void *cuda_stream);

/* ---- training through synthesis: saved contexts and the synthesis backward (DESIGN.md section 7i) --------------------
 * A caller's network between analyze and synthesize can be trained on a loss of the output samples.  The saving call
 * below synthesizes like rnnoise_batch_synthesize_device with float output (the same output and state bits) and also
 * stores, per (stream, frame), a context record of what synthesis read before the frame changed anything.  The backward
 * turns dL/d(output samples) of a window of saved frames into dL/d(raw band gains).
 *
 * Context record, RNNOISE_SYNTH_CONTEXT_BYTES bytes, 16-byte aligned sections (offsets in bytes):
 *      0  X       complex float [481] (re, im), padded to 964 floats: the frame's spectrum
 *   3856  P       complex float [400]: the pitch-lagged spectrum (bins >= 400 are never used)
 *   7056  ex      float [22], padded to 24
 *   7152  ep      float [22], padded to 24
 *   7248  exp     float [22], padded to 24: the pitch correlation
 *   7344  lastg   float [22], padded to 24: the gain floor's memory before the frame
 *   7440  g       float [22], padded to 24: the raw gains synthesis used
 *   7536  silence int32, padded to 16 bytes: 1 = silent frame
 *
 * Backward contract.  Frames 0..n_frames-1 of a stream are consecutive saved frames (a window).  The outputs of the
 * window's frames are taken as a function of the window's raw gains; the contexts' spectra, the lastg before frame 0
 * and the overlap memory before frame 0 are constants.  Output frame t holds the first half of frame t's windowed
 * inverse FFT plus the second half of frame t-1's, so frame t's gains receive gradient from grad_out[t] and
 * grad_out[t+1]; the overlap memory left after the last frame contributes nothing.  At the kinks, decided in f32 on the
 * stored values as synthesis decides them:
 *   - exp > g: r = 1, no gradient through the pitch filter; at exp == g the formula's derivative applies;
 *   - q = exp^2 (1 - g^2) / (0.001 + g^2 (1 - exp^2)) clamped to [0, 1]: gradient only for 0 < q < 1;
 *   - gg = max(g, 0.6f lastg): the gradient goes to g when g >= 0.6f lastg (ties included), else times 0.6 to the
 *     previous frame's gg, and so on back through a run of floored frames;
 *   - a silent frame's gains get 0, and its unchanged lastg passes the gradient through.
 * The same inputs give the same bits (fixed reduction order, no atomics). */
#define RNNOISE_SYNTH_CONTEXT_BYTES 7552
/* rnnoise_batch_synthesize_device (float output) that also writes the context record of (s, t) at
 * ctx + (s*ctx_stream_stride + t*ctx_frame_stride) * RNNOISE_SYNTH_CONTEXT_BYTES (DEVICE memory, 16-byte aligned).
 * The split-frame rules, refusals and ordering apply; records of the call must not overlap. */
int rnnoise_batch_synthesize_saving_device(RNNoiseBatch *b, float *out, const float *gains, int n_frames,
                                           long stream_stride, long sample_stride, long frame_stride,
                                           long gain_stream_stride, long gain_frame_stride,
                                           void *ctx, long ctx_stream_stride, long ctx_frame_stride, void *cuda_stream);
/* Bytes of workspace rnnoise_synthesis_backward_device needs for a window (0 if either count is < 1). */
size_t rnnoise_synthesis_backward_workspace_bytes(int n_streams, int n_frames);
/* dL/dg for every (stream, frame, band) of a window, given dL/dout for every output sample.  DEVICE pointers:
 *   ctx: record of (s, t) at ctx + (s*ctx_stream_stride + t*ctx_frame_stride) * RNNOISE_SYNTH_CONTEXT_BYTES
 *   grad_out: sample i of (s, t) at grad_out[s*go_stream_stride + t*go_frame_stride + i], i < 480
 *   grad_gains: band k of (s, t) at grad_gains[s*gg_stream_stride + t*gg_frame_stride + k], k < 22 (rows must not overlap)
 *   workspace: at least rnnoise_synthesis_backward_workspace_bytes(n_streams, n_frames) bytes, 16-byte aligned
 * Stateless (no handle): runs on `device` (< 0: the current device), after the work queued on cuda_stream, and
 * cuda_stream continues after it (without a stream the call returns when it has finished).  It allocates nothing, so it
 * can be captured in a CUDA graph.  Every argument is checked before any CUDA call. */
int rnnoise_synthesis_backward_device(const void *ctx, long ctx_stream_stride, long ctx_frame_stride,
                                      const float *grad_out, long go_stream_stride, long go_frame_stride,
                                      float *grad_gains, long gg_stream_stride, long gg_frame_stride,
                                      int n_streams, int n_frames, void *workspace, size_t workspace_bytes,
                                      int device, void *cuda_stream);

/* ---- window frames: split frames of any length, through caller-held records (DESIGN.md section 7j) -----------------
 * Split frames keep their spectra in the batch, which bounds them to RNNOISE_MAX_PENDING_FRAMES.  Window frames keep them
 * in the caller's context records instead (the layout above), so any number of frames may be analyzed before any is
 * synthesized: a sequence network over a whole window, offline or non-causal models, lookahead of any length.
 *   - Samples, features, silence flags and gains: as rnnoise_batch_analyze_device / _synthesize_device, and the
 *     split-frame rules apply (gains used as given, silent frames, GRU state untouched, the rest of the state record
 *     advancing as in a fused frame).
 *   - Records: (s, t) at ctx + (s*ctx_stream_stride + t*ctx_frame_stride) * RNNOISE_SYNTH_CONTEXT_BYTES, DEVICE memory,
 *     16-byte aligned, the records of one call not overlapping.  analyze_window writes X, P, ex, ep, exp, the silence
 *     flag and every padding word; synthesize_window reads those and writes lastg (before the frame) and g (the raw
 *     gains it used).  After both, a record holds the bytes rnnoise_batch_synthesize_saving_device writes for the same
 *     frame and gains, so rnnoise_synthesis_backward_device takes window records as they are.
 *   - Owed frames: a window frame is owed from its analysis until its synthesis, without a bound.  analyze_window may be
 *     called any number of times; synthesize_window(n) finishes the n oldest owed frames, and ctx must point at the
 *     records their analysis wrote.  Other records give unspecified samples; the kernels read only within the records.
 *     Streaming with L frames of lookahead: analyze one frame, synthesize one frame L behind.
 *   - Split and window frames are never mixed: analyze_window and synthesize_window are refused while split frames are
 *     pending, and analyze_device, synthesize_device and synthesize_saving_device while window frames are owed.  Every
 *     call refused with split frames pending is refused with window frames owed; rnnoise_batch_reset drops owed frames.
 *     After a window frame the taps return an error until the next fused full-batch frame.
 * Ordering, argument checks (before anything runs; a refused call changes nothing) and n_frames == 0 as for split
 * frames; a null or unaligned ctx, overlapping records, and a synthesize_window of more frames than are owed are
 * refused too. */
/* Frames analyzed by analyze_window and not yet synthesized by synthesize_window (0 .. INT_MAX). */
int rnnoise_batch_window_frames(const RNNoiseBatch *b);
int rnnoise_batch_analyze_window_device(RNNoiseBatch *b, const void *in, int pcm16, float *features, int *silence, int n_frames,
                                        long stream_stride, long sample_stride, long frame_stride,
                                        long feature_stream_stride, long feature_frame_stride,
                                        void *ctx, long ctx_stream_stride, long ctx_frame_stride, void *cuda_stream);
/* ctx is read and written (lastg and g). */
int rnnoise_batch_synthesize_window_device(RNNoiseBatch *b, void *out, int pcm16, const float *gains, int n_frames,
                                           long stream_stride, long sample_stride, long frame_stride,
                                           long gain_stream_stride, long gain_frame_stride,
                                           void *ctx, long ctx_stream_stride, long ctx_frame_stride, void *cuda_stream);

/* Clone of a legacy state (the reference's `impl Clone for DenoiseState`, src/denoise.rs:36): a new state with the same
 * weights whose next frames give the same bits as the original's.  Free it with rnnoise_destroy.  NULL on error. */
DenoiseState *rnnoise_clone(const DenoiseState *st);

/* Profiling aid: advance every stream by ONE frame like rnnoise_batch_process_device, with CUDA events
 * recorded between the kernels of the path on the launching stream; synchronises and writes each
 * kernel's duration in milliseconds to ms[0..n) (n = return value <= cap; negative on error).
 * rnnoise_kernel_name(i) names kernel i of the path (NULL past the end). */
int rnnoise_batch_profile_step(RNNoiseBatch *b, float *out, const float *in, float *vad, long stream_stride,
                               void *cuda_stream, float *ms, int cap);
const char *rnnoise_kernel_name(int i);

/* Pitch-kernel certification statistics, cumulative since the handle was created (synchronises): out[0] = stream-frames
 * whose coarse pitch search recomputed all 147 lags in the reference's operation order because the fast (FMA) values
 * could not certify find_best_pitch's decisions (src/pitch.rs:372-405); a stream that recomputes only its (at most 8)
 * candidate lags is not counted.  out[1] = stream-frames whose remove_doubling ladder (src/pitch.rs:144-203) was
 * recomputed in that order, out[2] = stream-frames processed.  The integer period is bit-identical either way. */
int rnnoise_batch_pitch_stats(RNNoiseBatch *b, unsigned long long out[3]);

/* ---- training-data rows on the GPU (additive; the arithmetic of the reference's `nnnoiseless-gen-training-data`
 * binary, src/training.rs:113-161 main loop + :399-432 NoiseSimulator::next_frame) ------------------------------
 * A lane is one NoiseSimulator with its three DenoiseFeatures (clean, noise, combined).  File reading and the random
 * draws of NoiseSimulator::randomize (:352-377) stay with the caller, who passes their outcome as RNNoiseSimParams
 * (initially NoiseSimulator::new: gains 1, zero filters, band_lp 21) and may change it between calls.  Per frame and
 * lane the library consumes one raw 480-sample signal frame and one noise frame (i16-valued floats as
 * SignalReader::frame yields them, :237-262) and produces the 87-float row
 *   [42 features of the combined signal | 22 band gains (-1 = masked) | 22 log10 noise levels | vad]. */
#define RNNOISE_TRAIN_ROW 87
typedef struct RNNoiseSimParams {
    float signal_gain, noise_gain;     /* NoiseSimulator::{signal_gain, noise_gain} */
    float sig_a[2], sig_b[2];          /* sig_filter (Biquad {a, b}, src/util.rs:82-93) */
    float noise_a[2], noise_b[2];      /* noise_filter */
    int band_lp;                       /* NoiseSimulator::band_lp */
} RNNoiseSimParams;
typedef struct RNNoiseTrainer RNNoiseTrainer;
RNNoiseTrainer *rnnoise_train_create(int n_lanes, int device);      /* NULL on error */
void rnnoise_train_destroy(RNNoiseTrainer *t);
int rnnoise_train_lanes(const RNNoiseTrainer *t);
/* Debug view: the trainer's own batch of 3 n_lanes feature extractors (stream l = lane l's clean signal, n_lanes + l its
 * noise, 2 n_lanes + l its combined signal), borrowed: it lives as long as t and must not be destroyed.  The only calls
 * allowed on it are the reads rnnoise_batch_get_taps, rnnoise_batch_get_spectral_taps, rnnoise_batch_get_states and
 * rnnoise_batch_state_bytes; they describe the trainer's most recent frame. */
RNNoiseBatch *rnnoise_train_feature_batch(RNNoiseTrainer *t);
int rnnoise_train_set_params(RNNoiseTrainer *t, int first_lane, int n, const RNNoiseSimParams *params);
/* EBAND_5MS.position(|x| x << 2 > lowpass).unwrap_or(21), src/training.rs:373-376 */
int rnnoise_train_band_lp(int lowpass);
/* HOST buffers: signal, noise [n_frames][n_lanes][480]; rows [n_frames][n_lanes][87]. */
int rnnoise_train_process_host(RNNoiseTrainer *t, float *rows, const float *signal, const float *noise, int n_frames);
/* DEVICE buffers: signal/noise sample (l, f, i) at ptr[l*stream_stride + f*frame_stride + i]; row (l, f) at
 * rows[l*row_lane_stride + f*row_frame_stride].  Asynchronous with respect to the host like
 * rnnoise_batch_process_device (cuda_stream NULL: synchronises before returning). */
int rnnoise_train_process_device(RNNoiseTrainer *t, float *rows, const float *signal, const float *noise, int n_frames,
                                 long stream_stride, long frame_stride, long row_lane_stride, long row_frame_stride,
                                 void *cuda_stream);
/* HOST buffers, 16-bit input: pool holds pool_len int16 samples (at most 2^27, 256 MiB); sig_at / noise_at
 * [n_frames][n_lanes] give each lane-frame's 480 samples as pool[at .. at + 480), or -1 for a frame of zeros.
 * rows [n_frames][n_lanes][87].  The rows are bit-identical to rnnoise_train_process_host fed the same samples as
 * floats.  Every offset is checked before anything runs: one outside [0, pool_len - 480] (and not -1) fails the call,
 * naming its frame and lane, and leaves the trainer as it was.  The pool is copied to the device once per call; the
 * offsets and rows go through in chunks of at most 256 MiB of rows. */
int rnnoise_train_process_pool_host(RNNoiseTrainer *t, float *rows, const short *pool, long pool_len,
                                    const long long *sig_at, const long long *noise_at, int n_frames);

/* ---- waveform windows for training through synthesis (additive; DESIGN.md section 7k) -------------------------------
 * The same simulators make, instead of rows, the waveforms a loss on the denoiser's output needs: per lane and frame
 * noisy = s + n (the mix a DenoiseState receives, before any high-pass), clean = hp(s) (what the denoiser passes at a
 * gain of 1, one frame later), optionally noise = hp(n) and the rows' VAD column, from samples in a device-resident
 * int16 pool the trainer owns (uploaded once, read every epoch).
 *   - Modes: a trainer's first frame call fixes its mode.  One that has made waveform frames refuses the row calls, and
 *     one that has made rows refuses rnnoise_train_waves_device, until rnnoise_train_reset.  set_params applies to both.
 *   - Every refusal leaves the trainer as it was. */
/* Every lane back to NoiseSimulator::new: default parameters, filter memories, VAD counter and the three streams' state
 * zeroed; the mode is cleared, the pool kept.  Waits for the trainer's work in flight. */
int rnnoise_train_reset(RNNoiseTrainer *t);
/* Replaces the pool by n_samples zeroed int16 samples on the trainer's device (0: no pool).  Refused, naming the bytes,
 * when the device cannot hold it.  Waits for the trainer's work in flight. */
int rnnoise_train_pool_reserve(RNNoiseTrainer *t, long long n_samples);
/* HOST src: n samples into pool[at .. at + n), which must lie within the reservation.  Synchronous. */
int rnnoise_train_pool_write(RNNoiseTrainer *t, long long at, const short *src, long long n);
/* Samples in the pool (0 without one). */
long long rnnoise_train_pool_samples(const RNNoiseTrainer *t);
/* Bytes a pool reservation may take on the trainer's device (its free memory plus the current pool) and the device's
 * total memory. */
int rnnoise_train_pool_room(const RNNoiseTrainer *t, size_t *room_bytes, size_t *total_bytes);
/* n_frames frames of every lane.  HOST sig_at / noise_at [n_frames][n_lanes]: each lane-frame's 480 samples are
 * pool[at .. at + 480), or zeros for -1; every offset is checked first, and one outside [0, pool_samples - 480] fails the
 * call naming its frame and lane.  DEVICE outputs, float32: sample (l, t, i) of noisy, clean and noise (may be NULL) at
 * ptr[l*stream_stride + t*frame_stride + i] (the sample layout of rnnoise_batch_analyze_window_device; rows must not
 * overlap), vad (may be NULL) (l, t) at vad[l*vad_stream_stride + t*vad_frame_stride].  Frame t continues each lane from
 * the previous call's last frame.  Ordered after cuda_stream, which continues after the call; the call returns without
 * waiting for the kernel when a stream is given (NULL: it returns when the frames are written).  The offsets are staged
 * in trainer-owned buffers that no call reuses while an earlier call may read them. */
int rnnoise_train_waves_device(RNNoiseTrainer *t, const long long *sig_at, const long long *noise_at, int n_frames,
                               float *noisy, float *clean, float *noise, float *vad, long stream_stride, long frame_stride,
                               long vad_stream_stride, long vad_frame_stride, void *cuda_stream);

/* ---- fitting denoise models to training rows on the GPU (additive; what train/rnn_train.py does with Keras, then
 * train/dump_rnn.py; DESIGN.md section 7e) ----------------------------------------------------------------------------
 * The network of rnn_train.py with layer widths nd (input_dense), nv (vad_gru), nn (noise_gru), ndn (denoise_gru), each
 * 1..96, exact activations (tanh, tanh, relu, tanh, sigmoid, sigmoid unless set from a model), every sequence from
 * a zero state.  Parameters are one flat f32 vector in the order of the
 * .rnn file (input_dense, vad_gru, noise_gru, denoise_gru, denoise_output, vad_output), each layer as kernel
 * [inputs][gates * neurons] row-major, then (GRUs) recurrent [neurons][3 * neurons], then bias; GRU gates z | r | h~.
 * Rows are [n_seq][window][87] training rows (rnnoise_train_*), weights [n_seq][window] sample weights, both in host or
 * device memory.  Loss: 10 mycost + 0.5 my_crossentropy (weighted sums over the n_seq * window frames, divided by
 * their number) + 1e-6 sum w^2 over the GRUs' kernel and recurrent matrices.  Optimiser: tf.keras Adam (lr 1e-3,
 * 0.9, 0.999, eps 1e-7), then every parameter clipped to +-0.499.  Calls restore the caller's device; errors return
 * a negative code (0 for the size_t calls) and rnnoise_last_error() says why. */
typedef struct RNNoiseFit RNNoiseFit;
/* Parameters start at zero: set them before the first step.  max_sequences bounds n_seq of every call. */
RNNoiseFit *rnnoise_fit_create(int nd, int nv, int nn, int ndn, int max_sequences, int window, int device);
void rnnoise_fit_destroy(RNNoiseFit *f);
long rnnoise_fit_n_params(const RNNoiseFit *f);
int rnnoise_fit_get_params(RNNoiseFit *f, float *params);                /* HOST [n_params] */
int rnnoise_fit_set_params(RNNoiseFit *f, const float *params);          /* HOST [n_params]; resets Adam */
/* Weights int8 / 256 (NULL: built-in), to fine-tune a model.  The fit also takes the model's activations for
 * input_dense and the GRUs (the built-in model's vad and denoise GRUs use relu), so that an export of an unchanged model
 * gives back its bytes; both output layers must be sigmoid.  Resets Adam. */
int rnnoise_fit_set_params_from_model(RNNoiseFit *f, const RNNModel *model);
/* One Adam step on n_seq sequences; *loss (may be NULL) = the loss before the step. */
int rnnoise_fit_step(RNNoiseFit *f, const float *rows, const float *weights, int n_seq, double *loss);
/* The loss without a step: out = {total, mycost, my_crossentropy, msse} (msse unweighted, of the gains). */
int rnnoise_fit_evaluate(RNNoiseFit *f, const float *rows, const float *weights, int n_seq, double out[4]);
/* Debug taps (HOST buffers): the gradient of the most recent step's loss, L2 term included, [n_params]; and the most
 * recent forward pass's outputs, gains [n_seq][window][22], vad [n_seq][window], GRU states [n_seq][window][nv+nn+ndn]
 * (any pointer may be NULL). */
int rnnoise_fit_get_grads(RNNoiseFit *f, float *grads);
int rnnoise_fit_get_activations(RNNoiseFit *f, float *gains, float *vad, float *state);
/* Stage taps, to test each kernel from its own inputs (HOST buffers, any pointer may be NULL), over the n_seq sequences of
 * the most recent forward (n_seq must be its count), rows r = s * window + t, R = n_seq * window.  After the forward: the
 * input_dense output d [R][nd] and, per GRU, the three GRUs' arrays one after another in vad | noise | denoise order:
 * gates z | r | h~ [R][3n], r * h_{t-1} [R][n] and the states hbuf [n_seq][window + 1][n] (row 0: the initial state).
 * After a backward of that forward: input_dense's pre-activation gradient dd [R][nd], the output-layer gradients
 * dzo [R][22], dzv [R] and per GRU the gradient dh [R][n] the later layers pass to h_t; and, when that backward ran with
 * taps on, the gate pre-activation gradients dG [R][3n] and the total dL/dh_t the recurrence read at each step,
 * dht [R][n].  A request for a backward's array without that backward is refused.  rnnoise_fit_set_taps(f, 1) makes every later backward keep dG
 * and dht (one device-to-device copy per GRU; the buffers are allocated on the first call); off, a step issues exactly
 * the work it does without taps.  Taps never change a computed value. */
int rnnoise_fit_set_taps(RNNoiseFit *f, int on);
int rnnoise_fit_get_taps(RNNoiseFit *f, int n_seq, float *d, float *dd, float *gates, float *rh, float *hbuf, float *dh, float *dzo,
                         float *dzv, float *dG, float *dht);
/* The .rnn model bytes of the current parameters (dump_rnn.py: clip(round_half_even(256 w), -128, 127)); returns the
 * size (buf NULL: the size only).  The format stores input counts in a signed byte: 42 + nd + nv and 42 + nv + nn must
 * be at most 127. */
size_t rnnoise_fit_export(RNNoiseFit *f, unsigned char *buf, size_t cap);
/* The same from a HOST parameter vector, without a fit handle or a GPU. */
size_t rnnoise_fit_export_params(int nd, int nv, int nn, int ndn, const float *params, unsigned char *buf, size_t cap);
/* Training the network on any loss (DESIGN.md section 7l): forward and backward over windows of DEVICE features, e.g.
 * those of rnnoise_batch_analyze_window_device, so that the gradients with respect to gains and vad can come from a
 * loss of the synthesized output (rnnoise_synthesis_backward_device) or any other.  The network and activations are the
 * fit's (the script's, or a model's after set_params_from_model); the parameters are read from `params`, DEVICE
 * [n_params] in the flat layout above, not from the fit's own vector; no L2 term and no clip.  Every call covers n_seq
 * (1..max_sequences) sequences of `window` frames.
 * Layouts (element strides): feature j of (s, t) at features[s*feature_seq_stride + t*feature_frame_stride + j],
 * band k of the gains likewise, vad (s, t) at vad[s*vad_seq_stride + t*vad_frame_stride], silence (s, t) likewise
 * (int32; rnnoise_batch_analyze_window_device's [n_frames][n_streams] array is seq stride 1, frame stride n_streams).
 * Output rows must not overlap.
 * Silent frames (silence != 0; silence NULL: none) are what the fused network does with them: nothing is evaluated,
 * every GRU state is carried (h_t = h_{t-1}), and gains and vad are written as 0, the vad synthesis reports for a
 * silent frame.  In the backward their incoming gradients are not read, they add nothing to any weight gradient, and
 * dL/dh passes through them unchanged.
 * State: state_in and state_out are [n_seq][nv + nn + ndn] (vad | noise | denoise GRU, rnn_taps' gru_state order),
 * contiguous; state_in NULL means zeros, state_out NULL is not written, and the two may be the same array.  No gradient
 * flows to state_in (truncated backpropagation through time), nor to the features.
 * Work is ordered after cuda_stream, and cuda_stream continues after it (NULL: the call returns when it is done).  The
 * same inputs give the same bits.  A refused call changes nothing. */
int rnnoise_fit_forward_device(RNNoiseFit *f, const float *params, int n_seq, const float *features, long feature_seq_stride,
                               long feature_frame_stride, const int *silence, long silence_seq_stride, long silence_frame_stride,
                               const float *state_in, float *state_out, float *gains, long gain_seq_stride, long gain_frame_stride,
                               float *vad, long vad_seq_stride, long vad_frame_stride, void *cuda_stream);
/* grad_params (DEVICE [n_params], overwritten) = dL/dparams for L = sum(grad_gains * gains) + sum(grad_vad * vad) of the
 * most recent rnnoise_fit_forward_device on this fit, whose n_seq and silence it uses.  grad_vad NULL means zero.
 * Refused when no forward_device ran, when rnnoise_fit_step or rnnoise_fit_evaluate ran since (they overwrite the same
 * activations), when `params` is not the pointer that forward ran with, or when grad_params overlaps params. */
int rnnoise_fit_backward_device(RNNoiseFit *f, const float *params, const float *grad_gains, long gg_seq_stride, long gg_frame_stride,
                                const float *grad_vad, long gv_seq_stride, long gv_frame_stride, float *grad_params, void *cuda_stream);

/* ---- file front-end (additive; what the reference's `nnnoiseless` binary does around the path, src/nnnoiseless.rs) --
 * decode (raw little-endian i16, or RIFF/WAVE: 8/16/24/32-bit integer and 32-bit float) -> resample to 48 kHz when
 * the rate differs (dasp `Sinc<[f32; 16]>` at ratio rate/48000, on the GPU) -> one DenoiseState per channel ->
 * the first frame's output is discarded, a trailing partial frame dropped -> clamp + round to i16 -> raw or 48 kHz
 * 16-bit WAV.  Every file call runs on the corpus engine below at its default options, and takes its contract and
 * refusals.  With one file, rnnoise_denoise_file and rnnoise_denoise_files first open the input and create the output,
 * as the reference binary does, so a refused one-file call may leave an empty output.  A call none of whose files has
 * two whole 48 kHz frames makes no CUDA call: it writes each file's empty output. */
typedef struct RNNoiseFileOptions {
    int wav_in;            /* non-zero: inputs are WAV; 0: decided per file by a ".wav" extension (--wav-in)  */
    int wav_out;           /* same for the outputs (--wav-out)                                                */
    double sample_rate;    /* raw input only (--sample-rate); <= 0: 48000                                     */
    int channels;          /* raw input only (--channels); <= 0: 1                                            */
    const RNNModel *model; /* NULL: built-in (--model)                                                        */
    int device;            /* CUDA device, -1: current                                                        */
} RNNoiseFileOptions;
int rnnoise_denoise_file(const char *in_path, const char *out_path, const RNNoiseFileOptions *opt);
int rnnoise_denoise_files(int n_files, const char *const *in_paths, const char *const *out_paths,
                          const RNNoiseFileOptions *opt);
/* rnnoise_denoise_files with the channels of every multi-channel file linked as one group (DESIGN.md section 7n):
 * link_mode RNNOISE_LINK_MAX or RNNOISE_LINK_MEAN (--link-channels), or 0 for rnnoise_denoise_files' behaviour.  Mono
 * files are unaffected; a file of more than RNNOISE_LINK_MAX_MEMBERS channels is refused when link_mode is not 0. */
int rnnoise_denoise_files_linked(int n_files, const char *const *in_paths, const char *const *out_paths,
                                 const RNNoiseFileOptions *opt, int link_mode);

/* ---- a corpus of files on recycled stream slots (additive; DESIGN.md section 7o) ------------------------------------
 * rnnoise_denoise_corpus denoises any number of files on one batch of `slots` streams; rnnoise_denoise_files is this
 * call with every default.  Files enter in list order, each
 * when as many slots as it has channels are free; all of a file's channels enter together, at a chunk boundary, on
 * streams reset by rnnoise_batch_reset_streams (and, with a link mode, linked as one group).  Every output file is byte
 * for byte what the call writes for that input alone with the same options, whatever the slot count, chunk length and
 * file order: one DenoiseState per channel (one linked group per file with a link mode) run over the file's whole
 * frames.
 * Refused before any output is created and before any CUDA call: bad option values; an output that is also an input,
 * or one output listed twice; an input that cannot be opened or whose WAV header fails (rnnoise_audio_probe's texts);
 * a file of more channels than `slots` (1048576 when `slots` is 0), or of more than RNNOISE_LINK_MAX_MEMBERS channels
 * with a link mode.  A later
 * error (a decoder refusing a file's data, a write or CUDA failure) fails the call naming the file; every file listed
 * before a file the decoder refuses is still written.  An output is created only once its file is complete, so no
 * output is left half written; a write error names the file, and an existing file that could not be opened is left
 * as it was.  The device holds the sources of the files in slots plus decode-ahead within device_pool_bytes (a file
 * larger than the budget runs when the pool is otherwise empty).  Each output is handed to a writer thread as soon as
 * its last frame is back; the outputs waiting to be written hold at most device_pool_bytes of host memory (one larger
 * output is taken alone), and the call waits for room.  Besides them the host holds the outputs of the files in slots
 * and up to decode_threads decoded files. */
/* slots 0: max(the widest file's channels, min(256, the channels of all files)), so a short list runs on exactly its
 * own channels.  chunk_frames 0: min(64, 2097152 / slots).  An explicit slots * chunk_frames is at most 2097152. */
typedef struct RNNoiseCorpusOptions {
    int slots;                   /* streams of the batch, fixed for the call; 0: the rule above                     */
    int chunk_frames;            /* 10 ms frames per device call; 0: the rule above                                 */
    long long device_pool_bytes; /* budget for decoded sources on the device (float32 samples); 0: 1 GiB           */
    int decode_threads;          /* host threads decoding ahead; 0: the hardware threads, at most 8                */
} RNNoiseCorpusOptions;
typedef struct RNNoiseCorpusStats {
    long long files;                /* outputs written                                                          */
    long long useful_stream_frames; /* sum of channels * frames over the files that took slots                 */
    long long issued_slot_frames;   /* slots * frames of every chunk run                                        */
    long long chunks;               /* device calls                                                             */
    long long peak_pool_bytes;      /* most bytes of decoded sources held in the pool at once                  */
    double decode_wait_seconds;     /* host time the scheduler waited for decoded input                        */
    double device_wait_seconds;     /* host time the scheduler waited for the device                           */
    double write_wait_seconds;      /* host time the call waited for the writer: for room, and for the last outputs */
} RNNoiseCorpusStats;
/* copt NULL: every default.  stats may be NULL; it is filled on success and on a failure found after the checks. */
int rnnoise_denoise_corpus(int n_files, const char *const *in_paths, const char *const *out_paths, const RNNoiseFileOptions *opt,
                           int link_mode, const RNNoiseCorpusOptions *copt, RNNoiseCorpusStats *stats);
/* The decoders / encoders alone (host code).  wav: 1 = RIFF/WAVE, -1 = raw, 0 = by ".wav" extension.  Decoded samples are
 * interleaved floats in the i16 range exactly as the binary feeds them to the path (src/nnnoiseless.rs:57-77, 190-228);
 * *samples is malloc'ed: release with rnnoise_audio_free.  Writers: raw little-endian i16 or 48 kHz 16-bit WAV. */
int rnnoise_audio_read(const char *path, int wav, int raw_channels, double raw_rate, float **samples, long *n_frames,
                       int *channels, double *sample_rate);
void rnnoise_audio_free(float *samples);
/* A RIFF/WAVE file's header alone, with read_audio's checks and error texts: the format, and where the samples are.
 * Sample i of channel c is at byte data_offset + (i * channels + c) * bits_per_sample / 8 (container bytes). */
typedef struct RNNoiseAudioInfo {
    int channels, sample_rate, bits_per_sample;
    int is_float;             /* 1: IEEE float samples; 0: integer PCM */
    long long data_offset;    /* byte offset of the data chunk's first sample */
    long long n_frames;       /* samples per channel */
} RNNoiseAudioInfo;
int rnnoise_audio_probe(const char *path, RNNoiseAudioInfo *info);
int rnnoise_audio_write(const char *path, int wav, const short *pcm, long n_frames, int channels);
/* The resampler alone, HOST buffers: in [n_in][channels] interleaved -> out [<= cap][channels]; returns the number of
 * output sample frames (Resample::next_sample until the source runs dry, src/nnnoiseless.rs:104-131), < 0 on error. */
long rnnoise_resample_host(float *out, long cap, const float *in, long n_in, int channels, double ratio, int device);

/* ---- streams at their own sample rate (additive; DESIGN.md section 7g) ----------------------------------------------
 * The denoise path runs on 48 kHz frames of 480 samples.  A resampler holds, for each of n_streams streams, a rate R
 * (8000 <= R <= 48000, R % 100 == 0: 8, 12, 16, 24, 32, 44.1, 48 kHz ...) and the filter history of two stages:
 *   up:   R/100 native samples of a 10 ms frame -> 480 samples at 48 kHz,
 *   down: 480 samples at 48 kHz -> R/100 native samples.
 * With g = gcd(48000, R), U = 48000/g and D = R/g, the up stage is scipy.signal.upfirdn(h, x, U, D) and the down
 * stage upfirdn(h', y, D, U): polyphase, causal, no delay compensation, with scipy.signal.resample_poly's default
 * filter firwin(20 max(up, down) + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up, designed in double, stored as
 * float.  After frames 0..t the concatenated output of a stage is the prefix of that upfirdn, up to float rounding: each
 * output sample is a sum of float products in ascending tap index (FMA allowed).  A stream's bits depend on its own rate
 * and samples only: not on how its frames are split into calls, nor on the batch size, row, subset or the other streams.
 * 48 kHz streams pass through unchanged.  Resampler and batch are separate handles: the batch and its state records
 * are unchanged by this section.  Every call leaves the caller's current device as it found it; errors return a
 * negative code and rnnoise_last_error() says why. */
typedef struct RNNoiseResampler RNNoiseResampler;
/* The filter of one stage, direction 0 = up (R -> 48 kHz), 1 = down (48 kHz -> R), in tap order: returns the number of
 * taps and writes min(taps, cap) of them to taps (may be NULL), the stage's factors to *up and *down (may be NULL).
 * 48 kHz: one tap of 1, up = down = 1.  Host code; needs no GPU. */
int rnnoise_resampler_filter(int rate, int direction, float *taps, int cap, int *up, int *down);
/* The delay the up and down stages add together, in 48 kHz samples: 960000 / R (60 at 16 kHz, 21.77... at 44.1 kHz),
 * 0 at 48 kHz; negative for an invalid rate.  The denoiser's own delay (one 480-sample frame) is not included. */
double rnnoise_resampler_delay(int rate);
/* n_streams streams on CUDA device `device` (-1: current), stream s at rates[s] (rates NULL: every stream at 48000),
 * histories zero.  The rates are checked before the device is touched; a bad one is named with its stream. */
RNNoiseResampler *rnnoise_resampler_create(int n_streams, const int *rates, int device);
void rnnoise_resampler_destroy(RNNoiseResampler *r);
/* Stream streams[i] (streams NULL: i) gets rate rates[i], and its histories are reset to zero, even when the rate is
 * unchanged: this is also the reset.  Every index and rate is checked first; on an error nothing changes. */
int rnnoise_resampler_set_stream_rates(RNNoiseResampler *r, const int *streams, int n, const int *rates);
int rnnoise_resampler_get_stream_rates(const RNNoiseResampler *r, const int *streams, int n, int *rates);
/* The stages alone, DEVICE pointers.  Row i of the call is stream streams[i] (NULL: i), distinct indices.  Native
 * sample (i, t, k), k < R/100, is at ptr[i * stream_stride + t * frame_stride + k] (element strides; pcm16 0: float,
 * 1: int16, converted like the batch's int16 output: clamp, then round half away from zero); the 48 kHz side is compact
 * [n_frames][n][480] float.  With a cuda_stream the call is asynchronous and ordered on it; without one it synchronises. */
int rnnoise_resampler_up_device(RNNoiseResampler *r, const int *streams, int n, float *out, const void *in, int pcm16, int n_frames,
                                long stream_stride, long frame_stride, void *cuda_stream);
int rnnoise_resampler_down_device(RNNoiseResampler *r, const int *streams, int n, void *out, const float *in, int pcm16, int n_frames,
                                  long stream_stride, long frame_stride, void *cuda_stream);
/* State records of single streams, HOST memory, RNNOISE_RESAMPLER_STATE_BYTES each, little-endian:
 *   offset 0: u32 magic RNNOISE_RESAMPLER_STATE_MAGIC ("RSST"), i32 version 1, i32 rate, i32 0
 *         16: f32 up history[20], the last native samples the up stage read, oldest first
 *         96: f32 down history[120], the last 48 kHz samples the down stage read, oldest first
 * With the stream's batch record (rnnoise_batch_get_states) it moves or restores a native-rate stream bit for bit.
 * set_states checks every record (magic, version, rate) and index before anything is written; it sets the rates. */
#define RNNOISE_RESAMPLER_STATE_MAGIC 0x54535352u
#define RNNOISE_RESAMPLER_STATE_VERSION 1
#define RNNOISE_RESAMPLER_STATE_BYTES 576
int rnnoise_resampler_get_states(RNNoiseResampler *r, const int *streams, int n, void *dst);
int rnnoise_resampler_set_states(RNNoiseResampler *r, const int *streams, int n, const void *src);
/* Denoise native-rate streams: up -> rnnoise_batch_process_device (streams NULL and n == n_streams) or
 * rnnoise_batch_process_streams_device -> down, on one CUDA stream, in place on 48 kHz scratch owned by the resampler
 * (at most 256 MiB: longer calls go through in chunks of frames).  Subset semantics and per-stream models apply as in
 * those calls.  The handles must have the same n_streams and device.  Layout and pcm16 as the stage calls; vad
 * [n_frames][n] or NULL.  Every argument is checked first; on an error nothing changes. */
int rnnoise_batch_process_native_device(RNNoiseBatch *b, RNNoiseResampler *r, const int *streams, int n, void *out, const void *in, int pcm16,
                                        float *vad, int n_frames, long stream_stride, long frame_stride, void *cuda_stream);
/* The same through HOST buffers of [n_frames][n][480] slots: the first R/100 samples of a slot are the stream's frame,
 * the rest are ignored on input and written as 0 on output.  vad [n_frames][n] or NULL.  Synchronises. */
int rnnoise_batch_process_native_host(RNNoiseBatch *b, RNNoiseResampler *r, const int *streams, int n, void *out, const void *in, int pcm16,
                                      float *vad, int n_frames);

/* ---- quality metrics against clean speech (additive; DESIGN.md section 7p) -----------------------------------------
 * A metrics handle scores n_streams denoised streams against their clean speech on the GPU, frame by frame, into one
 * record per stream.  Output frame t of a stream is paired with clean frame t - 1 (the denoiser's one-frame delay); the
 * pairing state (the last clean frame and its target, the previous output and clean half-windows) lives on the device,
 * so any split of a stream's frames into calls gives the same records bit for bit.  The first output frame after
 * creation pairs with nothing and is not counted.
 * A counted frame (y = output frame, c = the clean frame paired with it) is in class "all", and in "speech" when c's
 * target is 1 or "noise" when it is 0 (0.5, another value, or no target pointer in the call that brought c: neither).
 * Every counted frame adds to its classes Ec = sum c^2, Ey = sum y^2, Ecy = sum c y and Ed = sum (y - c)^2 (products
 * exact in double, sums in double, frame order).  Band energies Yb, Cb (b < 22) are computed as the analysis kernel's
 * `ex` of the 960-sample windows [previous half | this frame], and Lb = 10 log10(E_b + 0.01) in double.  A speech frame adds its
 * segmental SNR (35 when Ed = 0, else 10 log10(Ec / Ed) clamped to [-10, 35]), its log-spectral distance
 * sqrt(mean_b (Ly_b - Lc_b)^2) and per band Ly_b - Lc_b; a noise frame adds Ly_b per band.  With both vad pointers,
 * a counted frame whose own target (no lag) is 0 or 1 adds one of tp, fp, fn, tn (the network's vad >= 0.5: speech).
 * Sample (s, t, i) of out and clean is at ptr[s * stream_stride + t * frame_stride + i]; vad (s, t) and vad_target
 * (s, t) at ptr[s * vad_stream_stride + t * vad_frame_stride] (each may be NULL).  Rows must not overlap.  Every call
 * leaves the caller's current device as it found it; errors return -1 and rnnoise_last_error() says why, with nothing
 * changed. */
typedef struct RNNoiseMetrics RNNoiseMetrics;
typedef struct RNNoiseMetricsRecord {
    long long frames[3];              /* counted frames: all, speech, noise */
    double ec[3], ey[3], ecy[3], ed[3]; /* per class, as frames */
    double seg_snr, lsd;              /* sums over speech frames */
    double speech_dev[22];            /* speech frames: sum of Ly_b - Lc_b */
    double noise_level[22];           /* noise frames: sum of Ly_b */
    long long vad_counts[4];          /* tp, fp, fn, tn */
    float last_bands[2][22];          /* Yb, Cb of the last counted frame */
} RNNoiseMetricsRecord;               /* 696 bytes */
/* n_streams streams on CUDA device `device` (-1: current), records and pairing state zero.  NULL on error. */
RNNoiseMetrics *rnnoise_metrics_create(int n_streams, int device);
void rnnoise_metrics_destroy(RNNoiseMetrics *m);
/* Scores n_frames frames of every stream.  Ordered after cuda_stream, which continues after the call; without one the
 * call returns when the work has finished. */
int rnnoise_metrics_accumulate_device(RNNoiseMetrics *m, const float *out, const float *clean, long stream_stride, long frame_stride,
                                      const float *vad, const float *vad_target, long vad_stream_stride, long vad_frame_stride,
                                      int n_frames, void *cuda_stream);
/* Zeroes the records of streams[i] (streams NULL: i < n) and keeps their pairing state: frames before the clear are
 * dropped without breaking the pairing.  Ordered after the handle's accumulate calls; returns when done. */
int rnnoise_metrics_clear(RNNoiseMetrics *m, const int *streams, int n);
/* The records of streams[i] (streams NULL: i < n) to dst[i], host memory, after every call issued so far. */
int rnnoise_metrics_get(RNNoiseMetrics *m, const int *streams, int n, RNNoiseMetricsRecord *dst);

/* ---- intelligibility: STOI and ESTOI of clips (additive; DESIGN.md section 7q) --------------------------------------
 * Scores n_pairs pairs (y = processed `out`, x = `clean`) of n_samples float samples each, all at one rate R (a
 * multiple of 100 in 8000..48000), with STOI (Taal et al., IEEE TASLP 2011) and ESTOI (Jensen & Taal, IEEE TASLP
 * 2016).  EPS = 2^-52.
 *   1. Both signals to 10 kHz: g = gcd(R, 10000), up = 10000/g, down = R/g, half = 10 max(up, down), h = the float taps
 *      of firwin(2 half + 1, 1/max(up, down), window=('kaiser', 5.0)) * up designed in double (the resampler's filter
 *      design), x10[m] = sum_n x[n] h[half + m down - n up] over the taps, samples outside the clip 0, m < n10 =
 *      ceil(n up / down); a float sum of float products in ascending tap order, FMA allowed.  At 10 kHz x10 = x.
 *   2. Frames w x10[128 f .. 128 f + 256), w[i] = 0.5 - 0.5 cos(2 pi (i + 1) / 257), f < F = n10 >= 256 ?
 *      (n10 - 256) / 128 + 1 : 0.
 *   3. Frame f of the clean signal has E_f = 20 log10(||w x10 frame||_2 + EPS) in double; it is kept when
 *      E_f > max E - 40.  The K kept frames of each signal are overlap-added at hop 128 in kept order.
 *   4. STFT of the result: M = K - 1 frames of 256 samples at hop 128, windowed by w, 512-point DFT.
 *   5. 15 third-octave bands from 150 Hz, bins [7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219):
 *      X[b][m] = sqrt(sum of |X_m(k)|^2 over the band), stored as float; everything after it runs in double.
 *   6. STOI: over the S = M - 29 segments of 30 consecutive frames and the 15 bands, the mean of the correlations of
 *      x and y' = min(alpha y, c x), alpha = ||x|| / (||y|| + EPS), c = 1 + 10^(15/20); a correlation is
 *      <x - mean x, y' - mean y'> / ((||x - mean x|| + EPS) (||y' - mean y'|| + EPS)).
 *   7. ESTOI: each segment's 15 x 30 matrices have their rows, then their columns, centred and divided by their
 *      norm + EPS; ESTOI = sum of the products / (30 S).
 *   8. S < 1: both scores are NaN; the counts are still written.
 * Sample i of pair p is at ptr[p * stream_stride + i] (DEVICE memory; rows must not overlap: stream_stride >=
 * n_samples).  Stateless: runs on `device` (< 0: the current device) after the work queued on cuda_stream, which
 * continues after it (without a stream the call returns when the work has finished).  Every argument is checked
 * before any CUDA call; a refused call changes nothing, and rnnoise_last_error() says why.  Four kernel launches.
 * Workspace (DEVICE memory, 256-byte aligned), regions in this order, each starting at a multiple of 256 bytes:
 *   x10, y10:  float [2][n_pairs][n10]          (0: clean, 1: out)
 *   kept:      int [n_pairs][F]                 entry k < K: the index of the k-th kept frame; -1 after
 *   bands:     float [2][n_pairs][15][max(F - 1, 0)]   band b of STFT frame m at [b][m], m < M
 *   tables:    the polyphase taps, the window and the FFT twiddles (internal). */
typedef struct RNNoiseIntelligibility {
    double stoi, estoi;      /* NaN when segments < 1 */
    int frames;              /* F: 10 kHz frames of the clip */
    int kept;                /* K: frames kept by the silence rule */
    int segments;            /* S = max(K - 30, 0) */
    int reserved;            /* 0 */
} RNNoiseIntelligibility;    /* 32 bytes */
/* Bytes of workspace for the call (host only); 0 on bad arguments or a size past SIZE_MAX. */
size_t rnnoise_intelligibility_workspace_bytes(int n_pairs, long n_samples, int rate);
int rnnoise_intelligibility_device(const float *out, const float *clean, int n_pairs, long n_samples, long stream_stride,
                                   int rate, RNNoiseIntelligibility *result /* DEVICE, n_pairs */,
                                   void *workspace, size_t workspace_bytes, int device, void *cuda_stream);

/* Backward (DESIGN.md section 7r): after rnnoise_intelligibility_device(out, clean, n_pairs, n_samples, ., rate,
 * result, fwd_workspace, ...), writes grad_out[p * grad_stride + i] = dL/d out[p][i] for every i < n_samples of every
 * pair, L = sum_p (grad_stoi[p] stoi_p + grad_estoi[p] estoi_p) (grad_stoi or grad_estoi NULL: that term is 0).  It
 * overwrites grad_out, it does not accumulate into it.
 *   - It differentiates steps 1-7 as written, with the float rounding of step 5's bands taken as the identity.
 *   - clean is a constant: the silence rule depends on clean alone, so the kept list is constant and needs no gradient.
 *   - Kinks: min(alpha y, c x) follows the y branch when alpha y <= c x.  A zero band magnitude, a zero ||y|| of a
 *     band-segment and a zero centred norm contribute 0 there (the subgradient at the square root's zero).
 *     d by[b] / by[b] is formed in double, so a band just above 0 (where d by nears 1/EPS) still gives a finite float
 *     gradient.
 *   - Pairs with segments < 1 get +0.0 in every sample, whatever their grad_stoi and grad_estoi (NaN included).
 *   - A sample whose 10 kHz filter support meets no sample that an STFT frame reads gets +0.0.
 * It reads the forward workspace's x10 / y10, kept and bands regions and its tables, and the records; not the signals.
 * The conventions are the forward's: stateless, no allocation (graph-capturable); every argument (nulls, alignment,
 * sizes, grad_stride >= n_samples, both workspaces' bytes for (n_pairs, n_samples, rate)) is checked before any CUDA
 * call and a refused call changes nothing; ordered after the work queued on cuda_stream (without one it returns when
 * done).  Deterministic: no floating-point atomics, every output element is summed by one thread in a fixed order, so
 * the result is bit-reproducible under any permutation of the pairs and any grid size.  Four kernel launches.
 * Workspace (DEVICE memory, 256-byte aligned), regions in this order, each starting at a multiple of 256 bytes:
 *   dbands:  double [n_pairs][15][max(F - 1, 0)]  dL/d (out's band b of STFT frame m) at [b][m], m < M
 *   inverse: int [n_pairs][F]                     the kept index of 10 kHz frame f, or -1
 *   dframes: float [n_pairs][max(F - 1, 0)][256]  dL/d (sample i of the overlap-added out before STFT frame m's
 *                                                 window) at [m][i], m < M
 *   dy10:    float [n_pairs][n10]                 dL/d y10 */
size_t rnnoise_intelligibility_backward_workspace_bytes(int n_pairs, long n_samples, int rate);
int rnnoise_intelligibility_backward_device(int n_pairs, long n_samples, int rate,
                                            const RNNoiseIntelligibility *result /* DEVICE: the forward's records */,
                                            const void *fwd_workspace, size_t fwd_workspace_bytes /* as the forward left it */,
                                            const double *grad_stoi, const double *grad_estoi /* DEVICE [n_pairs] or NULL */,
                                            float *grad_out, long grad_stride, void *workspace, size_t workspace_bytes,
                                            int device, void *cuda_stream);

/* Number of kernel launches issued by this library since load (bench evidence). */
unsigned long long rnnoise_kernel_launches(void);

/* Text of the most recent error on this thread ("" if none). */
const char *rnnoise_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* RNNOISE_H */
