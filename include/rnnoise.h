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
 * without one it synchronises.  The cost grows with n: the listed streams' live state (8,396 bytes per stream for the
 * built-in model) is gathered into a compact work state, advanced there by the frame kernels, and scattered back
 * (10,316 bytes: the full 1728-sample input_mem of the record).
 * Device memory: the work state is allocated on first use and grows to the largest n used so far, about
 * 4 * (4523 + nv + nn + nd) bytes per row (18,764 bytes for the built-in model: 1.23 GB at n = 65,536); it is freed by
 * rnnoise_batch_destroy.  The frames' intermediates reuse the batch's own buffers.
 * rnnoise_batch_get_taps / get_rnn_taps / get_spectral_taps describe full-batch frames: after a subset call they return an error until the
 * next full-batch frame. */
int rnnoise_batch_process_streams_device(RNNoiseBatch *b, const int *streams, int n, void *out, const void *in, int pcm16, float *vad,
                                         int n_frames, long stream_stride, long sample_stride, long frame_stride, void *cuda_stream);
/* Same through HOST buffers, float samples, compact layout in/out [n_frames][n][480], vad [n_frames][n] (may be NULL).
 * Frames stream through the batch's staging ring: the device memory does not grow with n_frames. */
int rnnoise_batch_process_streams_host(RNNoiseBatch *b, const int *streams, int n, float *out, const float *in, float *vad,
                                       int n_frames);

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
 * whose coarse pitch search had to be recomputed in the reference's operation order because the fast (FMA) values could
 * not certify find_best_pitch's decisions (src/pitch.rs:372-405), out[1] = the same for remove_doubling's ladder
 * (src/pitch.rs:144-203), out[2] = stream-frames processed.  The integer period is bit-identical either way. */
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

/* ---- file front-end (additive; what the reference's `nnnoiseless` binary does around the path, src/nnnoiseless.rs) --
 * decode (raw little-endian i16, or RIFF/WAVE: 8/16/24/32-bit integer and 32-bit float) -> resample to 48 kHz when
 * the rate differs (dasp `Sinc<[f32; 16]>` at ratio rate/48000, on the GPU) -> one DenoiseState per channel ->
 * the first frame's output is discarded, a trailing partial frame dropped -> clamp + round to i16 -> raw or 48 kHz
 * 16-bit WAV.  All channels of all files of one call are streams of one batch. */
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
/* The decoders / encoders alone (host code).  wav: 1 = RIFF/WAVE, -1 = raw, 0 = by ".wav" extension.  Decoded samples are
 * interleaved floats in the i16 range exactly as the binary feeds them to the path (src/nnnoiseless.rs:57-77, 190-228);
 * *samples is malloc'ed: release with rnnoise_audio_free.  Writers: raw little-endian i16 or 48 kHz 16-bit WAV. */
int rnnoise_audio_read(const char *path, int wav, int raw_channels, double raw_rate, float **samples, long *n_frames,
                       int *channels, double *sample_rate);
void rnnoise_audio_free(float *samples);
int rnnoise_audio_write(const char *path, int wav, const short *pcm, long n_frames, int channels);
/* The resampler alone, HOST buffers: in [n_in][channels] interleaved -> out [<= cap][channels]; returns the number of
 * output sample frames (Resample::next_sample until the source runs dry, src/nnnoiseless.rs:104-131), < 0 on error. */
long rnnoise_resample_host(float *out, long cap, const float *in, long n_in, int channels, double ratio, int device);

/* Number of kernel launches issued by this library since load (bench evidence). */
unsigned long long rnnoise_kernel_launches(void);

/* Text of the most recent error on this thread ("" if none). */
const char *rnnoise_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* RNNOISE_H */
