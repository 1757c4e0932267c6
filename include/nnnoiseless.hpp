// nnnoiseless.hpp -- C++ mirror of the reference's Rust API for the per-frame denoise path, layered on
// the C ABI of rnnoise.h.  The reference is compiled code (Rust); no Rust toolchain exists in this
// image, so the host side above the C ABI is C++ with the same names, argument meaning and error
// behaviour as:
//   nnnoiseless::RnnModel      src/rnn.rs:55-94, 235-240   (from_bytes -> Option, Default, Clone)
//   nnnoiseless::DenoiseState  src/denoise.rs:37-116        (FRAME_SIZE, new, from_model, with_model,
//                                                             process_frame; panics on wrong length)
// plus the additive batched type (N independent DenoiseStates advanced by one call).
//
// Header-only; link with libnnnoiseless_b200.so.  There is no CPU fallback: constructors throw
// std::runtime_error when no CUDA device is usable.
#pragma once
#include <cstddef>
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "rnnoise.h"

namespace nnnoiseless {

/// `RnnModel` (src/rnn.rs:55-62).  Default-constructed = the built-in model (`impl Default`, :235-240).
class RnnModel {
  public:
    RnnModel() = default;  // built-in weights (NULL at the C ABI)

    /// `RnnModel::from_bytes(&[u8]) -> Option<RnnModel>` (src/rnn.rs:75): nullopt on malformed bytes.
    static std::optional<RnnModel> from_bytes(const uint8_t* bytes, size_t len) {
        ::RNNModel* h = rnnoise_model_from_bytes(bytes, len);
        if (!h) return std::nullopt;
        return RnnModel(h);
    }
    static std::optional<RnnModel> from_bytes(const std::vector<uint8_t>& v) { return from_bytes(v.data(), v.size()); }
    /// `from_static_bytes` (src/rnn.rs:92): same validation; the C ABI copies, so it is an alias here.
    static std::optional<RnnModel> from_static_bytes(const uint8_t* bytes, size_t len) { return from_bytes(bytes, len); }
    /// RNNoise text format (train/convert_rnnoise.py) -> model.
    static std::optional<RnnModel> from_text(const std::string& text) {
        ::RNNModel* h = rnnoise_model_from_text(text.data(), text.size());
        if (!h) return std::nullopt;
        return RnnModel(h);
    }

    /// `Clone`: re-parses the exact byte image.
    RnnModel clone() const {
        std::vector<uint8_t> b = to_bytes();
        return *from_bytes(b);
    }
    std::vector<uint8_t> to_bytes() const {
        std::vector<uint8_t> b(rnnoise_model_bytes(h_.get(), nullptr, 0));
        rnnoise_model_bytes(h_.get(), b.data(), b.size());
        return b;
    }
    ::RNNModel* raw() const { return h_.get(); }

  private:
    explicit RnnModel(::RNNModel* h) : h_(h, &rnnoise_model_free) {}
    std::shared_ptr<::RNNModel> h_;  // shared so that states can keep a borrowed model alive
};

/// `DenoiseState<'model>` (src/denoise.rs:37-42): one mono 48 kHz stream.
class DenoiseState {
  public:
    static constexpr size_t FRAME_SIZE = 480;  // src/denoise.rs:46

    /// `DenoiseState::new()` (src/denoise.rs:53): built-in model.
    static std::unique_ptr<DenoiseState> new_() { return std::unique_ptr<DenoiseState>(new DenoiseState(RnnModel())); }
    /// `DenoiseState::from_model(model)` (src/denoise.rs:61): the state owns the model.
    static std::unique_ptr<DenoiseState> from_model(RnnModel model) {
        return std::unique_ptr<DenoiseState>(new DenoiseState(std::move(model)));
    }
    /// `DenoiseState::with_model(&model)` (src/denoise.rs:72): the model is shared (kept alive by refcount,
    /// which is what the Rust lifetime guarantees statically).
    static std::unique_ptr<DenoiseState> with_model(const RnnModel& model) {
        return std::unique_ptr<DenoiseState>(new DenoiseState(model));
    }

    /// `process_frame(&mut self, output: &mut [f32], input: &[f32]) -> f32` (src/denoise.rs:95-116).
    /// Samples are floats in the i16 range.  Throws (the reference panics, src/features.rs:98) unless both
    /// slices hold exactly FRAME_SIZE samples.  output may alias input.
    float process_frame(float* output, size_t output_len, const float* input, size_t input_len) {
        if (input_len != FRAME_SIZE || output_len != FRAME_SIZE) throw std::invalid_argument("process_frame: 480 samples required");
        return rnnoise_process_frame(st_, output, const_cast<float*>(input));
    }

    /// `impl Clone for DenoiseState` (src/denoise.rs:36): an independent state sharing the model, whose next frames give
    /// the same bits as this one's.  (Copy construction stays deleted: a copy allocates GPU state and can fail.)
    std::unique_ptr<DenoiseState> clone() const {
        ::DenoiseState* c = rnnoise_clone(st_);
        if (!c) throw std::runtime_error(std::string("rnnoise_clone: ") + rnnoise_last_error());
        return std::unique_ptr<DenoiseState>(new DenoiseState(model_, c));
    }

    ~DenoiseState() { rnnoise_destroy(st_); }
    DenoiseState(const DenoiseState&) = delete;
    DenoiseState& operator=(const DenoiseState&) = delete;

  private:
    explicit DenoiseState(RnnModel m) : model_(std::move(m)), st_(rnnoise_create(model_.raw())) {
        if (!st_) throw std::runtime_error(std::string("rnnoise_create: ") + rnnoise_last_error());
    }
    DenoiseState(RnnModel m, ::DenoiseState* st) : model_(std::move(m)), st_(st) {}
    RnnModel model_;
    ::DenoiseState* st_;
};

class Resampler;

/// N independent `DenoiseState`s on one GPU (additive; see rnnoise_batch_* in rnnoise.h).
class DenoiseBatch {
  public:
    DenoiseBatch(int n_streams, const RnnModel& model = RnnModel(), int device = -1)
        : b_(rnnoise_batch_create(model.raw(), n_streams, device)) {
        if (!b_) throw std::runtime_error(std::string("rnnoise_batch_create: ") + rnnoise_last_error());
    }
    ~DenoiseBatch() { rnnoise_batch_destroy(b_); }
    DenoiseBatch(const DenoiseBatch&) = delete;
    DenoiseBatch& operator=(const DenoiseBatch&) = delete;

    int streams() const { return rnnoise_batch_streams(b_); }
    void reset() { check(rnnoise_batch_reset(b_)); }
    /// host buffers, layout [n_frames][n_streams][480]; vad (optional) [n_frames][n_streams]
    void process_frames(float* out, const float* in, float* vad, int n_frames) { check(rnnoise_batch_process_host(b_, out, in, vad, n_frames)); }
    void process_frames_pcm16(short* out, const short* in, float* vad, int n_frames) {
        check(rnnoise_batch_process_pcm16_host(b_, out, in, vad, n_frames));
    }
    /// device buffers with explicit strides (floats); asynchronous on `cuda_stream` when given
    void process_frames_device(float* out, const float* in, float* vad, int n_frames, long stream_stride, long frame_stride,
                               void* cuda_stream = nullptr) {
        check(rnnoise_batch_process_device(b_, out, in, vad, n_frames, stream_stride, frame_stride, cuda_stream));
    }

    /// Per-stream state records (layout in rnnoise.h).  streams: n indices, or nullptr for streams 0..n-1; records in host
    /// memory or in device memory (asynchronous on `cuda_stream` when given).
    size_t state_bytes() const { return rnnoise_batch_state_bytes(b_); }
    void get_states(const int* streams, int n, void* dst, void* cuda_stream = nullptr) {
        check(rnnoise_batch_get_states(b_, streams, n, dst, cuda_stream));
    }
    /// Validates every record and index first; throws, with no stream changed, if one is bad.
    void set_states(const int* streams, int n, const void* src, void* cuda_stream = nullptr) {
        check(rnnoise_batch_set_states(b_, streams, n, src, cuda_stream));
    }
    void reset_streams(const int* streams, int n, void* cuda_stream = nullptr) { check(rnnoise_batch_reset_streams(b_, streams, n, cuda_stream)); }

    /// Advance only streams[0..n) (nullptr: 0..n-1) by n_frames frames; the other streams are not touched.  Row r of the
    /// buffers belongs to streams[r].  Host buffers [n_frames][n][480], vad (optional) [n_frames][n]:
    void process_streams(const int* streams, int n, float* out, const float* in, float* vad, int n_frames) {
        check(rnnoise_batch_process_streams_host(b_, streams, n, out, in, vad, n_frames));
    }
    /// device buffers, sample (r, t, i) at ptr[r*stream_stride + t*frame_stride + i*sample_stride]; pcm16 as
    /// rnnoise_batch_process_device_strided; asynchronous on `cuda_stream` when given
    void process_streams(const int* streams, int n, void* out, const void* in, int pcm16, float* vad, int n_frames, long stream_stride,
                         long sample_stride, long frame_stride, void* cuda_stream = nullptr) {
        check(rnnoise_batch_process_streams_device(b_, streams, n, out, in, pcm16, vad, n_frames, stream_stride, sample_stride, frame_stride,
                                                   cuda_stream));
    }

    /// Add a model of this batch's geometry to its model table; returns its index (the batch's own model is 0).
    int add_model(const RnnModel& model) {
        const int k = rnnoise_batch_add_model(b_, model.raw());
        check(k < 0 ? k : 0);
        return k;
    }
    /// Stream streams[r] (nullptr: r) runs on model model_ids[r] from the next frame on; the streams keep their state.
    void set_stream_models(const int* streams, int n, const int* model_ids) { check(rnnoise_batch_set_stream_models(b_, streams, n, model_ids)); }
    std::vector<int> stream_models(const int* streams, int n) const {
        std::vector<int> ids((size_t)n);
        check(rnnoise_batch_get_stream_models(b_, streams, n, ids.data()));
        return ids;
    }
    ::RNNoiseBatch* raw() const { return b_; }

    /// Denoise streams at their own sample rates (the resampler's; it must have this batch's size and device): row r is
    /// stream streams[r] (nullptr: r), its frames R/100 samples at rate R, float (pcm16 0) or int16 (pcm16 1).
    /// Host buffers of [n_frames][n][480] slots, the first R/100 samples of each valid; vad (optional) [n_frames][n]:
    void process_native(Resampler& rs, const int* streams, int n, void* out, const void* in, int pcm16, float* vad, int n_frames);
    /// device buffers, native sample (r, t, k) at ptr[r*stream_stride + t*frame_stride + k]; asynchronous on `cuda_stream`
    /// when given
    void process_native(Resampler& rs, const int* streams, int n, void* out, const void* in, int pcm16, float* vad, int n_frames,
                        long stream_stride, long frame_stride, void* cuda_stream = nullptr);

  private:
    static void check(int rc) {
        if (rc != 0) throw std::runtime_error(rnnoise_last_error());
    }
    ::RNNoiseBatch* b_;
};

/// Per-stream sample rates (8000..48000 Hz, multiples of 100) for a DenoiseBatch of the same size: the up and down
/// resampling stages with each stream's filter history (see rnnoise_resampler_* in rnnoise.h).
class Resampler {
  public:
    /// rates: n_streams rates, or nullptr for 48 kHz everywhere
    explicit Resampler(int n_streams, const int* rates = nullptr, int device = -1) : r_(rnnoise_resampler_create(n_streams, rates, device)) {
        if (!r_) throw std::runtime_error(std::string("rnnoise_resampler_create: ") + rnnoise_last_error());
    }
    ~Resampler() { rnnoise_resampler_destroy(r_); }
    Resampler(const Resampler&) = delete;
    Resampler& operator=(const Resampler&) = delete;

    /// Stream streams[i] (nullptr: i) gets rates[i] and zero histories (also the reset).
    void set_stream_rates(const int* streams, int n, const int* rates) { check(rnnoise_resampler_set_stream_rates(r_, streams, n, rates)); }
    std::vector<int> stream_rates(const int* streams, int n) const {
        std::vector<int> rates((size_t)n);
        check(rnnoise_resampler_get_stream_rates(r_, streams, n, rates.data()));
        return rates;
    }
    /// The stages alone, device buffers (layout in rnnoise.h); asynchronous on `cuda_stream` when given.
    void up(const int* streams, int n, float* out, const void* in, int pcm16, int n_frames, long stream_stride, long frame_stride,
            void* cuda_stream = nullptr) {
        check(rnnoise_resampler_up_device(r_, streams, n, out, in, pcm16, n_frames, stream_stride, frame_stride, cuda_stream));
    }
    void down(const int* streams, int n, void* out, const float* in, int pcm16, int n_frames, long stream_stride, long frame_stride,
              void* cuda_stream = nullptr) {
        check(rnnoise_resampler_down_device(r_, streams, n, out, in, pcm16, n_frames, stream_stride, frame_stride, cuda_stream));
    }
    /// State records of RNNOISE_RESAMPLER_STATE_BYTES each, host memory; set_states validates every record first.
    void get_states(const int* streams, int n, void* dst) { check(rnnoise_resampler_get_states(r_, streams, n, dst)); }
    void set_states(const int* streams, int n, const void* src) { check(rnnoise_resampler_set_states(r_, streams, n, src)); }
    /// The stage's float filter (direction 0: up, 1: down) and its up / down factors; needs no GPU.
    static std::vector<float> filter(int rate, int direction, int* up = nullptr, int* down = nullptr) {
        const int n = rnnoise_resampler_filter(rate, direction, nullptr, 0, up, down);
        check(n < 0 ? n : 0);
        std::vector<float> h((size_t)n);
        rnnoise_resampler_filter(rate, direction, h.data(), n, nullptr, nullptr);
        return h;
    }
    /// Delay of both stages together in 48 kHz samples (not counting the denoiser's).
    static double delay(int rate) {
        const double d = rnnoise_resampler_delay(rate);
        if (d < 0) throw std::runtime_error(rnnoise_last_error());
        return d;
    }
    ::RNNoiseResampler* raw() const { return r_; }

  private:
    static void check(int rc) {
        if (rc != 0) throw std::runtime_error(rnnoise_last_error());
    }
    ::RNNoiseResampler* r_;
};

inline void DenoiseBatch::process_native(Resampler& rs, const int* streams, int n, void* out, const void* in, int pcm16, float* vad,
                                         int n_frames) {
    check(rnnoise_batch_process_native_host(b_, rs.raw(), streams, n, out, in, pcm16, vad, n_frames));
}
inline void DenoiseBatch::process_native(Resampler& rs, const int* streams, int n, void* out, const void* in, int pcm16, float* vad,
                                         int n_frames, long stream_stride, long frame_stride, void* cuda_stream) {
    check(rnnoise_batch_process_native_device(b_, rs.raw(), streams, n, out, in, pcm16, vad, n_frames, stream_stride, frame_stride,
                                              cuda_stream));
}

/// Training-data rows (src/training.rs): n_lanes x (NoiseSimulator + 3 DenoiseFeatures) on one GPU; see rnnoise_train_*.
class TrainingBatch {
  public:
    static constexpr int ROW = RNNOISE_TRAIN_ROW;  // 87 = 42 features + 22 gains + 22 noise levels + vad (src/training.rs:90)
    explicit TrainingBatch(int n_lanes, int device = -1) : t_(rnnoise_train_create(n_lanes, device)) {
        if (!t_) throw std::runtime_error(std::string("rnnoise_train_create: ") + rnnoise_last_error());
    }
    ~TrainingBatch() { rnnoise_train_destroy(t_); }
    TrainingBatch(const TrainingBatch&) = delete;
    TrainingBatch& operator=(const TrainingBatch&) = delete;
    int lanes() const { return rnnoise_train_lanes(t_); }
    /// the outcome of NoiseSimulator::randomize (src/training.rs:352-377) for lanes [first, first + n)
    void set_params(int first_lane, int n, const RNNoiseSimParams* params) { check(rnnoise_train_set_params(t_, first_lane, n, params)); }
    /// host buffers: signal, noise [n_frames][lanes][480] -> rows [n_frames][lanes][87]
    void process_frames(float* rows, const float* signal, const float* noise, int n_frames) {
        check(rnnoise_train_process_host(t_, rows, signal, noise, n_frames));
    }

  private:
    static void check(int rc) {
        if (rc != 0) throw std::runtime_error(rnnoise_last_error());
    }
    ::RNNoiseTrainer* t_;
};

/// The `nnnoiseless` binary's main() (src/nnnoiseless.rs:230-334) for a set of files denoised as one batch.
inline void denoise_files(const std::vector<std::pair<std::string, std::string>>& in_out, const RNNoiseFileOptions* opt = nullptr) {
    std::vector<const char*> ins, outs;
    for (const auto& p : in_out) {
        ins.push_back(p.first.c_str());
        outs.push_back(p.second.c_str());
    }
    if (rnnoise_denoise_files((int)in_out.size(), ins.data(), outs.data(), opt) != 0) throw std::runtime_error(rnnoise_last_error());
}

}  // namespace nnnoiseless
