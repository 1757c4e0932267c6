// model.hpp -- host-side RnnModel: parser for the nnnoiseless binary model format
// (src/rnn.rs:96-232) and the built-in weights (src/rnn.rs:235-240).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace nnb {

struct HostDense {
    int ni = 0, nn = 0, act = 0;
    size_t w_off = 0, b_off = 0;  // offsets into HostModel::bytes
};
struct HostGru {
    int ni = 0, nn = 0, act = 0;
    size_t w_off = 0, r_off = 0, b_off = 0;
};

struct HostModel {
    std::vector<int8_t> bytes;  // the exact image accepted by from_bytes
    HostDense input_dense, denoise_output, vad_output;
    HostGru vad_gru, noise_gru, denoise_gru;

    // floats of GRU state per stream: vad | noise | denoise
    int state_size() const { return vad_gru.nn + noise_gru.nn + denoise_gru.nn; }

    // RnnModel::from_bytes: false on any violation of src/rnn.rs:116-222.
    static bool parse(const uint8_t* data, size_t len, HostModel* out);
    // RNNoise text format -> binary image (train/convert_rnnoise.py:18-29) -> parse.
    static bool parse_text(const char* text, size_t len, HostModel* out);
    // RnnModel::default(): the embedded weights.rnn.
    static const HostModel& builtin();
};

// The tanh table of src/util.rs:3-27, which every packed model image carries.
extern const float kTansigTable[201];

}  // namespace nnb
