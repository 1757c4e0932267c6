// audio_io.hpp -- file formats of the reference's `nnnoiseless` binary (src/nnnoiseless.rs:34-102, 133-228):
// headerless little-endian 16-bit PCM and RIFF/WAVE (integer 8/16/24/32-bit and 32-bit float, as hound 3.x reads
// them), decoded to interleaved f32 in the i16 range; 16-bit PCM WAV / raw writers.  Host code, no CUDA.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace nnb {

struct AudioData {
    std::vector<float> samples;  // interleaved [n_frames][channels], i16-range values
    int channels = 1;
    double sample_rate = 48000.0;
    long frames() const { return channels > 0 ? (long)(samples.size() / (size_t)channels) : 0; }
};

// A RIFF/WAVE file's format and the place of its samples, from the header alone.
struct WavHeader {
    int fmt_tag = 0;           // 1 = integer PCM, 3 = IEEE float (WAVE_FORMAT_EXTENSIBLE resolved)
    int channels = 0;
    uint32_t sample_rate = 0;
    int bits = 0;              // bits per sample
    int bytes = 0;             // bytes per sample
    size_t data_offset = 0;    // byte offset of the first sample
    size_t n_frames = 0;       // samples per channel
};

// All three return false and set *err (the reference's / hound's wording where a test greps for it).
bool read_wav_file(const std::string& path, AudioData* out, std::string* err);
bool read_raw_file(const std::string& path, int channels, double sample_rate, AudioData* out, std::string* err);
// The header checks of read_wav_file (same error texts) without reading the samples.
bool probe_wav_file(const std::string& path, WavHeader* h, std::string* err);

// pcm: interleaved [n_frames][channels] int16.  WAV = 48 kHz 16-bit PCM (WavSpec at src/nnnoiseless.rs:278-283).
// *opened (when given): whether the file was opened for writing, i.e. whether a failure may have left it truncated.
bool write_wav_file(const std::string& path, const int16_t* pcm, long n_frames, int channels, std::string* err, bool* opened = nullptr);
bool write_raw_file(const std::string& path, const int16_t* pcm, long n_frames, int channels, std::string* err, bool* opened = nullptr);

// `Path::extension() == Some("wav")` (src/nnnoiseless.rs:260-263)
bool has_wav_extension(const std::string& path);

}  // namespace nnb
