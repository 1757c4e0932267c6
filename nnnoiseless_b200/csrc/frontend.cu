// frontend.cu -- the host calls around the file front-end of the reference's `nnnoiseless` binary (src/nnnoiseless.rs,
// SURVEY §8(f) N2): the resampler alone on the GPU (rnnoise_resample_host) and the audio decoders and encoders.  The
// file calls themselves run in corpus.cu.  The resampler is described in frontend.cuh.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/rnnoise.h"
#include "abi.hpp"
#include "audio_io.hpp"
#include "common.cuh"
#include "frontend.cuh"
#include "owners.hpp"

using namespace nnb;

namespace {

// One thread per (output sample k, channel c) of one file.  src: [n_in][C] interleaved.  mk/posk: per output sample,
// source frames pushed so far and the interpolation position (NULL: 48 kHz input, samples pass through).  Output
// samples k in [k0, k0 + nk) go to out[(k - k0) * S + c0 + c]; k >= K (past the end of this file) are zero.
__global__ void __launch_bounds__(256) resample_kernel(const float* __restrict__ src, int C, const int* __restrict__ mk,
                                                       const double* __restrict__ posk, long K, long k0, long nk, float* __restrict__ out,
                                                       long S, int c0) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nk * C) return;
    const long kk = t / C;
    const int c = (int)(t - kk * C);
    const long k = k0 + kk;
    out[kk * S + c0 + c] = k < K ? dasp_sample(src, C, c, mk, posk, k) : 0.0f;
}

int launch_resample(const float* d_src, int C, const PosTable* t, long K, long k0, long nk, float* d_out, long S, int c0, cudaStream_t st) {
    const long n = nk * C;
    if (n <= 0) return 0;
    resample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_src, C, t ? t->d_m : nullptr, t ? t->d_pos : nullptr, K, k0, nk, d_out, S, c0);
    CK(cudaGetLastError());
    count_launches(1);
    return 0;
}

}  // namespace

extern "C" {

long rnnoise_resample_host(float* out, long cap, const float* in, long n_in, int channels, double ratio, int device) {
    if (!out || !in || channels < 1 || n_in < 0 || cap < 0) return fail("rnnoise_resample_host: bad argument");
    if (open_device(device, &device)) return -1;
    ON_DEVICE(device);
    PosTable t;
    build_pos_table(ratio, n_in, &t);
    const long K = std::min<long>((long)t.m.size(), cap);
    if (K == 0) return 0;
    DeviceWork dw;
    float *d_src = nullptr, *d_out = nullptr;
    CK(dalloc(&dw.dev, &d_src, std::max<size_t>(1, (size_t)n_in * channels)));
    CK(dalloc(&dw.dev, &d_out, (size_t)K * channels));
    CK(dalloc(&dw.dev, &t.d_m, (size_t)K));
    CK(dalloc(&dw.dev, &t.d_pos, (size_t)K));
    CK(cudaMemcpy(d_src, in, (size_t)n_in * channels * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(t.d_m, t.m.data(), (size_t)K * sizeof(int), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(t.d_pos, t.pos.data(), (size_t)K * sizeof(double), cudaMemcpyHostToDevice));
    if (launch_resample(d_src, channels, &t, K, 0, K, d_out, channels, 0, nullptr)) return -1;
    CK(cudaMemcpy(out, d_out, (size_t)K * channels * sizeof(float), cudaMemcpyDeviceToHost));
    return K;
}

int rnnoise_audio_read(const char* path, int wav, int raw_channels, double raw_rate, float** samples, long* n_frames, int* channels,
                       double* sample_rate) {
    if (!path || !samples || !n_frames || !channels || !sample_rate) return fail("rnnoise_audio_read: null argument");
    AudioData a;
    std::string err;
    const bool is_wav = wav > 0 || (wav == 0 && has_wav_extension(path));
    const bool ok = is_wav ? read_wav_file(path, &a, &err)
                           : read_raw_file(path, raw_channels > 0 ? raw_channels : 1, raw_rate > 0.0 ? raw_rate : 48000.0, &a, &err);
    if (!ok) return fail(err);
    float* p = static_cast<float*>(malloc(std::max<size_t>(1, a.samples.size()) * sizeof(float)));
    if (!p) return fail("out of memory");
    std::copy(a.samples.begin(), a.samples.end(), p);
    *samples = p;
    *n_frames = a.frames();
    *channels = a.channels;
    *sample_rate = a.sample_rate;
    return 0;
}

void rnnoise_audio_free(float* samples) { free(samples); }

int rnnoise_audio_probe(const char* path, RNNoiseAudioInfo* info) {
    if (!path || !info) return fail("rnnoise_audio_probe: null argument");
    WavHeader h;
    std::string err;
    if (!probe_wav_file(path, &h, &err)) return fail(err);
    info->channels = h.channels;
    info->sample_rate = (int)h.sample_rate;
    info->bits_per_sample = h.bits;
    info->is_float = h.fmt_tag == 3;
    info->data_offset = (long long)h.data_offset;
    info->n_frames = (long long)h.n_frames;
    return 0;
}

int rnnoise_audio_write(const char* path, int wav, const short* pcm, long n_frames, int channels) {
    if (!path || (!pcm && n_frames > 0) || n_frames < 0 || channels < 1) return fail("rnnoise_audio_write: bad argument");
    std::string err;
    const bool is_wav = wav > 0 || (wav == 0 && has_wav_extension(path));
    const bool ok = is_wav ? write_wav_file(path, pcm, n_frames, channels, &err) : write_raw_file(path, pcm, n_frames, channels, &err);
    return ok ? 0 : fail(err);
}

}  // extern "C"
