// frontend.cu -- the file front-end of the reference's `nnnoiseless` binary (src/nnnoiseless.rs) on the GPU
// (SURVEY §8(f) N2): decode -> [resample to 48 kHz] -> 480-sample frames per channel -> denoise -> drop the first
// frame -> clamp/round to i16 -> raw / WAV.  Every channel of every file is one stream of ONE batch, so a set of
// files is denoised together ("many files = many streams").  The resampler is described in frontend.cuh.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <sys/stat.h>
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

struct Job {
    AudioData a;
    double ratio = 1.0;
    int c0 = 0;
    long K = 0, F = 0;
    float* d_src = nullptr;
    std::vector<int16_t> out;  // [(F-1)*480][C]
};

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

static bool same_file(const char* a, const char* b) {
    if (std::string(a) == b) return true;
    struct stat sa, sb;
    if (stat(a, &sa) != 0 || stat(b, &sb) != 0) return false;
    return sa.st_dev == sb.st_dev && sa.st_ino == sb.st_ino;
}

int rnnoise_denoise_files(int n_files, const char* const* in_paths, const char* const* out_paths, const RNNoiseFileOptions* opt) {
    return rnnoise_denoise_files_linked(n_files, in_paths, out_paths, opt, 0);
}

int rnnoise_denoise_files_linked(int n_files, const char* const* in_paths, const char* const* out_paths, const RNNoiseFileOptions* opt,
                                 int link_mode) {
    if (n_files < 0 || (n_files > 0 && (!in_paths || !out_paths))) return fail("rnnoise_denoise_files: bad argument");
    if (link_mode != 0 && link_mode != RNNOISE_LINK_MAX && link_mode != RNNOISE_LINK_MEAN)
        return fail("link mode " + std::to_string(link_mode) + " is neither 0, RNNOISE_LINK_MAX (1) nor RNNOISE_LINK_MEAN (2)");
    if (n_files == 0) return 0;
    RNNoiseFileOptions o{};
    o.device = -1;
    if (opt) o = *opt;
    const double raw_rate = o.sample_rate > 0.0 ? o.sample_rate : 48000.0;  // :270
    const int raw_channels = o.channels > 0 ? o.channels : 1;               // :271

    // ---- decode (host) ----------------------------------------------------------------------------
    // One file: like the reference, the output is created before the input is parsed (src/nnnoiseless.rs:251-258).
    // A batch (additive mode) must not amplify that: an output that is also an input of the batch is refused, every input
    // is decoded first, and only then are the outputs created -- a malformed file leaves the other files untouched.
    const bool batch_mode = n_files > 1;
    if (batch_mode)
        for (int i = 0; i < n_files; i++)
            for (int k = 0; k < n_files; k++)
                if (same_file(out_paths[i], in_paths[k]))
                    return fail(std::string("output file \"") + out_paths[i] + "\" is also an input of this batch");
    std::vector<Job> jobs((size_t)n_files);
    std::vector<bool> wav_out((size_t)n_files);
    long S = 0;
    for (int i = 0; i < n_files; i++) {
        const std::string in = in_paths[i], outp = out_paths[i];
        const bool wav_in = o.wav_in || has_wav_extension(in);  // :260-261
        wav_out[i] = o.wav_out || has_wav_extension(outp);      // :262-263
        std::string err;
        FILE* probe = fopen(in.c_str(), "rb");
        if (!probe) return fail("Failed to open input file \"" + in + "\"");  // :251-253
        fclose(probe);
        if (!batch_mode) {
            FILE* created = fopen(outp.c_str(), "wb");  // the reference creates the output before it parses the input (:255-258)
            if (!created) return fail("Failed to open output file \"" + outp + "\"");
            fclose(created);
        }
        Job& j = jobs[i];
        const bool ok = wav_in ? read_wav_file(in, &j.a, &err) : read_raw_file(in, raw_channels, raw_rate, &j.a, &err);
        if (!ok) return fail(err);
        if (link_mode && j.a.channels > RNNOISE_LINK_MAX_MEMBERS)
            return fail("\"" + in + "\" has " + std::to_string(j.a.channels) + " channels: linked channels are at most " +
                        std::to_string(RNNOISE_LINK_MAX_MEMBERS) + " per file");
        j.ratio = j.a.sample_rate / 48000.0;  // :182-186, :209-213
        j.c0 = (int)S;
        S += j.a.channels;
        if (S > (1 << 28)) return fail("too many channels in one call");
    }
    if (batch_mode)
        for (int i = 0; i < n_files; i++) {
            FILE* created = fopen(out_paths[i], "wb");
            if (!created) return fail(std::string("Failed to open output file \"") + out_paths[i] + "\"");
            fclose(created);
        }

    // ---- position tables, one per distinct rate -------------------------------------------------------
    std::map<double, PosTable> tables;
    for (Job& j : jobs)
        if (j.a.sample_rate != 48000.0) {
            PosTable& t = tables[j.ratio];
            t.n_in_max = std::max(t.n_in_max, j.a.frames());
        }
    for (auto& kv : tables) build_pos_table(kv.first, kv.second.n_in_max, &kv.second);
    long Tmax = 0;
    for (Job& j : jobs) {
        if (j.a.sample_rate == 48000.0) {
            j.K = j.a.frames();
        } else {
            const PosTable& t = tables[j.ratio];
            j.K = (long)(std::upper_bound(t.m.begin(), t.m.end(), (int)std::min<long>(j.a.frames(), 0x7fffffff)) - t.m.begin());
        }
        j.F = j.K / FRAME_SIZE;  // a trailing partial frame is dropped (:303-311)
        Tmax = std::max(Tmax, j.F);
        if (j.F > 1) j.out.resize((size_t)(j.F - 1) * FRAME_SIZE * (size_t)j.a.channels);
    }

    // ---- device: sources, tables, one chunk of interleaved frames in / out -----------------------------------
    if (Tmax > 1) {  // inputs shorter than two frames produce no output (src/nnnoiseless.rs:319-327) and need no device
        // format errors above are reported even on a machine without a GPU; from here on CUDA is required
        int device;
        if (open_device(o.device, &device)) return -1;
        ON_DEVICE(device);
        DeviceWork cl;  // declared after the guard: the device stays selected while cl's destructor frees
        CK(cudaStreamCreateWithFlags(cl.st.put(), cudaStreamNonBlocking));
        for (Job& j : jobs) {
            const size_t n = j.a.samples.size();
            CK(dalloc(&cl.dev, &j.d_src, std::max<size_t>(1, n)));
            CK(cudaMemcpyAsync(j.d_src, j.a.samples.data(), n * sizeof(float), cudaMemcpyHostToDevice, cl.st));
        }
        for (auto& kv : tables) {
            PosTable& t = kv.second;
            const size_t n = std::max<size_t>(1, t.m.size());
            CK(dalloc(&cl.dev, &t.d_m, n));
            CK(dalloc(&cl.dev, &t.d_pos, n));
            CK(cudaMemcpyAsync(t.d_m, t.m.data(), t.m.size() * sizeof(int), cudaMemcpyHostToDevice, cl.st));
            CK(cudaMemcpyAsync(t.d_pos, t.pos.data(), t.pos.size() * sizeof(double), cudaMemcpyHostToDevice, cl.st));
        }
        const size_t per_frame = (size_t)S * FRAME_SIZE;
        const long Fc = (long)std::max<size_t>(1, std::min<size_t>((size_t)Tmax, (size_t(1) << 30) / (per_frame * 6)));
        float* d_in = nullptr;
        int16_t* d_out = nullptr;
        CK(dalloc(&cl.dev, &d_in, (size_t)Fc * per_frame));
        CK(dalloc(&cl.dev, &d_out, (size_t)Fc * per_frame));
        CK(cudaMallocHost(cl.pinned.put(), (size_t)Fc * per_frame * sizeof(int16_t)));
        const int16_t* h_out = static_cast<const int16_t*>(static_cast<void*>(cl.pinned));
        cl.batch.reset(rnnoise_batch_create(o.model, (int)S, o.device));
        if (!cl.batch) return -1;
        if (link_mode)  // the channels of each multi-channel file are one group
            for (const Job& j : jobs)
                if (j.a.channels > 1) {
                    std::vector<int> ch((size_t)j.a.channels);
                    for (int c = 0; c < j.a.channels; c++) ch[(size_t)c] = j.c0 + c;
                    if (rnnoise_batch_link_streams(cl.batch.get(), ch.data(), j.a.channels, link_mode) != 0) return -1;
                }
        for (long f0 = 0; f0 < Tmax; f0 += Fc) {
            const long nf = std::min(Fc, Tmax - f0);
            for (Job& j : jobs) {
                const PosTable* t = j.a.sample_rate == 48000.0 ? nullptr : &tables[j.ratio];
                // only whole frames of this file are audio; everything after them is padding for the longer files
                if (launch_resample(j.d_src, j.a.channels, t, j.F * FRAME_SIZE, f0 * FRAME_SIZE, nf * FRAME_SIZE, d_in, S, j.c0, cl.st)) return -1;
            }
            // every channel is a stream: float in, int16 out, interleaved (stream_stride 1, sample_stride S)
            if (rnnoise_batch_process_device_strided(cl.batch.get(), d_out, d_in, 2, nullptr, (int)nf, 1, S, (long)per_frame, cl.st) != 0) return -1;
            CK(cudaMemcpyAsync(cl.pinned, d_out, (size_t)nf * per_frame * sizeof(int16_t), cudaMemcpyDeviceToHost, cl.st));
            CK(cudaStreamSynchronize(cl.st));
            for (Job& j : jobs) {
                const int C = j.a.channels;
                for (long f = std::max<long>(f0, 1); f < std::min(f0 + nf, j.F); f++)  // frame 0 is discarded (:319-327)
                    for (int i = 0; i < FRAME_SIZE; i++) {
                        const int16_t* srow = h_out + ((size_t)(f - f0) * FRAME_SIZE + i) * (size_t)S + j.c0;
                        int16_t* drow = j.out.data() + ((size_t)(f - 1) * FRAME_SIZE + i) * (size_t)C;
                        for (int c = 0; c < C; c++) drow[c] = srow[c];
                    }
            }
        }
    }

    // ---- encode (host) ----------------------------------------------------------------------------
    for (int i = 0; i < n_files; i++) {
        Job& j = jobs[i];
        std::string err;
        const long n = j.F > 1 ? (j.F - 1) * FRAME_SIZE : 0;
        const bool ok = wav_out[i] ? write_wav_file(out_paths[i], j.out.data(), n, j.a.channels, &err)
                                   : write_raw_file(out_paths[i], j.out.data(), n, j.a.channels, &err);
        if (!ok) return fail(err);
    }
    return 0;
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

int rnnoise_denoise_file(const char* in_path, const char* out_path, const RNNoiseFileOptions* opt) {
    if (!in_path || !out_path) return fail("rnnoise_denoise_file: null path");
    return rnnoise_denoise_files(1, &in_path, &out_path, opt);
}

}  // extern "C"
