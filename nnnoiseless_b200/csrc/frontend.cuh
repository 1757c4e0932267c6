// frontend.cuh -- what the file calls share (frontend.cu: the resampler alone; corpus.cu: every file call, on recycled
// stream slots): the dasp resampler's per-sample evaluation, its position tables and the device side of a call.
//
// Resampler = dasp_interpolate 0.11.0 `Sinc<[f32; 16]>` as driven by Resample::next_sample (:104-131): a depth-8
// Hann-windowed sinc evaluated in f64 per tap, taps accumulated in f32 in the order left(n), right(n).  The
// fractional position is a sequential f64 accumulation (`pos += ratio; while pos >= 1 { pos -= 1; push }`), so the
// host replays it once per distinct rate and hands the kernels (source frames consumed, pos) per output sample; the
// kernels then evaluate all output samples of all channels in parallel.
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "../../include/rnnoise.h"
#include "owners.hpp"

namespace nnb {

// Output sample k of channel c of a source src [n_in][C] (interleaved).  mk/posk: per output sample, source frames
// pushed so far and the interpolation position (NULL: 48 kHz input, samples pass through).
__device__ __forceinline__ float dasp_sample(const float* __restrict__ src, int C, int c, const int* __restrict__ mk,
                                             const double* __restrict__ posk, long k) {
    if (!mk) return __ldg(src + k * C + c);
    const double PI = 3.14159265358979323846264338327950288;
    const int depth = 8, len = 16;
    const long m = mk[k];                       // Sinc::next_source_frame calls so far
    const double phil = posk[k], phir = __dsub_rn(1.0, phil);
    const int idx = m < depth ? (int)m : depth;  // saturates at depth
    const int nl = idx, nr = idx + 1;
    const int rightmost = nl + depth, leftmost = nr - depth;
    const int max_depth = rightmost >= len ? len - depth : (leftmost < 0 ? depth + leftmost : depth);
    // ring frame j (0 = oldest) is source frame m - 16 + j; frames the source has not reached yet are the
    // ring's initial zeros; Fixed's index wraps modulo 16
    auto frame = [&](int j) -> double {
        const long si = m - len + (j & (len - 1));
        return si >= 0 ? (double)__ldg(src + si * C + c) : 0.0;
    };
    float v = 0.0f;
    for (int n = 0; n < max_depth; n++) {
        double a = __dmul_rn(PI, __dadd_rn(phil, (double)n));
        double first = a == 0.0 ? 1.0 : __ddiv_rn(sin(a), a);
        double second = __dadd_rn(0.5, __dmul_rn(0.5, cos(__ddiv_rn(a, (double)depth))));
        v = __fadd_rn(v, __double2float_rn(__dmul_rn(__dmul_rn(first, second), frame(nl - n))));
        a = __dmul_rn(PI, __dadd_rn(phir, (double)n));
        first = a == 0.0 ? 1.0 : __ddiv_rn(sin(a), a);
        second = __dadd_rn(0.5, __dmul_rn(0.5, cos(__ddiv_rn(a, (double)depth))));
        v = __fadd_rn(v, __double2float_rn(__dmul_rn(__dmul_rn(first, second), frame(nr + n))));
    }
    return v;
}

// Resample::next_sample's position recurrence (src/nnnoiseless.rs:105-118) replayed until more than n_in source
// frames would be needed, or for max_out outputs.  m[k] = source frames consumed before output k is interpolated; pos[k]
// its position.  The recurrence does not depend on n_in, so a table built for a longer source starts with the shorter
// one's entries.
struct PosTable {
    std::vector<int> m;
    std::vector<double> pos;
    int* d_m = nullptr;
    double* d_pos = nullptr;
    long n_in_max = 0;
};

inline void build_pos_table(double ratio, long n_in, PosTable* t, size_t max_out = SIZE_MAX) {
    double pos = 0.0;
    long m = 0;
    t->m.clear();
    t->pos.clear();
    if (!(ratio > 0.0)) return;  // a non-positive rate never consumes input: no output (the reference would spin)
    for (;;) {
        pos += ratio;
        while (pos >= 1.0) {
            pos -= 1.0;
            m++;
        }
        if (m > n_in || t->m.size() >= max_out) break;
        t->m.push_back((int)m);
        t->pos.push_back(pos);
    }
    t->n_in_max = n_in;
}

// The device side of a file call.  Its destructor waits for the stream; then the members free what they own.
struct DeviceWork {
    Stream st;
    std::vector<DeviceMem> dev;
    std::unique_ptr<RNNoiseBatch, void (*)(RNNoiseBatch*)> batch{nullptr, rnnoise_batch_destroy};
    ~DeviceWork() {
        if (st) cudaStreamSynchronize(st);
    }
};

}  // namespace nnb
