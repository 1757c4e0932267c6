// train.cu -- training-data rows on the GPU (SURVEY §8(f) N4): the per-frame arithmetic of the reference's
// `nnnoiseless-gen-training-data` main loop (src/training.rs:113-161) and NoiseSimulator::next_frame (:399-432)
// for n_lanes independent simulators.  Lane l owns three feature extractors of the batch (streams l = clean,
// L + l = noise, 2L + l = combined), so the pitch and analysis kernels of the denoise path run unchanged on 3L
// streams; this file adds the two kernels either side of them:
//
//   train_front : raw signal / noise frames -> gains, random-filter biquads, mix, VAD counter, and the DC-blocking
//                 high-pass of all three (five f64 biquad chains per lane, fused: the intermediate frames never
//                 reach HBM) -> history ring of the three streams.
//   train_rows  : band energies / features of the three streams -> the 87-float row
//                 [42 features | 22 gains | 22 noise levels | vad].
//
// Compiled with -fmad=false: the biquads and the frame energy are rounded and ordered exactly like the scalar code.
// tests/test_training_kernels.py holds both kernels to that frame by frame (histories, VAD and gain columns as bits).
#include <type_traits>

#include "common.cuh"

namespace nnb {

constexpr int TF_LANES = 64;
constexpr int TF_CHUNK = 80;
constexpr int TF_LD = TF_CHUNK + 1;
static_assert(FRAME_SIZE % TF_CHUNK == 0 && TF_CHUNK % 4 == 0, "chunking must tile the frame");

struct Biquad64 {
    double a0, a1, b0, b1;
    float m0, m1;
    // Biquad::filter / filter_in_place, src/util.rs:95-124
    __device__ __forceinline__ float step(float x) {
        const double x64 = (double)x;
        const double y64 = __dadd_rn(x64, (double)m0);
        const double t0 = __dsub_rn(__dmul_rn(b0, x64), __dmul_rn(a0, y64));
        const double t1 = __dsub_rn(__dmul_rn(b1, x64), __dmul_rn(a1, y64));
        m0 = __double2float_rn(__dadd_rn((double)m1, t0));
        m1 = __double2float_rn(t1);
        return __double2float_rn(y64);
    }
};

// Where a frame's raw samples come from (the template argument of train_front_kernel):
//   F32Frames : lane l's 480 floats at signal / noise + l * stream_stride; aux = vec_ok (16-byte float4 loads).
//   PoolFrames: lane l's 480 int16 samples at aux + signal[l] / aux + noise[l] (signal / noise are the frame's row of
//               offsets into the sample pool aux, -1 = a frame of zeros); stream_stride is unused.
// Only the tile load differs; the kernel's parameter list keeps the F32 layout, so that instantiation is the kernel
// it was before the template.
struct F32Frames {
    using Src = float;
    using Aux = int;
};
struct PoolFrames {
    using Src = long long;
    using Aux = const short*;
};

template <class In>
__global__ void __launch_bounds__(TF_LANES) train_front_kernel(const typename In::Src* __restrict__ signal,
                                                               const typename In::Src* __restrict__ noise, long stream_stride,
                                                               TrainBuffers tb, int set, float* __restrict__ hist,
                                                               float* __restrict__ hp_mem, int slot, typename In::Aux aux) {
    extern __shared__ float tf_smem[];
    float* ts = tf_smem;                       // signal -> clean (high-passed)
    float* tn = ts + TF_LANES * TF_LD;         // noise  -> noise (high-passed)
    float* tc = tn + TF_LANES * TF_LD;         // combined (high-passed)
    const int L = tb.n_lanes;
    const int l0 = blockIdx.x * TF_LANES;
    const int tid = threadIdx.x;
    const int nl = min(TF_LANES, L - l0);
    const int lane = l0 + tid;
    const bool act = tid < nl;

    TrainLaneParams p{};
    Biquad64 fs{}, fn{}, hs{}, hn{}, hc{};
    float sig_e = 0.0f;
    if (act) {
        p = tb.params[lane];
        fs = {(double)p.sig_a[0], (double)p.sig_a[1], (double)p.sig_b[0], (double)p.sig_b[1], tb.resp_mem[4 * lane], tb.resp_mem[4 * lane + 1]};
        fn = {(double)p.noise_a[0], (double)p.noise_a[1], (double)p.noise_b[0], (double)p.noise_b[1], tb.resp_mem[4 * lane + 2],
              tb.resp_mem[4 * lane + 3]};
        const double a0 = (double)-1.99599f, a1 = (double)0.99600f, b0 = (double)-2.0f, b1 = (double)1.0f;  // BIQUAD_HP, src/util.rs:68-71
        hs = {a0, a1, b0, b1, hp_mem[2 * lane], hp_mem[2 * lane + 1]};
        hn = {a0, a1, b0, b1, hp_mem[2 * (L + lane)], hp_mem[2 * (L + lane) + 1]};
        hc = {a0, a1, b0, b1, hp_mem[2 * (2 * L + lane)], hp_mem[2 * (2 * L + lane) + 1]};
    }
    constexpr int Q = TF_CHUNK / 4;
    long long* s_at = reinterpret_cast<long long*>(tc + TF_LANES * TF_LD);  // PoolFrames: the block's [2][64] offsets
    if constexpr (std::is_same_v<In, PoolFrames>) {
        if (act) {
            s_at[tid] = signal[lane];
            s_at[TF_LANES + tid] = noise[lane];
        }
        __syncthreads();
    }
    for (int c = 0; c < FRAME_SIZE / TF_CHUNK; c++) {
        if constexpr (std::is_same_v<In, PoolFrames>) {
            // arbitrary (2-byte aligned) offsets: consecutive threads read consecutive samples of one lane's chunk
#pragma unroll 4
            for (int idx = tid; idx < nl * TF_CHUNK; idx += TF_LANES) {
                const int row = idx / TF_CHUNK, i = idx - row * TF_CHUNK;
                const long long as = s_at[row], an = s_at[TF_LANES + row];
                ts[row * TF_LD + i] = as < 0 ? 0.0f : (float)aux[as + c * TF_CHUNK + i];
                tn[row * TF_LD + i] = an < 0 ? 0.0f : (float)aux[an + c * TF_CHUNK + i];
            }
        } else if (aux) {  // vec_ok
            for (int idx = tid; idx < nl * Q; idx += TF_LANES) {
                const int row = idx / Q, q = idx - row * Q;
                const long off = (long)(l0 + row) * stream_stride + c * TF_CHUNK;
                const float4 a = __ldg(reinterpret_cast<const float4*>(signal + off) + q);
                const float4 b = __ldg(reinterpret_cast<const float4*>(noise + off) + q);
                float* t = ts + row * TF_LD + 4 * q;
                t[0] = a.x; t[1] = a.y; t[2] = a.z; t[3] = a.w;
                t = tn + row * TF_LD + 4 * q;
                t[0] = b.x; t[1] = b.y; t[2] = b.z; t[3] = b.w;
            }
        } else {
            for (int idx = tid; idx < nl * TF_CHUNK; idx += TF_LANES) {
                const int row = idx / TF_CHUNK, i = idx - row * TF_CHUNK;
                const long off = (long)(l0 + row) * stream_stride + c * TF_CHUNK + i;
                ts[row * TF_LD + i] = signal[off];
                tn[row * TF_LD + i] = noise[off];
            }
        }
        __syncthreads();
        if (act) {
            float* rs = ts + tid * TF_LD;
            float* rn = tn + tid * TF_LD;
            float* rc = tc + tid * TF_LD;
#pragma unroll 2
            for (int i = 0; i < TF_CHUNK; i++) {
                const float x = rs[i];
                sig_e = __fadd_rn(sig_e, __fmul_rn(x, x));                 // read_signal: energy before the gain (:351-359)
                const float s = fs.step(__fmul_rn(x, p.signal_gain));       // sig_filter.filter_in_place (:406-407)
                const float n = fn.step(__fmul_rn(rn[i], p.noise_gain));    // read_noise + noise_filter (:342-348, :408-409)
                const float z = __fadd_rn(s, n);                            // combined (:411-413)
                rs[i] = hs.step(s);                                         // shift_and_filter_input x3 (:127-129)
                rn[i] = hn.step(n);
                rc[i] = hc.step(z);
            }
        }
        __syncthreads();
        for (int idx = tid; idx < 3 * nl * Q; idx += TF_LANES) {
            const int which = idx / (nl * Q), r = idx - which * (nl * Q);
            const int row = r / Q, q = r - row * Q;
            const float* t = (which == 0 ? ts : which == 1 ? tn : tc) + row * TF_LD + 4 * q;
            reinterpret_cast<float4*>(hist + (size_t)(which * L + l0 + row) * HIST_CAP + slot * FRAME_SIZE + c * TF_CHUNK)[q] =
                make_float4(t[0], t[1], t[2], t[3]);
        }
        __syncthreads();
    }
    if (act) {
        tb.resp_mem[4 * lane] = fs.m0;
        tb.resp_mem[4 * lane + 1] = fs.m1;
        tb.resp_mem[4 * lane + 2] = fn.m0;
        tb.resp_mem[4 * lane + 3] = fn.m1;
        hp_mem[2 * lane] = hs.m0;
        hp_mem[2 * lane + 1] = hs.m1;
        hp_mem[2 * (L + lane)] = hn.m0;
        hp_mem[2 * (L + lane) + 1] = hn.m1;
        hp_mem[2 * (2 * L + lane)] = hc.m0;
        hp_mem[2 * (2 * L + lane) + 1] = hc.m1;
        // NoiseSimulator::vad, src/training.rs:380-397
        int vc = tb.vad_count[lane];
        if (sig_e > 1e9f) vc = 0;
        else if (sig_e > 1e8f) vc -= 5;
        else if (sig_e > 1e7f) vc += 1;
        else vc += 2;
        vc = max(0, min(15, vc));
        tb.vad_count[lane] = vc;
        const float vad = vc >= 10 ? 0.0f : (vc > 0 ? 0.5f : 1.0f);
        tb.vad[(size_t)set * L + lane] = vad;
        tb.cutoff[(size_t)set * L + lane] = (vad == 0.0f && p.noise_gain == 0.0f) ? 0 : p.band_lp + 1;  // :420-424
    }
}

// src/training.rs:132-159: one thread per row element
__global__ void __launch_bounds__(128) train_rows_kernel(BatchBuffers b, TrainBuffers tb, int set, float* __restrict__ rows, long lane_stride) {
    const int L = tb.n_lanes;
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long)L * TRAIN_ROW) return;
    const int lane = (int)(idx / TRAIN_ROW), j = (int)(idx - (long)lane * TRAIN_ROW);
    const size_t sc = lane, sn = (size_t)L + lane, sm = 2 * (size_t)L + lane;
    float v;
    if (j < NB_FEATURES) {
        v = b.features[sm * NB_FEATURES + j];
    } else if (j < NB_FEATURES + NB_BANDS) {
        const int i = j - NB_FEATURES;
        const int cutoff = b.silence[sm] ? 0 : tb.cutoff[(size_t)set * L + lane];
        if (i < cutoff) {
            const float ce = b.ex[sc * NB_BANDS + i], me = b.ex[sm * NB_BANDS + i];
            v = (ce < 5e-2f && me < 5e-2f) ? -1.0f : fminf(sqrtf(__fdiv_rn(__fadd_rn(ce, 1e-3f), __fadd_rn(me, 1e-3f))), 1.0f);
        } else {
            v = -1.0f;
        }
    } else if (j < NB_FEATURES + 2 * NB_BANDS) {
        v = log10f(__fadd_rn(b.ex[sn * NB_BANDS + (j - NB_FEATURES - NB_BANDS)], 1e-2f));
    } else {
        v = tb.vad[(size_t)set * L + lane];
    }
    rows[(long)lane * lane_stride + j] = v;
}

template <class In>
static cudaError_t launch_front(const BatchBuffers& b, const TrainBuffers& tb, int set, const typename In::Src* signal,
                                const typename In::Src* noise, long stream_stride, typename In::Aux aux, int slot, cudaStream_t st) {
    const size_t smem = 3 * TF_LANES * TF_LD * sizeof(float) + (std::is_same_v<In, PoolFrames> ? 2 * TF_LANES * sizeof(long long) : 0);
    {  // per device; cheap next to a frame of work
        cudaError_t e = cudaFuncSetAttribute(train_front_kernel<In>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    const int grid = (tb.n_lanes + TF_LANES - 1) / TF_LANES;
    train_front_kernel<In><<<grid, TF_LANES, smem, st>>>(signal, noise, stream_stride, tb, set, b.hist, b.hp_mem, slot, aux);
    return cudaGetLastError();
}

cudaError_t launch_train_front(const BatchBuffers& b, const TrainBuffers& tb, int set, const float* signal, const float* noise,
                               long stream_stride, int slot, cudaStream_t st) {
    const int vec_ok = ((reinterpret_cast<uintptr_t>(signal) & 15) == 0) && ((reinterpret_cast<uintptr_t>(noise) & 15) == 0) &&
                       (stream_stride % 4 == 0);
    return launch_front<F32Frames>(b, tb, set, signal, noise, stream_stride, vec_ok, slot, st);
}

cudaError_t launch_train_front_pool(const BatchBuffers& b, const TrainBuffers& tb, int set, const short* pool, const long long* sig_at,
                                    const long long* noise_at, int slot, cudaStream_t st) {
    return launch_front<PoolFrames>(b, tb, set, sig_at, noise_at, 0, pool, slot, st);
}

cudaError_t launch_train_rows(const BatchBuffers& b, const TrainBuffers& tb, int set, float* rows, long lane_stride, cudaStream_t st) {
    const long n = (long)tb.n_lanes * TRAIN_ROW;
    train_rows_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(b, tb, set, rows, lane_stride);
    return cudaGetLastError();
}

}  // namespace nnb
