// metrics.cu -- quality metrics of denoised streams against clean speech (rnnoise_metrics_*, DESIGN.md §7p).
//
// metrics_kernel: one warp per stream, a grid-stride loop over streams, and each warp walks the call's frames in order,
// so every stream's double sums are formed in frame order whatever the split of its frames into calls.  A frame is
// the analysis kernel's band-energy computation run twice: the 960-sample windows [previous half | this frame] of the
// output y and of the paired clean frame c go through fft480_warp<true> (y as X, c as P), the even/odd split and
// band_sums_warp<3>, so Yb and Cb are the analysis kernel's `ex` for those windows up to rounding: the compiler
// contracts the shared FFT and band-sum source into FMAs differently in the two kernels.  The time-domain sums
// come from the same loaded samples.
//
// Lane b holds the complex samples z[32 a + b] = (w[64 a + 2 b], w[64 a + 2 b + 1]) of a window w, a = 0..14 (the
// analysis kernel's layout).  Window samples >= 480 are the frame itself: slots a = 7 (lanes 16..31) and a = 8..14,
// kept as the lane's "current" registers cur[k], a = 7 + k.  The next frame's previous half is this frame: sample n of
// the half sits in lane b ^ 16, so the halves move by one shuffle per slot and only the first frame of a call reads the
// half-windows from the pairing state.  The next frame's own samples are loaded before this frame's FFT.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/rnnoise.h"
#include "abi.hpp"
#include "owners.hpp"
#include "spectral_warp.cuh"

namespace nnb {

namespace {

static_assert(sizeof(RNNoiseMetricsRecord) == 696, "record layout");
constexpr int kCur = 8;  // current-frame slots a = 7 .. 14

struct MetricsArgs {
    const float* out;
    const float* clean;
    long ss, fs;
    const float* vad;
    const float* tgt;
    long vss, vfs;
    int n_frames, n_streams;
    float* yh;   // [B][480] output frame before the next one
    float* ch;   // [B][480] clean frame before the last one
    float* cl;   // [B][480] last clean frame
    float* tl;   // [B] its target (0.5: none)
    int* started;  // [B] a frame has been seen
    RNNoiseMetricsRecord* rec;
};

// the lane's current-frame slots of frame p (480 samples): slot k holds samples 64 k + 2 lane - 32 and the next one
__device__ __forceinline__ void load_cur(const float* __restrict__ p, float2 (&v)[kCur], int lane) {
#pragma unroll
    for (int k = 0; k < kCur; k++) {
        const int n = 64 * k + 2 * lane - 32;
        v[k] = (k > 0 || lane >= 16) ? make_float2(__ldg(p + n), __ldg(p + n + 1)) : make_float2(0.f, 0.f);
    }
}

// the lane's half-window slots a = 0..7 of a previous frame p: samples 64 a + 2 lane (< 480) and the next one
__device__ __forceinline__ void load_half(const float* __restrict__ p, float2 (&v)[kCur], int lane) {
#pragma unroll
    for (int a = 0; a < kCur; a++) {
        const int n = 64 * a + 2 * lane;
        v[a] = (a < 7 || lane < 16) ? make_float2(p[n], p[n + 1]) : make_float2(0.f, 0.f);
    }
}

// this frame's current slots as the next frame's half-window slots: half slot a of lane b is current slot a + 1 of
// lane b + 16 (b < 16) or current slot a of lane b - 16
__device__ __forceinline__ void cur_to_half(const float2 (&cur)[kCur], float2 (&h)[kCur], int lane) {
#pragma unroll
    for (int a = 0; a < kCur; a++) {
        const float2 v = lane < 16 ? cur[a < 7 ? a + 1 : 7] : cur[a];
        h[a] = make_float2(__shfl_xor_sync(0xffffffffu, v.x, 16), __shfl_xor_sync(0xffffffffu, v.y, 16));
    }
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float target_at(const MetricsArgs& a, int s, int t) {
    return a.tgt ? __ldg(a.tgt + (long)s * a.vss + (long)t * a.vfs) : 0.5f;
}

__global__ void __launch_bounds__(WPB * 32) metrics_kernel(MetricsArgs a, const DeviceTables* __restrict__ tab) {
    __shared__ __align__(16) float2 sbuf[WPB][WBUF];
    __shared__ float ssc[WPB][WSC];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* buf = sbuf[warp];
    float* sc = ssc[warp];
    const int T = a.n_frames;
    for (int s = blockIdx.x * WPB + warp; s < a.n_streams; s += gridDim.x * WPB) {
        RNNoiseMetricsRecord* r = a.rec + s;
        // the record's sums, spread over the lanes: class `lane` (< 3), band `lane` (< 22), vad count `lane` (< 4)
        const int q = lane < 3 ? lane : 0, bq = lane < NB_BANDS ? lane : 0, vq = lane & 3;
        long long frames = r->frames[q], vc = r->vad_counts[vq];
        double ec = r->ec[q], ey = r->ey[q], ecy = r->ecy[q], ed = r->ed[q];
        double seg = r->seg_snr, lsd = r->lsd, dev = r->speech_dev[bq], lev = r->noise_level[bq];
        float lastY = 0.0f, lastC = 0.0f;
        bool counted_any = false;
        const float* ys = a.out + (long)s * a.ss;
        const float* cs = a.clean + (long)s * a.ss;
        float* yhs = a.yh + (size_t)s * FRAME_SIZE;
        float* chs = a.ch + (size_t)s * FRAME_SIZE;
        float* cls = a.cl + (size_t)s * FRAME_SIZE;
        const bool started = a.started[s] != 0;
        float tgt_c = a.tl[s];  // target of the clean frame paired with frame j

        float2 hy[kCur], hc[kCur], ny[kCur], nc[kCur];
        load_half(yhs, hy, lane);
        load_half(chs, hc, lane);
        load_cur(ys, ny, lane);
        load_cur(cls, nc, lane);
        for (int j = 0; j < T; j++) {
            float2 cy[kCur], cc[kCur];
#pragma unroll
            for (int k = 0; k < kCur; k++) {
                cy[k] = ny[k];
                cc[k] = nc[k];
            }
            const bool counted = started || j > 0;
            const float tgt_now = target_at(a, s, j);
            const bool speech = tgt_c == 1.0f, noise = tgt_c == 0.0f;
            // the frame's time-domain sums from its own samples, reduced before the FFT so that only its segmental SNR
            // stays live across it
            double seg_f = 0.0;
            if (counted) {
                double pec = 0.0, pey = 0.0, pecy = 0.0, ped = 0.0;
#pragma unroll
                for (int k = 0; k < kCur; k++) {
                    const double c0 = cc[k].x, c1 = cc[k].y, y0 = cy[k].x, y1 = cy[k].y;
                    const double d0 = y0 - c0, d1 = y1 - c1;  // exact: both are floats
                    pec += c0 * c0 + c1 * c1;
                    pey += y0 * y0 + y1 * y1;
                    pecy += c0 * y0 + c1 * y1;
                    ped += d0 * d0 + d1 * d1;
                }
                const double fec = warp_sum(pec), fey = warp_sum(pey), fecy = warp_sum(pecy), fed = warp_sum(ped);
                if (q == lane && (lane == 0 || (lane == 1 && speech) || (lane == 2 && noise))) {
                    frames++;
                    ec += fec;
                    ey += fey;
                    ecy += fecy;
                    ed += fed;
                }
                seg_f = fed == 0.0 ? 35.0 : (fec == 0.0 ? -10.0 : fmin(fmax(10.0 * log10(fec / fed), -10.0), 35.0));
            }
            // the windowed samples
            float2 vx[15], vp[15];
#pragma unroll
            for (int s15 = 0; s15 < 15; s15++) {
                const int n2 = 64 * s15 + 2 * lane;
                const float2 w = __ldg(reinterpret_cast<const float2*>(tab->window) + (n2 >> 1));
                float2 y, c;
                if (s15 < 7) {
                    y = hy[s15];
                    c = hc[s15];
                } else if (s15 == 7) {
                    y = lane < 16 ? hy[7] : cy[0];
                    c = lane < 16 ? hc[7] : cc[0];
                } else {
                    y = cy[s15 - 7];
                    c = cc[s15 - 7];
                }
                vx[s15] = make_float2(y.x * w.x, y.y * w.y);
                vp[s15] = make_float2(c.x * w.x, c.y * w.y);
            }
            // the next frame's halves are this frame; its own samples are loaded ahead of the FFT
            cur_to_half(cy, hy, lane);
            cur_to_half(cc, hc, lane);
            if (j + 1 < T) {
                load_cur(ys + (long)(j + 1) * a.fs, ny, lane);
                load_cur(cs + (long)j * a.fs, nc, lane);
            }
            if (counted) {
                fft480_warp<true>(vx, vp, buf, tab, lane);
                {
                    const float wn = tab->wnorm;
#pragma unroll
                    for (int jj = 0; jj < 8; jj++) {
                        const int k = lane + 32 * jj;
                        if (k <= 240) {
                            const int kc = k == 0 ? 0 : 480 - k;
                            const float2 tw = __ldg(&tab->tw960[k]);
                            float2 x0, x1, p0, p1;
                            rfft_split_pair(buf[k], buf[kc], tw, wn, k == 0, x0, x1);
                            rfft_split_pair(buf[ZP_OFF + k], buf[ZP_OFF + kc], tw, wn, k == 0, p0, p1);
                            buf[k] = x0;
                            buf[ZP_OFF + k] = p0;
                            if (k != 240) {
                                buf[480 - k] = x1;
                                buf[ZP_OFF + 480 - k] = p1;
                            }
                        }
                    }
                }
                __syncwarp();
                float bs[3];
                band_sums_warp<3>(buf, tab, sc, lane, bs);
                const double ly = 10.0 * log10((double)bs[0] + 0.01), lc = 10.0 * log10((double)bs[1] + 0.01);
                const double d = lane < NB_BANDS ? ly - lc : 0.0;
                if (speech) {
                    const double sq = warp_sum(d * d);
                    seg += seg_f;
                    lsd += sqrt(sq / NB_BANDS);
                    dev += d;
                }
                if (noise) lev += ly;
                if (a.vad && a.tgt && (tgt_now == 0.0f || tgt_now == 1.0f)) {
                    const bool said = __ldg(a.vad + (long)s * a.vss + (long)j * a.vfs) >= 0.5f, is = tgt_now == 1.0f;
                    const int k = said ? (is ? 0 : 1) : (is ? 2 : 3);  // tp, fp, fn, tn
                    if (lane == k) vc++;
                }
                lastY = bs[0];
                lastC = bs[1];
                counted_any = true;
            }
            tgt_c = tgt_now;
        }
        // the pairing state after the call: the last output frame and the clean frame paired with it (now the halves
        // hy, hc), the last clean frame and its target
        __syncwarp();
#pragma unroll
        for (int k = 0; k < kCur; k++) {
            if (k < 7 || lane < 16) {
                const int n = 64 * k + 2 * lane;
                yhs[n] = hy[k].x;
                yhs[n + 1] = hy[k].y;
                chs[n] = hc[k].x;
                chs[n + 1] = hc[k].y;
            }
        }
        const float* last = cs + (long)(T - 1) * a.fs;
        for (int i = lane; i < FRAME_SIZE; i += 32) cls[i] = __ldg(last + i);
        if (lane == 0) {
            a.tl[s] = tgt_c;
            a.started[s] = 1;
        }
        if (lane < 3) {
            r->frames[lane] = frames;
            r->ec[lane] = ec;
            r->ey[lane] = ey;
            r->ecy[lane] = ecy;
            r->ed[lane] = ed;
        }
        if (lane == 0) {
            r->seg_snr = seg;
            r->lsd = lsd;
        }
        if (lane < NB_BANDS) {
            r->speech_dev[lane] = dev;
            r->noise_level[lane] = lev;
            if (counted_any) {
                r->last_bands[0][lane] = lastY;
                r->last_bands[1][lane] = lastC;
            }
        }
        if (lane < 4) r->vad_counts[lane] = vc;
    }
}

__global__ void metrics_clear_kernel(RNNoiseMetricsRecord* rec, const int* idx, int n) {
    constexpr int W = sizeof(RNNoiseMetricsRecord) / 8;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)n * W) return;
    const int r = (int)(i / W);
    reinterpret_cast<unsigned long long*>(rec + idx[r])[i % W] = 0ull;
}

}  // namespace

}  // namespace nnb

using namespace nnb;

struct RNNoiseMetrics {
    int device = 0, n_streams = 0, grid = 0;
    Stream st;
    Event ev_call, ev_done;
    DeviceMem tab, rec, yh, ch, cl, tl, started, idx;
};

static int check_handle(const RNNoiseMetrics* m) { return m ? 0 : fail("null metrics handle"); }

extern "C" {

RNNoiseMetrics* rnnoise_metrics_create(int n_streams, int device) {
    if (n_streams <= 0) {
        fail("n_streams must be positive");
        return nullptr;
    }
    if (open_device(device, &device)) return nullptr;
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) {
        fail("cudaSetDevice", guard.err);
        return nullptr;
    }
    std::unique_ptr<RNNoiseMetrics> m(new (std::nothrow) RNNoiseMetrics());
    std::unique_ptr<DeviceTables> ht(new (std::nothrow) DeviceTables());
    if (!m || !ht) {
        fail("out of memory");
        return nullptr;
    }
    m->device = device;
    m->n_streams = n_streams;
    const size_t S = (size_t)n_streams, half = S * FRAME_SIZE * sizeof(float);
    build_tables(ht.get());
    int sms = 0, per_sm = 0;
    cudaError_t e = cudaStreamCreateWithFlags(m->st.put(), cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(m->ev_call.put(), cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(m->ev_done.put(), cudaEventDisableTiming);
    if (e == cudaSuccess) e = m->tab.alloc(sizeof(DeviceTables));
    if (e == cudaSuccess) e = m->rec.alloc(S * sizeof(RNNoiseMetricsRecord));
    for (DeviceMem* d : {&m->yh, &m->ch, &m->cl})
        if (e == cudaSuccess) e = d->alloc(half);
    if (e == cudaSuccess) e = m->tl.alloc(S * sizeof(float));
    if (e == cudaSuccess) e = m->started.alloc(S * sizeof(int));
    for (DeviceMem* d : {&m->rec, &m->yh, &m->ch, &m->cl, &m->tl, &m->started})
        if (e == cudaSuccess) e = cudaMemsetAsync(d->get(), 0, d->bytes(), m->st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(m->tab.get(), ht.get(), sizeof(DeviceTables), cudaMemcpyHostToDevice, m->st);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, metrics_kernel, WPB * 32, 0);
    if (e == cudaSuccess) e = cudaStreamSynchronize(m->st);  // ht is the copy's source
    if (e != cudaSuccess) {
        fail("metrics of " + std::to_string(n_streams) + " streams", e);
        return nullptr;
    }
    m->grid = (int)std::min<long>((S + WPB - 1) / WPB, (long)std::max(per_sm, 1) * sms);
    return m.release();
}

void rnnoise_metrics_destroy(RNNoiseMetrics* m) {
    if (!m) return;
    DeviceGuard guard(m->device);
    if (m->st) cudaStreamSynchronize(m->st);
    delete m;
}

int rnnoise_metrics_accumulate_device(RNNoiseMetrics* m, const float* out, const float* clean, long stream_stride, long frame_stride,
                                      const float* vad, const float* vad_target, long vad_stream_stride, long vad_frame_stride,
                                      int n_frames, void* cuda_stream) {
    if (!out || !clean) return fail("null out or clean");
    if (n_frames < 0) return fail("negative n_frames");
    if (check_handle(m)) return -1;
    if (n_frames == 0) return 0;
    if (!rows_disjoint(m->n_streams, n_frames, stream_stride, frame_stride, FRAME_SIZE)) return fail("sample strides overlap frames");
    if ((vad || vad_target) && !rows_disjoint(m->n_streams, n_frames, vad_stream_stride, vad_frame_stride, 1))
        return fail("vad strides overlap");
    ON_DEVICE(m->device);
    cudaStream_t us = (cudaStream_t)cuda_stream;
    if (wait_for_caller(m->st, us, m->ev_call)) return -1;
    MetricsArgs a{out, clean, stream_stride, frame_stride, vad, vad_target, vad_stream_stride, vad_frame_stride, n_frames, m->n_streams,
                  m->yh.get<float>(), m->ch.get<float>(), m->cl.get<float>(), m->tl.get<float>(), m->started.get<int>(),
                  m->rec.get<RNNoiseMetricsRecord>()};
    metrics_kernel<<<m->grid, WPB * 32, 0, m->st>>>(a, m->tab.get<DeviceTables>());
    CK(cudaGetLastError());
    count_launches(1);
    return resume_caller(m->st, us, m->ev_done);
}

int rnnoise_metrics_clear(RNNoiseMetrics* m, const int* streams, int n) {
    if (check_handle(m)) return -1;
    if (check_streams(m->n_streams, streams, n, "metrics handle")) return -1;
    if (n == 0) return 0;
    ON_DEVICE(m->device);
    std::vector<int> idx((size_t)n);
    for (int r = 0; r < n; r++) idx[(size_t)r] = stream_of(streams, r);
    if (m->idx.bytes() < idx.size() * sizeof(int)) {
        CK(cudaStreamSynchronize(m->st));
        CK(m->idx.alloc(idx.size() * sizeof(int)));
    }
    CK(cudaMemcpyAsync(m->idx.get(), idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice, m->st));
    const long words = (long)n * (sizeof(RNNoiseMetricsRecord) / 8);
    metrics_clear_kernel<<<(unsigned)((words + 255) / 256), 256, 0, m->st>>>(m->rec.get<RNNoiseMetricsRecord>(), m->idx.get<int>(), n);
    CK(cudaGetLastError());
    count_launches(1);
    CK(cudaStreamSynchronize(m->st));  // idx is the copy's source
    return 0;
}

int rnnoise_metrics_get(RNNoiseMetrics* m, const int* streams, int n, RNNoiseMetricsRecord* dst) {
    if (check_handle(m)) return -1;
    if (check_streams(m->n_streams, streams, n, "metrics handle")) return -1;
    if (n == 0) return 0;
    if (!dst) return fail("null argument");
    ON_DEVICE(m->device);
    std::vector<RNNoiseMetricsRecord> all((size_t)m->n_streams);
    CK(cudaMemcpyAsync(all.data(), m->rec.get(), all.size() * sizeof(RNNoiseMetricsRecord), cudaMemcpyDeviceToHost, m->st));
    CK(cudaStreamSynchronize(m->st));
    for (int r = 0; r < n; r++) std::memcpy(dst + r, &all[(size_t)stream_of(streams, r)], sizeof(RNNoiseMetricsRecord));
    return 0;
}

}  // extern "C"
