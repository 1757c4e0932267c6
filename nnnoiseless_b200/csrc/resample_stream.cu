// resample_stream.cu -- streams at their own sample rate (DESIGN.md 7g): per-stream polyphase resampling of 10 ms
// frames to and from the 48 kHz, 480-sample frames of the denoise path, with each stream's filter history carried
// from call to call.
//
// A stream at rate R (8000..48000, a multiple of 100) gives and gets R/100 samples per frame.  With g = gcd(48000, R),
// U = 48000/g and D = R/g, the up stage is scipy.signal.upfirdn(h_up, x, U, D) and the down stage
// upfirdn(h_dn, y, D, U), where h = firwin(20 U + 1, 1/U, window=('kaiser', 5.0)) scaled by the stage's up factor:
// resample_poly's default filter, causal, without delay compensation.  Each stage makes a whole number of samples per
// frame, so the polyphase phase is 0 at every frame boundary and frame t depends on its own input and on the last 20
// (up) or floor(20 U / D) <= 120 (down) input samples before it.  Those come from frame t - 1 of the same call, or for
// frame 0 from the stream's stored history, so both kernels run every (stream, frame) of a call in parallel; the
// warp of frame 0 also stores the tail of the call's last frame as the new history.
//
// Output sample i of a frame is sum_m h[p + m * up] * x[j0 - m] with i * down = j0 * up + p, accumulated with fmaf
// in ascending m: the bits depend on the stream's rate and samples only.  48 kHz streams pass through unchanged.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <new>
#include <numeric>
#include <string>
#include <vector>

#include "../../include/rnnoise.h"
#include "abi.hpp"
#include "common.cuh"
#include "owners.hpp"

namespace nnb {
int batch_device(const RNNoiseBatch* b);  // host.cu
}  // namespace nnb

using namespace nnb;

namespace {

constexpr int kUpHist = 20;    // native samples before a frame that the up stage reads
constexpr int kDnHist = 120;   // 48 kHz samples before a frame that the down stage reads (floor(20 U / D) at 8 kHz)
constexpr int kUpTaps = 21;    // taps of up-stage phase 0 (the other phases have 20)
constexpr int kWarps = 8;      // rows of one frame per block, one per warp
constexpr int kMaxGridY = 65535;  // frames per launch (grid y); longer calls take several launches
constexpr size_t kChunkBytes = size_t(256) << 20;  // bound of the scratch of one process_native chunk
// state record (include/rnnoise.h): 16-byte head, then the up history, then the down history
constexpr int kRecFloats = RNNOISE_RESAMPLER_STATE_BYTES / 4, kRecUp = 4, kRecDn = kRecUp + kUpHist;
static_assert(kRecDn + kDnHist == kRecFloats, "resampler state record layout");

// One distinct rate: the two stages' taps, phase-major, in the resampler's tap table.
struct RsRate {
    int nin;        // R / 100: native samples per frame
    int U, D;       // 48000 / g, R / g (1, 1: 48 kHz, pass-through)
    int up_off;     // up stage: U phases of kUpTaps, up[p * kUpTaps + m] = h_up[p + m U]
    int dn_off;     // down stage: D phases of dn_stride, dn[p * dn_stride + m] = h_dn[p + m D]
    int dn_stride;  // 20 U / D + 1: taps of down-stage phase 0
};

struct RsArgs {
    const RsRate* rates;
    const float* taps;
    const int* rid;    // [n_streams] rate id of every stream
    float* hist;       // [n_streams][kUpHist] (up) or [n_streams][kDnHist] (down)
    const int* idx;    // [n] stream of each row, NULL: rows 0..n-1
    int n, T;          // rows, frames of the call
    int t0;            // first frame of this launch (blockIdx.y = frame - t0)
    long ss, fs;       // native side: element strides of a row and a frame
    int fill;          // down stage: samples written per frame, 0 = R / 100 (the rest, up to fill, are zeros)
};

__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(short v) { return (float)v; }
__device__ __forceinline__ void store(float* p, float v) { *p = v; }
__device__ __forceinline__ void store(short* p, float v) { *p = to_pcm16w(v); }

// native [row][frame][R/100] -> compact 48 kHz [frame][row][480]
template <typename TIn>
__global__ void __launch_bounds__(kWarps * 32) resample_up_kernel(RsArgs a, const TIn* __restrict__ in, float* __restrict__ out) {
    __shared__ float sbuf[kWarps][kUpHist + FRAME_SIZE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = blockIdx.x * kWarps + warp, t = a.t0 + blockIdx.y;
    if (r >= a.n) return;
    const int s = a.idx ? a.idx[r] : r;
    const RsRate q = a.rates[a.rid[s]];
    float* x = sbuf[warp] + kUpHist;  // x[-kUpHist .. nin)
    const TIn* row = in + (long)r * a.ss;
    for (int i = lane; i < q.nin; i += 32) x[i] = widen(row[(long)t * a.fs + i]);
    if (lane < kUpHist) {
        const int k = lane, tail = q.nin - kUpHist + k;
        float* h = a.hist + (size_t)s * kUpHist + k;
        x[k - kUpHist] = t == 0 ? *h : widen(row[(long)(t - 1) * a.fs + tail]);
        if (t == 0) *h = widen(row[(long)(a.T - 1) * a.fs + tail]);  // the same lane read the old value above
    }
    __syncwarp();
    float* o = out + ((size_t)t * a.n + r) * FRAME_SIZE;
    const float* taps = a.taps + q.up_off;
    for (int i = lane; i < FRAME_SIZE; i += 32) {
        float acc;
        if (q.U == 1) {
            acc = x[i];
        } else {
            const int num = i * q.D, j0 = num / q.U, p = num - j0 * q.U, nt = p == 0 ? kUpTaps : kUpTaps - 1;
            const float* h = taps + p * kUpTaps;
            acc = 0.0f;
            for (int m = 0; m < nt; m++) acc = fmaf(__ldg(h + m), x[j0 - m], acc);
        }
        o[i] = acc;
    }
}

// compact 48 kHz [frame][row][480] -> native [row][frame][R/100]
template <typename TOut>
__global__ void __launch_bounds__(kWarps * 32) resample_down_kernel(RsArgs a, const float* __restrict__ in, TOut* __restrict__ out) {
    __shared__ float sbuf[kWarps][kDnHist + FRAME_SIZE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = blockIdx.x * kWarps + warp, t = a.t0 + blockIdx.y;
    if (r >= a.n) return;
    const int s = a.idx ? a.idx[r] : r;
    const RsRate q = a.rates[a.rid[s]];
    float* x = sbuf[warp] + kDnHist;  // x[-kDnHist .. 480)
    const float* src = in + ((size_t)t * a.n + r) * FRAME_SIZE;
    for (int i = lane; i < FRAME_SIZE; i += 32) x[i] = src[i];
    for (int k = lane; k < kDnHist; k += 32) {
        const int tail = FRAME_SIZE - kDnHist + k;
        float* h = a.hist + (size_t)s * kDnHist + k;
        x[k - kDnHist] = t == 0 ? *h : in[((size_t)(t - 1) * a.n + r) * FRAME_SIZE + tail];
        if (t == 0) *h = in[((size_t)(a.T - 1) * a.n + r) * FRAME_SIZE + tail];
    }
    __syncwarp();
    TOut* o = out + (long)r * a.ss + (long)t * a.fs;
    const float* taps = a.taps + q.dn_off;
    const int fill = a.fill ? a.fill : q.nin;
    for (int i = lane; i < fill; i += 32) {
        float acc = 0.0f;
        if (i >= q.nin) {
        } else if (q.U == 1) {
            acc = x[i];
        } else {
            const int num = i * q.U, j0 = num / q.D, p = num - j0 * q.D, nt = (20 * q.U - p) / q.D + 1;
            const float* h = taps + p * q.dn_stride;
            for (int m = 0; m < nt; m++) acc = fmaf(__ldg(h + m), x[j0 - m], acc);
        }
        store(o + i, acc);
    }
}

// Sets the rate id of stream idx[r] (NULL: r) to ids[r] and its histories to record r's (rec NULL: zeros).
__global__ void __launch_bounds__(kWarps * 32) resample_set_kernel(const int* __restrict__ idx, int n, const int* __restrict__ ids,
                                                                 const float* __restrict__ rec, int* rid, float* hup, float* hdn) {
    const int lane = threadIdx.x & 31, r = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (r >= n) return;
    const int s = idx ? idx[r] : r;
    const float* src = rec ? rec + (size_t)r * kRecFloats : nullptr;
    if (lane == 0) rid[s] = ids[r];
    for (int k = lane; k < kUpHist; k += 32) hup[(size_t)s * kUpHist + k] = src ? src[kRecUp + k] : 0.0f;
    for (int k = lane; k < kDnHist; k += 32) hdn[(size_t)s * kDnHist + k] = src ? src[kRecDn + k] : 0.0f;
}

// The histories of stream idx[r] into record r (the head is the host's).
__global__ void __launch_bounds__(kWarps * 32) resample_get_kernel(const int* __restrict__ idx, int n, const float* __restrict__ hup,
                                                                 const float* __restrict__ hdn, float* __restrict__ rec) {
    const int lane = threadIdx.x & 31, r = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (r >= n) return;
    const int s = idx ? idx[r] : r;
    float* dst = rec + (size_t)r * kRecFloats;
    for (int k = lane; k < kUpHist; k += 32) dst[kRecUp + k] = hup[(size_t)s * kUpHist + k];
    for (int k = lane; k < kDnHist; k += 32) dst[kRecDn + k] = hdn[(size_t)s * kDnHist + k];
}

unsigned blocks(int items) { return (unsigned)((items + kWarps - 1) / kWarps); }

// ---- filter design (host, double) ----------------------------------------------------------------------------------
bool valid_rate(int rate) { return rate >= 8000 && rate <= 48000 && rate % 100 == 0; }

std::string rate_error(int rate) {
    return "rate " + std::to_string(rate) + " Hz: a stream rate must be a multiple of 100 in 8000..48000";
}

double bessel_i0(double x) {
    double sum = 1.0, term = 1.0;
    for (int k = 1; k < 1000; k++) {
        const double f = x / (2.0 * k);
        term *= f * f;
        sum += term;
        if (term < sum * 1e-18) break;
    }
    return sum;
}

// scipy.signal.firwin(n, 1 / M, window=('kaiser', 5.0)): windowed ideal low-pass, scaled to unit gain at DC
std::vector<double> firwin_kaiser(int n, int M) {
    const double pi = 3.14159265358979323846264338327950288, beta = 5.0, alpha = 0.5 * (n - 1), c = 1.0 / M;
    std::vector<double> h((size_t)n);
    double sum = 0.0;
    for (int i = 0; i < n; i++) {
        const double m = i - alpha, x = c * m;
        const double sinc = x == 0.0 ? 1.0 : std::sin(pi * x) / (pi * x);
        const double r = m / alpha;
        h[(size_t)i] = c * sinc * (bessel_i0(beta * std::sqrt(1.0 - r * r)) / bessel_i0(beta));
        sum += h[(size_t)i];
    }
    for (double& v : h) v /= sum;
    return h;
}

// The stage's factors and f32 filter: direction 0 = up (R -> 48 kHz), 1 = down.  48 kHz: one tap of 1.
void stage_filter(int rate, int direction, std::vector<float>* h, int* up, int* down) {
    const int g = std::gcd(48000, rate), U = 48000 / g, D = rate / g;
    *up = direction ? D : U;
    *down = direction ? U : D;
    h->clear();
    if (U == 1) {
        h->push_back(1.0f);
        return;
    }
    for (double v : firwin_kaiser(20 * U + 1, U)) h->push_back((float)(v * *up));
}

}  // namespace

struct RNNoiseResampler {
    int device = 0, n_streams = 0;
    Stream st;                      // every kernel of the resampler runs here
    Event ev_call, ev_done;
    std::vector<int> rates;         // host mirror: the rate of every stream
    std::vector<int> rate_list;     // distinct rates met so far; rate id k is rate_list[k]
    std::vector<RsRate> h_rates;
    std::vector<float> h_taps;
    DeviceMem d_rates, d_taps;      // device images of h_rates / h_taps
    DeviceMem rid, hup, hdn;        // per stream: rate id, up and down histories
    DeviceMem idx, ids, rec;        // per call: stream indices, rate ids, state records
    DeviceMem scratch;              // process_native: 48 kHz frames (+ the host call's native frames and vad)
};

namespace {

// m holds at least `bytes`; a reallocation waits for the work that may still use the old one
int grow(RNNoiseResampler* rs, DeviceMem* m, size_t bytes) {
    if (m->bytes() >= bytes) return 0;
    CK(cudaStreamSynchronize(rs->st));
    CK(m->alloc(bytes));
    return 0;
}

int check_rates(const int* streams, int n, const int* rates) {
    for (int r = 0; r < n; r++)
        if (!valid_rate(rates[r])) return fail("stream " + std::to_string(stream_of(streams, r)) + ": " + rate_error(rates[r]));
    return 0;
}

// The rate ids of `rates`, adding the rates not met before to the tap tables.
int rate_ids(RNNoiseResampler* rs, const int* rates, int n, std::vector<int>* ids) {
    const size_t before = rs->rate_list.size();
    ids->resize((size_t)n);
    for (int r = 0; r < n; r++) {
        const auto it = std::find(rs->rate_list.begin(), rs->rate_list.end(), rates[r]);
        (*ids)[(size_t)r] = (int)(it - rs->rate_list.begin());
        if (it != rs->rate_list.end()) continue;
        const int R = rates[r];
        std::vector<float> hu, hd;
        int U, D, up2, down2;
        stage_filter(R, 0, &hu, &U, &D);
        stage_filter(R, 1, &hd, &up2, &down2);
        RsRate q{R / 100, U, D, (int)rs->h_taps.size(), 0, 20 * U / D + 1};
        rs->h_taps.resize((size_t)q.up_off + (size_t)U * kUpTaps, 0.0f);
        for (int k = 0; k < (int)hu.size() && U > 1; k++) rs->h_taps[(size_t)q.up_off + (size_t)(k % U) * kUpTaps + k / U] = hu[(size_t)k];
        q.dn_off = (int)rs->h_taps.size();
        rs->h_taps.resize((size_t)q.dn_off + (size_t)D * q.dn_stride, 0.0f);
        for (int k = 0; k < (int)hd.size() && U > 1; k++) rs->h_taps[(size_t)q.dn_off + (size_t)(k % D) * q.dn_stride + k / D] = hd[(size_t)k];
        rs->rate_list.push_back(R);
        rs->h_rates.push_back(q);
    }
    if (rs->rate_list.size() == before) return 0;
    // kernels in flight read the old tables: they are replaced once the stream has drained
    CK(cudaStreamSynchronize(rs->st));
    CK(rs->d_rates.alloc(rs->h_rates.size() * sizeof(RsRate)));
    CK(rs->d_taps.alloc(rs->h_taps.size() * sizeof(float)));
    CK(cudaMemcpy(rs->d_rates.get(), rs->h_rates.data(), rs->h_rates.size() * sizeof(RsRate), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(rs->d_taps.get(), rs->h_taps.data(), rs->h_taps.size() * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

// Upload the rows' stream indices on rs->st; *d = NULL for streams NULL.
int upload_idx(RNNoiseResampler* rs, const int* streams, int n, const int** d) {
    *d = nullptr;
    if (!streams || n == 0) return 0;
    if (grow(rs, &rs->idx, (size_t)n * sizeof(int))) return -1;
    CK(cudaMemcpyAsync(rs->idx.get(), streams, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, rs->st));
    *d = rs->idx.get<int>();
    return 0;
}

// Streams streams[r] get rate rates[r] and the histories of record r (recs NULL: zeros).  Arguments are checked.
int assign(RNNoiseResampler* rs, const int* streams, int n, const int* rates, const float* recs) {
    std::vector<int> ids;
    if (rate_ids(rs, rates, n, &ids)) return -1;
    const int* d_idx;
    if (upload_idx(rs, streams, n, &d_idx)) return -1;
    if (grow(rs, &rs->ids, (size_t)n * sizeof(int)) || (recs && grow(rs, &rs->rec, (size_t)n * RNNOISE_RESAMPLER_STATE_BYTES))) return -1;
    CK(cudaMemcpyAsync(rs->ids.get(), ids.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, rs->st));
    if (recs) CK(cudaMemcpyAsync(rs->rec.get(), recs, (size_t)n * RNNOISE_RESAMPLER_STATE_BYTES, cudaMemcpyHostToDevice, rs->st));
    resample_set_kernel<<<blocks(n), kWarps * 32, 0, rs->st>>>(d_idx, n, rs->ids.get<int>(), recs ? rs->rec.get<float>() : nullptr,
                                                              rs->rid.get<int>(), rs->hup.get<float>(), rs->hdn.get<float>());
    CK(cudaGetLastError());
    count_launches(1);
    CK(cudaStreamSynchronize(rs->st));  // the host arrays above are the copies' sources
    for (int r = 0; r < n; r++) rs->rates[(size_t)stream_of(streams, r)] = rates[r];
    return 0;
}

RsArgs args(RNNoiseResampler* rs, const int* d_idx, int n, int T, long ss, long fs, float* hist) {
    return {rs->d_rates.get<RsRate>(), rs->d_taps.get<float>(), rs->rid.get<int>(), hist, d_idx, n, T, 0, ss, fs, 0};
}

// Launchers on rs->st; the rows' indices are uploaded already.
int launch_up(RNNoiseResampler* rs, const int* d_idx, int n, float* out, const void* in, int pcm16, int T, long ss, long fs) {
    RsArgs a = args(rs, d_idx, n, T, ss, fs, rs->hup.get<float>());
    for (a.t0 = 0; a.t0 < T; a.t0 += kMaxGridY) {
        const dim3 grid(blocks(n), (unsigned)std::min(kMaxGridY, T - a.t0));
        if (pcm16) resample_up_kernel<short><<<grid, kWarps * 32, 0, rs->st>>>(a, static_cast<const short*>(in), out);
        else resample_up_kernel<float><<<grid, kWarps * 32, 0, rs->st>>>(a, static_cast<const float*>(in), out);
        CK(cudaGetLastError());
        count_launches(1);
    }
    return 0;
}

int launch_down(RNNoiseResampler* rs, const int* d_idx, int n, void* out, const float* in, int pcm16, int T, long ss, long fs, int fill) {
    RsArgs a = args(rs, d_idx, n, T, ss, fs, rs->hdn.get<float>());
    a.fill = fill;
    for (a.t0 = 0; a.t0 < T; a.t0 += kMaxGridY) {
        const dim3 grid(blocks(n), (unsigned)std::min(kMaxGridY, T - a.t0));
        if (pcm16) resample_down_kernel<short><<<grid, kWarps * 32, 0, rs->st>>>(a, in, static_cast<short*>(out));
        else resample_down_kernel<float><<<grid, kWarps * 32, 0, rs->st>>>(a, in, static_cast<float*>(out));
        CK(cudaGetLastError());
        count_launches(1);
    }
    return 0;
}

// Checks shared by the stage calls; 1: nothing to do, 0: go ahead, -1: error.
int stage_check(const RNNoiseResampler* rs, const int* streams, int n, const void* out, const void* in, int pcm16, int n_frames) {
    if (!rs) return fail("null resampler");
    if (check_streams(rs->n_streams, streams, n, "resampler")) return -1;
    if (pcm16 != 0 && pcm16 != 1) return fail("pcm16 must be 0 (float) or 1 (int16)");
    if (n_frames < 0) return fail("negative n_frames");
    if (n == 0 || n_frames == 0) return 1;
    if (!out || !in) return fail("null argument");
    return 0;
}

// The up -> denoise -> down path of one chunk of frames, in place on the 48 kHz scratch `w48`.
int native_chunk(RNNoiseBatch* b, RNNoiseResampler* rs, const int* streams, const int* d_idx, int n, void* out, const void* in, int pcm16,
                 float* vad, int nf, long ss, long fs, int fill, float* w48) {
    if (launch_up(rs, d_idx, n, w48, in, pcm16, nf, ss, fs)) return -1;
    const long B = (long)n * FRAME_SIZE;
    const int rc = !streams && n == rs->n_streams
                       ? rnnoise_batch_process_device(b, w48, w48, vad, nf, FRAME_SIZE, B, rs->st)
                       : rnnoise_batch_process_streams_device(b, streams, n, w48, w48, 0, vad, nf, FRAME_SIZE, 1, B, rs->st);
    if (rc) return -1;
    return launch_down(rs, d_idx, n, out, w48, pcm16, nf, ss, fs, fill);
}

int native_check(RNNoiseBatch* b, RNNoiseResampler* rs, const int* streams, int n, const void* out, const void* in, int pcm16, int n_frames) {
    if (!b) return fail("null batch");
    const int rc = stage_check(rs, streams, n, out, in, pcm16, n_frames);
    if (rc) return rc;
    if (rnnoise_batch_streams(b) != rs->n_streams)
        return fail("the batch has " + std::to_string(rnnoise_batch_streams(b)) + " streams, the resampler " + std::to_string(rs->n_streams));
    if (batch_device(b) != rs->device)
        return fail("the batch is on device " + std::to_string(batch_device(b)) + ", the resampler on device " + std::to_string(rs->device));
    return 0;
}

}  // namespace

extern "C" {

int rnnoise_resampler_filter(int rate, int direction, float* taps, int cap, int* up, int* down) {
    if (!valid_rate(rate)) return fail(rate_error(rate));
    if (direction != 0 && direction != 1) return fail("direction must be 0 (up) or 1 (down)");
    std::vector<float> h;
    int u, d;
    stage_filter(rate, direction, &h, &u, &d);
    if (up) *up = u;
    if (down) *down = d;
    if (taps) std::copy(h.begin(), h.begin() + std::min<size_t>(h.size(), (size_t)std::max(cap, 0)), taps);
    return (int)h.size();
}

double rnnoise_resampler_delay(int rate) {
    if (!valid_rate(rate)) {
        fail(rate_error(rate));
        return -1.0;
    }
    return rate == 48000 ? 0.0 : 960000.0 / rate;  // (20 U / D) / 2 per stage, in 48 kHz samples
}

RNNoiseResampler* rnnoise_resampler_create(int n_streams, const int* rates, int device) {
    if (n_streams <= 0) {
        fail("n_streams must be positive");
        return nullptr;
    }
    if (rates && check_rates(nullptr, n_streams, rates)) return nullptr;
    if (open_device(device, &device)) return nullptr;
    DeviceGuard guard(device);
    if (guard.err != cudaSuccess) {
        fail("cudaSetDevice", guard.err);
        return nullptr;
    }
    std::unique_ptr<RNNoiseResampler> rs(new (std::nothrow) RNNoiseResampler());
    if (!rs) {
        fail("out of memory");
        return nullptr;
    }
    rs->device = device;
    rs->n_streams = n_streams;
    rs->rates.assign((size_t)n_streams, 48000);
    const size_t S = (size_t)n_streams;
    std::vector<int> all(rates ? rates : rs->rates.data(), (rates ? rates : rs->rates.data()) + S);
    cudaError_t e = cudaStreamCreateWithFlags(rs->st.put(), cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(rs->ev_call.put(), cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(rs->ev_done.put(), cudaEventDisableTiming);
    if (e == cudaSuccess) e = rs->rid.alloc(S * sizeof(int));
    if (e == cudaSuccess) e = rs->hup.alloc(S * kUpHist * sizeof(float));
    if (e == cudaSuccess) e = rs->hdn.alloc(S * kDnHist * sizeof(float));
    if (e != cudaSuccess) {
        fail("resampler of " + std::to_string(n_streams) + " streams", e);
        return nullptr;
    }
    if (assign(rs.get(), nullptr, n_streams, all.data(), nullptr)) return nullptr;
    return rs.release();
}

void rnnoise_resampler_destroy(RNNoiseResampler* rs) {
    if (!rs) return;
    DeviceGuard guard(rs->device);
    if (rs->st) cudaStreamSynchronize(rs->st);
    delete rs;
}

int rnnoise_resampler_set_stream_rates(RNNoiseResampler* rs, const int* streams, int n, const int* rates) {
    if (!rs) return fail("null resampler");
    if (check_streams(rs->n_streams, streams, n, "resampler")) return -1;
    if (n == 0) return 0;
    if (!rates) return fail("null argument");
    if (check_rates(streams, n, rates)) return -1;
    ON_DEVICE(rs->device);
    return assign(rs, streams, n, rates, nullptr);
}

int rnnoise_resampler_get_stream_rates(const RNNoiseResampler* rs, const int* streams, int n, int* rates) {
    if (!rs) return fail("null resampler");
    if (check_streams(rs->n_streams, streams, n, "resampler")) return -1;
    if (n == 0) return 0;
    if (!rates) return fail("null argument");
    for (int r = 0; r < n; r++) rates[r] = rs->rates[(size_t)stream_of(streams, r)];
    return 0;
}

int rnnoise_resampler_up_device(RNNoiseResampler* rs, const int* streams, int n, float* out, const void* in, int pcm16, int n_frames,
                                long stream_stride, long frame_stride, void* cuda_stream) {
    const int rc = stage_check(rs, streams, n, out, in, pcm16, n_frames);
    if (rc) return rc < 0 ? -1 : 0;
    ON_DEVICE(rs->device);
    cudaStream_t us = (cudaStream_t)cuda_stream;
    const int* d_idx;
    if (wait_for_caller(rs->st, us, rs->ev_call) || upload_idx(rs, streams, n, &d_idx)) return -1;
    if (launch_up(rs, d_idx, n, out, in, pcm16, n_frames, stream_stride, frame_stride)) return -1;
    return resume_caller(rs->st, us, rs->ev_done);
}

int rnnoise_resampler_down_device(RNNoiseResampler* rs, const int* streams, int n, void* out, const float* in, int pcm16, int n_frames,
                                  long stream_stride, long frame_stride, void* cuda_stream) {
    const int rc = stage_check(rs, streams, n, out, in, pcm16, n_frames);
    if (rc) return rc < 0 ? -1 : 0;
    ON_DEVICE(rs->device);
    cudaStream_t us = (cudaStream_t)cuda_stream;
    const int* d_idx;
    if (wait_for_caller(rs->st, us, rs->ev_call) || upload_idx(rs, streams, n, &d_idx)) return -1;
    if (launch_down(rs, d_idx, n, out, in, pcm16, n_frames, stream_stride, frame_stride, 0)) return -1;
    return resume_caller(rs->st, us, rs->ev_done);
}

int rnnoise_resampler_get_states(RNNoiseResampler* rs, const int* streams, int n, void* dst) {
    if (!rs) return fail("null resampler");
    if (check_streams(rs->n_streams, streams, n, "resampler")) return -1;
    if (n == 0) return 0;
    if (!dst) return fail("null argument");
    ON_DEVICE(rs->device);
    const size_t bytes = (size_t)n * RNNOISE_RESAMPLER_STATE_BYTES;
    const int* d_idx;
    if (grow(rs, &rs->rec, bytes) || upload_idx(rs, streams, n, &d_idx)) return -1;
    resample_get_kernel<<<blocks(n), kWarps * 32, 0, rs->st>>>(d_idx, n, rs->hup.get<float>(), rs->hdn.get<float>(), rs->rec.get<float>());
    CK(cudaGetLastError());
    count_launches(1);
    CK(cudaMemcpyAsync(dst, rs->rec.get(), bytes, cudaMemcpyDeviceToHost, rs->st));
    CK(cudaStreamSynchronize(rs->st));
    for (int r = 0; r < n; r++) {
        const int32_t head[4] = {(int32_t)RNNOISE_RESAMPLER_STATE_MAGIC, RNNOISE_RESAMPLER_STATE_VERSION, rs->rates[(size_t)stream_of(streams, r)], 0};
        std::memcpy(static_cast<unsigned char*>(dst) + (size_t)r * RNNOISE_RESAMPLER_STATE_BYTES, head, sizeof head);
    }
    return 0;
}

int rnnoise_resampler_set_states(RNNoiseResampler* rs, const int* streams, int n, const void* src) {
    if (!rs) return fail("null resampler");
    if (check_streams(rs->n_streams, streams, n, "resampler")) return -1;
    if (n == 0) return 0;
    if (!src) return fail("null argument");
    std::vector<int> rates((size_t)n);
    for (int r = 0; r < n; r++) {
        int32_t head[4];
        std::memcpy(head, static_cast<const unsigned char*>(src) + (size_t)r * RNNOISE_RESAMPLER_STATE_BYTES, sizeof head);
        const std::string at = "resampler state record " + std::to_string(r) + ": ";
        if ((uint32_t)head[0] != RNNOISE_RESAMPLER_STATE_MAGIC) return fail(at + "bad magic");
        if (head[1] != RNNOISE_RESAMPLER_STATE_VERSION) return fail(at + "unsupported version " + std::to_string(head[1]));
        if (!valid_rate(head[2])) return fail(at + rate_error(head[2]));
        rates[(size_t)r] = head[2];
    }
    ON_DEVICE(rs->device);
    return assign(rs, streams, n, rates.data(), static_cast<const float*>(src));
}

int rnnoise_batch_process_native_device(RNNoiseBatch* b, RNNoiseResampler* rs, const int* streams, int n, void* out, const void* in, int pcm16,
                                        float* vad, int n_frames, long stream_stride, long frame_stride, void* cuda_stream) {
    const int rc = native_check(b, rs, streams, n, out, in, pcm16, n_frames);
    if (rc) return rc < 0 ? -1 : 0;
    ON_DEVICE(rs->device);
    cudaStream_t us = (cudaStream_t)cuda_stream;
    const size_t frame_bytes = (size_t)n * FRAME_SIZE * sizeof(float);
    const int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_frames, kChunkBytes / frame_bytes));
    const int* d_idx;
    if (wait_for_caller(rs->st, us, rs->ev_call) || grow(rs, &rs->scratch, (size_t)chunk * frame_bytes) || upload_idx(rs, streams, n, &d_idx)) return -1;
    const size_t esz = pcm16 ? sizeof(short) : sizeof(float);
    for (int f0 = 0; f0 < n_frames; f0 += chunk) {
        const int nf = std::min(chunk, n_frames - f0);
        const size_t off = (size_t)f0 * frame_stride * esz;
        if (native_chunk(b, rs, streams, d_idx, n, (char*)out + off, (const char*)in + off, pcm16, vad ? vad + (size_t)f0 * n : nullptr, nf,
                         stream_stride, frame_stride, 0, rs->scratch.get<float>()))
            return -1;
    }
    return resume_caller(rs->st, us, rs->ev_done);
}

int rnnoise_batch_process_native_host(RNNoiseBatch* b, RNNoiseResampler* rs, const int* streams, int n, void* out, const void* in, int pcm16,
                                      float* vad, int n_frames) {
    const int rc = native_check(b, rs, streams, n, out, in, pcm16, n_frames);
    if (rc) return rc < 0 ? -1 : 0;
    ON_DEVICE(rs->device);
    const size_t esz = pcm16 ? sizeof(short) : sizeof(float), slots = (size_t)n * FRAME_SIZE;
    const size_t frame_bytes = slots * (sizeof(float) + esz) + (size_t)n * sizeof(float);
    const int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_frames, kChunkBytes / frame_bytes));
    const int* d_idx;
    if (grow(rs, &rs->scratch, (size_t)chunk * frame_bytes) || upload_idx(rs, streams, n, &d_idx)) return -1;
    float* w48 = rs->scratch.get<float>();
    char* nat = (char*)(w48 + (size_t)chunk * slots);
    float* dvad = (float*)(nat + (size_t)chunk * slots * esz);
    for (int f0 = 0; f0 < n_frames; f0 += chunk) {
        const int nf = std::min(chunk, n_frames - f0);
        const size_t bytes = (size_t)nf * slots * esz, off = (size_t)f0 * slots * esz;
        CK(cudaMemcpyAsync(nat, (const char*)in + off, bytes, cudaMemcpyHostToDevice, rs->st));
        if (native_chunk(b, rs, streams, d_idx, n, nat, nat, pcm16, vad ? dvad : nullptr, nf, FRAME_SIZE, (long)slots, FRAME_SIZE, w48)) return -1;
        CK(cudaMemcpyAsync((char*)out + off, nat, bytes, cudaMemcpyDeviceToHost, rs->st));
        if (vad) CK(cudaMemcpyAsync(vad + (size_t)f0 * n, dvad, (size_t)nf * n * sizeof(float), cudaMemcpyDeviceToHost, rs->st));
    }
    CK(cudaStreamSynchronize(rs->st));
    return 0;
}

}  // extern "C"
