// intelligibility.cu -- STOI and ESTOI of clips on the GPU (rnnoise_intelligibility_*, DESIGN.md §7q).
//
// Four kernels, each reading the previous one's output from the caller's workspace (the regions of include/rnnoise.h):
//   stoi_resample_kernel: out and clean to 10 kHz, one block per 256 outputs of a row, the row's input span staged in
//                         shared memory and the taps laid out polyphase ([phase][tap], zero-padded), as
//                         resample_down_kernel reads them;
//   stoi_mask_kernel:     one warp per pair: the clean frames' energies in double (twice: once for the maximum, once
//                         for the decisions), the strict 40 dB rule, and the kept list by ballot prefix sums;
//   stoi_bands_kernel:    one warp per (pair, STFT frame): the overlap-added frame rebuilt from kept frames j - 1..j + 1,
//                         windowed, each signal's 512-point real DFT as a radix-2 256-point complex FFT in shared
//                         memory and a split, and the 15 band magnitudes of both;
//   stoi_score_kernel:    one warp per pair, the segments in order: lanes 0..14 a band's STOI correlation, lanes 16..30 a
//                         band's ESTOI row normalisation, then lanes 0..29 a frame's column normalisation.
// The unit is compiled without FMA contraction (build.py), so the double tail's operations are the ones written: the
// float64 restatement in tests/stoi_ref.py performs them in the same order and gets the same bits from the same bands.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <numeric>
#include <string>
#include <vector>

#include "../../include/rnnoise.h"
#include "abi.hpp"

namespace nnb {
bool valid_rate(int rate);                        // resample_stream.cu
std::string rate_error(int rate);                 // resample_stream.cu
std::vector<double> firwin_kaiser(int n, int M);  // resample_stream.cu
}  // namespace nnb

using namespace nnb;

namespace {

static_assert(sizeof(RNNoiseIntelligibility) == 32, "record layout");

constexpr int kRate = 10000;
constexpr int kFrame = 256, kHop = 128, kFft = 512, kBands = 15, kSeg = 30;
constexpr int kLo = 7, kHi = 219;  // the bins the bands cover
constexpr double kEps = 2.220446049250313e-16;  // 2^-52
constexpr int kTile = 256;                        // outputs per resample block
constexpr int kMaskWarps = 4, kBandWarps = 8, kScoreWarps = 4;
__constant__ int kEdges[kBands + 1] = {7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219};

struct Tables {
    float wf[kFrame];    // the window in float (STFT)
    double wd[kFrame];   // the window in double (frame energies)
    float2 tw[kFft / 2]; // exp(-2 pi i t / 512)
    // then the polyphase taps: [up][P] floats
};

// The sizes and workspace offsets of one call.
struct Layout {
    int up = 1, down = 1, half = 0, ntaps = 1, P = 1;
    long n10 = 0, F = 0, maxM = 0;
    size_t off_x10 = 0, off_kept = 0, off_bands = 0, off_tab = 0, total = 0;
    bool ok = false;
};

size_t round256(size_t v) { return (v + 255) & ~size_t(255); }

// false on an overflow of size_t or of the kernels' int counts
bool mul_ok(size_t a, size_t b, size_t* r) {
    if (a != 0 && b > std::numeric_limits<size_t>::max() / a) return false;
    *r = a * b;
    return true;
}

Layout layout(int B, long n, int rate) {
    Layout L;
    if (B <= 0 || n < 0 || !valid_rate(rate)) return L;
    const int g = std::gcd(rate, kRate);
    L.up = kRate / g;
    L.down = rate / g;
    if (L.up != 1 || L.down != 1) {
        L.half = 10 * std::max(L.up, L.down);
        L.ntaps = 2 * L.half + 1;
        L.P = (L.ntaps + L.up - 1) / L.up;
    }
    if (n > std::numeric_limits<long>::max() / L.up) return L;
    L.n10 = (n * L.up + L.down - 1) / L.down;
    L.F = L.n10 >= kFrame ? (L.n10 - kFrame) / kHop + 1 : 0;
    if (L.F > std::numeric_limits<int>::max()) return L;
    L.maxM = std::max(L.F - 1, 0L);
    size_t a, b, c;
    if (!mul_ok((size_t)2 * B, (size_t)L.n10 * sizeof(float), &a) || !mul_ok((size_t)B, (size_t)L.F * sizeof(int), &b) ||
        !mul_ok((size_t)2 * B * kBands, (size_t)L.maxM * sizeof(float), &c))
        return L;
    const size_t tab = sizeof(Tables) + (size_t)L.up * L.P * sizeof(float);
    if (a > (size_t)1 << 60 || b > (size_t)1 << 60 || c > (size_t)1 << 60) return L;
    L.off_x10 = 0;
    L.off_kept = round256(a);
    L.off_bands = L.off_kept + round256(b);
    L.off_tab = L.off_bands + round256(c);
    L.total = L.off_tab + round256(tab);
    L.ok = true;
    return L;
}

struct StoiArgs {
    const float* y;  // out
    const float* x;  // clean
    long ss, n;
    int B, up, down, half, P, span;
    long n10, F, maxM;
    float* x10;      // [2][B][n10]: clean, then out
    int* kept;       // [B][F]
    float* bands;    // [2][B][15][maxM]
    const Tables* tab;
    const float* taps;  // [up][P]
    RNNoiseIntelligibility* rec;
    double c;           // 1 + 10^(15/20)
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// x10[m] = sum_j taps[p][j] x[n0 - j], q = half + m down = n0 up + p; one block per tile of 256 outputs of one row.
__global__ void __launch_bounds__(kTile) stoi_resample_kernel(StoiArgs a) {
    extern __shared__ float sx[];
    const long tiles = (a.n10 + kTile - 1) / kTile, total = 2L * a.B * tiles;
    for (long blk = blockIdx.x; blk < total; blk += gridDim.x) {
        const long row = blk / tiles, m0 = (blk - row * tiles) * kTile;  // row: signal * B + pair
        const int sig = (int)(row / a.B), p = (int)(row - (long)sig * a.B);
        const float* in = (sig == 0 ? a.x : a.y) + (long)p * a.ss;
        float* o = a.x10 + row * a.n10;
        const long m = m0 + threadIdx.x;
        if (a.up == 1 && a.down == 1) {
            if (m < a.n10) o[m] = __ldg(in + m);
            continue;
        }
        const long lo = ((long)a.half + m0 * a.down) / a.up - (a.P - 1);
        __syncthreads();  // the previous tile's reads of sx are done
        for (int i = threadIdx.x; i < a.span; i += kTile) {
            const long k = lo + i;
            sx[i] = (k >= 0 && k < a.n) ? __ldg(in + k) : 0.0f;
        }
        __syncthreads();
        if (m < a.n10) {
            const long q = (long)a.half + m * a.down, n0 = q / a.up;
            const int ph = (int)(q - n0 * a.up);
            const float* h = a.taps + (long)ph * a.P;
            const float* s = sx + (n0 - lo);
            float acc = 0.0f;
            for (int j = 0; j < a.P; j++) acc = fmaf(__ldg(h + j), s[-j], acc);
            o[m] = acc;
        }
    }
}

// ||w x10 frame||^2 of the frame at r, in double, on every lane
__device__ __forceinline__ double frame_energy(const float* __restrict__ r, const double* __restrict__ wd, int lane) {
    double e = 0.0;
#pragma unroll
    for (int t = 0; t < kFrame / 32; t++) {
        const int i = lane + 32 * t;
        const double v = wd[i] * (double)__ldg(r + i);
        e += v * v;
    }
    return warp_sum(e);
}

__device__ __forceinline__ double frame_db(const float* r, const double* wd, int lane) {
    return 20.0 * log10(sqrt(frame_energy(r, wd, lane)) + kEps);
}

__global__ void __launch_bounds__(kMaskWarps * 32) stoi_mask_kernel(StoiArgs a) {
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMaskWarps + (threadIdx.x >> 5); p < a.B; p += (long)gridDim.x * kMaskWarps) {
        const float* xr = a.x10 + p * a.n10;
        int* kl = a.kept + p * a.F;
        double top = -INFINITY;
        for (long f = 0; f < a.F; f++) top = fmax(top, frame_db(xr + f * kHop, a.tab->wd, lane));
        const double thr = top - 40.0;
        long K = 0;
        for (long f0 = 0; f0 < a.F; f0 += 32) {
            bool keep = false;
            for (int l = 0; l < 32 && f0 + l < a.F; l++) {
                const bool k = frame_db(xr + (f0 + l) * kHop, a.tab->wd, lane) > thr;
                if (lane == l) keep = k;
            }
            const unsigned bal = __ballot_sync(0xffffffffu, keep);
            if (keep) kl[K + __popc(bal & ((1u << lane) - 1u))] = (int)(f0 + lane);
            K += __popc(bal);
        }
        for (long k = K + lane; k < a.F; k += 32) kl[k] = -1;
        if (lane == 0) {
            RNNoiseIntelligibility* r = a.rec + p;
            r->frames = (int)a.F;
            r->kept = (int)K;
            r->segments = (int)(K > kSeg ? K - kSeg : 0);
            r->reserved = 0;
        }
    }
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

__global__ void __launch_bounds__(kBandWarps * 32) stoi_bands_kernel(StoiArgs a) {
    __shared__ float2 sbuf[kBandWarps][kFft];  // two 256-point transforms: clean, out
    __shared__ float spow[kBandWarps][2][kHi - kLo];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* s = sbuf[warp];
    const long items = (long)a.B * a.maxM;
    for (long it = (long)blockIdx.x * kBandWarps + warp; it < items; it += (long)gridDim.x * kBandWarps) {
        const long p = it / a.maxM, j = it - p * a.maxM;
        const long M = (long)__ldg(&a.rec[p].kept) - 1;
        if (j >= M) continue;  // warp-uniform
        const int* kl = a.kept + p * a.F;
        const long kj = __ldg(kl + j), kp = j > 0 ? __ldg(kl + j - 1) : 0, kn = __ldg(kl + j + 1);
        const float* xr = a.x10 + p * a.n10;
        const float* yr = a.x10 + ((long)a.B + p) * a.n10;
        __syncwarp();  // the previous item's reads of s are done
        // Each signal's 512-point real DFT is a 256-point complex FFT of z[n] = (v[2n], v[2n + 1]) (v: the windowed
        // frame, zero past 256, so z[n] = 0 for n >= 128), in s[sig * 256 ..], loaded in bit-reversed order.  Each
        // signal has a transform of its own, so scaling one by a power of two scales its bands exactly.
#pragma unroll
        for (int t = 0; t < 8; t++) {
            const int b = lane + 32 * t, sig = b >> 7, n = b & 127;
            const float* r = sig ? yr : xr;
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                // sample 128 j + i of the overlap-added signal: kept frame j at offset i plus its neighbour's overlap
                const int i = 2 * n + e;
                const float w = a.tab->wf[i];
                float u = w * __ldg(r + kj * kHop + i);
                if (i < kHop) {
                    if (j > 0) u += a.tab->wf[i + kHop] * __ldg(r + kp * kHop + i + kHop);
                } else {
                    u += a.tab->wf[i - kHop] * __ldg(r + kn * kHop + i - kHop);
                }
                v[e] = w * u;
            }
            s[sig * 256 + (__brev(n) >> 24)] = make_float2(v[0], v[1]);
            s[sig * 256 + (__brev(n + 128) >> 24)] = make_float2(0.0f, 0.0f);
        }
        __syncwarp();
#pragma unroll
        for (int lg = 0; lg < 8; lg++) {
            const int h = 1 << lg;
#pragma unroll
            for (int t = 0; t < 8; t++) {
                const int b = lane + 32 * t, sig = b >> 7, bb = b & 127, pos = bb & (h - 1);
                const int i0 = sig * 256 + ((bb >> lg) << (lg + 1)) + pos, i1 = i0 + h;
                const float2 u = s[i0], v = cmul(s[i1], a.tab->tw[pos << (8 - lg)]);
                s[i0] = make_float2(u.x + v.x, u.y + v.y);
                s[i1] = make_float2(u.x - v.x, u.y - v.y);
            }
            __syncwarp();
        }
        // V(k) = E(k) + W^k O(k), E = (Z(k) + conj Z(256 - k)) / 2, O = (Z(k) - conj Z(256 - k)) / 2i, W = e^(-2 pi i / 512)
        for (int q = lane; q < 2 * (kHi - kLo); q += 32) {
            const int sig = q >= kHi - kLo, k = kLo + q - sig * (kHi - kLo);
            const float2 u = s[sig * 256 + k], c = s[sig * 256 + 256 - k], w = a.tab->tw[k];
            const float er = 0.5f * (u.x + c.x), ei = 0.5f * (u.y - c.y), orr = 0.5f * (u.y + c.y), oi = -0.5f * (u.x - c.x);
            const float vr = er + (w.x * orr - w.y * oi), vi = ei + (w.x * oi + w.y * orr);
            spow[warp][sig][k - kLo] = vr * vr + vi * vi;
        }
        __syncwarp();
        if ((lane & 15) < kBands) {
            const int sig = lane >> 4, b = lane & 15;
            float e = 0.0f;
            for (int k = kEdges[b]; k < kEdges[b + 1]; k++) e += spow[warp][sig][k - kLo];
            a.bands[(((long)sig * a.B + p) * kBands + b) * a.maxM + j] = sqrtf(e);
        }
    }
}

// mean, then (v - mean) / (||v - mean|| + EPS) of n values in place, in order
template <int N, int STRIDE>
__device__ __forceinline__ void normalise(double* v) {
    double m = 0.0;
    for (int i = 0; i < N; i++) m += v[i * STRIDE];
    m /= N;
    double q = 0.0;
    for (int i = 0; i < N; i++) {
        v[i * STRIDE] -= m;
        q += v[i * STRIDE] * v[i * STRIDE];
    }
    const double d = sqrt(q) + kEps;
    for (int i = 0; i < N; i++) v[i * STRIDE] /= d;
}

__global__ void __launch_bounds__(kScoreWarps * 32) stoi_score_kernel(StoiArgs a) {
    __shared__ double sm[kScoreWarps][2][kBands][kSeg];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (long p = (long)blockIdx.x * kScoreWarps + warp; p < a.B; p += (long)gridDim.x * kScoreWarps) {
        const long S = (long)__ldg(&a.rec[p].segments);
        double stoi = 0.0, estoi = 0.0;
        const float* bx = a.bands + ((long)p * kBands) * a.maxM;
        const float* by = a.bands + (((long)a.B + p) * kBands) * a.maxM;
        for (long sg = 0; sg < S; sg++) {
            double term = 0.0;
            if (lane < kBands) {
                // STOI: band `lane`, frames sg .. sg + 29
                const float* rx = bx + lane * a.maxM + sg;
                const float* ry = by + lane * a.maxM + sg;
                double x[kSeg], y[kSeg], nx = 0.0, ny = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    x[i] = __ldg(rx + i);
                    y[i] = __ldg(ry + i);
                    nx += x[i] * x[i];
                    ny += y[i] * y[i];
                }
                const double alpha = sqrt(nx) / (sqrt(ny) + kEps);
                double mx = 0.0, my = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    y[i] = fmin(alpha * y[i], a.c * x[i]);
                    mx += x[i];
                    my += y[i];
                }
                mx /= kSeg;
                my /= kSeg;
                double sxy = 0.0, sxx = 0.0, syy = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    const double dx = x[i] - mx, dy = y[i] - my;
                    sxy += dx * dy;
                    sxx += dx * dx;
                    syy += dy * dy;
                }
                term = sxy / ((sqrt(sxx) + kEps) * (sqrt(syy) + kEps));
            } else if (lane >= 16 && lane < 16 + kBands) {
                // ESTOI: band lane - 16's rows, centred and normalised
                const int b = lane - 16;
                double* vx = sm[warp][0][b];
                double* vy = sm[warp][1][b];
                for (int i = 0; i < kSeg; i++) {
                    vx[i] = __ldg(bx + b * a.maxM + sg + i);
                    vy[i] = __ldg(by + b * a.maxM + sg + i);
                }
                normalise<kSeg, 1>(vx);
                normalise<kSeg, 1>(vy);
            }
            __syncwarp();
            double prod = 0.0;
            if (lane < kSeg) {
                double* cx = &sm[warp][0][0][lane];
                double* cy = &sm[warp][1][0][lane];
                normalise<kBands, kSeg>(cx);
                normalise<kBands, kSeg>(cy);
                for (int b = 0; b < kBands; b++) prod += cx[b * kSeg] * cy[b * kSeg];
            }
            __syncwarp();  // this segment's columns are read before the next segment's rows are written
            stoi += warp_sum(term);
            estoi += warp_sum(prod);
        }
        if (lane == 0) {
            RNNoiseIntelligibility* r = a.rec + p;
            r->stoi = S > 0 ? stoi / (double)(kBands * S) : NAN;
            r->estoi = S > 0 ? estoi / (double)(kSeg * S) : NAN;
        }
    }
}

// the host image of the tables region: Tables, then the polyphase taps
std::vector<unsigned char> host_tables(const Layout& L) {
    std::vector<unsigned char> img(sizeof(Tables) + (size_t)L.up * L.P * sizeof(float), 0);
    Tables* t = reinterpret_cast<Tables*>(img.data());
    const double pi = 3.14159265358979323846264338327950288;
    for (int i = 0; i < kFrame; i++) {
        t->wd[i] = 0.5 - 0.5 * std::cos(2.0 * pi * (i + 1) / (kFrame + 1));
        t->wf[i] = (float)t->wd[i];
    }
    for (int i = 0; i < kFft / 2; i++)
        t->tw[i] = make_float2((float)std::cos(2.0 * pi * i / kFft), (float)-std::sin(2.0 * pi * i / kFft));
    float* taps = reinterpret_cast<float*>(img.data() + sizeof(Tables));
    if (L.up == 1 && L.down == 1) {
        taps[0] = 1.0f;
    } else {
        const std::vector<double> h = firwin_kaiser(L.ntaps, std::max(L.up, L.down));
        for (int k = 0; k < L.ntaps; k++) taps[(size_t)(k % L.up) * L.P + k / L.up] = (float)(h[(size_t)k] * L.up);
    }
    return img;
}

unsigned grid_of(long items, int per_block) {
    return (unsigned)std::max<long>(1, std::min<long>((items + per_block - 1) / per_block, 1L << 20));
}

}  // namespace

extern "C" {

size_t rnnoise_intelligibility_workspace_bytes(int n_pairs, long n_samples, int rate) {
    const Layout L = layout(n_pairs, n_samples, rate);
    return L.ok ? L.total : 0;
}

int rnnoise_intelligibility_device(const float* out, const float* clean, int n_pairs, long n_samples, long stream_stride, int rate,
                                   RNNoiseIntelligibility* result, void* workspace, size_t workspace_bytes, int device,
                                   void* cuda_stream) {
    if (!out || !clean || !result || !workspace) return fail("null argument");
    if (n_pairs <= 0) return fail("n_pairs must be positive");
    if (n_samples < 0) return fail("negative n_samples");
    if (!valid_rate(rate)) return fail(rate_error(rate));
    if (stream_stride < n_samples) return fail("stream_stride is less than n_samples: rows overlap");
    if ((reinterpret_cast<uintptr_t>(out) & 3) || (reinterpret_cast<uintptr_t>(clean) & 3)) return fail("out and clean must be float-aligned");
    if (reinterpret_cast<uintptr_t>(result) & 7) return fail("result must be 8-byte aligned");
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return fail("workspace must be 256-byte aligned");
    const Layout L = layout(n_pairs, n_samples, rate);
    if (!L.ok) return fail("a workspace for " + std::to_string(n_pairs) + " pairs of " + std::to_string(n_samples) + " samples is too large");
    if (workspace_bytes < L.total)
        return fail("workspace of " + std::to_string(workspace_bytes) + " bytes; " + std::to_string(L.total) + " needed");
    int dev = 0;
    if (open_device(device, &dev)) return -1;
    ON_DEVICE(dev);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    const std::vector<unsigned char> img = host_tables(L);
    // a copy from pageable memory returns once the source has been staged, so img may go when the call returns
    CK(cudaMemcpyAsync(ws + L.off_tab, img.data(), img.size(), cudaMemcpyHostToDevice, st));
    StoiArgs a{};
    a.y = out;
    a.x = clean;
    a.ss = stream_stride;
    a.n = n_samples;
    a.B = n_pairs;
    a.up = L.up;
    a.down = L.down;
    a.half = L.half;
    a.P = L.P;
    a.span = (int)(((long)(kTile - 1) * L.down) / L.up + L.P + 2);
    a.n10 = L.n10;
    a.F = L.F;
    a.maxM = L.maxM;
    a.x10 = reinterpret_cast<float*>(ws + L.off_x10);
    a.kept = reinterpret_cast<int*>(ws + L.off_kept);
    a.bands = reinterpret_cast<float*>(ws + L.off_bands);
    a.tab = reinterpret_cast<const Tables*>(ws + L.off_tab);
    a.taps = reinterpret_cast<const float*>(ws + L.off_tab + sizeof(Tables));
    a.rec = result;
    a.c = 1.0 + std::pow(10.0, 15.0 / 20.0);
    const long tiles = (L.n10 + kTile - 1) / kTile;
    const size_t smem = (L.up == 1 && L.down == 1) ? 0 : (size_t)a.span * sizeof(float);
    stoi_resample_kernel<<<grid_of(2L * n_pairs * tiles, 1), kTile, smem, st>>>(a);
    CK(cudaGetLastError());
    stoi_mask_kernel<<<grid_of(n_pairs, kMaskWarps), kMaskWarps * 32, 0, st>>>(a);
    CK(cudaGetLastError());
    stoi_bands_kernel<<<grid_of((long)n_pairs * L.maxM, kBandWarps), kBandWarps * 32, 0, st>>>(a);
    CK(cudaGetLastError());
    stoi_score_kernel<<<grid_of(n_pairs, kScoreWarps), kScoreWarps * 32, 0, st>>>(a);
    CK(cudaGetLastError());
    count_launches(4);
    if (!st) CK(cudaStreamSynchronize(st));
    return 0;
}

}  // extern "C"
