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

// ---- backward (rnnoise_intelligibility_backward_device) -------------------------------------------------------------
// Four kernels, each the adjoint of a forward stage written as a gather, so every output element has one writer that
// sums its terms in a fixed order:
//   stoi_score_bwd_kernel:    one warp per pair, the segments in order: lanes 0..14 a band's STOI correlation backward,
//                             lanes 16..30 then 0..29 the ESTOI row and column normalisations backward; lane b and then
//                             lane 16 + b add the segment's terms into d by[b][sg .. sg + 29] (double).  Also the inverse
//                             of the kept list;
//   stoi_bands_bwd_kernel:    one warp per (pair, STFT frame): out's spectrum recomputed as stoi_bands_kernel does,
//                             G(k) = d by[b] V(k) / by[b], the split's adjoint, the inverse FFT (the forward butterflies
//                             on the conjugate) and one window: d of the overlap-added frame's 256 samples;
//   stoi_ola_bwd_kernel:      one thread per 10 kHz sample: the second window and the sum over the (at most two) kept
//                             frames that contain it and the (at most two) STFT frames that read each;
//   stoi_resample_bwd_kernel: one block per 256 outputs of a row: d out[n] = sum_m d y10[m] h[half + m down - n up],
//                             the row's d y10 span staged in shared memory.
constexpr int kScoreBwdWarps = 4;

// The backward workspace's offsets.
struct BwdLayout {
    size_t off_dby = 0, off_inv = 0, off_du = 0, off_dy10 = 0, total = 0;
    bool ok = false;
};

BwdLayout bwd_layout(const Layout& L, int B) {
    BwdLayout W;
    if (!L.ok) return W;
    size_t a, b, c, d;
    if (!mul_ok((size_t)B * kBands, (size_t)L.maxM * sizeof(double), &a) || !mul_ok((size_t)B, (size_t)L.F * sizeof(int), &b) ||
        !mul_ok((size_t)B * kFrame, (size_t)L.maxM * sizeof(float), &c) || !mul_ok((size_t)B, (size_t)L.n10 * sizeof(float), &d))
        return W;
    if (a > (size_t)1 << 60 || b > (size_t)1 << 60 || c > (size_t)1 << 60 || d > (size_t)1 << 60) return W;
    W.off_dby = 0;
    W.off_inv = round256(a);
    W.off_du = W.off_inv + round256(b);
    W.off_dy10 = W.off_du + round256(c);
    W.total = std::max<size_t>(W.off_dy10 + round256(d), 256);  // never 0, the refusal's value
    W.ok = true;
    return W;
}

struct BwdArgs {
    int B, up, down, half, ntaps, P, span;
    long n, n10, F, maxM;
    const float* y10;    // [B][n10]: the forward's out at 10 kHz
    const int* kept;     // [B][F]
    const float* by;     // [B][15][maxM]: the forward's out bands
    const Tables* tab;
    const float* taps;   // [up][P]
    const RNNoiseIntelligibility* rec;
    const double* gs;    // [B] or null
    const double* ge;    // [B] or null
    double* dby;         // [B][15][maxM]
    int* inv;            // [B][F]
    float* du;           // [B][maxM][256]
    float* dy10;         // [B][n10]
    float* g;            // grad_out
    long gst;            // its row stride
    double c;
};

// Given g = dL/d(v / (||v|| + EPS)) for v centred (d = v - mean v, D = ||d|| + EPS, r = ||d||), dL/dv in place of g:
// dd_i = g_i / D + coef d_i, coef = -(sum g d / D^2) / r (0 at r = 0), then dd - mean dd.  d and g strided by STRIDE.
template <int N, int STRIDE>
__device__ __forceinline__ void normalise_bwd(const double* d, double* g, double r) {
    const double D = r + kEps;
    double s = 0.0;
    for (int i = 0; i < N; i++) s += g[i * STRIDE] * d[i * STRIDE];
    const double coef = r > 0.0 ? -(s / (D * D)) / r : 0.0;
    double m = 0.0;
    for (int i = 0; i < N; i++) {
        g[i * STRIDE] = g[i * STRIDE] / D + coef * d[i * STRIDE];
        m += g[i * STRIDE];
    }
    m /= N;
    for (int i = 0; i < N; i++) g[i * STRIDE] -= m;
}

// centre n values in place, in order; -> the norm of the centred values
template <int N, int STRIDE>
__device__ __forceinline__ double centre(double* v) {
    double m = 0.0;
    for (int i = 0; i < N; i++) m += v[i * STRIDE];
    m /= N;
    double q = 0.0;
    for (int i = 0; i < N; i++) {
        v[i * STRIDE] -= m;
        q += v[i * STRIDE] * v[i * STRIDE];
    }
    return sqrt(q);
}

__global__ void __launch_bounds__(kScoreBwdWarps * 32) stoi_score_bwd_kernel(BwdArgs a) {
    __shared__ double sm[kScoreBwdWarps][3][kBands][kSeg];  // X (x rows, then x hat), A (y rows), G (gradients)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double(*X)[kSeg] = sm[warp][0];
    double(*A)[kSeg] = sm[warp][1];
    double(*G)[kSeg] = sm[warp][2];
    for (long p = (long)blockIdx.x * kScoreBwdWarps + warp; p < a.B; p += (long)gridDim.x * kScoreBwdWarps) {
        const RNNoiseIntelligibility* r = a.rec + p;
        const long S = (long)__ldg(&r->segments), K = (long)__ldg(&r->kept);
        int* inv = a.inv + p * a.F;
        for (long f = lane; f < a.F; f += 32) inv[f] = -1;
        __syncwarp();
        for (long k = lane; k < K; k += 32) inv[__ldg(a.kept + p * a.F + k)] = (int)k;
        double* grow = a.dby + (p * kBands + (lane < kBands ? lane : lane - 16)) * a.maxM;  // lanes b and 16 + b: row b
        if (lane < kBands)
            for (long m = 0; m < a.maxM; m++) grow[m] = 0.0;
        __syncwarp();
        if (S < 1) continue;
        const double gst = a.gs ? __ldg(a.gs + p) / (double)(kBands * S) : 0.0;
        const double gse = a.ge ? __ldg(a.ge + p) / (double)(kSeg * S) : 0.0;
        const float* bx = a.by - (long)a.B * kBands * a.maxM + p * kBands * a.maxM;  // the clean bands precede out's
        const float* by = a.by + p * kBands * a.maxM;
        for (long sg = 0; sg < S; sg++) {
            if (a.gs && lane < kBands) {
                // STOI: band `lane`, frames sg .. sg + 29, the forward's operations, then their adjoint
                const float* rx = bx + lane * a.maxM + sg;
                const float* ry = by + lane * a.maxM + sg;
                // the rows are read again in each pass (from L1) rather than held: 60 doubles of registers spill
                double nx = 0.0, ny = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    const double x = __ldg(rx + i), y = __ldg(ry + i);
                    nx += x * x;
                    ny += y * y;
                }
                const double sy = sqrt(ny), alpha = sqrt(nx) / (sy + kEps);
                double mx = 0.0, my = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    mx += (double)__ldg(rx + i);
                    my += fmin(alpha * (double)__ldg(ry + i), a.c * (double)__ldg(rx + i));
                }
                mx /= kSeg;
                my /= kSeg;
                double sxy = 0.0, sxx = 0.0, syy = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    const double dx = (double)__ldg(rx + i) - mx, dy = fmin(alpha * (double)__ldg(ry + i), a.c * (double)__ldg(rx + i)) - my;
                    sxy += dx * dy;
                    sxx += dx * dx;
                    syy += dy * dy;
                }
                const double ry_ = sqrt(syy), Dy = ry_ + kEps, den = (sqrt(sxx) + kEps) * Dy, term = sxy / den;
                const double dsxy = gst / den, coef = ry_ > 0.0 ? -(gst * term) / (Dy * ry_) : 0.0;
                double* h = G[lane];
                double mh = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    const double dx = (double)__ldg(rx + i) - mx, dy = fmin(alpha * (double)__ldg(ry + i), a.c * (double)__ldg(rx + i)) - my;
                    h[i] = dsxy * dx + coef * dy;
                    mh += h[i];
                }
                mh /= kSeg;
                double dalpha = 0.0;
#pragma unroll
                for (int i = 0; i < kSeg; i++) {
                    h[i] -= mh;  // d y'_i
                    if (alpha * (double)__ldg(ry + i) <= a.c * (double)__ldg(rx + i)) {  // y' = alpha y on the tie
                        dalpha += h[i] * (double)__ldg(ry + i);
                        h[i] = h[i] * alpha;
                    } else {
                        h[i] = 0.0;
                    }
                }
                const double cny = sy > 0.0 ? -(dalpha * alpha) / ((sy + kEps) * sy) : 0.0;
                double* o = grow + sg;
#pragma unroll
                for (int i = 0; i < kSeg; i++) o[i] += h[i] + cny * (double)__ldg(ry + i);
            } else if (a.ge && lane >= 16 && lane < 16 + kBands) {
                const int b = lane - 16;
                for (int i = 0; i < kSeg; i++) {
                    X[b][i] = __ldg(bx + b * a.maxM + sg + i);
                    A[b][i] = __ldg(by + b * a.maxM + sg + i);
                }
                normalise<kSeg, 1>(X[b]);
                normalise<kSeg, 1>(A[b]);
            }
            __syncwarp();
            if (!a.ge) continue;
            if (lane < kSeg) {
                // column `lane`: x hat, then the column normalisation of y backward from d yhat = gse x hat
                normalise<kBands, kSeg>(&X[0][lane]);
                const double rc = centre<kBands, kSeg>(&A[0][lane]);
                for (int b = 0; b < kBands; b++) G[b][lane] = gse * X[b][lane];
                normalise_bwd<kBands, kSeg>(&A[0][lane], &G[0][lane], rc);
            }
            __syncwarp();
            if (lane >= 16 && lane < 16 + kBands) {
                // row b: the row normalisation backward, from the raw row (in A's row, read by no one now), then into
                // d by after the STOI terms
                const int b = lane - 16;
                for (int i = 0; i < kSeg; i++) A[b][i] = __ldg(by + b * a.maxM + sg + i);
                const double rr = centre<kSeg, 1>(A[b]);
                normalise_bwd<kSeg, 1>(A[b], G[b], rr);
                double* o = grow + sg;
                for (int i = 0; i < kSeg; i++) o[i] += G[b][i];
            }
            __syncwarp();  // this segment's shared rows and d by terms are done before the next segment's
        }
    }
}

__global__ void __launch_bounds__(kBandWarps * 32) stoi_bands_bwd_kernel(BwdArgs a) {
    __shared__ float2 sbuf[kBandWarps][kFft / 2];
    __shared__ float2 sg[kBandWarps][kHi - kLo];
    __shared__ double ssc[kBandWarps][16];  // d by / by: in double, as it reaches 1/EPS over a band near 0
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* s = sbuf[warp];
    const long items = (long)a.B * a.maxM;
    for (long it = (long)blockIdx.x * kBandWarps + warp; it < items; it += (long)gridDim.x * kBandWarps) {
        const long p = it / a.maxM, j = it - p * a.maxM;
        const long M = (long)__ldg(&a.rec[p].kept) - 1;
        if (j >= M || __ldg(&a.rec[p].segments) < 1) continue;  // warp-uniform
        const int* kl = a.kept + p * a.F;
        const long kj = __ldg(kl + j), kp = j > 0 ? __ldg(kl + j - 1) : 0, kn = __ldg(kl + j + 1);
        const float* yr = a.y10 + p * a.n10;
        __syncwarp();  // the previous item's reads of s, sg and ssc are done
        // out's frame and spectrum, as stoi_bands_kernel computes them
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const int n = lane + 32 * t;
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int i = 2 * n + e;
                const float w = a.tab->wf[i];
                float u = w * __ldg(yr + kj * kHop + i);
                if (i < kHop) {
                    if (j > 0) u += a.tab->wf[i + kHop] * __ldg(yr + kp * kHop + i + kHop);
                } else {
                    u += a.tab->wf[i - kHop] * __ldg(yr + kn * kHop + i - kHop);
                }
                v[e] = w * u;
            }
            s[__brev(n) >> 24] = make_float2(v[0], v[1]);
            s[__brev(n + 128) >> 24] = make_float2(0.0f, 0.0f);
        }
        if (lane < kBands) {
            const float b = __ldg(a.by + (p * kBands + lane) * a.maxM + j);
            ssc[warp][lane] = b > 0.0f ? a.dby[(p * kBands + lane) * a.maxM + j] / (double)b : 0.0;
        }
        __syncwarp();
        for (int pass = 0; pass < 2; pass++) {
#pragma unroll
            for (int lg = 0; lg < 8; lg++) {
                const int h = 1 << lg;
#pragma unroll
                for (int t = 0; t < 4; t++) {
                    const int bb = lane + 32 * t, pos = bb & (h - 1);
                    const int i0 = ((bb >> lg) << (lg + 1)) + pos, i1 = i0 + h;
                    const float2 u = s[i0], v = cmul(s[i1], a.tab->tw[pos << (8 - lg)]);
                    s[i0] = make_float2(u.x + v.x, u.y + v.y);
                    s[i1] = make_float2(u.x - v.x, u.y - v.y);
                }
                __syncwarp();
            }
            if (pass == 1) break;
            // G(k) = d by[b] / by[b] * V(k), V as stoi_bands_kernel forms it
            for (int k = kLo + lane; k < kHi; k += 32) {
                const float2 u = s[k], c = s[256 - k], w = a.tab->tw[k];
                const float er = 0.5f * (u.x + c.x), ei = 0.5f * (u.y - c.y), orr = 0.5f * (u.y + c.y), oi = -0.5f * (u.x - c.x);
                const float vr = er + (w.x * orr - w.y * oi), vi = ei + (w.x * oi + w.y * orr);
                int b = 0;
                while (k >= kEdges[b + 1]) b++;
                // |V(k)| <= by[b], so the product, formed in double, is at most |d by[b]|: finite in float
                const double sc = ssc[warp][b];
                sg[warp][k - kLo] = make_float2((float)(sc * (double)vr), (float)(sc * (double)vi));
            }
            __syncwarp();
            // dZ(t): the split's adjoint, from V(t) (t as k) and V(256 - t) (t as 256 - k); conjugated, bit-reversed
#pragma unroll
            for (int q = 0; q < 8; q++) {
                const int t = lane + 32 * q;
                float zr = 0.0f, zi = 0.0f;
                if (t >= kLo && t < kHi) {
                    const float2 g = sg[warp][t - kLo], w = a.tab->tw[t];
                    const float dorr = g.x * w.x + g.y * w.y, doi = g.y * w.x - g.x * w.y;
                    zr += 0.5f * g.x - 0.5f * doi;
                    zi += 0.5f * g.y + 0.5f * dorr;
                }
                const int k = 256 - t;
                if (k >= kLo && k < kHi) {
                    const float2 g = sg[warp][k - kLo], w = a.tab->tw[k];
                    const float dorr = g.x * w.x + g.y * w.y, doi = g.y * w.x - g.x * w.y;
                    zr += 0.5f * g.x + 0.5f * doi;
                    zi += -0.5f * g.y + 0.5f * dorr;
                }
                s[__brev(t) >> 24] = make_float2(zr, -zi);
            }
            __syncwarp();
        }
        // z = conj(FFT(conj dZ)); d v[2n] = Re z[n], d v[2n + 1] = Im z[n]; d u = w d v
        float* o = a.du + (p * a.maxM + j) * kFrame;
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const int n = lane + 32 * t;
            const float2 z = s[n];
            o[2 * n] = a.tab->wf[2 * n] * z.x;
            o[2 * n + 1] = a.tab->wf[2 * n + 1] * -z.y;
        }
    }
}

// d y10[m] = sum over the kept frames k holding m (10 kHz frame f, offset o = m - 128 f) of w[o] times the sum of
// d u_j[128 (k - j) + o] over the STFT frames j < M that read it; f ascending, then j ascending.
__global__ void stoi_ola_bwd_kernel(BwdArgs a) {
    const long total = (long)a.B * a.n10;
    for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long p = e / a.n10, m = e - p * a.n10;
        float acc = 0.0f;
        if (__ldg(&a.rec[p].segments) >= 1) {
            const long M = (long)__ldg(&a.rec[p].kept) - 1;
            for (long f = m / kHop - 1; f <= m / kHop; f++) {
                if (f < 0 || f >= a.F) continue;
                const long k = __ldg(a.inv + p * a.F + f);
                if (k < 0) continue;
                const int o = (int)(m - f * kHop), hi = o >= kHop;
                float s = 0.0f;
                for (long j = k - 1 + hi; j <= k + hi; j++)
                    if (j >= 0 && j < M) s += __ldg(a.du + (p * a.maxM + j) * kFrame + (k - j) * kHop + o);
                acc += a.tab->wf[o] * s;
            }
        }
        a.dy10[e] = acc;
    }
}

// floor(a / b) for b > 0
__device__ __forceinline__ long floordiv(long x, long b) { return x >= 0 ? x / b : -((-x + b - 1) / b); }

// d out[n] = sum_m d y10[m] h[half + m down - n up], m ascending; one block per tile of 256 outputs of one row.
__global__ void __launch_bounds__(kTile) stoi_resample_bwd_kernel(BwdArgs a) {
    extern __shared__ float sd[];
    const long tiles = (a.n + kTile - 1) / kTile, total = (long)a.B * tiles;
    for (long blk = blockIdx.x; blk < total; blk += gridDim.x) {
        const long p = blk / tiles, n0 = (blk - p * tiles) * kTile, n = n0 + threadIdx.x;
        const float* d = a.dy10 + p * a.n10;
        float* o = a.g + p * a.gst;
        const bool live = __ldg(&a.rec[p].segments) >= 1;  // block-uniform
        if (a.up == 1 && a.down == 1) {
            if (n < a.n) o[n] = live ? d[n] : 0.0f;
            continue;
        }
        // the m whose taps reach the tile: ceil((n0 up - half) / down) ..
        const long lo = -floordiv(-(n0 * a.up - a.half), a.down);
        __syncthreads();  // the previous tile's reads of sd are done
        for (int i = threadIdx.x; i < a.span; i += kTile) {
            const long m = lo + i;
            sd[i] = (live && m >= 0 && m < a.n10) ? d[m] : 0.0f;
        }
        __syncthreads();
        if (n < a.n) {
            long m = -floordiv(-(n * a.up - a.half), a.down);  // the first m with half + m down - n up >= 0
            int k = (int)(a.half + m * a.down - n * a.up);
            if (m < 0) {
                k += (int)(-m * a.down);
                m = 0;
            }
            int ph = k % a.up, jj = k / a.up;
            const int dph = a.down % a.up, dj = a.down / a.up;
            float acc = 0.0f;
            for (; k < a.ntaps && m < a.n10; k += a.down, m++) {
                acc = fmaf(__ldg(a.taps + ph * a.P + jj), sd[m - lo], acc);
                ph += dph;
                jj += dj;
                if (ph >= a.up) {
                    ph -= a.up;
                    jj++;
                }
            }
            o[n] = acc;
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

size_t rnnoise_intelligibility_backward_workspace_bytes(int n_pairs, long n_samples, int rate) {
    const BwdLayout W = bwd_layout(layout(n_pairs, n_samples, rate), n_pairs);
    return W.ok ? W.total : 0;
}

int rnnoise_intelligibility_backward_device(int n_pairs, long n_samples, int rate, const RNNoiseIntelligibility* result,
                                            const void* fwd_workspace, size_t fwd_workspace_bytes, const double* grad_stoi,
                                            const double* grad_estoi, float* grad_out, long grad_stride, void* workspace,
                                            size_t workspace_bytes, int device, void* cuda_stream) {
    if (!result || !fwd_workspace || !grad_out || !workspace) return fail("null argument");
    if (n_pairs <= 0) return fail("n_pairs must be positive");
    if (n_samples < 0) return fail("negative n_samples");
    if (!valid_rate(rate)) return fail(rate_error(rate));
    if (grad_stride < n_samples) return fail("grad_stride is less than n_samples: rows overlap");
    if (reinterpret_cast<uintptr_t>(grad_out) & 3) return fail("grad_out must be float-aligned");
    if ((reinterpret_cast<uintptr_t>(result) & 7) || (reinterpret_cast<uintptr_t>(grad_stoi) & 7) || (reinterpret_cast<uintptr_t>(grad_estoi) & 7))
        return fail("result, grad_stoi and grad_estoi must be 8-byte aligned");
    if ((reinterpret_cast<uintptr_t>(fwd_workspace) & 255) || (reinterpret_cast<uintptr_t>(workspace) & 255))
        return fail("fwd_workspace and workspace must be 256-byte aligned");
    const Layout L = layout(n_pairs, n_samples, rate);
    const BwdLayout W = bwd_layout(L, n_pairs);
    if (!L.ok || !W.ok) return fail("a workspace for " + std::to_string(n_pairs) + " pairs of " + std::to_string(n_samples) + " samples is too large");
    if (fwd_workspace_bytes < L.total)
        return fail("forward workspace of " + std::to_string(fwd_workspace_bytes) + " bytes; " + std::to_string(L.total) + " needed");
    if (workspace_bytes < W.total)
        return fail("workspace of " + std::to_string(workspace_bytes) + " bytes; " + std::to_string(W.total) + " needed");
    int dev = 0;
    if (open_device(device, &dev)) return -1;
    ON_DEVICE(dev);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    const unsigned char* fw = static_cast<const unsigned char*>(fwd_workspace);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    BwdArgs a{};
    a.B = n_pairs;
    a.up = L.up;
    a.down = L.down;
    a.half = L.half;
    a.ntaps = L.ntaps;
    a.P = L.P;
    a.span = (int)(((long)(kTile - 1) * L.up) / L.down + L.ntaps / L.down + 3);
    a.n = n_samples;
    a.n10 = L.n10;
    a.F = L.F;
    a.maxM = L.maxM;
    a.y10 = reinterpret_cast<const float*>(fw + L.off_x10) + (size_t)n_pairs * L.n10;
    a.kept = reinterpret_cast<const int*>(fw + L.off_kept);
    a.by = reinterpret_cast<const float*>(fw + L.off_bands) + (size_t)n_pairs * kBands * L.maxM;
    a.tab = reinterpret_cast<const Tables*>(fw + L.off_tab);
    a.taps = reinterpret_cast<const float*>(fw + L.off_tab + sizeof(Tables));
    a.rec = result;
    a.gs = grad_stoi;
    a.ge = grad_estoi;
    a.dby = reinterpret_cast<double*>(ws + W.off_dby);
    a.inv = reinterpret_cast<int*>(ws + W.off_inv);
    a.du = reinterpret_cast<float*>(ws + W.off_du);
    a.dy10 = reinterpret_cast<float*>(ws + W.off_dy10);
    a.g = grad_out;
    a.gst = grad_stride;
    a.c = 1.0 + std::pow(10.0, 15.0 / 20.0);
    stoi_score_bwd_kernel<<<grid_of(n_pairs, kScoreBwdWarps), kScoreBwdWarps * 32, 0, st>>>(a);
    CK(cudaGetLastError());
    stoi_bands_bwd_kernel<<<grid_of((long)n_pairs * L.maxM, kBandWarps), kBandWarps * 32, 0, st>>>(a);
    CK(cudaGetLastError());
    stoi_ola_bwd_kernel<<<grid_of((long)n_pairs * L.n10, 256), 256, 0, st>>>(a);
    CK(cudaGetLastError());
    const long tiles = (n_samples + kTile - 1) / kTile;
    const size_t smem = (L.up == 1 && L.down == 1) ? 0 : (size_t)a.span * sizeof(float);
    stoi_resample_bwd_kernel<<<grid_of((long)n_pairs * std::max(tiles, 1L), 1), kTile, smem, st>>>(a);
    CK(cudaGetLastError());
    count_launches(4);
    if (!st) CK(cudaStreamSynchronize(st));
    return 0;
}

}  // extern "C"
