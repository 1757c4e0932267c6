// synth_grad.cu -- training through synthesis (DESIGN.md 7i): the synthesis contexts a saving split frame stores, and
// the backward of a window of saved frames, dL/d(raw band gains) from dL/d(output samples).
//
//   synth_context_kernel      one thread per 8 bytes of a record: copies what K5 of the frame is about to read (X, P,
//                             ex, ep, exp, lastg, the caller's gains, the silence flag) into the caller's record.  It runs
//                             on stage 4's stream just before K5, so lastg is the value before the frame.
//   grad_tables_kernel        the window, twiddles and band tables the backward reads, computed into the caller's
//                             workspace on every call (the backward belongs to no handle and allocates nothing).
//   synthesis_grad_warp_kernel one warp per (stream, frame), all frames of a window at once: recomputes K5's intermediates
//                             from the record, forms 0.5 window * (grad_out[t] | grad_out[t+1]) and applies the adjoint of
//                             the unnormalised inverse real FFT (a forward 960-point real FFT on fft480.cuh's 32 x 15 warp
//                             decomposition, bins 1..479 counted twice), then the adjoints of the gain interpolation, the
//                             renormalisation and the pitch filter.  Writes dL/dgg (through this frame's output) and the
//                             pitch filter's dL/dg per band.
//   synthesis_grad_scan_kernel one thread per (stream, band), frames in reverse: the gain floor gg = max(g, 0.6 lastg)
//                             routes dL/dgg to g, or (x 0.6) to the previous frame's gg; silent frames pass it through.
// Every sum runs in a fixed order and nothing is accumulated atomically: the same inputs give the same bits.
#include "../../include/rnnoise.h"
#include "abi.hpp"
#include "common.cuh"
#include "fft480.cuh"

namespace nnb {

namespace {

static_assert(CX_FLOATS * 4 == RNNOISE_SYNTH_CONTEXT_BYTES, "record layout");
constexpr int CX_UNITS = RNNOISE_SYNTH_CONTEXT_BYTES / 8;  // float2 units of a record

__global__ void synth_context_kernel(BatchBuffers bb, const float* __restrict__ gains, long gain_stride, unsigned char* __restrict__ ctx,
                                     long ctx_stride) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int s = (int)(i / CX_UNITS), u = (int)(i % CX_UNITS);
    if (s >= bb.n_streams) return;
    float2 v = make_float2(0.f, 0.f);
    if (u < CX_P / 2) {
        if (u < FREQ_SIZE) v = bb.X[(size_t)s * FREQ_SIZE + u];
    } else if (u < CX_EX / 2) {
        v = bb.P[(size_t)s * NB_BINS_BANDED + u - CX_P / 2];
    } else if (u < CX_SIL / 2) {
        const int sec = (u - CX_EX / 2) / (CX_BAND_SECTION / 2), j = 2 * ((u - CX_EX / 2) % (CX_BAND_SECTION / 2));
        if (j < NB_BANDS) {
            const size_t o = (size_t)s * NB_BANDS + j;
            switch (sec) {
                case 0: v = make_float2(bb.ex[o], bb.ex[o + 1]); break;
                case 1: v = make_float2(bb.ep[o], bb.ep[o + 1]); break;
                case 2: v = make_float2(bb.exp[o], bb.exp[o + 1]); break;
                case 3: v = make_float2(bb.lastg[o], bb.lastg[o + 1]); break;
                default: v = make_float2(gains[(size_t)s * gain_stride + j], gains[(size_t)s * gain_stride + j + 1]); break;
            }
        }
    } else if (u == CX_SIL / 2) {
        v.x = __int_as_float(bb.silence[s]);
    }
    reinterpret_cast<float2*>(ctx + (size_t)s * ctx_stride * RNNOISE_SYNTH_CONTEXT_BYTES)[u] = v;
}

// ---- tables of the backward ----
struct GradTables {
    float window[WINDOW_SIZE];
    float2 tw960[FREQ_SIZE + 3];  // exp(-2 pi i k / 960)
    float2 twl[15][32];           // exp(-2 pi i b k1 / 480)
    float band_frac[NB_BINS_BANDED];
    int band_of[NB_BINS_BANDED];
    // the band segments dealt to the 32 lanes as in build_tables (host.cu): lane l walks bins b0 .. b0 + n of segment seg
    int bp_seg[32], bp_b0[32], bp_n[32], bp_off[32];
    float bp_inv[32];
};
constexpr size_t TABLE_BYTES = (sizeof(GradTables) + 255) & ~(size_t)255;

__constant__ int c_eband[NB_BANDS] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 34, 40, 48, 60, 78, 100};

// The same values as build_tables (double, rounded once to f32).
__global__ void grad_tables_kernel(GradTables* t) {
    const double pi = 3.14159265358979323846264338327950288;
    for (int i = threadIdx.x; i < FRAME_SIZE; i += blockDim.x) {
        const double s = sin(0.5 * pi * ((double)i + 0.5) / (double)FRAME_SIZE);
        const float w = (float)sin(0.5 * pi * s * s);
        t->window[i] = w;
        t->window[WINDOW_SIZE - 1 - i] = w;
    }
    for (int k = threadIdx.x; k < FREQ_SIZE + 3; k += blockDim.x)
        t->tw960[k] = k < FREQ_SIZE ? make_float2((float)cos(-2.0 * pi * (double)k / 960.0), (float)sin(-2.0 * pi * (double)k / 960.0))
                                    : make_float2(0.f, 0.f);
    for (int i = threadIdx.x; i < 15 * 32; i += blockDim.x) {
        const int k1 = i / 32, b = i % 32;
        const double ang = -2.0 * pi * (double)(b * k1) / 480.0;
        t->twl[k1][b] = make_float2((float)cos(ang), (float)sin(ang));
    }
    for (int k = threadIdx.x; k < NB_BINS_BANDED; k += blockDim.x) {
        int i = 0;
        while ((c_eband[i + 1] << 2) <= k) i++;
        const int size = (c_eband[i + 1] - c_eband[i]) << 2;
        t->band_frac[k] = (float)(k - (c_eband[i] << 2)) / (float)size;
        t->band_of[k] = i;
    }
    if (threadIdx.x == 0) {
        int l = 0;
        for (int sg = 0; sg < NB_BANDS - 1; sg++) {
            const int first = c_eband[sg] << 2, size = (c_eband[sg + 1] << 2) - first;
            const int nl = size <= 16 ? 1 : (size <= 32 ? 2 : (size <= 48 ? 3 : 4));
            for (int q = 0; q < nl; q++, l++) {
                const int lo = first + size * q / nl, hi = first + size * (q + 1) / nl;
                t->bp_seg[l] = sg;
                t->bp_b0[l] = lo;
                t->bp_n[l] = hi - lo;
                t->bp_off[l] = lo - first;
                t->bp_inv[l] = 1.0f / (float)size;
            }
        }
    }
}

constexpr int GW = 4;                  // warps per block
constexpr int RS = 33;                 // transpose row stride in float2 (as spectral_warp.cu)
constexpr int FBUF = 15 * RS;          // the FFT's transpose area, then the band reductions' inputs (<= 2 x 400 floats)
constexpr int S_R = 0, S_GG = 32, S_S2 = 64, S_DNE = 96, S_SEG = 128;  // floats in the per-warp scratch
constexpr int WSC = S_SEG + (NB_BANDS - 1) * 4;
static_assert(2 * NB_BINS_BANDED <= 2 * FBUF, "two reduction inputs fit the transpose area");

// Band reductions of NQ per-bin values v[q * 400 + k], k < 400: the (1 - frac) parts go to band seg, the frac parts to
// band seg + 1 (no doubling of the first and last band).  Lane b < 22 returns band b in o[].  The lanes of one segment
// are combined in a fixed order.
template <int NQ>
__device__ __forceinline__ void band_reduce(const float* __restrict__ v, const GradTables* __restrict__ tb, float* __restrict__ sc, int lane,
                                            float (&o)[NQ]) {
    const int sg = tb->bp_seg[lane], b0 = tb->bp_b0[lane], n = tb->bp_n[lane], off0 = tb->bp_off[lane];
    const float inv = tb->bp_inv[lane];
    float a[NQ], b[NQ];
#pragma unroll
    for (int q = 0; q < NQ; q++) a[q] = b[q] = 0.0f;
#pragma unroll
    for (int i = 0; i < BP_MAXBINS; i++) {
        if (i < n) {
            const float f = (float)(off0 + i) * inv, g = 1.0f - f;
#pragma unroll
            for (int q = 0; q < NQ; q++) {
                const float e = v[q * NB_BINS_BANDED + b0 + i];
                a[q] = fmaf(g, e, a[q]);
                b[q] = fmaf(f, e, b[q]);
            }
        }
    }
    float a0[NQ], b0v[NQ];
#pragma unroll
    for (int q = 0; q < NQ; q++) {
        a0[q] = a[q];
        b0v[q] = b[q];
    }
#pragma unroll
    for (int off = 1; off < 4; off++) {
        const int osg = __shfl_down_sync(0xffffffffu, sg, off);
        const bool take = lane + off < 32 && osg == sg;
#pragma unroll
        for (int q = 0; q < NQ; q++) {
            const float va = __shfl_down_sync(0xffffffffu, a0[q], off), vb = __shfl_down_sync(0xffffffffu, b0v[q], off);
            if (take) {
                a[q] += va;
                b[q] += vb;
            }
        }
    }
    const int psg = __shfl_up_sync(0xffffffffu, sg, 1);
    if (lane == 0 || psg != sg) {
#pragma unroll
        for (int q = 0; q < NQ; q++) {
            sc[S_SEG + sg * 4 + q] = a[q];
            sc[S_SEG + sg * 4 + 2 + q] = b[q];
        }
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < NQ; q++) {
        float r = 0.0f;
        if (lane < NB_BANDS) {
            if (lane < NB_BANDS - 1) r = sc[S_SEG + lane * 4 + q];
            if (lane > 0) r += sc[S_SEG + (lane - 1) * 4 + 2 + q];
        }
        o[q] = r;
    }
    __syncwarp();
}

// band values sc[base + b] interpolated to bin k < 400 (src/lib.rs:84-97)
__device__ __forceinline__ float interp(const float* __restrict__ sc, int base, const GradTables* __restrict__ tb, int k) {
    const int bi = tb->band_of[k];
    const float fr = tb->band_frac[k];
    return (1.0f - fr) * sc[base + bi] + fr * sc[base + bi + 1];
}

// forward 480-point FFT of z[32 a + lane] held in v -> natural order in buf[0..480)
__device__ __forceinline__ void fft480_one(float2 (&v)[15], float2* __restrict__ buf, const GradTables* __restrict__ tb, int lane) {
    dft15(v);
#pragma unroll
    for (int k1 = 1; k1 < 15; k1++) v[k1] = c_mul(v[k1], tb->twl[k1][lane]);
#pragma unroll
    for (int k1 = 0; k1 < 15; k1++) buf[k1 * RS + lane] = v[k1];
    __syncwarp();
    float2 r[32];
    if (lane < 15) {
#pragma unroll
        for (int b = 0; b < 32; b++) r[b] = buf[lane * RS + b];
        fft32_dif(r);
    }
    __syncwarp();
    if (lane < 15) {
#pragma unroll
        for (int k2 = 0; k2 < 32; k2++) buf[lane + 15 * k2] = r[bitrev5(k2)];
    }
    __syncwarp();
}

__global__ void __launch_bounds__(GW * 32) synthesis_grad_warp_kernel(const unsigned char* __restrict__ ctx, long css, long cfs,
                                                                      const float* __restrict__ go, long gss, long gfs, int n_streams,
                                                                      int n_frames, const GradTables* __restrict__ tb,
                                                                      float* __restrict__ w_gg, float* __restrict__ w_g) {
    __shared__ __align__(16) float2 sbuf[GW][FBUF];
    __shared__ __align__(16) float2 shs[GW][FREQ_SIZE + 3];
    __shared__ float ssc[GW][WSC];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long item = (long)blockIdx.x * GW + warp;
    if (item >= (long)n_streams * n_frames) return;
    const int s = (int)(item / n_frames), t = (int)(item % n_frames);
    const float* c = reinterpret_cast<const float*>(ctx + ((size_t)s * css + (size_t)t * cfs) * RNNOISE_SYNTH_CONTEXT_BYTES);
    float* o_gg = w_gg + (size_t)item * NB_BANDS;
    float* o_g = w_g + (size_t)item * NB_BANDS;
    if (__float_as_int(c[CX_SIL])) {  // the output does not depend on a silent frame's gains
        if (lane < NB_BANDS) o_gg[lane] = o_g[lane] = 0.0f;
        return;
    }
    float2* buf = sbuf[warp];
    float2* hs = shs[warp];
    float* sc = ssc[warp];
    float* fb = reinterpret_cast<float*>(buf);

    // ---- H = rfft960(0.5 window (grad_out[t] | grad_out[t+1])): lane b packs z[32 a + b] = (h[64 a + 2 b], h[64 a + 2 b + 1]) ----
    {
        const float* g0 = go + (size_t)s * gss + (size_t)t * gfs;
        const float* g1 = t + 1 < n_frames ? go + (size_t)s * gss + (size_t)(t + 1) * gfs : nullptr;
        float2 v[15];
#pragma unroll
        for (int a = 0; a < 15; a++) {
            const int n = 64 * a + 2 * lane;  // n and n + 1 lie on one side of 480
            float2 d = make_float2(0.f, 0.f);
            if (n < FRAME_SIZE) d = make_float2(g0[n], g0[n + 1]);
            else if (g1) d = make_float2(g1[n - FRAME_SIZE], g1[n - FRAME_SIZE + 1]);
            v[a] = make_float2(0.5f * tb->window[n] * d.x, 0.5f * tb->window[n + 1] * d.y);
        }
        fft480_one(v, buf, tb, lane);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int k = lane + 32 * j;
            if (k <= 240) {
                float2 h0, h1;
                rfft_split_pair(buf[k], buf[k == 0 ? 0 : 480 - k], tb->tw960[k], 1.0f, k == 0, h0, h1);
                hs[k] = h0;
                if (k != 240) hs[480 - k] = h1;
            }
        }
        __syncwarp();  // the transpose area is free again
    }

    // ---- K5's intermediates from the record ----
    float ex = 0.f, e = 0.f, g = 0.f, cb = 0.f, q = 0.f;
    bool q_live = false;
    if (lane < NB_BANDS) {
        ex = c[CX_EX + lane];
        const float ep = c[CX_EP + lane], lastg = c[CX_LASTG + lane];
        e = c[CX_EXP + lane];
        g = c[CX_G + lane];
        cb = sqrtf(ex / (1e-8f + ep));
        float r;
        if (e > g) {
            r = 1.0f;
        } else {
            const float e2 = e * e, g2 = g * g;
            q = e2 * (1.0f - g2) / (0.001f + g2 * (1.0f - e2));
            q_live = q > 0.0f && q < 1.0f;
            r = q;
        }
        r = (r < 0.0f) ? 0.0f : r;
        r = (r > 1.0f) ? 1.0f : r;
        sc[S_R + lane] = sqrtf(r) * cb;
        sc[S_GG + lane] = fmaxf(g, 0.6f * lastg);
    }
    __syncwarp();
    const float2* Xc = reinterpret_cast<const float2*>(c + CX_X);
    const float2* Pc = reinterpret_cast<const float2*>(c + CX_P);
    float2 xv[13];  // x = X + P rf, bins k = lane + 32 j < 400 (bins >= 400 of y are zero)
#pragma unroll
    for (int j = 0; j < 13; j++) {
        const int k = lane + 32 * j;
        xv[j] = make_float2(0.f, 0.f);
        if (k < NB_BINS_BANDED) {
            const float rf = interp(sc, S_R, tb, k);
            const float2 xk = Xc[k], pk = Pc[k];
            xv[j] = make_float2(xk.x + pk.x * rf, k > 0 ? xk.y + pk.y * rf : xk.y);
            fb[k] = xv[j].x * xv[j].x + xv[j].y * xv[j].y;
        }
    }
    __syncwarp();
    float ne[1];
    band_reduce<1>(fb, tb, sc, lane, ne);
    if (lane == 0 || lane == NB_BANDS - 1) ne[0] *= 2.0f;  // compute_band_corr doubles the first and last band
    float s2 = 0.f;
    if (lane < NB_BANDS) {
        s2 = sqrtf(ex / (1e-8f + ne[0]));
        sc[S_S2 + lane] = s2;
    }
    __syncwarp();

    // ---- adjoints: y = x rf2 gf (per bin), gy = c_k H_k (c_0 = 1, the imaginary part of DC unused; else 2) ----
    float2 ga[13];  // gy rf2 gf: the part of dL/dx that does not pass through the renormalisation
#pragma unroll
    for (int j = 0; j < 13; j++) {
        const int k = lane + 32 * j;
        ga[j] = make_float2(0.f, 0.f);
        if (k < NB_BINS_BANDED) {
            const float rf2 = interp(sc, S_S2, tb, k), gf = interp(sc, S_GG, tb, k);
            const float2 h = hs[k];
            const float2 gy = k == 0 ? make_float2(h.x, 0.0f) : make_float2(2.0f * h.x, 2.0f * h.y);
            const float u = gy.x * xv[j].x + gy.y * xv[j].y;
            fb[k] = rf2 * u;                   // -> dL/dgg
            fb[NB_BINS_BANDED + k] = gf * u;   // -> dL/ds2
            const float a = rf2 * gf;
            ga[j] = make_float2(gy.x * a, gy.y * a);
        }
    }
    __syncwarp();
    float d2[2];
    band_reduce<2>(fb, tb, sc, lane, d2);
    if (lane < NB_BANDS) {
        o_gg[lane] = d2[0];
        // s2 = sqrt(ex / (1e-8 + ne)): ds2/dne = -s2 / (2 (1e-8 + ne)); ne's first and last band count twice
        float dne = d2[1] * (-0.5f * s2 / (1e-8f + ne[0]));
        if (lane == 0 || lane == NB_BANDS - 1) dne *= 2.0f;
        sc[S_DNE + lane] = dne;
    }
    __syncwarp();
    // dL/dx = ga + 2 x W^T dne;  dL/drf = dL/dx . P (bin 0: real part only)
#pragma unroll
    for (int j = 0; j < 13; j++) {
        const int k = lane + 32 * j;
        if (k < NB_BINS_BANDED) {
            const float wd = 2.0f * interp(sc, S_DNE, tb, k);
            const float2 pk = Pc[k];
            const float gxr = ga[j].x + wd * xv[j].x, gxi = ga[j].y + wd * xv[j].y;
            fb[k] = k > 0 ? gxr * pk.x + gxi * pk.y : gxr * pk.x;
        }
    }
    __syncwarp();
    float dr[1];
    band_reduce<1>(fb, tb, sc, lane, dr);
    if (lane < NB_BANDS) {
        // r = sqrt(clamp(q, 0, 1)) cb: gradient only on the formula's branch (exp <= g) strictly inside the clamp (the
        // decision is K5's q).  The value uses 1 - x^2 = (1 - x)(1 + x), exact up to one rounding: near g = 1 or exp = 1
        // the derivative is large and 1 - x*x would lose most of its bits.
        float dg = 0.0f;
        if (q_live) {
            const float e2 = e * e, g2 = g * g, omg = (1.0f - g) * (1.0f + g), ome = (1.0f - e) * (1.0f + e);
            const float num = e2 * omg, den = 0.001f + g2 * ome;
            const float dq = -2.0f * g * (e2 * den + num * ome) / (den * den);
            dg = dr[0] * cb * 0.5f / sqrtf(num / den) * dq;
        }
        o_g[lane] = dg;
    }
}

__global__ void synthesis_grad_scan_kernel(const unsigned char* __restrict__ ctx, long css, long cfs, const float* __restrict__ w_gg,
                                           const float* __restrict__ w_g, float* __restrict__ gg_out, long ggs, long ggf, int n_streams,
                                           int n_frames) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const int s = (int)(i / NB_BANDS), b = (int)(i % NB_BANDS);
    if (s >= n_streams) return;
    float carry = 0.0f;  // dL/dlastg after frame t, i.e. dL/dgg_t through the later frames
    for (int t = n_frames - 1; t >= 0; t--) {
        const float* c = reinterpret_cast<const float*>(ctx + ((size_t)s * css + (size_t)t * cfs) * RNNOISE_SYNTH_CONTEXT_BYTES);
        const size_t w = ((size_t)s * n_frames + t) * NB_BANDS + b;
        float d = 0.0f;
        if (!__float_as_int(c[CX_SIL])) {  // a silent frame leaves lastg as it was: the carry passes through
            const float g = c[CX_G + b], lastg = c[CX_LASTG + b];
            const float dgg = w_gg[w] + carry;
            if (g >= 0.6f * lastg) {
                d = w_g[w] + dgg;
                carry = 0.0f;
            } else {
                d = w_g[w];
                carry = 0.6f * dgg;
            }
        }
        gg_out[(size_t)s * ggs + (size_t)t * ggf + b] = d;
    }
}

size_t grad_vector_bytes(int n_streams, int n_frames) {
    return (((size_t)n_streams * (size_t)n_frames * NB_BANDS * sizeof(float)) + 255) & ~(size_t)255;
}

}  // namespace

cudaError_t launch_synth_context(const BatchBuffers& b, const float* gains, long gain_stride, void* ctx, long ctx_stride, cudaStream_t st) {
    const long n = (long)b.n_streams * CX_UNITS;
    synth_context_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(b, gains, gain_stride, static_cast<unsigned char*>(ctx), ctx_stride);
    return cudaGetLastError();
}

// Rows of `len` elements at s * ss + t * ts (s < ns, t < nt) overlap nowhere and have positive strides.
bool rows_disjoint(int ns, int nt, long ss, long ts, long len) {
    if ((ns > 1 && ss < 1) || (nt > 1 && ts < 1)) return false;
    long s1 = ss, s2 = ts, n1 = ns, n2 = nt;  // s1: the inner dimension
    if (ns <= 1 || (nt > 1 && ts < ss)) {
        s1 = ts, s2 = ss, n1 = nt, n2 = ns;
    }
    if (n1 > 1 && s1 < len) return false;
    return n2 <= 1 || s2 >= s1 * (n1 - 1) + len;
}

}  // namespace nnb

using namespace nnb;

extern "C" {

size_t rnnoise_synthesis_backward_workspace_bytes(int n_streams, int n_frames) {
    if (n_streams < 1 || n_frames < 1) return 0;
    return TABLE_BYTES + 2 * grad_vector_bytes(n_streams, n_frames);
}

int rnnoise_synthesis_backward_device(const void* ctx, long ctx_stream_stride, long ctx_frame_stride, const float* grad_out,
                                      long go_stream_stride, long go_frame_stride, float* grad_gains, long gg_stream_stride,
                                      long gg_frame_stride, int n_streams, int n_frames, void* workspace, size_t workspace_bytes, int device,
                                      void* cuda_stream) {
    if (!ctx || !grad_out || !grad_gains || !workspace) return fail("null argument");
    if (n_streams < 1) return fail("n_streams must be >= 1");
    if (n_frames < 1) return fail("n_frames must be >= 1");
    if ((reinterpret_cast<uintptr_t>(ctx) & 15) || (reinterpret_cast<uintptr_t>(workspace) & 15))
        return fail("ctx and workspace must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(grad_out) & 3) || (reinterpret_cast<uintptr_t>(grad_gains) & 3))
        return fail("grad_out and grad_gains must be float-aligned");
    if ((n_streams > 1 && ctx_stream_stride < 1) || (n_frames > 1 && ctx_frame_stride < 1) || (n_streams > 1 && go_stream_stride < 1) ||
        (n_frames > 1 && go_frame_stride < 1))
        return fail("context and grad_out strides must be positive");
    if (!rows_disjoint(n_streams, n_frames, gg_stream_stride, gg_frame_stride, NB_BANDS))
        return fail("grad_gains strides overlap rows of 22 gains");
    const size_t need = rnnoise_synthesis_backward_workspace_bytes(n_streams, n_frames);
    if (workspace_bytes < need) return fail("workspace of " + std::to_string(workspace_bytes) + " bytes; " + std::to_string(need) + " needed");
    int dev = 0;
    if (open_device(device, &dev)) return -1;
    ON_DEVICE(dev);
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    GradTables* tb = static_cast<GradTables*>(workspace);
    float* w_gg = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + TABLE_BYTES);
    float* w_g = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(w_gg) + grad_vector_bytes(n_streams, n_frames));
    const unsigned char* c = static_cast<const unsigned char*>(ctx);
    grad_tables_kernel<<<1, 512, 0, st>>>(tb);
    CK(cudaGetLastError());
    const long items = (long)n_streams * n_frames;
    synthesis_grad_warp_kernel<<<(unsigned)((items + GW - 1) / GW), GW * 32, 0, st>>>(c, ctx_stream_stride, ctx_frame_stride, grad_out,
                                                                                      go_stream_stride, go_frame_stride, n_streams,
                                                                                      n_frames, tb, w_gg, w_g);
    CK(cudaGetLastError());
    const long lanes = (long)n_streams * NB_BANDS;
    synthesis_grad_scan_kernel<<<(unsigned)((lanes + 127) / 128), 128, 0, st>>>(c, ctx_stream_stride, ctx_frame_stride, w_gg, w_g, grad_gains,
                                                                                gg_stream_stride, gg_frame_stride, n_streams, n_frames);
    CK(cudaGetLastError());
    count_launches(3);
    if (!st) CK(cudaStreamSynchronize(st));
    return 0;
}

}  // extern "C"
