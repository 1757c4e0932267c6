// fit.cu -- fitting the denoise network to training rows on the GPU: what the reference's train/rnn_train.py does with
// Keras (tf.keras 2.x semantics, DESIGN.md §7e), and the .rnn export of train/dump_rnn.py.
//
// The work is split at the sequential dependency, layer by layer, in f32 (no TF32) and without float atomics:
//   fit_gemm       : every dense product -- a GRU's input projection over all (sequence, frame) rows, the dense layers,
//                    dX = dG W^T, and the weight gradients X^T dG over the rows as split-K partials summed in a fixed
//                    order by fit_reduce.  Operands are views over up to three column blocks, so concatenated inputs
//                    ([dense | vad_h | x], ...) are read in place and dX is scattered back onto its sources.
//   fit_gru_fwd    : a GRU's recurrence over the window with U in shared memory; writes z, r, h~, r*h_{t-1} and h_t.
//   fit_gru_bwd    : the reverse-time recurrence: carries dh and writes the gate pre-activation gradients dG.
//   fit_loss       : per-frame loss terms and the gradients at the two output layers; fit_finish reduces them
//                    (and the L2 term) in a fixed order in f64.
//   fit_adam       : L2 gradient, tf.keras Adam and the WeightClip(0.499) constraint over the flat parameter vector.
#include <algorithm>
#include <cmath>
#include <initializer_list>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/rnnoise.h"
#include "abi.hpp"
#include "common.cuh"
#include "model.hpp"
#include "owners.hpp"

using namespace nnb;

namespace {

constexpr int FIT_TILE = 64;
constexpr int FIT_BK = 16;
constexpr int FIT_G = 8;            // sequences per recurrence CTA at most
constexpr int FIT_SPLIT_ROWS = 2048;  // rows per split-K partial of a weight gradient
constexpr int FIT_SPLITS_MAX = 256;
constexpr int FIT_MAX_WIDTH = 96;
constexpr int ACT_TANH = 0, ACT_SIGMOID = 1, ACT_RELU = 2, ACT_NONE = -1;

// A matrix of rows r = s * T + t (sequence s, frame t) made of up to three column blocks.  Block i holds columns
// [c0[i], c0[i + 1]) at p[i][row_i * ld[i] + c - c0[i]], with row_i = r, or r + s when pad[i] (a [S][T + 1] buffer
// whose row 0 of each sequence is the zero initial state).  p[i] == nullptr reads as 1 (a column of ones for bias
// gradients) and is skipped as an output.
struct View {
    float* p[3];
    int ld[3];
    int pad[3];
    int c0[4];
    int nb;
    int T;
};

__device__ __forceinline__ int view_block(const View& v, int c) {
    int i = 0;
    while (i + 1 < v.nb && c >= v.c0[i + 1]) i++;
    return i;
}
__device__ __forceinline__ long view_row(const View& v, int i, long r) { return v.pad[i] ? r + r / v.T : r; }
__device__ __forceinline__ float view_get(const View& v, long r, int c) {
    const int i = view_block(v, c);
    const float* p = v.p[i];
    return p ? p[view_row(v, i, r) * v.ld[i] + (c - v.c0[i])] : 1.0f;
}

__device__ __forceinline__ float fit_act(int act, float x) {
    if (act == ACT_TANH) return tanhf(x);
    if (act == ACT_SIGMOID) return 1.0f / (1.0f + expf(-x));
    if (act == ACT_RELU) return fmaxf(x, 0.0f);
    return x;
}

// d act / d x expressed through y = act(x); relu' is 0 at 0, as TensorFlow's
__device__ __forceinline__ float fit_dact(int act, float y) {
    if (act == ACT_TANH) return 1.0f - y * y;
    if (act == ACT_SIGMOID) return y * (1.0f - y);
    return y > 0.0f ? 1.0f : 0.0f;
}

// C(m, n) [+]= act(sum_k A(m, k) B(k, n) + bias[n]);  A(m, k) = a(m, k), or a(k, m) when trans_a;  B(k, n) at
// b[k * sbk + n * sbn].  With split-K (gridDim.z > 1) each z sums its own k range into part[z][M][N].
struct Gemm {
    View a;
    int trans_a;
    const float* b;
    long sbk, sbn;
    View c;
    const float* bias;
    int act;
    int accumulate;
    int M, N;
    long K, kchunk;
    float* part;
};

__device__ __forceinline__ void gemm_store(const Gemm& g, int m, int n, float v) {
    if (g.bias) v += g.bias[n];
    v = fit_act(g.act, v);
    const int i = view_block(g.c, n);
    float* p = g.c.p[i];
    if (!p) return;
    float* q = p + view_row(g.c, i, m) * g.c.ld[i] + (n - g.c.c0[i]);
    *q = g.accumulate ? *q + v : v;
}

__global__ void __launch_bounds__(256) fit_gemm_kernel(Gemm g) {
    __shared__ float As[FIT_BK][FIT_TILE + 4];
    __shared__ float Bs[FIT_BK][FIT_TILE + 4];
    const int m0 = blockIdx.y * FIT_TILE, n0 = blockIdx.x * FIT_TILE;
    const long k_begin = (long)blockIdx.z * g.kchunk;
    const long k_end = min(g.K, k_begin + g.kchunk);
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    float acc[4][4] = {};
    for (long k0 = k_begin; k0 < k_end; k0 += FIT_BK) {
        for (int e = tid; e < FIT_BK * FIT_TILE; e += 256) {
            int kk, mm;
            if (g.trans_a) kk = e / FIT_TILE, mm = e % FIT_TILE;  // consecutive threads walk the view's columns
            else mm = e / FIT_BK, kk = e % FIT_BK;
            const long k = k0 + kk;
            const int m = m0 + mm;
            float v = 0.0f;
            if (k < k_end && m < g.M) v = g.trans_a ? view_get(g.a, k, m) : view_get(g.a, m, (int)k);
            As[kk][mm] = v;
            int kb, nn;
            if (g.sbn == 1) kb = e / FIT_TILE, nn = e % FIT_TILE;
            else nn = e / FIT_BK, kb = e % FIT_BK;
            const long kg = k0 + kb;
            const int n = n0 + nn;
            Bs[kb][nn] = (kg < k_end && n < g.N) ? g.b[kg * g.sbk + (long)n * g.sbn] : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < FIT_BK; kk++) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) a[i] = As[kk][ty * 4 + i], b[i] = Bs[kk][tx * 4 + i];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
            if (m >= g.M || n >= g.N) continue;
            if (gridDim.z > 1) g.part[((size_t)blockIdx.z * g.M + m) * g.N + n] = acc[i][j];
            else gemm_store(g, m, n, acc[i][j]);
        }
}

// The split-K partials of one product, summed in split order.
__global__ void __launch_bounds__(256) fit_reduce_kernel(Gemm g, int splits) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= g.M * g.N) return;
    float s = 0.0f;
    for (int z = 0; z < splits; z++) s += g.part[(size_t)z * g.M * g.N + idx];
    gemm_store(g, idx / g.N, idx % g.N, s);
}

// One GRU layer's device arrays; rows r = s * T + t.
struct GruArgs {
    int n, act;
    const float* U;      // [n][3n]
    const float* xw;     // [R][3n] x W + b (forward)
    float* gates;        // [R][3n] z | r | h~
    float* rh;           // [R][n]  r * h_{t-1}
    float* hbuf;         // [S][T + 1][n], row 0 of each sequence = 0
    const float* dh;     // [R][n]  dLoss/dh_t from the layers that read h_t (backward)
    float* dG;           // [R][3n] dLoss/d(z, r, h~ pre-activations) (backward)
};

__device__ __forceinline__ int fit_ldu(int n) { return (3 * n) | 1; }  // odd: the backward's column reads hit distinct banks

__global__ void __launch_bounds__(3 * FIT_MAX_WIDTH) fit_gru_fwd_kernel(GruArgs L, int S, int T, int G) {
    extern __shared__ float fsm[];
    const int n = L.n, n3 = 3 * n, ldu = fit_ldu(n);
    // the unrolled loops read all FIT_G slots: the buffers hold FIT_G sequences, the slots past gs stay zero
    float* Us = fsm;                // [n][ldu]
    float* hs = Us + n * ldu;       // [FIT_G][n]
    float* zs = hs + FIT_G * n;     // [FIT_G][n]
    float* rhs = zs + FIT_G * n;    // [FIT_G][n]
    const int s0 = blockIdx.x * G, gs = min(G, S - s0);
    const int j = threadIdx.x;
    for (int i = j; i < n * n3; i += blockDim.x) Us[(i / n3) * ldu + i % n3] = L.U[i];
    for (int i = j; i < 3 * FIT_G * n; i += blockDim.x) hs[i] = 0.0f;
    for (int i = j; i < gs * n; i += blockDim.x) L.hbuf[(size_t)(s0 + i / n) * (T + 1) * n + i % n] = 0.0f;
    float xcur[FIT_G];
#pragma unroll
    for (int g = 0; g < FIT_G; g++) xcur[g] = (g < gs && j < n3) ? L.xw[((size_t)(s0 + g) * T) * n3 + j] : 0.0f;
    __syncthreads();
    for (int t = 0; t < T; t++) {
        float xnxt[FIT_G];
#pragma unroll
        for (int g = 0; g < FIT_G; g++)
            xnxt[g] = (g < gs && j < n3 && t + 1 < T) ? L.xw[((size_t)(s0 + g) * T + t + 1) * n3 + j] : 0.0f;
        if (j < 2 * n) {  // z and r; the r threads also form r * h_{t-1}
            float acc[FIT_G];
#pragma unroll
            for (int g = 0; g < FIT_G; g++) acc[g] = xcur[g];
            for (int k = 0; k < n; k++) {
                const float u = Us[k * ldu + j];
#pragma unroll
                for (int g = 0; g < FIT_G; g++) acc[g] = fmaf(hs[g * n + k], u, acc[g]);
            }
#pragma unroll
            for (int g = 0; g < FIT_G; g++) {
                if (g >= gs) break;
                const size_t row = (size_t)(s0 + g) * T + t;
                const float v = fit_act(ACT_SIGMOID, acc[g]);
                L.gates[row * n3 + j] = v;
                if (j < n) {
                    zs[g * n + j] = v;
                } else {
                    const float rh = v * hs[g * n + j - n];
                    rhs[g * n + j - n] = rh;
                    L.rh[row * n + j - n] = rh;
                }
            }
        }
        __syncthreads();
        if (j >= 2 * n && j < n3) {  // h~ and the new state; nothing reads hs in this phase
            const int jj = j - 2 * n;
            float acc[FIT_G];
#pragma unroll
            for (int g = 0; g < FIT_G; g++) acc[g] = xcur[g];
            for (int k = 0; k < n; k++) {
                const float u = Us[k * ldu + j];
#pragma unroll
                for (int g = 0; g < FIT_G; g++) acc[g] = fmaf(rhs[g * n + k], u, acc[g]);
            }
#pragma unroll
            for (int g = 0; g < FIT_G; g++) {
                if (g >= gs) break;
                const size_t row = (size_t)(s0 + g) * T + t;
                const float hc = fit_act(L.act, acc[g]);
                const float z = zs[g * n + jj];
                const float h = z * hs[g * n + jj] + (1.0f - z) * hc;
                L.gates[row * n3 + j] = hc;
                hs[g * n + jj] = h;
                L.hbuf[((size_t)(s0 + g) * (T + 1) + t + 1) * n + jj] = h;
            }
        }
        __syncthreads();
#pragma unroll
        for (int g = 0; g < FIT_G; g++) xcur[g] = xnxt[g];
    }
}

__global__ void __launch_bounds__(FIT_MAX_WIDTH) fit_gru_bwd_kernel(GruArgs L, int S, int T, int G) {
    extern __shared__ float fsm[];
    const int n = L.n, n3 = 3 * n, ldu = fit_ldu(n);
    float* Us = fsm;           // [n][ldu]
    float* das = Us + n * ldu;  // [G][3n]
    const int s0 = blockIdx.x * G, gs = min(G, S - s0);
    const int k = threadIdx.x;
    for (int i = k; i < n * n3; i += blockDim.x) Us[(i / n3) * ldu + i % n3] = L.U[i];
    float carry[FIT_G], rr[FIT_G], hp[FIT_G], daz[FIT_G], dar[FIT_G], dah[FIT_G];
#pragma unroll
    for (int g = 0; g < FIT_G; g++) carry[g] = 0.0f;
    __syncthreads();
    for (int t = T - 1; t >= 0; t--) {
        if (k < n) {
#pragma unroll
            for (int g = 0; g < FIT_G; g++) {
                if (g >= gs) break;
                const size_t row = (size_t)(s0 + g) * T + t;
                const float dh = carry[g] + L.dh[row * n + k];
                const float z = L.gates[row * n3 + k], r = L.gates[row * n3 + n + k], hc = L.gates[row * n3 + 2 * n + k];
                hp[g] = L.hbuf[((size_t)(s0 + g) * (T + 1) + t) * n + k];
                rr[g] = r;
                daz[g] = dh * (hp[g] - hc) * z * (1.0f - z);
                dah[g] = dh * (1.0f - z) * fit_dact(L.act, hc);
                das[g * n3 + k] = daz[g];
                das[g * n3 + 2 * n + k] = dah[g];
                carry[g] = dh * z;
            }
        }
        __syncthreads();
        if (k < n) {  // d(r * h_{t-1}) = dah U_h^T
#pragma unroll
            for (int g = 0; g < FIT_G; g++) {
                if (g >= gs) break;
                float drh = 0.0f;
                for (int j = 0; j < n; j++) drh = fmaf(das[g * n3 + 2 * n + j], Us[k * ldu + 2 * n + j], drh);
                dar[g] = drh * hp[g] * rr[g] * (1.0f - rr[g]);
                das[g * n3 + n + k] = dar[g];
                carry[g] += drh * rr[g];
            }
        }
        __syncthreads();
        if (k < n) {  // dh_{t-1} += (daz | dar) U_zr^T
#pragma unroll
            for (int g = 0; g < FIT_G; g++) {
                if (g >= gs) break;
                float acc = carry[g];
                for (int j = 0; j < 2 * n; j++) acc = fmaf(das[g * n3 + j], Us[k * ldu + j], acc);
                carry[g] = acc;
                const size_t row = (size_t)(s0 + g) * T + t;
                L.dG[row * n3 + k] = daz[g];
                L.dG[row * n3 + n + k] = dar[g];
                L.dG[row * n3 + 2 * n + k] = dah[g];
            }
        }
        __syncthreads();
    }
}

// Per (sequence, frame) row: the weighted terms of the loss and its gradients at the output pre-activations
// (rnn_train.py:33-43, 79-81).  rows [R][87]: [42 features | 22 gains | 22 noise | vad].
__global__ void __launch_bounds__(256) fit_loss_kernel(const float* __restrict__ rows, const float* __restrict__ wts,
                                                       const float* __restrict__ gains, const float* __restrict__ vad, float* dzo,
                                                       float* dzv, float* rowloss, long R, float inv_rows) {
    const long r = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const float eps = 1e-7f, one_m = 1.0f - eps;
    const float w = wts[r];
    const float* y = rows + r * TRAIN_ROW + NB_FEATURES;
    float cost = 0.0f, msse = 0.0f;
    for (int j = 0; j < NB_BANDS; j++) {
        const float g = gains[r * NB_BANDS + j], t = y[j];
        const float mask = fminf(t + 1.0f, 1.0f);                       // mymask
        const float sg = sqrtf(fmaxf(g, 0.0f)), d = sg - sqrtf(fmaxf(t, 0.0f));  // K.sqrt clips at 0
        const float tc = fminf(fmaxf(t, eps), one_m);
        const float la = logf(tc + eps), lb = logf(1.0f - tc + eps);
        const float bce = -(g * la + (1.0f - g) * lb);                  // K.binary_crossentropy(y_pred, y_true)
        const float d2 = d * d;
        cost += mask * (10.0f * d2 * d2 + d2 + 0.01f * bce);
        msse += mask * d2;
        const float dcost = mask * ((40.0f * d2 * d + 2.0f * d) * (0.5f / sg) - 0.01f * (la - lb)) / NB_BANDS;
        dzo[r * NB_BANDS + j] = w * inv_rows * 10.0f * dcost * g * (1.0f - g);
    }
    cost /= NB_BANDS;
    msse /= NB_BANDS;
    const float v = vad[r], t = rows[r * TRAIN_ROW + TRAIN_ROW - 1];
    const float tc = fminf(fmaxf(t, eps), one_m);
    const float la = logf(tc + eps), lb = logf(1.0f - tc + eps);
    const float c = 2.0f * fabsf(t - 0.5f);
    const float xent = c * -(v * la + (1.0f - v) * lb);                  // my_crossentropy
    dzv[r] = w * inv_rows * 0.5f * c * -(la - lb) * v * (1.0f - v);
    rowloss[r * 3 + 0] = w * cost;
    rowloss[r * 3 + 1] = w * xent;
    rowloss[r * 3 + 2] = msse;
}

struct Ranges {
    long off[6], len[6];  // the kernel and recurrent matrices of the three GRUs
};

// out = {10 mycost + 0.5 crossentropy + L2, mycost, crossentropy, msse}: weighted sums over the rows / R, in a fixed order.
__global__ void __launch_bounds__(512) fit_finish_kernel(const float* rowloss, long R, const float* params, Ranges l2, double* out) {
    __shared__ double red[4][512];
    const int tid = threadIdx.x;
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (long r = tid; r < R; r += 512)
        for (int q = 0; q < 3; q++) s[q] += (double)rowloss[r * 3 + q];
    for (int i = 0; i < 6; i++)
        for (long e = tid; e < l2.len[i]; e += 512) {
            const double p = params[l2.off[i] + e];
            s[3] += p * p;
        }
    for (int q = 0; q < 4; q++) red[q][tid] = s[q];
    __syncthreads();
    for (int h = 256; h > 0; h >>= 1) {
        if (tid < h)
            for (int q = 0; q < 4; q++) red[q][tid] += red[q][tid + h];
        __syncthreads();
    }
    if (tid == 0) {
        const double cost = red[0][0] / (double)R, xent = red[1][0] / (double)R;
        out[0] = 10.0 * cost + 0.5 * xent + 1e-6 * red[3][0];
        out[1] = cost;
        out[2] = xent;
        out[3] = red[2][0] / (double)R;
    }
}

// input_dense: dLoss/d pre-activation = dLoss/d out * act'
__global__ void fit_dense_bwd_kernel(float* dd, const float* d, long n, int act) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dd[i] *= fit_dact(act, d[i]);
}

// L2 (1e-6 sum w^2 over the GRU matrices), tf.keras Adam (ResourceApplyAdam: eps outside the bias correction),
// WeightClip(0.499).  grads holds the data-loss gradient on entry and the full gradient on exit.
__global__ void fit_adam_kernel(float* params, float* grads, float* m, float* v, long n, Ranges l2, float lr_t) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float w = params[i], g = grads[i];
    for (int q = 0; q < 6; q++)
        if (i >= l2.off[q] && i < l2.off[q] + l2.len[q]) g += 2e-6f * w;
    grads[i] = g;
    float mi = m[i], vi = v[i];
    mi += (g - mi) * (1.0f - 0.9f);
    vi += (g * g - vi) * (1.0f - 0.999f);
    m[i] = mi;
    v[i] = vi;
    w -= lr_t * mi / (sqrtf(vi) + 1e-7f);
    params[i] = fminf(fmaxf(w, -0.499f), 0.499f);
}

// ---- host side ---------------------------------------------------------------------------------------------------

struct Layer {
    int ni, nn, gates, act;
    long w, u, b;  // offsets into the flat parameter vector (u = -1: dense)
};

// The six layers in the order of the .rnn file (src/rnn.rs from_bytes), Keras shapes: kernel [ni][gates nn],
// recurrent [nn][3 nn], bias [gates nn].
long layout(int nd, int nv, int nn, int ndn, Layer out[6]) {
    const int spec[6][4] = {{NB_FEATURES, nd, 1, ACT_TANH},
                            {nd, nv, 3, ACT_TANH},
                            {nd + nv + NB_FEATURES, nn, 3, ACT_RELU},
                            {nv + nn + NB_FEATURES, ndn, 3, ACT_TANH},
                            {ndn, NB_BANDS, 1, ACT_SIGMOID},
                            {nv, 1, 1, ACT_SIGMOID}};
    long p = 0;
    for (int i = 0; i < 6; i++) {
        Layer& L = out[i];
        L.ni = spec[i][0], L.nn = spec[i][1], L.gates = spec[i][2], L.act = spec[i][3];
        L.w = p;
        p += (long)L.ni * L.gates * L.nn;
        L.u = -1;
        if (L.gates == 3) {
            L.u = p;
            p += 3L * L.nn * L.nn;
        }
        L.b = p;
        p += (long)L.gates * L.nn;
    }
    return p;
}

struct Src {
    float* p;
    int ld, pad, cols;
};

View view(std::initializer_list<Src> s, int T) {
    View v{};
    int c = 0;
    for (const Src& x : s) {
        v.p[v.nb] = x.p;
        v.ld[v.nb] = x.ld;
        v.pad[v.nb] = x.pad;
        v.c0[v.nb] = c;
        c += x.cols;
        v.nb++;
    }
    v.c0[v.nb] = c;
    v.T = T;
    return v;
}

}  // namespace

struct RNNoiseFit {
    int device = 0;
    int nd = 0, nv = 0, nn = 0, ndn = 0, max_seq = 0, T = 0;
    Layer L[6];
    long n_params = 0;
    long step_count = 0;
    int last_seq = 0;  // sequences of the most recent forward pass
    size_t part_elems = 0;
    Ranges l2{};
    float *params = nullptr, *grads = nullptr, *m = nullptr, *v = nullptr;
    float *rows = nullptr, *wts = nullptr, *d = nullptr, *scratch = nullptr, *gains = nullptr, *vad = nullptr;
    float *dzo = nullptr, *dzv = nullptr, *dd = nullptr, *rowloss = nullptr, *part = nullptr;
    float *gates[3] = {}, *rh[3] = {}, *hbuf[3] = {}, *dh[3] = {};
    double* out = nullptr;
    Stream stream;
    // Declared last, so destroyed first; the destructor runs with the device selected.
    std::vector<DeviceMem> mem;
};

namespace {

struct FitRelease {
    void operator()(RNNoiseFit* f) const {
        DeviceGuard guard(f->device);
        if (f->stream) cudaStreamSynchronize(f->stream);
        delete f;
    }
};

int launch_gemm(const RNNoiseFit* f, Gemm g) {
    if (g.M <= 0 || g.N <= 0) return 0;
    int splits = 1;
    g.kchunk = g.K;
    if (g.K > FIT_SPLIT_ROWS) {
        splits = (int)std::min<long>(FIT_SPLITS_MAX, (g.K + FIT_SPLIT_ROWS - 1) / FIT_SPLIT_ROWS);
        g.kchunk = ((g.K + splits - 1) / splits + FIT_BK - 1) / FIT_BK * FIT_BK;
        splits = (int)((g.K + g.kchunk - 1) / g.kchunk);
        if ((size_t)splits * g.M * g.N > f->part_elems) return fail("fit: split-K workspace too small");
    }
    g.part = f->part;
    const dim3 grid((g.N + FIT_TILE - 1) / FIT_TILE, (g.M + FIT_TILE - 1) / FIT_TILE, splits);
    fit_gemm_kernel<<<grid, 256, 0, f->stream>>>(g);
    count_launches(1);
    if (splits > 1) {
        fit_reduce_kernel<<<(g.M * g.N + 255) / 256, 256, 0, f->stream>>>(g, splits);
        count_launches(1);
    }
    CK(cudaGetLastError());
    return 0;
}

// C[M][N] (+)= act(A B + bias) with A a view of rows, B = W [K][N] row-major
int gemm_fwd(const RNNoiseFit* f, const View& a, const float* w, int K, int N, const View& c, const float* bias, int act, long R,
             int accumulate = 0) {
    Gemm g{};
    g.a = a;
    g.b = w;
    g.sbk = N;
    g.sbn = 1;
    g.c = c;
    g.bias = bias;
    g.act = act;
    g.accumulate = accumulate;
    g.M = (int)R;
    g.N = N;
    g.K = K;
    return launch_gemm(f, g);
}

// dX[R][N] += dG[R][K] W^T restricted to W's first N rows (W [rows][K] row-major)
int gemm_dx(const RNNoiseFit* f, const float* dg, int K, const float* w, int N, const View& dx, long R) {
    Gemm g{};
    g.a = view({{const_cast<float*>(dg), K, 0, K}}, f->T);
    g.b = w;
    g.sbk = 1;
    g.sbn = K;
    g.c = dx;
    g.act = ACT_NONE;
    g.accumulate = 1;
    g.M = (int)R;
    g.N = N;
    g.K = K;
    return launch_gemm(f, g);
}

// G[M][N] (row stride ldg) = A^T B over the R rows, B(r, n) = b[r * ldb + n]
int gemm_wgrad(const RNNoiseFit* f, const View& a, int M, const float* b, int ldb, int N, float* grad, int ldg, long R) {
    Gemm g{};
    g.a = a;
    g.trans_a = 1;
    g.b = b;
    g.sbk = ldb;
    g.sbn = 1;
    g.c = view({{grad, ldg, 0, N}}, f->T);
    g.act = ACT_NONE;
    g.M = M;
    g.N = N;
    g.K = R;
    return launch_gemm(f, g);
}

int gru_threads(int n, int per) { return (per * n + 31) / 32 * 32; }
int gru_group(int S) { return std::max(1, std::min(FIT_G, (S + 131) / 132)); }

GruArgs gru_args(const RNNoiseFit* f, int i) {
    const Layer& L = f->L[i + 1];
    GruArgs a{};
    a.n = L.nn;
    a.act = L.act;
    a.U = f->params + L.u;
    a.xw = f->scratch;
    a.gates = f->gates[i];
    a.rh = f->rh[i];
    a.hbuf = f->hbuf[i];
    a.dh = f->dh[i];
    a.dG = f->scratch;
    return a;
}

int gru_fwd(const RNNoiseFit* f, int i, int S) {
    const GruArgs a = gru_args(f, i);
    const int G = gru_group(S);
    const size_t smem = ((size_t)a.n * ((3 * a.n) | 1) + 3 * (size_t)FIT_G * a.n) * sizeof(float);
    CK(cudaFuncSetAttribute(fit_gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fit_gru_fwd_kernel<<<(S + G - 1) / G, gru_threads(a.n, 3), smem, f->stream>>>(a, S, f->T, G);
    count_launches(1);
    CK(cudaGetLastError());
    return 0;
}

int gru_bwd(const RNNoiseFit* f, int i, int S) {
    const GruArgs a = gru_args(f, i);
    const int G = gru_group(S);
    const size_t smem = ((size_t)a.n * ((3 * a.n) | 1) + 3 * (size_t)G * a.n) * sizeof(float);
    CK(cudaFuncSetAttribute(fit_gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fit_gru_bwd_kernel<<<(S + G - 1) / G, gru_threads(a.n, 1), smem, f->stream>>>(a, S, f->T, G);
    count_launches(1);
    CK(cudaGetLastError());
    return 0;
}

Src hsrc(const RNNoiseFit* f, int i) {  // h_t of GRU i as a view block
    const int n = f->L[i + 1].nn;
    return {f->hbuf[i] + n, n, 1, n};
}

// rows / weights -> the handle's buffers (host or device pointers)
int load_inputs(RNNoiseFit* f, const float* rows, const float* wts, int S) {
    const size_t R = (size_t)S * f->T;
    CK(cudaMemcpyAsync(f->rows, rows, R * TRAIN_ROW * sizeof(float), cudaMemcpyDefault, f->stream));
    CK(cudaMemcpyAsync(f->wts, wts, R * sizeof(float), cudaMemcpyDefault, f->stream));
    return 0;
}

// forward pass, loss terms and output gradients, reduction into f->out
int forward(RNNoiseFit* f, int S) {
    const int T = f->T;
    const long R = (long)S * T;
    const Layer* L = f->L;
    float* P = f->params;
    const Src x{f->rows, TRAIN_ROW, 0, NB_FEATURES};
    const Src dsrc{f->d, f->nd, 0, f->nd};
    auto plain = [&](float* p, int ld) { return view({{p, ld, 0, ld}}, T); };
    f->last_seq = S;
    if (gemm_fwd(f, view({x}, T), P + L[0].w, NB_FEATURES, f->nd, plain(f->d, f->nd), P + L[0].b, L[0].act, R)) return -1;
    if (gemm_fwd(f, view({dsrc}, T), P + L[1].w, f->nd, 3 * f->nv, plain(f->scratch, 3 * f->nv), P + L[1].b, ACT_NONE, R)) return -1;
    if (gru_fwd(f, 0, S)) return -1;
    if (gemm_fwd(f, view({hsrc(f, 0)}, T), P + L[5].w, f->nv, 1, plain(f->vad, 1), P + L[5].b, L[5].act, R)) return -1;
    if (gemm_fwd(f, view({dsrc, hsrc(f, 0), x}, T), P + L[2].w, L[2].ni, 3 * f->nn, plain(f->scratch, 3 * f->nn), P + L[2].b, ACT_NONE, R))
        return -1;
    if (gru_fwd(f, 1, S)) return -1;
    if (gemm_fwd(f, view({hsrc(f, 0), hsrc(f, 1), x}, T), P + L[3].w, L[3].ni, 3 * f->ndn, plain(f->scratch, 3 * f->ndn), P + L[3].b,
                 ACT_NONE, R))
        return -1;
    if (gru_fwd(f, 2, S)) return -1;
    if (gemm_fwd(f, view({hsrc(f, 2)}, T), P + L[4].w, f->ndn, NB_BANDS, plain(f->gains, NB_BANDS), P + L[4].b, L[4].act, R))
        return -1;
    fit_loss_kernel<<<(unsigned)((R + 255) / 256), 256, 0, f->stream>>>(f->rows, f->wts, f->gains, f->vad, f->dzo, f->dzv, f->rowloss, R,
                                                                        (float)(1.0 / (double)R));
    fit_finish_kernel<<<1, 512, 0, f->stream>>>(f->rowloss, R, P, f->l2, f->out);
    count_launches(2);
    CK(cudaGetLastError());
    return 0;
}

// weight gradients of GRU i (layer i + 1) from dG in scratch; X = its input view
int gru_wgrads(RNNoiseFit* f, int i, const View& X, long R) {
    const Layer& L = f->L[i + 1];
    const int n = L.nn, n3 = 3 * n;
    float* G = f->grads;
    if (gemm_wgrad(f, X, L.ni, f->scratch, n3, n3, G + L.w, n3, R)) return -1;
    if (gemm_wgrad(f, view({{f->hbuf[i], n, 1, n}}, f->T), n, f->scratch, n3, 2 * n, G + L.u, n3, R)) return -1;  // h_{t-1}^T dG_zr
    if (gemm_wgrad(f, view({{f->rh[i], n, 0, n}}, f->T), n, f->scratch + 2 * n, n3, n, G + L.u + 2 * n, n3, R)) return -1;
    return gemm_wgrad(f, view({{nullptr, 0, 0, 1}}, f->T), 1, f->scratch, n3, n3, G + L.b, n3, R);
}

int backward(RNNoiseFit* f, int S) {
    const int T = f->T;
    const long R = (long)S * T;
    const Layer* L = f->L;
    float *P = f->params, *G = f->grads;
    const int nd = f->nd, nv = f->nv, nn = f->nn, ndn = f->ndn;
    const Src x{f->rows, TRAIN_ROW, 0, NB_FEATURES};
    const Src dsrc{f->d, nd, 0, nd};
    const View ones = view({{nullptr, 0, 0, 1}}, T);
    CK(cudaMemsetAsync(f->dd, 0, (size_t)R * nd * sizeof(float), f->stream));
    for (int i = 0; i < 3; i++) CK(cudaMemsetAsync(f->dh[i], 0, (size_t)R * L[i + 1].nn * sizeof(float), f->stream));
    // denoise_output and vad_output
    if (gemm_wgrad(f, view({hsrc(f, 2)}, T), ndn, f->dzo, NB_BANDS, NB_BANDS, G + L[4].w, NB_BANDS, R) ||
        gemm_wgrad(f, ones, 1, f->dzo, NB_BANDS, NB_BANDS, G + L[4].b, NB_BANDS, R) ||
        gemm_dx(f, f->dzo, NB_BANDS, P + L[4].w, ndn, view({{f->dh[2], ndn, 0, ndn}}, T), R))
        return -1;
    if (gemm_wgrad(f, view({hsrc(f, 0)}, T), nv, f->dzv, 1, 1, G + L[5].w, 1, R) || gemm_wgrad(f, ones, 1, f->dzv, 1, 1, G + L[5].b, 1, R) ||
        gemm_dx(f, f->dzv, 1, P + L[5].w, nv, view({{f->dh[0], nv, 0, nv}}, T), R))
        return -1;
    // denoise_gru: input [vad_h | noise_h | x]
    if (gru_bwd(f, 2, S) || gru_wgrads(f, 2, view({hsrc(f, 0), hsrc(f, 1), x}, T), R) ||
        gemm_dx(f, f->scratch, 3 * ndn, P + L[3].w, nv + nn, view({{f->dh[0], nv, 0, nv}, {f->dh[1], nn, 0, nn}}, T), R))
        return -1;
    // noise_gru: input [dense | vad_h | x]
    if (gru_bwd(f, 1, S) || gru_wgrads(f, 1, view({dsrc, hsrc(f, 0), x}, T), R) ||
        gemm_dx(f, f->scratch, 3 * nn, P + L[2].w, nd + nv, view({{f->dd, nd, 0, nd}, {f->dh[0], nv, 0, nv}}, T), R))
        return -1;
    // vad_gru: input dense
    if (gru_bwd(f, 0, S) || gru_wgrads(f, 0, view({dsrc}, T), R) ||
        gemm_dx(f, f->scratch, 3 * nv, P + L[1].w, nd, view({{f->dd, nd, 0, nd}}, T), R))
        return -1;
    // input_dense
    fit_dense_bwd_kernel<<<(unsigned)((R * nd + 255) / 256), 256, 0, f->stream>>>(f->dd, f->d, R * nd, L[0].act);
    count_launches(1);
    CK(cudaGetLastError());
    if (gemm_wgrad(f, view({x}, T), NB_FEATURES, f->dd, nd, nd, G + L[0].w, nd, R) || gemm_wgrad(f, ones, 1, f->dd, nd, nd, G + L[0].b, nd, R))
        return -1;
    return 0;
}

int check_call(const RNNoiseFit* f, const float* rows, const float* wts, int S) {
    if (!f || !rows || !wts) return fail("null argument");
    if (S <= 0 || S > f->max_seq) return fail("n_seq must be in 1.." + std::to_string(f->max_seq));
    return 0;
}

int fit_init(RNNoiseFit* f) {
    ON_DEVICE(f->device);
    const size_t R = (size_t)f->max_seq * f->T;
    const int w[3] = {f->nv, f->nn, f->ndn};
    const int nmax = std::max(f->nv, std::max(f->nn, f->ndn));
    size_t mn = 0;
    for (int i = 0; i < 6; i++) mn = std::max(mn, (size_t)std::max(f->L[i].ni, f->L[i].nn) * f->L[i].gates * f->L[i].nn);
    f->part_elems = (size_t)FIT_SPLITS_MAX * mn;
    CK(cudaStreamCreateWithFlags(f->stream.put(), cudaStreamNonBlocking));
    CK(dalloc(&f->mem, &f->params, f->n_params));
    CK(dalloc(&f->mem, &f->grads, f->n_params));
    CK(dalloc(&f->mem, &f->m, f->n_params));
    CK(dalloc(&f->mem, &f->v, f->n_params));
    CK(dalloc(&f->mem, &f->rows, R * TRAIN_ROW));
    CK(dalloc(&f->mem, &f->wts, R));
    CK(dalloc(&f->mem, &f->d, R * f->nd));
    CK(dalloc(&f->mem, &f->dd, R * f->nd));
    CK(dalloc(&f->mem, &f->scratch, R * 3 * nmax));
    CK(dalloc(&f->mem, &f->gains, R * NB_BANDS));
    CK(dalloc(&f->mem, &f->vad, R));
    CK(dalloc(&f->mem, &f->dzo, R * NB_BANDS));
    CK(dalloc(&f->mem, &f->dzv, R));
    CK(dalloc(&f->mem, &f->rowloss, R * 3));
    CK(dalloc(&f->mem, &f->part, f->part_elems));
    CK(dalloc(&f->mem, &f->out, 4));
    for (int i = 0; i < 3; i++) {
        CK(dalloc(&f->mem, &f->gates[i], R * 3 * w[i]));
        CK(dalloc(&f->mem, &f->rh[i], R * w[i]));
        CK(dalloc(&f->mem, &f->hbuf[i], (size_t)f->max_seq * (f->T + 1) * w[i]));
        CK(dalloc(&f->mem, &f->dh[i], R * w[i]));
    }
    CK(cudaMemset(f->params, 0, f->n_params * sizeof(float)));
    CK(cudaMemset(f->grads, 0, f->n_params * sizeof(float)));
    CK(cudaMemset(f->m, 0, f->n_params * sizeof(float)));
    CK(cudaMemset(f->v, 0, f->n_params * sizeof(float)));
    for (int i = 0; i < 3; i++) {
        const Layer& L = f->L[i + 1];
        f->l2.off[2 * i] = L.w;
        f->l2.len[2 * i] = (long)L.ni * 3 * L.nn;
        f->l2.off[2 * i + 1] = L.u;
        f->l2.len[2 * i + 1] = 3L * L.nn * L.nn;
    }
    return 0;
}

int reset_adam(RNNoiseFit* f) {
    f->step_count = 0;
    CK(cudaMemsetAsync(f->m, 0, f->n_params * sizeof(float), f->stream));
    CK(cudaMemsetAsync(f->v, 0, f->n_params * sizeof(float), f->stream));
    return 0;
}

int read_out(RNNoiseFit* f, double* out, int n) {
    double h[4];
    CK(cudaMemcpyAsync(h, f->out, sizeof(h), cudaMemcpyDeviceToHost, f->stream));
    CK(cudaStreamSynchronize(f->stream));
    for (int i = 0; i < n; i++) out[i] = h[i];
    return 0;
}

}  // namespace

extern "C" {

RNNoiseFit* rnnoise_fit_create(int nd, int nv, int nn, int ndn, int max_sequences, int window, int device) {
    const int w[4] = {nd, nv, nn, ndn};
    for (int x : w)
        if (x < 1 || x > FIT_MAX_WIDTH) {
            fail("layer widths must be in 1..96");
            return nullptr;
        }
    if (max_sequences < 1 || window < 1 || (double)max_sequences * window > 1e9) {
        fail("max_sequences and window must be positive (and their product at most 1e9)");
        return nullptr;
    }
    if (open_device(device, &device)) return nullptr;
    std::unique_ptr<RNNoiseFit, FitRelease> f(new (std::nothrow) RNNoiseFit());
    if (!f) {
        fail("out of memory");
        return nullptr;
    }
    f->device = device;
    f->nd = nd, f->nv = nv, f->nn = nn, f->ndn = ndn;
    f->max_seq = max_sequences;
    f->T = window;
    f->n_params = layout(nd, nv, nn, ndn, f->L);
    return fit_init(f.get()) ? nullptr : f.release();
}

void rnnoise_fit_destroy(RNNoiseFit* f) {
    if (f) FitRelease()(f);
}

long rnnoise_fit_n_params(const RNNoiseFit* f) { return f ? f->n_params : 0; }

int rnnoise_fit_get_params(RNNoiseFit* f, float* params) {
    if (!f || !params) return fail("null argument");
    ON_DEVICE(f->device);
    CK(cudaMemcpyAsync(params, f->params, f->n_params * sizeof(float), cudaMemcpyDeviceToHost, f->stream));
    CK(cudaStreamSynchronize(f->stream));
    return 0;
}

int rnnoise_fit_set_params(RNNoiseFit* f, const float* params) {
    if (!f || !params) return fail("null argument");
    ON_DEVICE(f->device);
    CK(cudaMemcpyAsync(f->params, params, f->n_params * sizeof(float), cudaMemcpyHostToDevice, f->stream));
    if (reset_adam(f)) return -1;
    CK(cudaStreamSynchronize(f->stream));
    return 0;
}

int rnnoise_fit_set_params_from_model(RNNoiseFit* f, const RNNModel* model) {
    if (!f) return fail("null argument");
    const size_t nb = rnnoise_model_bytes(model, nullptr, 0);
    std::vector<unsigned char> bytes(nb);
    rnnoise_model_bytes(model, bytes.data(), nb);
    HostModel hm;
    if (!HostModel::parse(bytes.data(), nb, &hm)) return fail("model does not parse");
    const HostDense* dense[3] = {&hm.input_dense, &hm.denoise_output, &hm.vad_output};
    const HostGru* gru[3] = {&hm.vad_gru, &hm.noise_gru, &hm.denoise_gru};
    if (hm.input_dense.nn != f->nd || hm.vad_gru.nn != f->nv || hm.noise_gru.nn != f->nn || hm.denoise_gru.nn != f->ndn)
        return fail("model widths differ from the fit's");
    if (hm.denoise_output.act != ACT_SIGMOID || hm.vad_output.act != ACT_SIGMOID)
        return fail("the loss needs sigmoid output layers (activation 1)");
    const int acts[4] = {hm.input_dense.act, hm.vad_gru.act, hm.noise_gru.act, hm.denoise_gru.act};
    for (int a : acts)
        if (a < ACT_TANH || a > ACT_RELU) return fail("unknown activation in the model");
    std::vector<float> p(f->n_params);
    auto put = [&](long off, size_t src, size_t n) {
        for (size_t i = 0; i < n; i++) p[off + i] = (float)hm.bytes[src + i] / 256.0f;
    };
    const int di[3] = {0, 4, 5};
    for (int i = 0; i < 3; i++) {
        const Layer& L = f->L[di[i]];
        put(L.w, dense[i]->w_off, (size_t)L.ni * L.nn);
        put(L.b, dense[i]->b_off, L.nn);
    }
    for (int i = 0; i < 3; i++) {
        const Layer& L = f->L[i + 1];
        put(L.w, gru[i]->w_off, (size_t)L.ni * 3 * L.nn);
        put(L.u, gru[i]->r_off, (size_t)3 * L.nn * L.nn);
        put(L.b, gru[i]->b_off, (size_t)3 * L.nn);
    }
    if (rnnoise_fit_set_params(f, p.data())) return -1;
    for (int i = 0; i < 4; i++) f->L[i].act = acts[i];
    return 0;
}

int rnnoise_fit_step(RNNoiseFit* f, const float* rows, const float* weights, int n_seq, double* loss) {
    if (check_call(f, rows, weights, n_seq)) return -1;
    ON_DEVICE(f->device);
    if (load_inputs(f, rows, weights, n_seq) || forward(f, n_seq) || backward(f, n_seq)) return -1;
    f->step_count++;
    const double t = (double)f->step_count;
    const float lr_t = (float)(1e-3 * std::sqrt(1.0 - std::pow(0.999, t)) / (1.0 - std::pow(0.9, t)));
    fit_adam_kernel<<<(unsigned)((f->n_params + 255) / 256), 256, 0, f->stream>>>(f->params, f->grads, f->m, f->v, f->n_params, f->l2,
                                                                                 lr_t);
    count_launches(1);
    CK(cudaGetLastError());
    double out[1];
    if (read_out(f, out, 1)) return -1;
    if (loss) *loss = out[0];
    return 0;
}

int rnnoise_fit_evaluate(RNNoiseFit* f, const float* rows, const float* weights, int n_seq, double out[4]) {
    if (check_call(f, rows, weights, n_seq)) return -1;
    if (!out) return fail("null argument");
    ON_DEVICE(f->device);
    if (load_inputs(f, rows, weights, n_seq) || forward(f, n_seq)) return -1;
    return read_out(f, out, 4);
}

int rnnoise_fit_get_grads(RNNoiseFit* f, float* grads) {
    if (!f || !grads) return fail("null argument");
    ON_DEVICE(f->device);
    CK(cudaMemcpyAsync(grads, f->grads, f->n_params * sizeof(float), cudaMemcpyDeviceToHost, f->stream));
    CK(cudaStreamSynchronize(f->stream));
    return 0;
}

int rnnoise_fit_get_activations(RNNoiseFit* f, float* gains, float* vad, float* state) {
    if (!f) return fail("null argument");
    ON_DEVICE(f->device);
    const int S = f->last_seq, T = f->T;
    const size_t R = (size_t)S * T;
    if (gains) CK(cudaMemcpyAsync(gains, f->gains, R * NB_BANDS * sizeof(float), cudaMemcpyDeviceToHost, f->stream));
    if (vad) CK(cudaMemcpyAsync(vad, f->vad, R * sizeof(float), cudaMemcpyDeviceToHost, f->stream));
    if (state) {
        const int w[3] = {f->nv, f->nn, f->ndn}, ld = f->nv + f->nn + f->ndn;
        int c = 0;
        for (int i = 0; i < 3; i++) {  // h_t of sequence s, frame t: hbuf row s * (T + 1) + t + 1
            for (int s = 0; s < S; s++)
                CK(cudaMemcpy2DAsync(state + ((size_t)s * T) * ld + c, ld * sizeof(float), f->hbuf[i] + ((size_t)s * (T + 1) + 1) * w[i],
                                      w[i] * sizeof(float), w[i] * sizeof(float), T, cudaMemcpyDeviceToHost, f->stream));
            c += w[i];
        }
    }
    CK(cudaStreamSynchronize(f->stream));
    return 0;
}

}  // extern "C"

namespace {

size_t export_layers(const Layer L[6], long np, const float* params, unsigned char* buf, size_t cap) {
    if (L[2].ni > 127 || L[3].ni > 127) {
        fail("the .rnn format stores a layer's input count in a signed byte: 42 + nd + nv and 42 + nv + nn must be <= 127");
        return 0;
    }
    const size_t size = 6 * 3 + (size_t)np;
    if (!buf) return size;
    if (!params) {
        fail("null argument");
        return 0;
    }
    if (cap < size) {
        fail("buffer too small: " + std::to_string(size) + " bytes needed");
        return 0;
    }
    // dump_rnn.py: header [inputs, neurons, activation], then every weight as clip(round(256 w), -128, 127) with
    // round half to even (Python's round); the parameter vector is already in file order.
    size_t p = 0;
    long q = 0;
    for (int i = 0; i < 6; i++) {
        buf[p++] = (unsigned char)L[i].ni;
        buf[p++] = (unsigned char)L[i].nn;
        buf[p++] = (unsigned char)L[i].act;
        const long end = i + 1 < 6 ? L[i + 1].w : np;
        for (; q < end; q++) {
            const float r = std::nearbyint(256.0f * params[q]);
            buf[p++] = (unsigned char)(signed char)std::fmin(std::fmax(r, -128.0f), 127.0f);
        }
    }
    return size;
}

}  // namespace

extern "C" {

size_t rnnoise_fit_export_params(int nd, int nv, int nn, int ndn, const float* params, unsigned char* buf, size_t cap) {
    const int w[4] = {nd, nv, nn, ndn};
    for (int x : w)
        if (x < 1 || x > FIT_MAX_WIDTH) {
            fail("layer widths must be in 1..96");
            return 0;
        }
    Layer L[6];
    const long np = layout(nd, nv, nn, ndn, L);
    return export_layers(L, np, params, buf, cap);
}

size_t rnnoise_fit_export(RNNoiseFit* f, unsigned char* buf, size_t cap) {
    if (!f) {
        fail("null argument");
        return 0;
    }
    std::vector<float> p(f->n_params);
    if (buf && rnnoise_fit_get_params(f, p.data())) return 0;
    return export_layers(f->L, f->n_params, p.data(), buf, cap);
}

}  // extern "C"
