// rnn_mma.cu -- the GRU network (src/rnn.rs:251-379) on tensor cores, batched across streams.
//
// One block advances TS = 32 streams.  With 32 streams side by side every layer is a real dense contraction
// [32 x K] x [K x N] (K up to 224, N up to 192), so it runs as mma.sync.m16n8k16 (f16 inputs, f32 accumulate):
//   * weights are int8 -> exactly representable in f16; pre-packed on the host in B-fragment order, so a warp
//     fetches a whole 16x8 fragment with one coalesced 256-byte load and reuses it for both 16-stream row tiles
//     and for the hi and lo halves of the activations;
//   * activations are f32; each is split x = hi + lo (two f16, ~22 significant bits) and both halves are
//     multiplied -- products are exact in f32, only the summation order differs from the reference's;
//   * per GRU a warp owns the same output columns for z, r and the candidate, so z stays in registers and the
//     update h = z h + (1-z) h~ happens in the accumulator layout without a transpose.
// Activations: src/util.rs:29-53 (table tanh, sigmoid = .5 + .5 tanh(x/2), relu) chosen per layer at run time.
// GRU semantics: src/rnn.rs:292-327 (reset gate applied to the state BEFORE the recurrent product).
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_fp16.h>

#include "common.cuh"
#include "model.hpp"

namespace nnb {

namespace {

constexpr int TS = 32;      // streams per block = two m16 row tiles
constexpr int NWARP = 8;
constexpr int NT = NWARP * 32;
constexpr int MIN_BLOCKS = 2;  // per SM (__launch_bounds__)
constexpr int MAXOT = 16 / NWARP;  // output tiles (8 neurons) per warp: NWARP * MAXOT tiles cover layers up to 128 neurons
constexpr float WEIGHTS_SCALE = 1.0f / 256.0f;

// src/util.rs:3-27, branch-free (the lanes of a warp hold different neurons): same arithmetic on |x| clamped to 8, the
// saturations (NaN -> 1 like the reference's `!(x < 8)`) applied as selects at the end.
__device__ __forceinline__ float tansig_approx(float x, const float* __restrict__ table) {
    const float sign = (x < 0.0f) ? -1.0f : 1.0f;
    float ax = fminf(fabsf(x), 8.0f);  // fminf(NaN, 8) = 8: the table index stays in range
    const float fi = floorf(0.5f + 25.0f * ax);
    ax -= 0.04f * fi;
    float y = table[(int)fi];
    const float dy = 1.0f - y * y;
    y = y + ax * dy * (1.0f - y * ax);
    y = sign * y;
    y = !(x > -8.0f) ? -1.0f : y;
    return !(x < 8.0f) ? 1.0f : y;
}
__device__ __forceinline__ float sigmoid_approx(float x, const float* __restrict__ table) {
    return 0.5f + 0.5f * tansig_approx(0.5f * x, table);
}
__device__ __forceinline__ float activate(int act, float x, const float* __restrict__ table) {
    if (act == 0) return tansig_approx(x, table);
    if (act == 1) return sigmoid_approx(x, table);
    return fmaxf(x, 0.0f);
}

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], const uint2 b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}

// x = hi + lo with hi, lo in f16.  No clamp: |x| >= 65520 (only an unbounded ReLU layer of a custom model can get
// there; below it hi rounds to 65504 and stays finite) becomes +-inf in hi and -+inf in lo, i.e. NaN in every product.
// The tables map a NaN pre-activation to 1 (as the reference does) and ReLU maps it to 0, which would hide it, so the
// split reports the overflow (true): the stream's vad and gains of the frame are then NaN.  The bundled models
// (tanh / sigmoid, |x| <= 1) and the 42 features are far inside the range.
__device__ __forceinline__ bool split_f16(float x, __half& hi, __half& lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
    return __hisinf(hi) != 0;
}
// two adjacent columns (col even) of one row; an f16 overflow marks the row in ovf
__device__ __forceinline__ void store_pair(__half* Ahi, __half* Alo, int idx, float v0, float v1, int* ovf, int row) {
    __half h0, l0, h1, l1;
    const bool o0 = split_f16(v0, h0, l0), o1 = split_f16(v1, h1, l1);
    if (o0 || o1) ovf[row] = 1;
    *reinterpret_cast<__half2*>(Ahi + idx) = __halves2half2(h0, h1);
    *reinterpret_cast<__half2*>(Alo + idx) = __halves2half2(l0, l1);
}

__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t smem_addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr)
                 : "memory");
}

// Output tiles of a warp: tile(i, gate) = gate * ot + warp + i * NWARP for i < cnt (gate 0 only, or z | r of a GRU).
// acc[i * NGATE + gate][mt][.] += A[:, phase columns] x W[:, tile(i, gate)], both 16-stream row tiles mt.
// One fragment pointer per GATE walks the chunks; the warp's other tiles sit at compile-time offsets from it.
template <int NGATE, int MO>
__device__ __forceinline__ void run_tiles(const MmaPhase& ph, const unsigned char* img, const __half* Ahi, const __half* Alo, int kp, int lane, int warp,
                                          int ot, int cnt, float (&acc)[NGATE * MO][2][4]) {
    constexpr int TSTEP = NWARP * 32;  // fragments between a warp's consecutive tiles
    const uint2* wg[NGATE];
#pragma unroll
    for (int gt = 0; gt < NGATE; gt++) wg[gt] = reinterpret_cast<const uint2*>(img + ph.w_off) + (size_t)(gt * ot + warp) * 32 + lane;
    const int wstep = ph.ntiles * 32;
    uint2 bn[NGATE * MO];
#pragma unroll
    for (int i = 0; i < MO; i++)
#pragma unroll
        for (int gt = 0; gt < NGATE; gt++) bn[i * NGATE + gt] = (i < cnt) ? __ldg(wg[gt] + i * TSTEP) : make_uint2(0u, 0u);
    // A fragments by ldmatrix: one x4 load = the 16x16 f16 tile in mma fragment order.  Lane l supplies the address of
    // row (l & 7) + 8 ((l >> 3) & 1), column 8 (l >> 4) of the tile; rows are kp halves apart (kp = 8 mod 16: 16-byte
    // aligned rows whose 8 addresses fall into 8 different 16-byte bank groups).
    const int rb = ((lane & 7) + ((lane >> 3) & 1) * 8) * kp + (lane >> 4) * 8;
    const uint32_t ah_base = (uint32_t)__cvta_generic_to_shared(Ahi + rb);
    const uint32_t al_base = (uint32_t)__cvta_generic_to_shared(Alo + rb);
    const uint32_t r16b = 32u * (uint32_t)kp;  // 16 rows further, in bytes
    const int nch = ph.nchunks;
    auto chunk = [&](int kc, const uint2 (&b)[NGATE * MO]) {
        const uint32_t cb = 2u * (uint32_t)ph.col[kc];
        uint32_t ah[2][4], al[2][4];
        ldsm4(ah[0], ah_base + cb);
        ldsm4(ah[1], ah_base + cb + r16b);
        ldsm4(al[0], al_base + cb);
        ldsm4(al[1], al_base + cb + r16b);
#pragma unroll
        for (int i = 0; i < MO; i++) {
            if (i < cnt) {
#pragma unroll
                for (int gt = 0; gt < NGATE; gt++)
#pragma unroll
                    for (int mt = 0; mt < 2; mt++) {
                        mma16816(acc[i * NGATE + gt][mt], ah[mt], b[i * NGATE + gt]);
                        mma16816(acc[i * NGATE + gt][mt], al[mt], b[i * NGATE + gt]);
                    }
            }
        }
    };
    auto fetch = [&](uint2 (&dst)[NGATE * MO]) {  // fragments of the next chunk
#pragma unroll
        for (int gt = 0; gt < NGATE; gt++) wg[gt] += wstep;
#pragma unroll
        for (int i = 0; i < MO; i++)
#pragma unroll
            for (int gt = 0; gt < NGATE; gt++)
                if (i < cnt) dst[i * NGATE + gt] = __ldg(wg[gt] + i * TSTEP);
    };
    // two fragment buffers used alternately (chunk loop unrolled by two): the next chunk's fragments are in flight
    // while this chunk's MMAs run, and no register copies are needed between iterations
    uint2 bm[NGATE * MO];
#pragma unroll
    for (int i = 0; i < NGATE * MO; i++) bm[i] = make_uint2(0u, 0u);
    int kc = 0;
#pragma unroll 1
    for (; kc + 1 < nch; kc += 2) {
        fetch(bm);
        chunk(kc, bn);
        if (kc + 2 < nch) fetch(bn);
        chunk(kc + 1, bm);
    }
    if (kc < nch) chunk(kc, bn);
}

template <int NGATE, int MO>
__device__ __forceinline__ void init_bias(const MmaPhase& ph, const unsigned char* img, int lane, int warp, int ot, int cnt, float (&acc)[NGATE * MO][2][4]) {
    const int t = lane & 3;
#pragma unroll
    for (int i = 0; i < MO; i++)
#pragma unroll
        for (int gt = 0; gt < NGATE; gt++) {
            float b0 = 0.0f, b1 = 0.0f;
            if (i < cnt) {
                const float2 bv = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(img + ph.b_off) + (gt * ot + warp + i * NWARP) * 8 + 2 * t));
                b0 = bv.x;
                b1 = bv.y;
            }
#pragma unroll
            for (int mt = 0; mt < 2; mt++) {
                acc[i * NGATE + gt][mt][0] = b0;
                acc[i * NGATE + gt][mt][1] = b1;
                acc[i * NGATE + gt][mt][2] = b0;
                acc[i * NGATE + gt][mt][3] = b1;
            }
        }
}

// One GRU layer for the block's 32 streams.  c_state: A columns of this layer's state; s_off: its offset in Hf.
#ifdef RNN_NOINLINE
#define RNN_GRU_ATTR __noinline__
#else
#define RNN_GRU_ATTR
#endif
__device__ RNN_GRU_ATTR void gru_layer(const MmaPhase& pzr, const MmaPhase& ph, const unsigned char* img, int act, int nn, int c_state, int c_rh, int s_off,
                          __half* Ahi, __half* Alo, int kp, float* Hf, int hs, const float* table, int* ovf) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int ot = (nn + 7) >> 3;  // output tiles of this layer
    int own[MAXOT], cnt = 0;
#pragma unroll
    for (int i = 0; i < MAXOT; i++) {
        own[i] = warp + i * NWARP;
        if (own[i] < ot) cnt = i + 1;
    }
    float zreg[MAXOT][2][4];
    {
        // z | r gates: tiles {z_j, r_j} for the owned output tiles j
        float acc[2 * MAXOT][2][4];
        init_bias<2, MAXOT>(pzr, img, lane, warp, ot, cnt, acc);
        run_tiles<2, MAXOT>(pzr, img, Ahi, Alo, kp, lane, warp, ot, cnt, acc);
#pragma unroll
        for (int i = 0; i < MAXOT; i++) {
            if (i < cnt) {
#pragma unroll
                for (int mt = 0; mt < 2; mt++) {
#pragma unroll
                    for (int hf = 0; hf < 2; hf++) {  // rows g and g + 8
                        const int row = mt * 16 + g + 8 * hf, o = own[i] * 8 + 2 * t;
                        float rh[2];
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            const float z = sigmoid_approx(WEIGHTS_SCALE * acc[2 * i][mt][2 * hf + c], table);
                            const float r = sigmoid_approx(WEIGHTS_SCALE * acc[2 * i + 1][mt][2 * hf + c], table);
                            zreg[i][mt][2 * hf + c] = z;
                            rh[c] = r * Hf[row * hs + s_off + o + c];  // reset gate scales the previous state
                        }
                        store_pair(Ahi, Alo, row * kp + c_rh + o, rh[0], rh[1], ovf, row);
                    }
                }
            }
        }
    }
    __syncthreads();
    {
        float acc[MAXOT][2][4];
        init_bias<1, MAXOT>(ph, img, lane, warp, 0, cnt, acc);
        run_tiles<1, MAXOT>(ph, img, Ahi, Alo, kp, lane, warp, 0, cnt, acc);
#pragma unroll
        for (int i = 0; i < MAXOT; i++) {
            if (i < cnt) {
#pragma unroll
                for (int mt = 0; mt < 2; mt++) {
#pragma unroll
                    for (int hf = 0; hf < 2; hf++) {
                        const int row = mt * 16 + g + 8 * hf, o = own[i] * 8 + 2 * t;
                        float hn[2];
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            const float z = zreg[i][mt][2 * hf + c];
                            const float hh = activate(act, WEIGHTS_SCALE * acc[i][mt][2 * hf + c], table);
                            const float hp = Hf[row * hs + s_off + o + c];
                            hn[c] = (o + c < nn) ? z * hp + (1.0f - z) * hh : 0.0f;
                            Hf[row * hs + s_off + o + c] = hn[c];
                        }
                        store_pair(Ahi, Alo, row * kp + c_state + o, hn[0], hn[1], ovf, row);
                    }
                }
            }
        }
    }
    __syncthreads();
}

// kMulti = false: block b advances batch rows [32 b, 32 b + 32) on the model at `image` with activation codes `acts`.
// kMulti = true (DESIGN.md 7c): block b advances tile b of the table mtab, on its own model of the table whose model 0
// is at `image` (same geometry, so the same descriptor m; the model's image lies model x stride bytes further, its
// activation codes come with the tile).
template <bool kMulti>
__global__ void __launch_bounds__(NT, MIN_BLOCKS) rnn_mma_kernel(BatchBuffers bb, DeviceModelMma m, const unsigned char* image, int acts,
                                                                 ModelTiles mtab) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int kp = m.kp, hs = m.hs;
    __half* Ahi = reinterpret_cast<__half*>(smraw);
    __half* Alo = Ahi + TS * kp;
    float* Hf = reinterpret_cast<float*>(Alo + TS * kp);
    float* table = Hf + TS * hs;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int s0 = blockIdx.x * TS;
    // kMulti: the tile's model (image and activation codes) and rows.  The TILE_STREAM select below folds at compile
    // time: the kMulti = false instantiation reads batch row s0 + row exactly as the one-model kernel always has.
    int t_first = 0, t_count = 0;
    if constexpr (kMulti) {
        const int4 tl = __ldg(reinterpret_cast<const int4*>(mtab.tile + blockIdx.x));  // {model, first, count, acts}
        image += (size_t)tl.x * mtab.stride;
        t_first = tl.y;
        t_count = tl.z;
        acts = tl.w;
    }
#define TILE_STREAM(row) (kMulti ? __ldg(mtab.rows + t_first + (row)) : s0 + (row))
    const int ns = kMulti ? t_count : min(TS, bb.n_streams - s0);
    const int SS = m.state_size;
    const int so_v = 0, so_n = (m.nv + 7) & ~7, so_d = so_n + ((m.nn + 7) & ~7);  // state offsets inside an Hf row

    // zero A (padding columns must hold finite values) and Hf, load the tanh table
    {
        uint32_t* z = reinterpret_cast<uint32_t*>(smraw);
        const int nz = (TS * kp * 2 * 2 + TS * hs * 4) / 4;
        for (int i = tid; i < nz; i += NT) z[i] = 0u;
        for (int i = tid; i < 201; i += NT) table[i] = __ldg(reinterpret_cast<const float*>(image + m.table_off) + i);
    }
    __shared__ int ovf[TS];  // rows with an f16 overflow in an operand (split_f16)
    if (tid < TS) ovf[tid] = 0;
    __syncthreads();
    {
        // features [ns][42] and GRU state [ns][SS]: warp w takes rows w, w + NWARP, ...; lane l the columns l, l + 32, ...
        // (coalesced row segments, no index divisions); every load of a thread is in flight before the first use.
        constexpr int RPW = TS / NWARP;                 // rows per warp
        constexpr int SK = (3 * MAX_NEURONS + 31) / 32;  // column slots per lane for the state (SS <= 3 * 128)
        const float* fsrc = bb.features + (size_t)s0 * NB_FEATURES;
        const float* ssrc = bb.gru_state + (size_t)s0 * SS;
        const int nsk = (SS + 31) >> 5;
        // A column / Hf column of state element j (the three GRU states are packed back to back in HBM)
        int acol[SK], hcol[SK];
#pragma unroll
        for (int k = 0; k < SK; k++) {
            const int j = lane + 32 * k;
            if (j < m.nv) { acol[k] = m.c_vad + j; hcol[k] = so_v + j; }
            else if (j < m.nv + m.nn) { acol[k] = m.c_noise + (j - m.nv); hcol[k] = so_n + (j - m.nv); }
            else { acol[k] = m.c_den + (j - m.nv - m.nn); hcol[k] = so_d + (j - m.nv - m.nn); }
        }
#pragma unroll 1
        for (int r = 0; r < RPW; r++) {
            const int row = warp + r * NWARP;
            if (row >= ns) break;
            float sv[SK], f0, f1 = 0.0f;
#pragma unroll
            for (int k = 0; k < SK; k++)
                sv[k] = (k < nsk && lane + 32 * k < SS)
                            ? __ldg((kMulti ? bb.gru_state + (size_t)TILE_STREAM(row) * SS : ssrc + (size_t)row * SS) + lane + 32 * k)
                            : 0.0f;
            f0 = __ldg((kMulti ? bb.features + (size_t)TILE_STREAM(row) * NB_FEATURES : fsrc + row * NB_FEATURES) + lane);
            if (lane + 32 < NB_FEATURES)
                f1 = __ldg((kMulti ? bb.features + (size_t)TILE_STREAM(row) * NB_FEATURES : fsrc + row * NB_FEATURES) + lane + 32);
            __half* ahr = Ahi + row * kp;
            __half* alr = Alo + row * kp;
            float* hfr = Hf + row * hs;
#pragma unroll
            for (int k = 0; k < SK; k++) {
                if (k < nsk && lane + 32 * k < SS) {
                    hfr[hcol[k]] = sv[k];
                    __half hi, lo;
                    if (split_f16(sv[k], hi, lo)) ovf[row] = 1;
                    ahr[acol[k]] = hi;
                    alr[acol[k]] = lo;
                }
            }
            {
                __half hi, lo;
                if (split_f16(f0, hi, lo)) ovf[row] = 1;
                ahr[m.c_feat + lane] = hi;
                alr[m.c_feat + lane] = lo;
                if (lane + 32 < NB_FEATURES) {
                    if (split_f16(f1, hi, lo)) ovf[row] = 1;
                    ahr[m.c_feat + lane + 32] = hi;
                    alr[m.c_feat + lane + 32] = lo;
                }
            }
        }
    }
    __syncthreads();

    // ---- input_dense (src/rnn.rs:353-355) ----
    {
        const int ntile = (m.nd + 7) >> 3;
        int tiles[MAXOT], cnt = 0;
#pragma unroll
        for (int i = 0; i < MAXOT; i++) {
            tiles[i] = warp + i * NWARP;
            if (tiles[i] < ntile) cnt = i + 1;
        }
        float acc[MAXOT][2][4];
        init_bias<1, MAXOT>(m.dense, image, lane, warp, 0, cnt, acc);
        run_tiles<1, MAXOT>(m.dense, image, Ahi, Alo, kp, lane, warp, 0, cnt, acc);
#pragma unroll
        for (int i = 0; i < MAXOT; i++)
            if (i < cnt)
#pragma unroll
                for (int mt = 0; mt < 2; mt++)
#pragma unroll
                    for (int hf = 0; hf < 2; hf++) {
                        const int row = mt * 16 + g + 8 * hf, o = tiles[i] * 8 + 2 * t;
                        float v[2];
#pragma unroll
                        for (int c = 0; c < 2; c++)
                            v[c] = (o + c < m.nd) ? activate(tile_act(acts, 0), WEIGHTS_SCALE * acc[i][mt][2 * hf + c], table) : 0.0f;
                        store_pair(Ahi, Alo, row * kp + m.c_dense + o, v[0], v[1], ovf, row);
                    }
    }
    __syncthreads();

    // ---- vad_gru (src/rnn.rs:356-358) ----
    gru_layer(m.vad_zr, m.vad_h, image, tile_act(acts, 1), m.nv, m.c_vad, m.c_rh, so_v, Ahi, Alo, kp, Hf, hs, table, ovf);

    // ---- vad_output (src/rnn.rs:359): one neuron -> tile 0, warp 0 (no barrier needed: it only reads the vad state) ----
    if (warp == 0) {
        float acc[1][2][4];
        init_bias<1, 1>(m.vad_out, image, lane, 0, 0, 1, acc);
        run_tiles<1, 1>(m.vad_out, image, Ahi, Alo, kp, lane, 0, 0, 1, acc);
        if (t == 0) {
#pragma unroll
            for (int mt = 0; mt < 2; mt++)
#pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    const int row = mt * 16 + g + 8 * hf;
                    if (row < ns && !bb.silence[TILE_STREAM(row)])
                        bb.vad[TILE_STREAM(row)] =
                            ovf[row] ? __int_as_float(0x7fc00000) : activate(tile_act(acts, 5), WEIGHTS_SCALE * acc[0][mt][2 * hf], table);
                }
        }
    }

    // ---- noise_gru, denoise_gru (src/rnn.rs:361-377) ----
    gru_layer(m.noise_zr, m.noise_h, image, tile_act(acts, 2), m.nn, m.c_noise, m.c_rh, so_n, Ahi, Alo, kp, Hf, hs, table, ovf);
    gru_layer(m.den_zr, m.den_h, image, tile_act(acts, 3), m.ndn, m.c_den, m.c_rh, so_d, Ahi, Alo, kp, Hf, hs, table, ovf);

    // ---- denoise_output (src/rnn.rs:378): 22 band gains ----
    {
        if (warp < (NB_BANDS + 7) / 8) {
            float acc[1][2][4];
            init_bias<1, 1>(m.out, image, lane, warp, 0, 1, acc);
            run_tiles<1, 1>(m.out, image, Ahi, Alo, kp, lane, warp, 0, 1, acc);
#pragma unroll
            for (int mt = 0; mt < 2; mt++)
#pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    const int row = mt * 16 + g + 8 * hf;
                    if (row < ns && !bb.silence[TILE_STREAM(row)]) {
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            const int o = warp * 8 + 2 * t + c;
                            if (o < NB_BANDS)
                                bb.gains[(size_t)TILE_STREAM(row) * NB_BANDS + o] =
                                    ovf[row] ? __int_as_float(0x7fc00000) : activate(tile_act(acts, 4), WEIGHTS_SCALE * acc[0][mt][2 * hf + c], table);
                        }
                    }
                }
        }
    }
    // ---- state write-back; silent frames leave the RNN state untouched (src/denoise.rs:102) ----
    for (int row = warp; row < ns; row += NWARP) {
        if (bb.silence[TILE_STREAM(row)]) continue;
        float* dst = bb.gru_state + (size_t)TILE_STREAM(row) * SS;
        const float* hfr = Hf + row * hs;
        for (int j = lane; j < SS; j += 32) {
            int ho;
            if (j < m.nv) ho = so_v + j;
            else if (j < m.nv + m.nn) ho = so_n + (j - m.nv);
            else ho = so_d + (j - m.nv - m.nn);
            dst[j] = hfr[ho];
        }
    }
#undef TILE_STREAM
}

static_assert(TS == MMA_TILE_ROWS, "tile tables are cut for this kernel's tile");

template <bool kMulti>
cudaError_t launch_mma(const BatchBuffers& b, const DeviceModelMma& m, const unsigned char* image, int acts, const ModelTiles& mt, int grid,
                       cudaStream_t st) {
    const size_t smem = (size_t)TS * m.kp * 2 * 2 + (size_t)TS * m.hs * 4 + 208 * 4;
    static std::atomic<size_t> attr_smem[64];  // zero-initialised; concurrent host threads may race to raise it (idempotent)
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 64 || smem > attr_smem[dev].load(std::memory_order_acquire)) {
        e = cudaFuncSetAttribute(rnn_mma_kernel<kMulti>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        if (dev < 64) {
            size_t cur = attr_smem[dev].load(std::memory_order_relaxed);
            while (cur < smem && !attr_smem[dev].compare_exchange_weak(cur, smem, std::memory_order_release)) {}
        }
    }
    rnn_mma_kernel<kMulti><<<grid, NT, smem, st>>>(b, m, image, acts, mt);
    return cudaGetLastError();
}

// ---- host: the model's weights packed in mma.sync m16n8k16 B-fragment order (see common.cuh MmaPhase) ----
struct Seg {
    int acol, len, recurrent, src_off;  // A column, valid rows, 0 = input matrix / 1 = recurrent matrix, first source row
};

inline int pad16(int n) { return (n + 15) & ~15; }
inline uint32_t pack_h2(int a, int b) {
    return (uint32_t)__half_as_ushort(__float2half((float)a)) | ((uint32_t)__half_as_ushort(__float2half((float)b)) << 16);
}

struct PhaseBuilder {
    std::vector<unsigned char>& blob;  // the image

    // weight(i_seg_row, out_col) -> int8 value; nout valid outputs per gate; ngates gates laid out as consecutive tile groups
    template <typename WF, typename BF>
    void add(MmaPhase* ph, const std::vector<Seg>& segs, int nout, int ngates, WF weight, BF bias) {
        const int ot = (nout + 7) / 8;
        ph->ntiles = ngates * ot;
        ph->nchunks = 0;
        std::vector<std::pair<int, int>> chunks;  // (segment index, first row in segment)
        for (size_t si = 0; si < segs.size(); si++)
            for (int c = 0; c < pad16(segs[si].len); c += 16) {
                if (ph->nchunks >= MMA_MAX_CHUNKS) abort();
                ph->col[ph->nchunks++] = (short)(segs[si].acol + c);
                chunks.push_back({(int)si, c});
            }
        while (blob.size() % 16) blob.push_back(0);
        ph->w_off = (uint32_t)blob.size();
        blob.resize(ph->w_off + (size_t)ph->nchunks * ph->ntiles * 32 * sizeof(uint2));
        uint2* wf = reinterpret_cast<uint2*>(blob.data() + ph->w_off);
        for (int kc = 0; kc < ph->nchunks; kc++) {
            const Seg& sg = segs[chunks[kc].first];
            const int r0 = chunks[kc].second;
            for (int nt = 0; nt < ph->ntiles; nt++) {
                const int gate = nt / ot, o0 = (nt % ot) * 8;
                for (int lane = 0; lane < 32; lane++) {
                    const int g = lane >> 2, t = lane & 3, n = o0 + g;
                    auto w = [&](int kr) -> int {
                        const int i = r0 + kr;
                        if (i >= sg.len || n >= nout) return 0;
                        return weight(sg, i, gate, n);
                    };
                    wf[((size_t)kc * ph->ntiles + nt) * 32 + lane] =
                        make_uint2(pack_h2(w(2 * t), w(2 * t + 1)), pack_h2(w(2 * t + 8), w(2 * t + 9)));
                }
            }
        }
        ph->b_off = (uint32_t)blob.size();
        blob.resize(ph->b_off + (size_t)ph->ntiles * 8 * sizeof(float));
        float* bf = reinterpret_cast<float*>(blob.data() + ph->b_off);
        for (int nt = 0; nt < ph->ntiles; nt++)
            for (int j = 0; j < 8; j++) {
                const int gate = nt / ot, o = (nt % ot) * 8 + j;
                bf[nt * 8 + j] = o < nout ? (float)bias(gate, o) : 0.0f;
            }
    }
};

}  // namespace

bool pack_model(const HostModel& m, DeviceModelMma* dp, std::vector<unsigned char>* blob) {
    std::memset(dp, 0, sizeof *dp);
    blob->clear();
    DeviceModelMma& d = *dp;
    const int nd = m.input_dense.nn, nv = m.vad_gru.nn, nn = m.noise_gru.nn, ndn = m.denoise_gru.nn;
    d.nd = nd; d.nv = nv; d.nn = nn; d.ndn = ndn;
    d.c_feat = 0;
    d.c_dense = pad16(NB_FEATURES);
    d.c_vad = d.c_dense + pad16(nd);
    d.c_noise = d.c_vad + pad16(nv);
    d.c_den = d.c_noise + pad16(nn);
    d.c_rh = d.c_den + pad16(ndn);
    int cols = d.c_rh + pad16(std::max(nv, std::max(nn, ndn)));
    int kp = cols;
    while ((kp / 2) % 8 != 4) kp += 2;
    d.kp = kp;
    int hs = ((nv + 7) & ~7) + ((nn + 7) & ~7) + ((ndn + 7) & ~7);
    while (hs % 32 != 8) hs++;
    d.hs = hs;
    d.state_size = nv + nn + ndn;

    const int8_t* B = m.bytes.data();
    PhaseBuilder pb{*blob};
    auto dense_w = [&](const HostDense& L) {
        return [&, B](const Seg& sg, int i, int, int n) -> int { return B[L.w_off + (size_t)(sg.src_off + i) * L.nn + n]; };
    };
    auto dense_b = [&](const HostDense& L) { return [&, B](int, int o) -> int { return B[L.b_off + o]; }; };
    auto gru_w = [&](const HostGru& L, int gate0) {
        return [&, B, gate0](const Seg& sg, int i, int gate, int n) -> int {
            const size_t st3 = (size_t)3 * L.nn;
            const size_t base = sg.recurrent ? L.r_off : L.w_off;
            return B[base + (size_t)(sg.src_off + i) * st3 + (size_t)(gate0 + gate) * L.nn + n];
        };
    };
    auto gru_b = [&](const HostGru& L, int gate0) { return [&, B, gate0](int gate, int o) -> int { return B[L.b_off + (size_t)(gate0 + gate) * L.nn + o]; }; };

    pb.add(&d.dense, {{d.c_feat, NB_FEATURES, 0, 0}}, nd, 1, dense_w(m.input_dense), dense_b(m.input_dense));
    pb.add(&d.vad_zr, {{d.c_dense, nd, 0, 0}, {d.c_vad, nv, 1, 0}}, nv, 2, gru_w(m.vad_gru, 0), gru_b(m.vad_gru, 0));
    pb.add(&d.vad_h, {{d.c_dense, nd, 0, 0}, {d.c_rh, nv, 1, 0}}, nv, 1, gru_w(m.vad_gru, 2), gru_b(m.vad_gru, 2));
    pb.add(&d.vad_out, {{d.c_vad, nv, 0, 0}}, 1, 1, dense_w(m.vad_output), dense_b(m.vad_output));
    pb.add(&d.noise_zr, {{d.c_dense, nd, 0, 0}, {d.c_vad, nv, 0, nd}, {d.c_feat, NB_FEATURES, 0, nd + nv}, {d.c_noise, nn, 1, 0}}, nn, 2,
           gru_w(m.noise_gru, 0), gru_b(m.noise_gru, 0));
    pb.add(&d.noise_h, {{d.c_dense, nd, 0, 0}, {d.c_vad, nv, 0, nd}, {d.c_feat, NB_FEATURES, 0, nd + nv}, {d.c_rh, nn, 1, 0}}, nn, 1,
           gru_w(m.noise_gru, 2), gru_b(m.noise_gru, 2));
    pb.add(&d.den_zr, {{d.c_vad, nv, 0, 0}, {d.c_noise, nn, 0, nv}, {d.c_feat, NB_FEATURES, 0, nv + nn}, {d.c_den, ndn, 1, 0}}, ndn, 2,
           gru_w(m.denoise_gru, 0), gru_b(m.denoise_gru, 0));
    pb.add(&d.den_h, {{d.c_vad, nv, 0, 0}, {d.c_noise, nn, 0, nv}, {d.c_feat, NB_FEATURES, 0, nv + nn}, {d.c_rh, ndn, 1, 0}}, ndn, 1,
           gru_w(m.denoise_gru, 2), gru_b(m.denoise_gru, 2));
    pb.add(&d.out, {{d.c_den, ndn, 0, 0}}, NB_BANDS, 1, dense_w(m.denoise_output), dense_b(m.denoise_output));
    while (blob->size() % 16) blob->push_back(0);
    d.table_off = (uint32_t)blob->size();
    blob->resize(blob->size() + sizeof kTansigTable);
    std::memcpy(blob->data() + d.table_off, kTansigTable, sizeof kTansigTable);
    while (blob->size() % 16) blob->push_back(0);
    return true;
}

cudaError_t launch_gru(const BatchBuffers& b, const DeviceModelMma& m, const unsigned char* image, int acts, const ModelTiles* tiles,
                       cudaStream_t st) {
    if (tiles) return launch_mma<true>(b, m, image, acts, *tiles, tiles->n_tiles, st);
    return launch_mma<false>(b, m, image, acts, ModelTiles{}, (b.n_streams + TS - 1) / TS, st);
}

}  // namespace nnb
