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
#include <atomic>

#include <cuda_fp16.h>

#include "common.cuh"

namespace nnb {

namespace {

constexpr int TS = 32;      // streams per block = two m16 row tiles
#ifndef RNN_NWARP
#define RNN_NWARP 8
#endif
constexpr int NWARP = RNN_NWARP;
constexpr int NT = NWARP * 32;
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

// p moved by moff bytes: the same phase of another model of the table (moff = model x stride)
template <typename T>
__device__ __forceinline__ const T* at_model(const T* p, size_t moff) {
    return reinterpret_cast<const T*>(reinterpret_cast<const char*>(p) + moff);
}

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], const uint2 b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}

// x = hi + lo with hi, lo in f16.  No clamp: NaN stays NaN, and |x| > 65504 (only an unbounded ReLU layer of a custom
// model can get there) becomes +-inf in hi and -+inf in lo, i.e. NaN in every product -- a loud failure instead of a
// silently clamped activation.  The bundled models (tanh / sigmoid, |x| <= 1) and the 42 features are far inside the range.
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}
// two adjacent columns (col even) of one row
__device__ __forceinline__ void store_pair(__half* Ahi, __half* Alo, int idx, float v0, float v1) {
    __half h0, l0, h1, l1;
    split_f16(v0, h0, l0);
    split_f16(v1, h1, l1);
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
__device__ __forceinline__ void run_tiles(const MmaPhase& ph, size_t moff, const __half* Ahi, const __half* Alo, int kp, int lane, int warp,
                                          int ot, int cnt, float (&acc)[NGATE * MO][2][4]) {
    constexpr int TSTEP = NWARP * 32;  // fragments between a warp's consecutive tiles
    const uint2* wg[NGATE];
#pragma unroll
    for (int gt = 0; gt < NGATE; gt++) wg[gt] = at_model(ph.wfrag, moff) + (size_t)(gt * ot + warp) * 32 + lane;
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
__device__ __forceinline__ void init_bias(const MmaPhase& ph, size_t moff, int lane, int warp, int ot, int cnt, float (&acc)[NGATE * MO][2][4]) {
    const int t = lane & 3;
#pragma unroll
    for (int i = 0; i < MO; i++)
#pragma unroll
        for (int gt = 0; gt < NGATE; gt++) {
            float b0 = 0.0f, b1 = 0.0f;
            if (i < cnt) {
                const float2 bv = __ldg(reinterpret_cast<const float2*>(at_model(ph.bias, moff) + (gt * ot + warp + i * NWARP) * 8 + 2 * t));
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
__device__ RNN_GRU_ATTR void gru_layer(const MmaPhase& pzr, const MmaPhase& ph, size_t moff, int act, int nn, int c_state, int c_rh, int s_off,
                          __half* Ahi, __half* Alo, int kp, float* Hf, int hs, const float* table) {
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
        init_bias<2, MAXOT>(pzr, moff, lane, warp, ot, cnt, acc);
        run_tiles<2, MAXOT>(pzr, moff, Ahi, Alo, kp, lane, warp, ot, cnt, acc);
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
                        store_pair(Ahi, Alo, row * kp + c_rh + o, rh[0], rh[1]);
                    }
                }
            }
        }
    }
    __syncthreads();
    {
        float acc[MAXOT][2][4];
        init_bias<1, MAXOT>(ph, moff, lane, warp, 0, cnt, acc);
        run_tiles<1, MAXOT>(ph, moff, Ahi, Alo, kp, lane, warp, 0, cnt, acc);
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
                        store_pair(Ahi, Alo, row * kp + c_state + o, hn[0], hn[1]);
                    }
                }
            }
        }
    }
    __syncthreads();
}

#ifndef RNN_MINB
#define RNN_MINB 2
#endif
// kMulti = false: block b advances batch rows [32 b, 32 b + 32) on model m.  kMulti = true (DESIGN.md 7c): block b advances
// tile b of the table mtab, on its own model of the table whose model 0 is m (same geometry, so the same layout; the
// model's fragments and biases lie model x stride bytes further, its activation codes come with the tile).
template <bool kMulti>
__global__ void __launch_bounds__(NT, RNN_MINB) rnn_mma_kernel(BatchBuffers bb, DeviceModelMma m, const DeviceTables* __restrict__ tab,
                                                               ModelTiles mtab) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int kp = m.kp, hs = m.hs;
    __half* Ahi = reinterpret_cast<__half*>(smraw);
    __half* Alo = Ahi + TS * kp;
    float* Hf = reinterpret_cast<float*>(Alo + TS * kp);
    float* table = Hf + TS * hs;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int s0 = blockIdx.x * TS;
    // kMulti: the tile's model offset, rows and activation codes.  The TILE_* selects below fold at compile time: the
    // kMulti = false instantiation reads m and batch row s0 + row exactly as the one-model kernel always has.
    size_t t_moff = 0;
    int t_first = 0, t_count = 0, t_acts = 0;
    if constexpr (kMulti) {
        const int4 tl = __ldg(reinterpret_cast<const int4*>(mtab.tile + blockIdx.x));  // {model, first, count, acts}
        t_moff = (size_t)tl.x * mtab.stride;
        t_first = tl.y;
        t_count = tl.z;
        t_acts = tl.w;
    }
#define TILE_MOFF (kMulti ? t_moff : (size_t)0)
#define TILE_ACT(i, field) (kMulti ? tile_act(t_acts, i) : m.field)
#define TILE_STREAM(row) (kMulti ? __ldg(mtab.rows + t_first + (row)) : s0 + (row))
    const int ns = kMulti ? t_count : min(TS, bb.n_streams - s0);
    const int SS = m.state_size;
    const int so_v = 0, so_n = (m.nv + 7) & ~7, so_d = so_n + ((m.nn + 7) & ~7);  // state offsets inside an Hf row

    // zero A (padding columns must hold finite values) and Hf, load the tanh table
    {
        uint32_t* z = reinterpret_cast<uint32_t*>(smraw);
        const int nz = (TS * kp * 2 * 2 + TS * hs * 4) / 4;
        for (int i = tid; i < nz; i += NT) z[i] = 0u;
        for (int i = tid; i < 201; i += NT) table[i] = tab->tansig[i];
    }
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
                    split_f16(sv[k], hi, lo);
                    ahr[acol[k]] = hi;
                    alr[acol[k]] = lo;
                }
            }
            {
                __half hi, lo;
                split_f16(f0, hi, lo);
                ahr[m.c_feat + lane] = hi;
                alr[m.c_feat + lane] = lo;
                if (lane + 32 < NB_FEATURES) {
                    split_f16(f1, hi, lo);
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
        init_bias<1, MAXOT>(m.dense, TILE_MOFF, lane, warp, 0, cnt, acc);
        run_tiles<1, MAXOT>(m.dense, TILE_MOFF, Ahi, Alo, kp, lane, warp, 0, cnt, acc);
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
                            v[c] = (o + c < m.nd) ? activate(TILE_ACT(0, act_dense), WEIGHTS_SCALE * acc[i][mt][2 * hf + c], table) : 0.0f;
                        store_pair(Ahi, Alo, row * kp + m.c_dense + o, v[0], v[1]);
                    }
    }
    __syncthreads();

    // ---- vad_gru (src/rnn.rs:356-358) ----
    gru_layer(m.vad_zr, m.vad_h, TILE_MOFF, TILE_ACT(1, act_vad), m.nv, m.c_vad, m.c_rh, so_v, Ahi, Alo, kp, Hf, hs, table);

    // ---- vad_output (src/rnn.rs:359): one neuron -> tile 0, warp 0 (no barrier needed: it only reads the vad state) ----
    if (warp == 0) {
        float acc[1][2][4];
        init_bias<1, 1>(m.vad_out, TILE_MOFF, lane, 0, 0, 1, acc);
        run_tiles<1, 1>(m.vad_out, TILE_MOFF, Ahi, Alo, kp, lane, 0, 0, 1, acc);
        if (t == 0) {
#pragma unroll
            for (int mt = 0; mt < 2; mt++)
#pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    const int row = mt * 16 + g + 8 * hf;
                    if (row < ns && !bb.silence[TILE_STREAM(row)])
                        bb.vad[TILE_STREAM(row)] = activate(TILE_ACT(5, act_vadout), WEIGHTS_SCALE * acc[0][mt][2 * hf], table);
                }
        }
    }

    // ---- noise_gru, denoise_gru (src/rnn.rs:361-377) ----
    gru_layer(m.noise_zr, m.noise_h, TILE_MOFF, TILE_ACT(2, act_noise), m.nn, m.c_noise, m.c_rh, so_n, Ahi, Alo, kp, Hf, hs, table);
    gru_layer(m.den_zr, m.den_h, TILE_MOFF, TILE_ACT(3, act_den), m.ndn, m.c_den, m.c_rh, so_d, Ahi, Alo, kp, Hf, hs, table);

    // ---- denoise_output (src/rnn.rs:378): 22 band gains ----
    {
        if (warp < (NB_BANDS + 7) / 8) {
            float acc[1][2][4];
            init_bias<1, 1>(m.out, TILE_MOFF, lane, warp, 0, 1, acc);
            run_tiles<1, 1>(m.out, TILE_MOFF, Ahi, Alo, kp, lane, warp, 0, 1, acc);
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
                                    activate(TILE_ACT(4, act_out), WEIGHTS_SCALE * acc[0][mt][2 * hf + c], table);
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
#undef TILE_MOFF
#undef TILE_ACT
#undef TILE_STREAM
}

static_assert(TS == MMA_TILE_ROWS, "tile tables are cut for this kernel's tile");

template <bool kMulti>
cudaError_t launch_mma(const BatchBuffers& b, const DeviceModelMma& m, const DeviceTables* tab, const ModelTiles& mt, int grid, cudaStream_t st) {
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
    rnn_mma_kernel<kMulti><<<grid, NT, smem, st>>>(b, m, tab, mt);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_rnn_mma(const BatchBuffers& b, const DeviceModelMma& m, const DeviceTables* tab, cudaStream_t st) {
    return launch_mma<false>(b, m, tab, ModelTiles{}, (b.n_streams + TS - 1) / TS, st);
}

cudaError_t launch_rnn_mma_multi(const BatchBuffers& b, const DeviceModelMma& m, const DeviceTables* tab, const ModelTiles& mt,
                                 cudaStream_t st) {
    return launch_mma<true>(b, m, tab, mt, mt.n_tiles, st);
}

}  // namespace nnb
