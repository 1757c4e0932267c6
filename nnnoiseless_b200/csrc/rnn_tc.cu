// rnn_tc.cu -- the GRU network (src/rnn.rs:251-379) on the Hopper tensor cores: wgmma with the accumulators in
// registers, the activations of 64 streams in shared memory as the A operand, the weights streamed through shared
// memory by the TMA bulk-copy engine.
//
// One consumer warpgroup (128 threads) advances a tile of M = 64 streams.  Every layer is D[64 x N] += A[64 x K] * W[K x N]:
//   * W: int8 weights are exact in f16; the host packs each layer phase as an [N][K] K-major, no-swizzle operand
//     (16-byte core-matrix rows: ((8,n),2):((1,SBO),LBO) in 16-byte units).  All nine phases (185 KB for the built-in
//     model) do not fit next to the activations, so the phases are cut into slabs of at most STAGE_BYTES (whole K
//     chunks).  A producer warp streams them with cp.async.bulk into a ring of STAGES buffers (full / empty
//     mbarriers); every tile uses the same slab sequence, so the producer runs ahead across phase and tile boundaries;
//   * A: activations are f32; each is split x = hi + lo (two f16, ~22 significant bits) and both halves are multiplied
//     (products exact in f32).  The halves live in shared memory in the same canonical K-major layout (8-column groups
//     of 64 rows x 16 bytes); the epilogue thread that owns an accumulator writes the next layer's operand there;
//   * D: f32 accumulators in registers, one m64nNk16 per K chunk and half with N the phase width (thread = two streams
//     x N / 4 neurons), for the epilogue: bias, 1/256 scale, table tanh / sigmoid (src/util.rs:29-53), the GRU update
//     in f32 against the f32 state in HBM.  The z | r phase of a GRU interleaves the two gates in blocks of 8 columns,
//     so the thread that holds z of neuron o also holds r of neuron o and, in the candidate phase, the candidate of
//     neuron o: the update gate waits in registers.  GRU semantics: src/rnn.rs:292-327 (reset gate applied to the
//     state BEFORE the recurrent product).
// The grid is persistent: each CTA loops over tiles, each fed by one pass of the weight ring.  109 KB of shared memory
// per CTA, two CTAs per SM, so one CTA's MMAs overlap the other's epilogue (DESIGN.md section 3, K4, has the measured
// comparison with two consumer warpgroups per CTA and one CTA per SM).
// Models whose layers do not fit this budget fall back to the mma.sync kernel (rnn_mma.cu).
#include <cuda_fp16.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "model.hpp"

namespace nnb {

extern const float kTansigTable[201];  // host.cu (src/util.rs:3-27)

namespace {

constexpr int TM = 64;            // streams per tile = MMA M
constexpr int NT = 128 + 32;      // threads: the consumer warpgroup, then the producer warp
constexpr int CTAS_PER_SM = 2;
constexpr int A_MAX_HALVES = 288; // 18 K-chunks of 16
constexpr int MAX_N = 192;        // accumulator columns of one phase (MAX_N / 2 registers per thread)
constexpr int NB_MAX = MAX_N / 8; // 8-column accumulator blocks
constexpr int ZB_MAX = 12;        // GRU width / 8 (padded): the update gate's registers
constexpr int FEAT_CHUNKS = 3;    // 48 feature columns (42 used)
constexpr int GROUP_BYTES = TM * 16;  // one 8-column group of a K-major operand
// weight ring: STAGES slabs of at most STAGE_BYTES (a K chunk of the widest phase is MAX_N * 32 = 6 KB)
constexpr int STAGES = 3;
constexpr uint32_t STAGE_BYTES = 8192;
static_assert(STAGE_BYTES >= MAX_N * 32, "a slab holds at least one K chunk of the widest phase");
// shared memory: the operand [A hi | A lo | features hi | features lo], then weight ring | tanh table |
// full mbarriers | empty mbarriers
constexpr uint32_t OP_AHI = 0, OP_ALO = OP_AHI + (A_MAX_HALVES / 8) * GROUP_BYTES;
constexpr uint32_t OP_FHI = OP_ALO + (A_MAX_HALVES / 8) * GROUP_BYTES, OP_FLO = OP_FHI + 2 * FEAT_CHUNKS * GROUP_BYTES;
constexpr uint32_t OP_BYTES = OP_FLO + 2 * FEAT_CHUNKS * GROUP_BYTES;
constexpr uint32_t SM_RING = OP_BYTES;
constexpr uint32_t SM_TABLE = SM_RING + STAGES * STAGE_BYTES;
constexpr uint32_t SM_BAR = SM_TABLE + 208 * 4;
constexpr uint32_t SMEM_BYTES = SM_BAR + 2 * 8 * STAGES;
constexpr float WEIGHTS_SCALE = 1.0f / 256.0f;

#ifdef RNN_TC_PROFILE
// NNB_VARIANT=prof: clock64 split of every tile (tools/rnn_phase_profile.py):
// [0] HBM loads into the operand, [1] waiting for weight slabs, [2] MMA issue and wait, [3] epilogue (barriers,
// activations, HBM stores), [4] tiles
__device__ unsigned long long g_rnn_prof[8];
#define RPROF(k)                              \
    do {                                      \
        const long long now_ = clock64();     \
        rprof_[k] += now_ - rprof_t_;         \
        rprof_t_ = now_;                      \
    } while (0)
#else
#define RPROF(k) \
    do {         \
    } while (0)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// src/util.rs:3-27, branch-free: same arithmetic on |x| clamped to 8, the saturations (NaN -> 1 like the reference's
// `!(x < 8)`) applied as selects at the end.
// The table is written once before the CTA's warps part ways and only read after: its loads carry no memory clobber,
// so the compiler may schedule them across the epilogue's operand and HBM stores (which cannot alias it).
__device__ __forceinline__ float table_at(uint32_t table, int i) {
    float v;
    asm("ld.shared.f32 %0, [%1];\n" : "=f"(v) : "r"(table + 4 * i));
    return v;
}
__device__ __forceinline__ float tansig_approx(float x, uint32_t table) {
    const float sign = (x < 0.0f) ? -1.0f : 1.0f;
    float ax = fminf(fabsf(x), 8.0f);
    const float fi = floorf(0.5f + 25.0f * ax);
    ax -= 0.04f * fi;
    float y = table_at(table, (int)fi);
    const float dy = 1.0f - y * y;
    y = y + ax * dy * (1.0f - y * ax);
    y = sign * y;
    y = !(x > -8.0f) ? -1.0f : y;
    return !(x < 8.0f) ? 1.0f : y;
}
__device__ __forceinline__ float sigmoid_approx(float x, uint32_t table) { return 0.5f + 0.5f * tansig_approx(0.5f * x, table); }
// act is the same for a whole layer; the selects (instead of branches) keep an epilogue's activations in one basic
// block, so the compiler can interleave their table loads and dependent chains.  Same values as the three functions.
__device__ __forceinline__ float activate(int act, float x, uint32_t table) {
    const float y = tansig_approx(act == 1 ? 0.5f * x : x, table);
    return act == 0 ? y : (act == 1 ? 0.5f + 0.5f * y : fmaxf(x, 0.0f));
}

// ---- wgmma shared-memory matrix descriptors (PTX ISA, "Matrix Descriptor Format"): K-major, no swizzle ----
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3fff);            // start address, bits [0,14)
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;  // leading byte offset (between the two 8-element K halves)
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;  // stride byte offset (between 8-row groups)
    return d;                                          // base offset 0, layout type 0 (no swizzle)
}
// D[64 x N] += A[64 x 16] * B[16 x N], f16 inputs, f32 accumulate: d[b] = the 8-column block b of the wgmma D fragment
// (rows g and g + 8 of the warp's 16, columns 8 b + 2 t, + 1).  One specialisation per phase width N = 16 ... 192.
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[NB_MAX][4], uint64_t a, uint64_t b);
#define WGMMA_HEAD "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned."
#define D4(b) "+f"(d[b][0]), "+f"(d[b][1]), "+f"(d[b][2]), "+f"(d[b][3])
template <> __device__ __forceinline__ void wgmma_f16<16>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n16k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7"
                 "}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<32>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n32k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
                 "}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<48>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n48k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23"
                 "}, %24, %25, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<64>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n64k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31"
                 "}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<80>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n80k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39"
                 "}, %40, %41, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<96>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n96k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
                 "}, %48, %49, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9), D4(10), D4(11)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<112>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n112k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55"
                 "}, %56, %57, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9), D4(10), D4(11),
                   D4(12), D4(13)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<128>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n128k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
                 "}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9), D4(10), D4(11),
                   D4(12), D4(13), D4(14), D4(15)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<144>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n144k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71"
                 "}, %72, %73, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9), D4(10), D4(11),
                   D4(12), D4(13), D4(14), D4(15), D4(16), D4(17)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<160>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n160k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, "
                 "%72, %73, %74, %75, %76, %77, %78, %79"
                 "}, %80, %81, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9), D4(10), D4(11),
                   D4(12), D4(13), D4(14), D4(15), D4(16), D4(17), D4(18), D4(19)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<176>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n176k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, "
                 "%72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87"
                 "}, %88, %89, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9), D4(10), D4(11),
                   D4(12), D4(13), D4(14), D4(15), D4(16), D4(17), D4(18), D4(19), D4(20), D4(21)
                 : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<192>(float (&d)[NB_MAX][4], uint64_t a, uint64_t b) {
    asm volatile(WGMMA_HEAD "m64n192k16.f32.f16.f16 {"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, "
                 "%72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
                 "}, %96, %97, p, 1, 1, 0, 0;\n\t}\n"
                 : D4(0), D4(1), D4(2), D4(3), D4(4), D4(5), D4(6), D4(7), D4(8), D4(9), D4(10), D4(11),
                   D4(12), D4(13), D4(14), D4(15), D4(16), D4(17), D4(18), D4(19), D4(20), D4(21), D4(22), D4(23)
                 : "l"(a), "l"(b));
}
#undef D4
#undef WGMMA_HEAD
// The accumulators are valid only after wgmma.wait_group: the empty volatile asm statements with "+" operands pin every
// use of them behind the wait.
__device__ __forceinline__ void fence_acc(float (&v)[4]) { asm volatile("" : "+f"(v[0]), "+f"(v[1]), "+f"(v[2]), "+f"(v[3])::"memory"); }

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\tbra WAIT_LOOP;\n\tDONE:\n\t}\n" ::"r"(bar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory"); }
// barrier over the 128 threads of the consumer warpgroup only (id 0 is __syncthreads)
__device__ __forceinline__ void wg_sync() { asm volatile("bar.sync %0, 128;\n" ::"r"(1) : "memory"); }
// L2 prefetch of the 16-byte aligned part of [p, p + bytes) (a hint: the next tile's rows, in flight during this one)
__device__ __forceinline__ void prefetch_l2(const void* p, size_t bytes) {
    const uintptr_t a0 = ((uintptr_t)p + 15) & ~(uintptr_t)15, a1 = ((uintptr_t)p + bytes) & ~(uintptr_t)15;
    if (a1 > a0) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;\n" ::"l"(a0), "r"((uint32_t)(a1 - a0)) : "memory");
}

// x = hi + lo with hi, lo in f16, two adjacent columns -> one packed register each.  No clamp: NaN stays NaN and
// |x| > 65504 (an unbounded ReLU layer of a custom model) becomes +-inf / NaN downstream: loud, not silent.
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __half h0 = __float2half_rn(a), h1 = __float2half_rn(b);
    const __half l0 = __float2half_rn(a - __half2float(h0)), l1 = __float2half_rn(b - __half2float(h1));
    hi = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
    lo = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
}
__device__ __forceinline__ float2 join2(uint32_t hi, uint32_t lo) {
    return make_float2(__half2float(__ushort_as_half((unsigned short)(hi & 0xffffu))) + __half2float(__ushort_as_half((unsigned short)(lo & 0xffffu))),
                       __half2float(__ushort_as_half((unsigned short)(hi >> 16))) + __half2float(__ushort_as_half((unsigned short)(lo >> 16))));
}
// byte offset of (row, column) in a K-major operand (column even for pairs)
__device__ __forceinline__ uint32_t opnd_off(int row, int col) { return (uint32_t)((col >> 3) * GROUP_BYTES + row * 16 + (col & 7) * 2); }

// The MMAs of one slab: K chunks [kc0, kc1) of phase `ph` into the first N / 8 accumulator blocks, hi and lo halves of
// the activations against the same weights (K chunk outer, hi then lo inner), then wait for them.  `op`: the
// activation operand, `wb`: the ring stage holding the slab.
template <int N>
__device__ __forceinline__ void mma_slab(float (&acc)[NB_MAX][4], const TcPhase& ph, const TcSlab& sl, uint32_t op, uint32_t wb) {
#pragma unroll
    for (int b = 0; b < N / 8; b++) fence_acc(acc[b]);
    // descriptors built once per slab; a K chunk moves the start address (16-byte units, bits [0,14))
    const uint64_t a_hi = make_desc(op + OP_AHI, GROUP_BYTES, 128), a_lo = make_desc(op + OP_ALO, GROUP_BYTES, 128);
    const uint64_t f_hi = make_desc(op + OP_FHI, GROUP_BYTES, 128), f_lo = make_desc(op + OP_FLO, GROUP_BYTES, 128);
    uint64_t b_desc = make_desc(wb, N * 16, 128);
    for (int kc = sl.kc0; kc < sl.kc1; kc++) {
        // the accumulators are carried around this run-time loop: fence them once per K chunk (CUTLASS does the same
        // per k-block) rather than leave ptxas to insert the fence in front of each MMA
        asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
        const int c = ph.chunk[kc];
        const uint64_t step = (uint64_t)((2 * (c >= 0 ? c : -c - 1) * GROUP_BYTES) >> 4);
        wgmma_f16<N>(acc, (c >= 0 ? a_hi : f_hi) + step, b_desc);
        wgmma_f16<N>(acc, (c >= 0 ? a_lo : f_lo) + step, b_desc);
        b_desc += (N * 32) >> 4;
    }
    asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
#pragma unroll
    for (int b = 0; b < N / 8; b++) fence_acc(acc[b]);
}

// f(std::integral_constant<int, n>()) for the run-time phase width n (a multiple of 16 in [N, M]): the phase width as a
// template constant, so no run-time guard sits around a wgmma
template <int N, int M, class F>
__device__ __forceinline__ void with_width(int n, F& f) {
    if constexpr (N >= M) {
        f(std::integral_constant<int, M>());
    } else {
        if (n == N) f(std::integral_constant<int, N>());
        else with_width<N + 16, M>(n, f);
    }
}

__global__ void __launch_bounds__(NT, CTAS_PER_SM) rnn_tc_kernel(BatchBuffers bb, DeviceModelTc m) {
    extern __shared__ __align__(1024) unsigned char smraw[];
    const uint32_t sbase = smem_u32(smraw), table = sbase + SM_TABLE;
    const uint32_t full_bar = sbase + SM_BAR, empty_bar = full_bar + 8 * STAGES;  // + 8 * stage

    // the warp index through a shuffle: ptxas then knows it is warp-uniform, so the role branch below is not a divergent
    // path around the wgmma (which would serialise them)
    const int tid = threadIdx.x, lane = tid & 31, warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int n_tiles = (bb.n_streams + TM - 1) / TM;

    if (tid == 0) {
        for (int s = 0; s < STAGES; s++) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" ::"r"(full_bar + 8 * s));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(empty_bar + 8 * s), "r"(4));  // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    // zero the activation operand once (padding columns that a K chunk spans must hold zeros: tiles write only zeros
    // there, except in the reset-gate columns, which every tile clears), load the table
    for (uint32_t i = tid; i < OP_FHI / 16; i += NT) reinterpret_cast<uint4*>(smraw)[i] = make_uint4(0u, 0u, 0u, 0u);
    for (int i = tid; i < 201; i += NT) reinterpret_cast<float*>(smraw + SM_TABLE)[i] = __ldg(reinterpret_cast<const float*>(m.blob + m.table_off) + i);
    __syncthreads();  // the only CTA-wide barrier: the warps part ways below

    if (warp == 4) {  // ---- producer: the slab sequence of every tile, STAGES slabs ahead of the consumers ----
        if (lane == 0) {
            int stage = 0;
            uint32_t par = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)
                for (int si = 0; si < m.n_slabs; si++) {
                    const TcSlab& sl = m.slab[si];
                    mbar_wait(empty_bar + 8 * stage, par ^ 1);  // every consumer warp has released the stage
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(full_bar + 8 * stage), "r"(sl.bytes) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                                     sbase + SM_RING + stage * STAGE_BYTES),
                                 "l"(m.blob + sl.off), "r"(sl.bytes), "r"(full_bar + 8 * stage)
                                 : "memory");
                    if (++stage == STAGES) { stage = 0; par ^= 1; }
                }
        }
        return;
    }

    // ---- consumer warpgroup: every tile of this CTA ----
    const int wt = tid & 127, g = lane >> 2, t = lane & 3;
    unsigned char* opb = smraw;  // the activation operand
    const uint32_t op = sbase;
    // accumulator rows of this thread: 16 warp + g and 16 warp + g + 8 (wgmma D fragment)
    const int rows[2] = {16 * (warp & 3) + g, 16 * (warp & 3) + g + 8};
    const int SS = m.state_size;
    const int so_n = m.nv, so_d = m.nv + m.nn;  // state offsets in HBM (vad | noise | denoise)
#ifdef RNN_TC_PROFILE
    long long rprof_[4] = {0, 0, 0, 0}, rprof_t_ = clock64();
    unsigned long long rprof_tiles_ = 0;
#endif

    auto get2 = [&](int row, int col) {
        const uint32_t o = opnd_off(row, col);
        return join2(*reinterpret_cast<const uint32_t*>(opb + OP_AHI + o), *reinterpret_cast<const uint32_t*>(opb + OP_ALO + o));
    };
    auto put2 = [&](int row, int col, float a, float b) {
        const uint32_t o = opnd_off(row, col);
        uint32_t hi, lo;
        split2(a, b, hi, lo);
        *reinterpret_cast<uint32_t*>(opb + OP_AHI + o) = hi;
        *reinterpret_cast<uint32_t*>(opb + OP_ALO + o) = lo;
    };

    float acc[NB_MAX][4];
    int stage = 0;
    uint32_t par = 0;  // ring position of the consumers (the same slab sequence as the producer's)
    // one phase: the warpgroup multiplies every slab of the phase into acc (hi and lo halves of every K chunk against
    // the same weights) and hands each ring stage back as soon as its MMAs have completed
    // max_width: the widest this phase can be for any model that build_model_tc accepts (a compile-time bound on the
    // registers the phase's accumulators take next to whatever else is live).  epilogue(width) runs with the phase width
    // as a template constant too: its loops over accumulator blocks have compile-time trip counts and no run-time guard
    // around the activations, so they form one basic block.
    auto run_phase = [&](int p, auto max_width, auto&& epilogue) __attribute__((always_inline)) {
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");  // the epilogue's operand stores -> wgmma
        wg_sync();
        RPROF(3);
        const TcPhase& ph = m.ph[p];
        // the slabs of a phase of width N: only its N / 8 accumulator blocks are carried through the slab loop, the
        // others stay the constant 0
        auto slabs = [&](auto width) __attribute__((always_inline)) {
            constexpr int N = decltype(width)::value;
#pragma unroll
            for (int b = 0; b < NB_MAX; b++) acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.0f;
            for (int si = m.slab0[p]; si < m.slab0[p + 1]; si++) {
                mbar_wait(full_bar + 8 * stage, par);
                RPROF(1);
                mma_slab<N>(acc, ph, m.slab[si], op, sbase + SM_RING + stage * STAGE_BYTES);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar + 8 * stage);  // this warp is done with the stage
                if (++stage == STAGES) { stage = 0; par ^= 1; }
                RPROF(2);
            }
            wg_sync();  // every warp's MMAs have read the operand before the epilogue rewrites it
            epilogue(width);
        };
        with_width<16, decltype(max_width)::value>(ph.n, slabs);
    };

    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int s0 = tile * TM;  // rows past n_streams compute on zeros and store nothing
        // ---- features -> shared-memory operand (64 rows x 6 groups of 8 columns) ----
        for (int it = wt; it < TM * 2 * FEAT_CHUNKS; it += 128) {
            const int row = it % TM, grp = it / TM, s = s0 + row;
            const float* fsrc = bb.features + (size_t)s * NB_FEATURES;
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int j = 8 * grp + 2 * i;
                float2 v = make_float2(0.f, 0.f);
                if (s < bb.n_streams && j < NB_FEATURES) v = __ldg(reinterpret_cast<const float2*>(fsrc + j));  // 42 is even
                split2(v.x, v.y, hi[i], lo[i]);
            }
            *reinterpret_cast<uint4*>(opb + OP_FHI + grp * GROUP_BYTES + row * 16) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<uint4*>(opb + OP_FLO + grp * GROUP_BYTES + row * 16) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        // ---- GRU states -> activation operand ----
        auto load_state = [&](int nn_, int p8, int s_off, int a_off) {
            for (int it = wt; it < TM * (p8 / 8); it += 128) {
                const int row = it % TM, grp = it / TM, s = s0 + row;
                const float* hsrc = bb.gru_state + (size_t)s * SS + s_off;
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int j = 8 * grp + 2 * i;
                    const float a = (s < bb.n_streams && j < nn_) ? __ldg(hsrc + j) : 0.0f;
                    const float b = (s < bb.n_streams && j + 1 < nn_) ? __ldg(hsrc + j + 1) : 0.0f;
                    split2(a, b, hi[i], lo[i]);
                }
                const uint32_t o = opnd_off(row, a_off + 8 * grp);
                *reinterpret_cast<uint4*>(opb + OP_AHI + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<uint4*>(opb + OP_ALO + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            }
        };
        load_state(m.nv, m.p_v, 0, m.o_vad);
        load_state(m.nn, m.p_n, so_n, m.o_noise);
        load_state(m.ndn, m.p_dn, so_d, m.o_den);
        // the reset-gate columns are shared by the three GRUs, and a narrow layer's last K chunk reaches into what the
        // widest layer of the previous tile left there: zero them as in a fresh operand, so tiles stay independent
        for (int it = wt; it < TM * ((A_MAX_HALVES - m.o_rh) / 8); it += 128) {
            const uint32_t o = opnd_off(it % TM, m.o_rh + 8 * (it / TM));
            *reinterpret_cast<uint4*>(opb + OP_AHI + o) = make_uint4(0u, 0u, 0u, 0u);
            *reinterpret_cast<uint4*>(opb + OP_ALO + o) = make_uint4(0u, 0u, 0u, 0u);
        }

        bool upd[2];
        float* hdst[2];
        int srow[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int s = s0 + rows[h];
            const bool live = s < bb.n_streams;
            srow[h] = live ? s : 0;
            upd[h] = live && !bb.silence[srow[h]];  // silent frames leave the RNN state and outputs untouched
            hdst[h] = bb.gru_state + (size_t)srow[h] * SS;
        }
        RPROF(0);

        // ---- input_dense (src/rnn.rs:353-355) ----
        run_phase(PH_DENSE, std::integral_constant<int, MAX_N>(), [&](auto width) __attribute__((always_inline)) {
            constexpr int NB = decltype(width)::value / 8;
            const float* bias = reinterpret_cast<const float*>(m.blob + m.ph[PH_DENSE].b_off);
#pragma unroll
            for (int b = 0; b < NB; b++) {
                const int o = 8 * b + 2 * t;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    float v[2];
#pragma unroll
                    for (int c = 0; c < 2; c++)
                        v[c] = (o + c < m.nd) ? activate(m.act_dense, WEIGHTS_SCALE * (acc[b][2 * h + c] + __ldg(bias + o + c)), table) : 0.0f;
                    // the last block of a width padded to 16 can lie past the layer, in the next one's columns
                    if (b + 1 < NB || 8 * b < m.p_d) put2(rows[h], m.o_dense + o, v[0], v[1]);
                }
            }
        });

        // ---- one GRU layer: z | r phase then candidate phase (src/rnn.rs:292-327) ----
        float z[ZB_MAX][4];
        auto gru = [&](int pzr, int phh, int act, int nn_, int p8, int s_off, int a_off) __attribute__((always_inline)) {
            // z of the previous layer is dead: the constant 0 keeps it out of registers during this layer's z | r MMAs
#pragma unroll
            for (int b = 0; b < ZB_MAX; b++) z[b][0] = z[b][1] = z[b][2] = z[b][3] = 0.0f;
            run_phase(pzr, std::integral_constant<int, MAX_N>(), [&](auto width) __attribute__((always_inline)) {
                constexpr int NZ = decltype(width)::value / 16;  // z | r block pairs: the width is exactly 2 p8
                const float* bias = reinterpret_cast<const float*>(m.blob + m.ph[pzr].b_off);
#pragma unroll
                for (int b = 0; b < NZ; b++) {
                    const int o = 8 * b + 2 * t;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const float2 hp = get2(rows[h], a_off + o);  // previous state as the tensor core sees it (hi + lo)
                        float r[2];
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            z[b][2 * h + c] = sigmoid_approx(WEIGHTS_SCALE * (acc[2 * b][2 * h + c] + __ldg(bias + 16 * b + 2 * t + c)), table);
                            r[c] = (o + c < nn_) ? sigmoid_approx(WEIGHTS_SCALE * (acc[2 * b + 1][2 * h + c] + __ldg(bias + 16 * b + 8 + 2 * t + c)), table) *
                                                       (c ? hp.y : hp.x)
                                                 : 0.0f;  // reset gate scales the previous state
                        }
                        put2(rows[h], m.o_rh + o, r[0], r[1]);
                    }
                }
            });
            // z is live: at most 48 + 48 registers
            run_phase(phh, std::integral_constant<int, 8 * ZB_MAX>(), [&](auto width) __attribute__((always_inline)) {
                constexpr int NB = decltype(width)::value / 8;
                const float* bias = reinterpret_cast<const float*>(m.blob + m.ph[phh].b_off);
#pragma unroll
                for (int b = 0; b < NB; b++) {
                    const int o = 8 * b + 2 * t;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const float2 hp = get2(rows[h], a_off + o);
                        float hn[2];
#pragma unroll
                        for (int c = 0; c < 2; c++) {
                            const float cand = activate(act, WEIGHTS_SCALE * (acc[b][2 * h + c] + __ldg(bias + o + c)), table);
                            const float zz = z[b][2 * h + c];
                            hn[c] = (o + c < nn_) ? zz * (c ? hp.y : hp.x) + (1.0f - zz) * cand : 0.0f;
                            if (upd[h] && o + c < nn_) hdst[h][s_off + o + c] = hn[c];
                        }
                        // the last block of a width padded to 16 can lie past the layer, in the next one's columns
                        if (b + 1 < NB || 8 * b < p8) put2(rows[h], a_off + o, hn[0], hn[1]);
                    }
                }
            });
        };
        // vad_gru (src/rnn.rs:356-358)
        gru(PH_VAD_ZR, PH_VAD_H, m.act_vad, m.nv, m.p_v, 0, m.o_vad);
        // vad_output (:359): one neuron from the new vad state
        run_phase(PH_VAD_OUT, std::integral_constant<int, 16>(), [&](auto) __attribute__((always_inline)) {
            if (t == 0) {
                const float* bias = reinterpret_cast<const float*>(m.blob + m.ph[PH_VAD_OUT].b_off);
#pragma unroll
                for (int h = 0; h < 2; h++)
                    if (upd[h]) bb.vad[srow[h]] = activate(m.act_vadout, WEIGHTS_SCALE * (acc[0][2 * h] + __ldg(bias)), table);
            }
        });
        // noise_gru (:361-369)
        gru(PH_NOISE_ZR, PH_NOISE_H, m.act_noise, m.nn, m.p_n, so_n, m.o_noise);
        // the next tile's features, states and silence flags: L2 prefetches, in flight during the denoise layers
        if (wt == 0 && tile + (int)gridDim.x < n_tiles) {
            const int sn = (tile + (int)gridDim.x) * TM, ns = min(TM, bb.n_streams - sn);
            if (ns > 0) {
                prefetch_l2(bb.features + (size_t)sn * NB_FEATURES, (size_t)ns * NB_FEATURES * 4);
                prefetch_l2(bb.gru_state + (size_t)sn * SS, (size_t)ns * SS * 4);
                prefetch_l2(bb.silence + sn, (size_t)ns * 4);
            }
        }
        // denoise_gru (:370-377)
        gru(PH_DEN_ZR, PH_DEN_H, m.act_den, m.ndn, m.p_dn, so_d, m.o_den);
        // denoise_output (:378): 22 band gains
        run_phase(PH_OUT, std::integral_constant<int, (NB_BANDS + 15) / 16 * 16>(), [&](auto) __attribute__((always_inline)) {
            const float* bias = reinterpret_cast<const float*>(m.blob + m.ph[PH_OUT].b_off);
#pragma unroll
            for (int b = 0; b < (NB_BANDS + 7) / 8; b++) {
#pragma unroll
                for (int h = 0; h < 2; h++) {
#pragma unroll
                    for (int c = 0; c < 2; c++) {
                        const int o = 8 * b + 2 * t + c;
                        const float v = activate(m.act_out, WEIGHTS_SCALE * (acc[b][2 * h + c] + __ldg(bias + o)), table);
                        if (upd[h] && o < NB_BANDS) bb.gains[(size_t)srow[h] * NB_BANDS + o] = v;
                    }
                }
            }
        });
        RPROF(3);
#ifdef RNN_TC_PROFILE
        rprof_tiles_++;
#endif
    }
#ifdef RNN_TC_PROFILE
    if (wt == 0) {
        for (int k = 0; k < 4; k++) atomicAdd(&g_rnn_prof[k], (unsigned long long)rprof_[k]);
        atomicAdd(&g_rnn_prof[4], rprof_tiles_);
    }
#endif
}

inline int pad8(int n) { return (n + 7) & ~7; }
inline int pad16(int n) { return (n + 15) & ~15; }
// accumulator column of (gate, neuron o) in a phase of `ngates` gates interleaved in blocks of 8 columns, and back
inline int gate_col(int gate, int o, int ngates) { return (o / 8) * 8 * ngates + gate * 8 + o % 8; }
inline void col_gate(int n, int ngates, int* gate, int* o) {
    *gate = (n / 8) % ngates;
    *o = (n / 8 / ngates) * 8 + n % 8;
}

}  // namespace

// ---- host: pack the model for the kernel.  Returns false if the model does not fit the register / shared-memory budget. ----
bool build_model_tc(const HostModel& hm, DeviceModelTc* d, std::vector<unsigned char>* blob) {
    const int nd = hm.input_dense.nn, nv = hm.vad_gru.nn, nn = hm.noise_gru.nn, ndn = hm.denoise_gru.nn;
    d->nd = nd; d->nv = nv; d->nn = nn; d->ndn = ndn;
    d->p_d = pad8(nd); d->p_v = pad8(nv); d->p_n = pad8(nn); d->p_dn = pad8(ndn);
    d->o_dense = 0;
    d->o_vad = d->o_dense + d->p_d;
    d->o_noise = d->o_vad + d->p_v;
    d->o_den = d->o_noise + d->p_n;
    d->o_rh = pad16(d->o_den + d->p_dn);
    const int rh = std::max(d->p_v, std::max(d->p_n, d->p_dn));
    if (d->o_rh + rh > A_MAX_HALVES) return false;
    if (d->p_d > MAX_N || rh > 8 * ZB_MAX) return false;
    d->act_dense = hm.input_dense.act; d->act_vad = hm.vad_gru.act; d->act_noise = hm.noise_gru.act; d->act_den = hm.denoise_gru.act;
    d->act_out = hm.denoise_output.act; d->act_vadout = hm.vad_output.act;
    d->state_size = nv + nn + ndn;
    const int8_t* B = hm.bytes.data();

    // which source does activation column a (in halves) of the operand hold?  seg: 0 dense, 1 vad, 2 noise, 3 den, 4 rh
    auto col_src = [&](int a, int* seg, int* j) {
        *seg = -1;
        if (a >= d->o_rh) { *seg = 4; *j = a - d->o_rh; }
        else if (a >= d->o_den) { *seg = 3; *j = a - d->o_den; }
        else if (a >= d->o_noise) { *seg = 2; *j = a - d->o_noise; }
        else if (a >= d->o_vad) { *seg = 1; *j = a - d->o_vad; }
        else { *seg = 0; *j = a; }
    };
    const int seg_off[5] = {d->o_dense, d->o_vad, d->o_noise, d->o_den, d->o_rh};
    // chunks (of 16 halves) covering segment `seg` restricted to its first `len` columns
    auto chunks_of = [&](int seg, int len, std::vector<int>* out) {
        const int a0 = seg_off[seg], a1 = seg_off[seg] + len;
        for (int c = a0 / 16; c * 16 < a1; c++)
            if (std::find(out->begin(), out->end(), c) == out->end()) out->push_back(c);
    };

    // weight(seg, j, gate, o): int8 weight of input (seg, j) for output neuron o of `gate`, or 0 if that input is not wired
    struct Wire { int seg; int len; int row0; bool recurrent; };  // rows of W (or R) that segment seg feeds
    auto add_phase = [&](int pi, const std::vector<Wire>& wires, bool use_feat, int feat_row0, int nout, int ngates, int gate0, int p8,
                         size_t w_off, size_t r_off, size_t b_off, int row_stride) -> bool {
        TcPhase& ph = d->ph[pi];
        std::vector<int> chunks;
        for (const Wire& w : wires) chunks_of(w.seg, w.len, &chunks);
        std::sort(chunks.begin(), chunks.end());
        std::vector<int> entries(chunks.begin(), chunks.end());
        if (use_feat)
            for (int f = 0; f < FEAT_CHUNKS; f++) entries.push_back(-(f + 1));
        if ((int)entries.size() > 16) return false;
        ph.nk = (int)entries.size();
        for (int i = 0; i < ph.nk; i++) ph.chunk[i] = (short)entries[i];
        ph.n = pad16(ngates * p8);
        // a layer of 0 neurons leaves a phase of width 0, which no wgmma shape covers (the mma.sync kernel runs it)
        if (ph.n == 0 || ph.n > MAX_N) return false;
        while (blob->size() % 128) blob->push_back(0);
        ph.w_off = (uint32_t)blob->size();
        const int K = 16 * ph.nk;
        blob->resize(blob->size() + (size_t)ph.n * K * 2, 0);
        __half* wb = reinterpret_cast<__half*>(blob->data() + ph.w_off);
        for (int kc = 0; kc < ph.nk; kc++)
            for (int kk = 0; kk < 16; kk++) {
                // source row of this K column
                const int8_t* src = nullptr;  // start of the weight row (all gates), or null = not wired
                if (entries[kc] >= 0) {
                    int seg, j;
                    col_src(entries[kc] * 16 + kk, &seg, &j);
                    for (const Wire& w : wires)
                        if (w.seg == seg && j < w.len) src = B + (w.recurrent ? r_off : w_off) + (size_t)(w.row0 + j) * row_stride;
                } else {
                    const int j = (-entries[kc] - 1) * 16 + kk;
                    if (j < NB_FEATURES) src = B + w_off + (size_t)(feat_row0 + j) * row_stride;
                }
                const int k = kc * 16 + kk;
                for (int n = 0; n < ph.n; n++) {
                    int gate, o;
                    col_gate(n, ngates, &gate, &o);
                    int val = 0;
                    if (src && gate < ngates && o < nout) val = src[(gate0 + gate) * nout + o];
                    // canonical K-major operand: element (n, k) at (k / 8) * (N * 16 B) + n * 16 B + (k % 8) * 2 B
                    wb[(size_t)(k / 8) * (ph.n * 8) + (size_t)n * 8 + (k % 8)] = __float2half((float)val);
                }
            }
        while (blob->size() % 16) blob->push_back(0);
        ph.b_off = (uint32_t)blob->size();
        blob->resize(blob->size() + (size_t)ph.n * 4, 0);
        float* bf = reinterpret_cast<float*>(blob->data() + ph.b_off);
        for (int n = 0; n < ph.n; n++) {
            int gate, o;
            col_gate(n, ngates, &gate, &o);
            bf[n] = (gate < ngates && o < nout) ? (float)B[b_off + (size_t)(gate0 + gate) * nout + o] : 0.0f;
        }
        return true;
    };

    bool ok = true;
    const HostDense& L0 = hm.input_dense;
    const HostGru &G1 = hm.vad_gru, &G2 = hm.noise_gru, &G3 = hm.denoise_gru;
    const HostDense &LO = hm.denoise_output, &LV = hm.vad_output;
    // dense: features only
    ok = ok && add_phase(PH_DENSE, {}, true, 0, nd, 1, 0, d->p_d, L0.w_off, 0, L0.b_off, nd);
    // vad_gru: input = dense_out
    ok = ok && add_phase(PH_VAD_ZR, {{0, nd, 0, false}, {1, nv, 0, true}}, false, 0, nv, 2, 0, d->p_v, G1.w_off, G1.r_off, G1.b_off, 3 * nv);
    ok = ok && add_phase(PH_VAD_H, {{0, nd, 0, false}, {4, nv, 0, true}}, false, 0, nv, 1, 2, d->p_v, G1.w_off, G1.r_off, G1.b_off, 3 * nv);
    // vad_output: one neuron from the vad state
    ok = ok && add_phase(PH_VAD_OUT, {{1, nv, 0, false}}, false, 0, 1, 1, 0, 8, LV.w_off, 0, LV.b_off, 1);
    // noise_gru: input = [dense_out | vad_state | features]
    ok = ok && add_phase(PH_NOISE_ZR, {{0, nd, 0, false}, {1, nv, nd, false}, {2, nn, 0, true}}, true, nd + nv, nn, 2, 0, d->p_n, G2.w_off, G2.r_off,
                         G2.b_off, 3 * nn);
    ok = ok && add_phase(PH_NOISE_H, {{0, nd, 0, false}, {1, nv, nd, false}, {4, nn, 0, true}}, true, nd + nv, nn, 1, 2, d->p_n, G2.w_off, G2.r_off,
                         G2.b_off, 3 * nn);
    // denoise_gru: input = [vad_state | noise_state | features]
    ok = ok && add_phase(PH_DEN_ZR, {{1, nv, 0, false}, {2, nn, nv, false}, {3, ndn, 0, true}}, true, nv + nn, ndn, 2, 0, d->p_dn, G3.w_off, G3.r_off,
                         G3.b_off, 3 * ndn);
    ok = ok && add_phase(PH_DEN_H, {{1, nv, 0, false}, {2, nn, nv, false}, {4, ndn, 0, true}}, true, nv + nn, ndn, 1, 2, d->p_dn, G3.w_off, G3.r_off,
                         G3.b_off, 3 * ndn);
    // denoise_output
    ok = ok && add_phase(PH_OUT, {{3, ndn, 0, false}}, false, 0, NB_BANDS, 1, 0, pad8(NB_BANDS), LO.w_off, 0, LO.b_off, NB_BANDS);
    if (!ok) return false;
    // slabs: whole K chunks of one phase, at most STAGE_BYTES (one ring stage) per bulk copy
    d->n_slabs = 0;
    for (int p = 0; p < TC_PHASES; p++) {
        const TcPhase& ph = d->ph[p];
        const int per = (int)(STAGE_BYTES / (uint32_t)(ph.n * 32));  // >= 1: n <= MAX_N
        d->slab0[p] = (short)d->n_slabs;
        for (int kc = 0; kc < ph.nk; kc += per) {
            if (d->n_slabs == TC_MAX_SLABS) return false;
            TcSlab& sl = d->slab[d->n_slabs++];
            sl.phase = (short)p;
            sl.kc0 = (short)kc;
            sl.kc1 = (short)std::min(ph.nk, kc + per);
            sl.off = ph.w_off + (uint32_t)(kc * ph.n * 32);
            sl.bytes = (uint32_t)((sl.kc1 - sl.kc0) * ph.n * 32);
        }
    }
    d->slab0[TC_PHASES] = (short)d->n_slabs;
    return true;
}

int upload_model_tc(const HostModel& hm, UploadedTc* u, cudaStream_t st) {
    u->ok = false;
    std::vector<unsigned char> blob;
    if (!build_model_tc(hm, &u->dm, &blob)) return 0;  // not an error: the caller uses the mma.sync kernel
    while (blob.size() % 16) blob.push_back(0);
    u->dm.table_off = (uint32_t)blob.size();
    blob.resize(blob.size() + 208 * 4, 0);
    std::memcpy(blob.data() + u->dm.table_off, kTansigTable, 201 * 4);
    while (blob.size() % 16) blob.push_back(0);
    u->dm.blob_bytes = (uint32_t)blob.size();
    u->smem_bytes = SMEM_BYTES;
    if (cudaMalloc(&u->d_blob, blob.size()) != cudaSuccess) return -1;
    if (cudaMemcpyAsync(u->d_blob, blob.data(), blob.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(st) != cudaSuccess) return -1;
    u->dm.blob = u->d_blob;
    u->ok = true;
    return 0;
}

// Persistent grid: min(tiles, resident CTAs per SM x SM count of the current device).
cudaError_t launch_rnn_tc(const BatchBuffers& b, const UploadedTc& u, cudaStream_t st) {
    static std::atomic<int> resident[64];  // per device, 0 = not yet known (the attribute is set on first use)
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    int ctas = dev < 64 ? resident[dev].load(std::memory_order_acquire) : 0;
    if (ctas == 0) {
        e = cudaFuncSetAttribute(rnn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)u.smem_bytes);
        if (e != cudaSuccess) return e;
        int sms = 0, per_sm = 0;
        e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return e;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rnn_tc_kernel, NT, u.smem_bytes);
        if (e != cudaSuccess) return e;
        ctas = std::max(1, per_sm) * sms;
        if (dev < 64) resident[dev].store(ctas, std::memory_order_release);
    }
    const int n_tiles = (b.n_streams + TM - 1) / TM;
    rnn_tc_kernel<<<std::min(n_tiles, ctas), NT, u.smem_bytes, st>>>(b, u.dm);
    return cudaGetLastError();
}

void free_model_tc(UploadedTc* u) {
    if (u->d_blob) cudaFree(u->d_blob);
    u->d_blob = nullptr;
    u->ok = false;
}

}  // namespace nnb

#ifdef RNN_TC_PROFILE
extern "C" void nnb_rnn_prof_read(unsigned long long* out8, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out8, nnb::g_rnn_prof, sizeof(unsigned long long) * 8);
    if (reset) {
        unsigned long long z[8] = {0};
        cudaMemcpyToSymbol(nnb::g_rnn_prof, z, sizeof z);
    }
}
#endif

// ---- host-side self test of the PACKING (no GPU): replays the kernel's phase structure in plain f32 from the packed
// blob and compares with a direct evaluation of src/rnn.rs:343-379 from the model bytes.  Returns the largest absolute
// difference over gains, vad and the new GRU states (-1: model rejected, -2: model does not fit the wgmma budget). ----
namespace nnb {
namespace {
float h_tansig(float x) {
    if (!(x < 8.0f)) return 1.0f;
    if (!(x > -8.0f)) return -1.0f;
    float sign = 1.0f;
    if (x < 0.0f) { x = -x; sign = -1.0f; }
    const int i = (int)std::floor(0.5f + 25.0f * x);
    x -= 0.04f * (float)i;
    const float y = kTansigTable[i], dy = 1.0f - y * y;
    return sign * (y + x * dy * (1.0f - y * x));
}
float h_act(int act, float x) { return act == 0 ? h_tansig(x) : (act == 1 ? 0.5f + 0.5f * h_tansig(0.5f * x) : std::max(x, 0.0f)); }
}  // namespace
}  // namespace nnb

extern "C" double nnb_tc_pack_selftest(const unsigned char* bytes, size_t len, int seed) {
    using namespace nnb;
    HostModel hm;
    if (!HostModel::parse(bytes, len, &hm)) return -1.0;
    DeviceModelTc d{};
    std::vector<unsigned char> blob;
    if (!build_model_tc(hm, &d, &blob)) return -2.0;
    const int8_t* B = hm.bytes.data();
    const int nd = d.nd, nv = d.nv, nn = d.nn, ndn = d.ndn;
    srand(seed);
    auto rnd = [](float a) { return a * ((float)(rand() % 20001) / 10000.0f - 1.0f); };
    std::vector<float> feat(NB_FEATURES), sv(nv), sn(nn), sd(ndn);
    for (auto& v : feat) v = rnd(3.0f);
    for (auto& v : sv) v = rnd(1.0f);
    for (auto& v : sn) v = rnd(1.0f);
    for (auto& v : sd) v = rnd(1.0f);

    // ---- direct evaluation (src/rnn.rs:251-379) ----
    auto dense = [&](const HostDense& L, const std::vector<float>& in) {
        std::vector<float> out(L.nn);
        for (int o = 0; o < L.nn; o++) {
            float acc = (float)B[L.b_off + o];
            for (int j = 0; j < L.ni; j++) acc += (float)B[L.w_off + (size_t)j * L.nn + o] * in[j];
            out[o] = h_act(L.act, acc * (1.0f / 256.0f));
        }
        return out;
    };
    auto grul = [&](const HostGru& L, const std::vector<float>& in, std::vector<float>& st) {
        const int n = L.nn, st3 = 3 * n;
        std::vector<float> z(n), r(n), h(n);
        for (int o = 0; o < n; o++) {
            float az = (float)B[L.b_off + o], ar = (float)B[L.b_off + n + o];
            for (int j = 0; j < L.ni; j++) { az += (float)B[L.w_off + (size_t)j * st3 + o] * in[j]; ar += (float)B[L.w_off + (size_t)j * st3 + n + o] * in[j]; }
            for (int j = 0; j < n; j++) { az += (float)B[L.r_off + (size_t)j * st3 + o] * st[j]; ar += (float)B[L.r_off + (size_t)j * st3 + n + o] * st[j]; }
            z[o] = h_act(1, az * (1.0f / 256.0f));
            r[o] = h_act(1, ar * (1.0f / 256.0f)) * st[o];
        }
        for (int o = 0; o < n; o++) {
            float ah = (float)B[L.b_off + 2 * n + o];
            for (int j = 0; j < L.ni; j++) ah += (float)B[L.w_off + (size_t)j * st3 + 2 * n + o] * in[j];
            for (int j = 0; j < n; j++) ah += (float)B[L.r_off + (size_t)j * st3 + 2 * n + o] * r[j];
            h[o] = z[o] * st[o] + (1.0f - z[o]) * h_act(L.act, ah * (1.0f / 256.0f));
        }
        st = h;
    };
    std::vector<float> rv = sv, rn = sn, rd = sd;
    std::vector<float> dout = dense(hm.input_dense, feat);
    grul(hm.vad_gru, dout, rv);
    const float rvad = dense(hm.vad_output, rv)[0];
    std::vector<float> nin(dout);
    nin.insert(nin.end(), rv.begin(), rv.end());
    nin.insert(nin.end(), feat.begin(), feat.end());
    grul(hm.noise_gru, nin, rn);
    std::vector<float> din(rv);
    din.insert(din.end(), rn.begin(), rn.end());
    din.insert(din.end(), feat.begin(), feat.end());
    grul(hm.denoise_gru, din, rd);
    std::vector<float> rg = dense(hm.denoise_output, rd);

    // ---- replay of the kernel's phases from the blob, slab by slab ----
    std::vector<float> A(A_MAX_HALVES + 16, 0.0f), F(16 * FEAT_CHUNKS, 0.0f), D(MAX_N, 0.0f);
    for (int j = 0; j < NB_FEATURES; j++) F[j] = feat[j];
    for (int j = 0; j < nv; j++) A[d.o_vad + j] = sv[j];
    for (int j = 0; j < nn; j++) A[d.o_noise + j] = sn[j];
    for (int j = 0; j < ndn; j++) A[d.o_den + j] = sd[j];
    auto run = [&](int p) {
        const TcPhase& ph = d.ph[p];
        std::fill(D.begin(), D.end(), 0.0f);
        for (int si = d.slab0[p]; si < d.slab0[p + 1]; si++) {
            const TcSlab& sl = d.slab[si];
            const __half* wb = reinterpret_cast<const __half*>(blob.data() + sl.off);  // the slab as the kernel receives it
            for (int n = 0; n < ph.n; n++)
                for (int kc = sl.kc0; kc < sl.kc1; kc++)
                    for (int kk = 0; kk < 16; kk++) {
                        const float a = ph.chunk[kc] >= 0 ? A[ph.chunk[kc] * 16 + kk] : F[(-ph.chunk[kc] - 1) * 16 + kk];
                        const int k = (kc - sl.kc0) * 16 + kk;
                        D[n] += a * __half2float(wb[(size_t)(k / 8) * (ph.n * 8) + (size_t)n * 8 + (k % 8)]);
                    }
        }
    };
    auto bias = [&](int p) { return reinterpret_cast<const float*>(blob.data() + d.ph[p].b_off); };
    run(PH_DENSE);
    for (int o = 0; o < d.p_d; o++) A[d.o_dense + o] = o < nd ? h_act(d.act_dense, (D[o] + bias(PH_DENSE)[o]) / 256.0f) : 0.0f;
    std::vector<float> ev = sv, en = sn, ed = sd;
    auto gru = [&](int pzr, int phh, int act, int n_, int p8, std::vector<float>& st, int a_off) {
        run(pzr);
        std::vector<float> z(p8);
        for (int o = 0; o < p8; o++) {
            const float hp = o < n_ ? st[o] : 0.0f;
            const int cz = gate_col(0, o, 2), cr = gate_col(1, o, 2);
            z[o] = h_act(1, (D[cz] + bias(pzr)[cz]) / 256.0f);
            A[d.o_rh + o] = o < n_ ? h_act(1, (D[cr] + bias(pzr)[cr]) / 256.0f) * hp : 0.0f;
        }
        run(phh);
        for (int o = 0; o < p8; o++) {
            const float hp = o < n_ ? st[o] : 0.0f;
            const float c = h_act(act, (D[o] + bias(phh)[o]) / 256.0f);
            const float hn = o < n_ ? z[o] * hp + (1.0f - z[o]) * c : 0.0f;
            if (o < n_) st[o] = hn;
            A[a_off + o] = hn;
        }
    };
    gru(PH_VAD_ZR, PH_VAD_H, d.act_vad, nv, d.p_v, ev, d.o_vad);
    run(PH_VAD_OUT);
    const float evad = h_act(d.act_vadout, (D[0] + bias(PH_VAD_OUT)[0]) / 256.0f);
    gru(PH_NOISE_ZR, PH_NOISE_H, d.act_noise, nn, d.p_n, en, d.o_noise);
    gru(PH_DEN_ZR, PH_DEN_H, d.act_den, ndn, d.p_dn, ed, d.o_den);
    run(PH_OUT);
    double worst = std::fabs(evad - rvad);
    for (int o = 0; o < NB_BANDS; o++) worst = std::max(worst, (double)std::fabs(h_act(d.act_out, (D[o] + bias(PH_OUT)[o]) / 256.0f) - rg[o]));
    for (int o = 0; o < nv; o++) worst = std::max(worst, (double)std::fabs(ev[o] - rv[o]));
    for (int o = 0; o < nn; o++) worst = std::max(worst, (double)std::fabs(en[o] - rn[o]));
    for (int o = 0; o < ndn; o++) worst = std::max(worst, (double)std::fabs(ed[o] - rd[o]));
    return worst;
}
