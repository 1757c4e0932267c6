// pitch.cu -- pitch analysis (src/pitch.rs:45-489) with a BIT-IDENTICAL integer period, 16 streams per block.
//
// Compiled with -fmad=false; every operation whose value reaches an output or the carried state is written
// with explicit round-to-nearest intrinsics in the reference's order (same roundings, same summation order).
//
// Two families of dot products dominate the path: the 147-lag coarse cross-correlation (src/pitch.rs:82,
// 296-363: 35k multiply-adds per stream-frame) and the sub-harmonic inner products of remove_doubling
// (src/pitch.rs:152-168: up to 23 x 480).  Neither value is an output: they only feed COMPARISONS
// (find_best_pitch's selection, the g1 > thresh ladder).  They are therefore computed with FMA in whatever
// order maps best onto the machine, and every comparison is certified:
//   for ANY order and any mix of fused / unfused roundings  |computed - exact| <= gamma_n sum|x_j y_j|
//   <= gamma_n ||x|| ||y||  (gamma_n = n u / (1 - n u), u = 2^-24), so a fast value and the reference's value
//   differ by at most kappa ||x|| ||y||, kappa = 2 gamma_n.
//   * coarse search: scores r_i = c_i^2 / y_i with intervals [lo_i, hi_i]; candidate set C = {j : hi_j (1+eta) >=
//     min(lo_F1, lo_F2)} around the approximate top two.  |C| = 2 with lo_F1 > hi_F2 (1+eta): (best, second) =
//     (F1, F2).  Otherwise the <= 8 candidates are recomputed in the reference's order, each must beat every
//     non-candidate's upper bound robustly, and the reference's sequential selection runs on C alone.  (If a set
//     "top" of >= 2 lags robustly beats every other lag, find_best_pitch ends in the same state as its scan
//     restricted to top: DESIGN.md section 4.)  Anything else: all 147 lags of that stream are recomputed exactly.
//   * remove_doubling: |g1^ - thresh^| > dg1 + 0.9 dg0 + 1e-6, else all inner products of that stream are
//     recomputed exactly and the ladder is replayed on them.
// What becomes STATE or OUTPUT (last_gain, the +-1 refinements, the fine search) is always order-exact.
// tools/pitch_fast_model.c is the CPU model of this logic (2.4M frames against the oracle: 0 mismatches, 0.56 % of
// stream-frames need an exact recomputation); tests/test_gpu_parity.py::test_pitch_mass_* is the GPU check.
//
// Why many streams per block: the path alternates strictly sequential recurrences (5-lag autocorrelation,
// Levinson, running energies with a clamp per step, the k = 2..15 ladder) with dense sums.  Recurrences run
// LANE-PER-STREAM (operands fetched as float4 rows of the shared-memory tile); dense sums are spread over
// (stream, lag-group) lane-tasks with register sliding windows, or one warp per stream with the 480 samples
// dealt to the lanes (15 each: conflict-free scalar reads for arbitrary lags, x held in registers).
//
// Shared-memory tile (dynamic, SB = 16 streams per block -> 75.7 KB, THREE blocks per SM: the serial phases of one block
// hide behind the dense phases of two others):
//   P   [SB][868]  2x-decimated, LPC-whitened history (pitch_buf); row stride 868 = 16B aligned and
//                  = 4 (mod 32) so that lane-per-stream float4 reads are bank-conflict free.  The 4x-decimated
//                  signal of the coarse search is P at stride 2 (no second copy: it cost 28 KB and the third block)
//   XC  [SB][149]  coarse cross-correlation; dead after the coarse search, then: IPR | LAGS | NLAG | YYS | YYK | YNF
//   YNK [SB][75]   coarse running energy (exact), every second lag (the odd lags are one replayed step away)
//   CK  [SB][39]   fine running energy, one checkpoint every 8 lags; dead after the fine search, then the ladder's gains
//   YYK [SB][49]   yy_lookup, one checkpoint every 8 lags; YYS [SB][24] its values at the lags the ladder reads
// All three running energies are sequential recurrences; a replay from a checkpoint repeats the same operations in the
// same order, hence the same bits.
#include <atomic>

#include "common.cuh"

namespace nnb {

namespace {

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }

#ifndef PITCH_SB
#define PITCH_SB 16
#endif
#ifndef PITCH_NT
#define PITCH_NT 256
#endif
constexpr int SB = PITCH_SB;    // streams per block (lane-per-stream phases use lanes 0..SB-1, the others predicated off)
constexpr int NT = PITCH_NT;    // threads per block
constexpr int NW = NT / 32;
static_assert(SB == 16 && NW >= 4, "phase-to-warp assignment below assumes 16 streams and >= 4 warps");
constexpr int PB = PITCH_BUF_SIZE / 2;                                 // 864
constexpr int MAXP = PITCH_MAX_PERIOD - 3 * PITCH_MIN_PERIOD;          // 588
constexpr int N4 = PITCH_FRAME_SIZE / 4;                               // 240
constexpr int NL4 = MAXP / 4;                                          // 147 coarse lags
constexpr int NL2 = MAXP / 2;                                          // 294 fine lags
constexpr int HALF_MAX = PITCH_MAX_PERIOD / 2;                         // 384
constexpr int HALF_N = PITCH_FRAME_SIZE / 2;                           // 480
constexpr int MIN_PERIOD2 = PITCH_MIN_PERIOD / 2;                      // 30

constexpr int P_LD = 868;
constexpr int XC_LD = 149;
constexpr int YNK_LD = 75;   // checkpoints of the coarse running energy (every second lag: 74 values)
constexpr int YYK_STEP = 8;
constexpr int FX_LD = 17;  // two fine windows per stream (6 even-aligned lags each, at offsets 0 and 8)
constexpr int NGRP = (NL4 + 3) / 4;  // 37 lag groups of 4
constexpr int CMAX = 8;              // coarse candidates recomputed exactly per stream
constexpr int LAG_LD = 24;           // remove_doubling lags per stream: 1 + 2 * 11 (k <= 12 because t1 >= 30, t0 <= 383)
constexpr int NSLOT = (NL4 + 31) / 32;  // 5 coarse lags per lane in the selection

// 2 gamma_n with head-room: n = 240 (+ the final adds) and n = 480
constexpr float KAPPA4 = 3.1e-5f;
constexpr float KAPPA2 = 6.0e-5f;
constexpr float ETA1 = 1.00001f;     // slack of every certified comparison (covers the float roundings of the check itself)

constexpr int CK_STEP = 8;                         // fine running energy: one checkpoint every 8 lags
constexpr int CK_N = (NL2 + CK_STEP - 1) / CK_STEP;  // 37
constexpr int CK_LD = 39;
constexpr int SF_LD = 19;                          // selection scratch (CAND 8 | CEX 8 | MB | NEEDX), then FX[17]
constexpr int OFF_P = 0;
constexpr int OFF_XC = OFF_P + SB * P_LD;
constexpr int OFF_YNK = OFF_XC + SB * XC_LD;
constexpr int OFF_CK = OFF_YNK + SB * YNK_LD;      // [SB][39]
constexpr int OFF_SF = OFF_CK + SB * CK_LD;        // [SB][26]
constexpr int OFF_AC = OFF_SF + SB * SF_LD;        // [5][SB]
constexpr int OFF_LPC = OFF_AC + 5 * SB;           // [5][SB]
constexpr int OFF_XX = OFF_LPC + 5 * SB;           // [SB]
constexpr int OFF_BND = OFF_XX + SB;               // [3][SB]: sum x_lp4^2 | sum P[0..384)^2 | sum of the even P[0..384)^2
constexpr int OFF_NZ = OFF_BND + 3 * SB;           // int [2][SB]: OR of the magnitude bits of P[384..864) | P[0..384)
constexpr int OFF_SI = OFF_NZ + 2 * SB;            // int [6][SB]: best4, second4, t0, t, t1b, position of t in LAGS
constexpr int OFF_CTR = OFF_SI + 6 * SB;           // int [8]
constexpr int OFF_FLAG = OFF_CTR + 8;              // int [SB]: bit 0 coarse all-exact, bit 1 remove_doubling all-exact, bit 2 coarse resolved
constexpr int OFF_CXL = OFF_FLAG + SB;             // int [SB]: streams whose coarse search is recomputed exactly
constexpr int OFF_RXL = OFF_CXL + SB;              // int [SB]: streams whose ladder is recomputed exactly
constexpr int OFF_XTL = OFF_RXL + SB;             // int [SB * CMAX]: exact single-lag tasks of the coarse search
constexpr int SMEM_FLOATS = OFF_XTL + SB * CMAX;
// inside a stream's XC row once the coarse search is over (all offsets in floats):
constexpr int XO_IPR = 0;                          // [31]
constexpr int XO_LAGS = 32;                        // int [24]
constexpr int XO_NLAG = 56;                        // int
constexpr int XO_YYS = 57;                         // [24]  yy_lookup at the lags of LAGS
constexpr int XO_YYK = 81;                         // [49]  yy_lookup checkpoints (lag 8 m)
constexpr int XO_YNF = 130;                        // [10]  fine running energy at the lags of the two fine windows
static_assert(XO_YYK + HALF_MAX / YYK_STEP + 1 <= XO_YNF && XO_YNF + 10 <= XC_LD, "ladder scratch must fit in the XC row");
// inside a stream's SF row
constexpr int SO_CAND = 0, SO_CEX = CMAX, SO_MB = 2 * CMAX, SO_NEEDX = 2 * CMAX + 1;
static_assert(CK_N <= CK_LD, "checkpoint row too short");
static_assert(FX_LD <= SF_LD && SO_NEEDX < SF_LD, "fine-window results reuse the selection scratch");
static_assert(3 * (SMEM_FLOATS * 4 + 1024) <= 228 * 1024, "three blocks per SM");


__device__ __forceinline__ float pitch_gain(float xy, float xx, float yy) {
    return __fdiv_rn(xy, __fsqrt_rn(fa(1.0f, fm(xx, yy))));  // src/pitch.rs:485-487
}

// Selection step of find_best_pitch (src/pitch.rs:383-400), written with selects instead of branches (the
// lanes of a warp are different streams): identical comparisons on identical values.
struct BestTwo {
    float best_num = -1.0f, second_num = -1.0f, best_den = 0.0f, second_den = 0.0f;
    int best = 0, second = 1;
    __device__ __forceinline__ void consider(int i, float corr, float ysq) {
        const float num = fm(corr, corr);
        const bool c2 = (corr > 0.0f) && (fm(num, second_den) > fm(second_num, ysq));
        const bool c1 = c2 && (fm(num, best_den) > fm(best_num, ysq));
        // c1: candidate becomes best, old best becomes second;  c2 && !c1: candidate becomes second
        second_num = c1 ? best_num : (c2 ? num : second_num);
        second_den = c1 ? best_den : (c2 ? ysq : second_den);
        second = c1 ? best : (c2 ? i : second);
        best_num = c1 ? num : best_num;
        best_den = c1 ? ysq : best_den;
        best = c1 ? i : best;
    }
};

// celt_autocorr lag K for one stream (lane-per-stream): sum_{j<860} p[j] p[j+K] in order, then the tail
// sum_{i=K+860}^{863} p[i] p[i-K] (src/pitch.rs:433-446, 296-363; empty for K = 4).  row = 217 float4.
template <int K>
__device__ __forceinline__ float autocorr_lag(const float4* __restrict__ row) {
    float c = 0.0f;
    float4 w0 = row[0];
#pragma unroll 5
    for (int m = 0; m < (PB - 4) / 4; m++) {
        const float4 w1 = row[m + 1];
        const float e[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int d = 0; d < 4; d++) c = fa(c, fm(e[d], e[d + K]));
        w0 = w1;
    }
    // w0 = p[860..863]
    const float e[4] = {w0.x, w0.y, w0.z, w0.w};
    float d = 0.0f;
#pragma unroll
    for (int i = K; i < 4; i++) d = fa(d, fm(e[i], e[i - K]));
    return fa(c, d);
}

// Barrier among a SUBSET of the block's warps (id 1..15; __syncthreads is id 0): the long serial chains run on their own
// warps past the barriers of phases that do not need their result.
__device__ __forceinline__ void bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// inner_prod(x, y, 480) of src/pitch.rs:225-244 for one (stream, lag) lane-task:
// xr = aligned float4 row of x (pbuf + 384), y = pbuf + 384 - lag (unaligned scalars).
__device__ __forceinline__ float inner_prod_480(const float4* __restrict__ xr, const float* __restrict__ y) {
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
#pragma unroll 4
    for (int m = 0; m < HALF_N / 4; m++) {
        const float4 x = xr[m];
        s0 = fa(s0, fm(x.x, y[4 * m]));
        s1 = fa(s1, fm(x.y, y[4 * m + 1]));
        s2 = fa(s2, fm(x.z, y[4 * m + 2]));
        s3 = fa(s3, fm(x.w, y[4 * m + 3]));
    }
    return fa(fa(fa(s0, s1), s2), s3);
}

// Two consecutive lags of inner_prod(x, y + lag, 480) starting at an 8-byte aligned y (64-bit reads):
// acc[c][u] is the reference's accumulator u of lag c.
__device__ __forceinline__ void inner_prod_window2_aligned(const float4* __restrict__ xr, const float2* __restrict__ yr, float* out) {
    float acc[2][4];
#pragma unroll
    for (int c = 0; c < 2; c++)
#pragma unroll
        for (int u = 0; u < 4; u++) acc[c][u] = 0.0f;
    float2 w0 = yr[0], w1 = yr[1];
#pragma unroll 4
    for (int m = 0; m < HALF_N / 4; m++) {
        const float4 x = xr[m];
        const float2 w2 = yr[2 * m + 2];
        const float e[5] = {w0.x, w0.y, w1.x, w1.y, w2.x};
        const float xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int u = 0; u < 4; u++)
#pragma unroll
            for (int c = 0; c < 2; c++) acc[c][u] = fa(acc[c][u], fm(xv[u], e[u + c]));
        w0 = w2;
        w1 = yr[2 * m + 3];
    }
#pragma unroll
    for (int c = 0; c < 2; c++) out[c] = fa(fa(fa(acc[c][0], acc[c][1]), acc[c][2]), acc[c][3]);
}

// Sixteen consecutive coarse lags 16g..16g+15 of one stream, FMA (certified afterwards).  The 4x-decimated operands are the
// even samples of the whitened row: x_lp4[j] = p[384 + 2 j], y_lp4[j] = p[2 j] (src/pitch.rs:74-79).  (ptxas splits the
// 128-bit reads into the two 32-bit halves that are used; forcing LDS.128 with ld.volatile removes 210 of the 1850
// shared-memory wavefronts per stream and was measured no faster -- the kernel is not wavefront-bound.)
__device__ __forceinline__ void coarse_group16(const float* __restrict__ prow, int g, float* __restrict__ xcrow) {
    const float4* xr = reinterpret_cast<const float4*>(prow + HALF_MAX);
    const float4* yr = reinterpret_cast<const float4*>(prow + 32 * g);
    float acc[16];
#pragma unroll
    for (int c = 0; c < 16; c++) acc[c] = 0.0f;
    float e[20];
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const float4 v = yr[q];
        e[2 * q] = v.x;
        e[2 * q + 1] = v.z;
    }
#pragma unroll 5  // the 20-sample window rotates with period 5: no register moves at the back-edge
    for (int m = 0; m < N4 / 4; m++) {
        const float4 xa = xr[2 * m], xb = xr[2 * m + 1];
        const float4 va = yr[2 * m + 8], vb = yr[2 * m + 9];
        e[16] = va.x; e[17] = va.z; e[18] = vb.x; e[19] = vb.z;
        const float xv[4] = {xa.x, xa.z, xb.x, xb.z};
#pragma unroll
        for (int u = 0; u < 4; u++)
#pragma unroll
            for (int c = 0; c < 16; c++) acc[c] = ffma(xv[u], e[u + c], acc[c]);
#pragma unroll
        for (int q = 0; q < 16; q++) e[q] = e[q + 4];
    }
#pragma unroll
    for (int c = 0; c < 16; c++)
        if (16 * g + c < NL4) xcrow[16 * g + c] = acc[c];
}

// Four consecutive coarse lags 4g..4g+3 of one stream in the REFERENCE's order (src/pitch.rs:82, 296-363): every accumulator
// sums x_lp4[j] * y_lp4[lag + j] with j ascending, separate multiply and add.  Used where the certificate of the FMA
// values fails.
__device__ __forceinline__ void coarse_group4_exact(const float* __restrict__ prow, int g, float* __restrict__ xcrow) {
    const float4* xr = reinterpret_cast<const float4*>(prow + HALF_MAX);
    const float4* yr = reinterpret_cast<const float4*>(prow + 8 * g);
    float c0 = 0.0f, c1 = 0.0f, c2 = 0.0f, c3 = 0.0f;
    float e[8];
    {
        const float4 v0 = yr[0], v1 = yr[1];
        e[0] = v0.x; e[1] = v0.z; e[2] = v1.x; e[3] = v1.z;
    }
#pragma unroll 2
    for (int m = 0; m < N4 / 4; m++) {
        const float4 xa = xr[2 * m], xb = xr[2 * m + 1];
        const float4 va = yr[2 * m + 2], vb = yr[2 * m + 3];
        e[4] = va.x; e[5] = va.z; e[6] = vb.x; e[7] = vb.z;
        const float xv[4] = {xa.x, xa.z, xb.x, xb.z};
#pragma unroll
        for (int u = 0; u < 4; u++) {
            c0 = fa(c0, fm(xv[u], e[u]));
            c1 = fa(c1, fm(xv[u], e[u + 1]));
            c2 = fa(c2, fm(xv[u], e[u + 2]));
            c3 = fa(c3, fm(xv[u], e[u + 3]));
        }
#pragma unroll
        for (int q = 0; q < 4; q++) e[q] = e[q + 4];
    }
    float* o = xcrow + 4 * g;
    o[0] = c0;
    o[1] = c1;
    o[2] = c2;
    if (4 * g + 3 < NL4) o[3] = c3;
}

#ifdef PITCH_PROFILE
// Per-warp clock trace of one launch (profiling build only): lane 0 of every warp writes clock64() at each trace point,
// g_pitch_trace[(block * NW + warp) * PT_N + point], points = the warp's arrival at each barrier (a stamp right after a
// barrier would be taken before the warp blocks: BAR.SYNC.DEFER_BLOCKING).  Slot PT_N - 1 holds the SM.
// tools/pitch_phase_profile.py turns it into busy / barrier-wait cycles per phase and warp.
constexpr int PT_N = 32;
__device__ long long* g_pitch_trace;
#define PT(k)                                            \
    do {                                                 \
        if (pt_ && lane == 0) pt_[k] = clock64();        \
    } while (0)
#else
#define PT(k)
#endif

// stats[0] += streams whose coarse search was recomputed exactly, stats[1] += streams whose ladder was,
// stats[2] += streams processed (one atomic per block each); pf_ahead = blocks resident at once (0: no L2 prefetch)
__global__ void __launch_bounds__(NT, 3) pitch_kernel(const float* __restrict__ hist, int32_t* __restrict__ last_period,
                                                      float* __restrict__ last_gain, int32_t* __restrict__ pitch_out,
                                                      int n_streams, int hbase, int force_exact, int pf_ahead,
                                                      unsigned long long* __restrict__ stats) {
    extern __shared__ __align__(16) float sm[];
    float* P = sm + OFF_P;
    float* XC = sm + OFF_XC;
    float* YNK = sm + OFF_YNK;
    float* CK = sm + OFF_CK;
    float* SF = sm + OFF_SF;
    float* AC = sm + OFF_AC;
    float* LPC = sm + OFF_LPC;
    float* XX = sm + OFF_XX;
    float* BND = sm + OFF_BND;
    int* NZ = reinterpret_cast<int*>(sm + OFF_NZ);
    int* SI = reinterpret_cast<int*>(sm + OFF_SI);
    int* CTR = reinterpret_cast<int*>(sm + OFF_CTR);
    // CTR: [1] remove_doubling stream counter, [2] streams in CXL, [3] entries in XT, [4] streams in RXL,
    //      [7] CXL entries already recomputed
    int* FLAG = reinterpret_cast<int*>(sm + OFF_FLAG);
    int* CXL = reinterpret_cast<int*>(sm + OFF_CXL);
    int* RXL = reinterpret_cast<int*>(sm + OFF_RXL);
    int* XT = reinterpret_cast<int*>(sm + OFF_XTL);
    // per-stream views: selection scratch / fine-window results in SF, ladder scratch in the (dead) XC row
    auto CANDp = [&](int s_) { return reinterpret_cast<int*>(SF + s_ * SF_LD + SO_CAND); };
    auto CEXp = [&](int s_) { return SF + s_ * SF_LD + SO_CEX; };
    auto FXp = [&](int s_) { return SF + s_ * SF_LD; };
    auto IPRp = [&](int s_) { return XC + s_ * XC_LD + XO_IPR; };
    auto LAGSp = [&](int s_) { return reinterpret_cast<int*>(XC + s_ * XC_LD + XO_LAGS); };
    auto NLAGp = [&](int s_) { return reinterpret_cast<int*>(XC + s_ * XC_LD + XO_NLAG); };
    auto YYSp = [&](int s_) { return XC + s_ * XC_LD + XO_YYS; };
    auto YYKp = [&](int s_) { return XC + s_ * XC_LD + XO_YYK; };
    auto YNFp = [&](int s_) { return XC + s_ * XC_LD + XO_YNF; };
    // the fine search's lags of stream s_ (src/pitch.rs:88-97): two 5-lag windows around 2 best4 and 2 second4, clipped to
    // the valid range and scanned in ascending order without overlap; lag j < 5 is lo0 + j (up to hi0), j >= 5 is lo1 + j - 5
    struct FineLags { int cA, cB, lo0, hi0, lo1, hi1; };
    auto fine_lags = [&](int s_) {
        FineLags f;
        f.cA = 2 * SI[0 * SB + s_];
        f.cB = 2 * SI[1 * SB + s_];
        const int c0 = min(f.cA, f.cB) - 2, c1 = max(f.cA, f.cB) - 2;
        f.lo0 = max(c0, 0);
        f.hi0 = min(c0 + 4, NL2 - 1);
        f.lo1 = max(max(c1, 0), f.hi0 + 1);
        f.hi1 = min(c1 + 4, NL2 - 1);
        return f;
    };
    // coarse running energy at lag i of stream s_ (src/pitch.rs:379-382, 401-402), replayed from the checkpoint at or below it
    auto yn4_at = [&](int s_, int i) -> float {
        const float* prow_ = P + s_ * P_LD;
        float y = YNK[s_ * YNK_LD + (i >> 1)];
        if (i & 1) {
            const float a = prow_[2 * (N4 + i - 1)], b = prow_[2 * (i - 1)];
            y = fmaxf(fa(y, fs(fm(a, a), fm(b, b))), 1.0f);
        }
        return y;
    };

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ls = lane % SB;  // lane-per-stream phases: lanes >= SB mirror lanes < SB (same reads, same writes)
    const int s0 = blockIdx.x * SB;
    const int ns = min(SB, n_streams - s0);
#ifdef PITCH_PROFILE
    long long* pt_ = g_pitch_trace ? g_pitch_trace + ((size_t)blockIdx.x * NW + warp) * PT_N : nullptr;
    if (pt_ && lane == 0) {
        unsigned smid_;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid_));
        pt_[PT_N - 1] = smid_;
    }
    PT(0);
#endif

    // ---- Ph1: pitch_downsample part 1 (src/pitch.rs:455-458); all 128-bit loads of a row issued before use ----
    for (int r = warp; r < SB; r += NW) {
        float* prow = P + r * P_LD;
        constexpr int NQ = (PITCH_BUF_SIZE / 4 + 31) / 32;  // 14 float4 per lane
        if (r < ns) {
            const float* h = hist + (size_t)(s0 + r) * HIST_CAP;
            float4 v[NQ];
#pragma unroll
            for (int k = 0; k < NQ; k++) {
                const int m = lane + 32 * k;
                v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (m < PITCH_BUF_SIZE / 4) {
                    int pos = hbase + 4 * m;  // hbase is a multiple of 4: a float4 never straddles the ring wrap
                    if (pos >= HIST_CAP) pos -= HIST_CAP;
                    v[k] = __ldg(reinterpret_cast<const float4*>(h + pos));
                }
            }
#pragma unroll
            for (int k = 0; k < NQ; k++) {
                const int m = lane + 32 * k;
                // sample 4 m - 1 is the last of float4 m - 1: lane - 1's v[k], or lane 31's v[k - 1] for lane 0
                const float up = __shfl_up_sync(0xffffffffu, v[k].w, 1);
                const float wrap = __shfl_sync(0xffffffffu, v[k > 0 ? k - 1 : 0].w, 31);
                const float pv = lane > 0 ? up : wrap;
                if (m < PITCH_BUF_SIZE / 4) {
                    float o0;
                    if (m == 0) o0 = fm(fa(fm(v[k].y, 0.5f), v[k].x), 0.5f);
                    else o0 = fm(fa(fm(fa(pv, v[k].y), 0.5f), v[k].x), 0.5f);
                    const float o1 = fm(fa(fm(fa(v[k].y, v[k].w), 0.5f), v[k].z), 0.5f);
                    *reinterpret_cast<float2*>(prow + 2 * m) = make_float2(o0, o1);
                }
            }
        } else {
            for (int i = lane; i < PB; i += 32) prow[i] = 0.0f;  // absent streams: zero rows
        }
        if (lane < 4) prow[PB + lane] = 0.0f;
    }
    if (tid < 8) CTR[tid] = 0;
    if (tid < SB) FLAG[tid] = 0;
    PT(1);
    __syncthreads();

    // ---- Ph2: celt_autocorr, lane = stream: warp k = lag k (k = 0..4), one 128-bit read per four steps ----
    if (warp < 5 && lane < SB) {  // lanes 16-31 stay off: a mirrored lane would double the shared-memory wavefronts
        const float4* row = reinterpret_cast<const float4*>(P + ls * P_LD);
        float v;
        switch (warp) {
            case 0: v = autocorr_lag<0>(row); break;
            case 1: v = autocorr_lag<1>(row); break;
            case 2: v = autocorr_lag<2>(row); break;
            case 3: v = autocorr_lag<3>(row); break;
            default: v = autocorr_lag<4>(row); break;
        }
        AC[warp * SB + ls] = v;
    }
    PT(3);
    __syncthreads();

    // ---- Ph3: noise floor, lag window, LPC(4), bandwidth expansion, extra zero (src/pitch.rs:462-480, 257-292) ----
    if (warp == 0) {
        float a[5];
#pragma unroll
        for (int i = 0; i < 5; i++) a[i] = AC[i * SB + ls];
        a[0] = fm(a[0], 1.0001f);
#pragma unroll
        for (int i = 1; i < 5; i++) {
            float w = fm(0.008f, (float)i);
            a[i] = fs(a[i], fm(fm(a[i], w), w));
        }
        float lpc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        if (a[0] != 0.0f) {
            float error = a[0];
            bool live = true;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                if (live) {
                    float rr = 0.0f;
#pragma unroll
                    for (int j = 0; j < i; j++) rr = fa(rr, fm(lpc[j], a[i - j]));
                    rr = fa(rr, a[i + 1]);
                    float r = __fdiv_rn(-rr, error);
                    lpc[i] = r;
#pragma unroll
                    for (int j = 0; j < (i + 1) / 2; j++) {
                        float t1 = lpc[j], t2 = lpc[i - 1 - j];
                        lpc[j] = fa(t1, fm(r, t2));
                        lpc[i - 1 - j] = fa(t2, fm(r, t1));
                    }
                    error = fs(error, fm(fm(r, r), error));
                    if (error < fm(0.001f, a[0])) live = false;  // "bail out once we get 30 dB gain"
                }
            }
        }
        float tmp = 1.0f;
#pragma unroll
        for (int i = 0; i < 4; i++) {
            tmp = fm(tmp, 0.9f);
            lpc[i] = fm(lpc[i], tmp);
        }
        LPC[0 * SB + ls] = fa(lpc[0], 0.8f);
        LPC[1 * SB + ls] = fa(lpc[1], fm(0.8f, lpc[0]));
        LPC[2 * SB + ls] = fa(lpc[2], fm(0.8f, lpc[1]));
        LPC[3 * SB + ls] = fa(lpc[3], fm(0.8f, lpc[2]));
        LPC[4 * SB + ls] = fm(0.8f, lpc[3]);
    }
    PT(5);
    __syncthreads();

    // ---- Ph4: fir5_in_place (src/pitch.rs:407-429).  (The second decimation, src/pitch.rs:74-79, is P read at stride 2.)
    // One warp per two rows (warp, warp + NW), both in the same rounds so that their chains overlap; four samples per lane,
    // 128-sample rounds from the END of the row backwards, so the five older inputs a round needs are still un-filtered
    // when it runs. ----
    static_assert(SB == 2 * NW, "Ph4: two rows per warp");
    {
        float* prow[2] = {P + warp * P_LD, P + (warp + NW) * P_LD};
        float nc[2][5];
#pragma unroll
        for (int j = 0; j < 2; j++)
#pragma unroll
            for (int i = 0; i < 5; i++) nc[j][i] = LPC[i * SB + warp + j * NW];
        for (int rd = (PB / 4 + 31) / 32 - 1; rd >= 0; rd--) {
            const int q = 32 * rd + lane;
            const bool on = q < PB / 4;
            float o[2][4];
            if (on) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const float4* row4 = reinterpret_cast<const float4*>(prow[j]);
                    const float4 cur = row4[q];
                    const float4 prv = q >= 1 ? row4[q - 1] : make_float4(0.f, 0.f, 0.f, 0.f);
                    const float e[9] = {q >= 2 ? prow[j][4 * q - 5] : 0.0f, prv.x, prv.y, prv.z, prv.w, cur.x, cur.y, cur.z, cur.w};
#pragma unroll
                    for (int d = 0; d < 4; d++)
                        o[j][d] = fa(fa(fa(fa(fa(e[5 + d], fm(nc[j][0], e[4 + d])), fm(nc[j][1], e[3 + d])), fm(nc[j][2], e[2 + d])),
                                           fm(nc[j][3], e[1 + d])),
                                     fm(nc[j][4], e[d]));
                }
            }
            __syncwarp();
            if (on) {
#pragma unroll
                for (int j = 0; j < 2; j++) reinterpret_cast<float4*>(prow[j])[q] = make_float4(o[j][0], o[j][1], o[j][2], o[j][3]);
            }
        }
    }
    PT(7);
    __syncthreads();

    // ---- Warp roles from here on (NW = 8).  Three serial chains run on their own warps beside the dense work:
    //   CKW (warp 5): fine running energy (needed in Ph8), YNW (warp 6): coarse running energy -- both under the coarse
    //                 cross-correlation of warps 0-4 (Ph5);
    //   YYW (warp 7): energies in Ph5, then yy_lookup (needed from Ph9 on): it leaves after Ph6x and runs PAST the barrier
    //                 of the fine search (named barrier 2 over the other seven warps), rejoining before Ph9.
    constexpr int CKW = NW - 3, YNW = NW - 2, YYW = NW - 1;
    constexpr int G1N = NT;
    static_assert(NW == 8, "warp roles assume 8 warps");
    const int g1idx = warp;
    const int g1tid = tid;

    if (warp == CKW) {
      if (lane < SB) {
        // y_sq_norm of find_best_pitch(xcorr, y, 480) (the FINE search, src/pitch.rs:97): a 774-step chain that needs
        // nothing but the whitened buffer.  Only every 8th value is kept (CK[m] = value seen at fine lag 8 m); Ph8 replays
        // the few steps it needs from the nearest checkpoint -- same operations in the same order, hence the same values.
        const float4* row = reinterpret_cast<const float4*>(P + ls * P_LD);
        float y = 1.0f;
#pragma unroll 4
        for (int m = 0; m < HALF_N / 4; m++) {
            const float4 v = row[m];
            y = fa(y, fm(v.x, v.x));
            y = fa(y, fm(v.y, v.y));
            y = fa(y, fm(v.z, v.z));
            y = fa(y, fm(v.w, v.w));
        }
        float* ck = CK + ls * CK_LD;
        ck[0] = y;
        // The checkpoint stores go to the same shared memory as the operands, so the compiler cannot move a later read
        // above them: the next iteration's operands are read before this iteration's store (in the YNW chain below too).
        float4 va = row[HALF_N / 4], vb = row[0];
#pragma unroll 2
        for (int m = 0; m < (CK_N - 1) * CK_STEP / 4; m++) {
            const float4 na = row[HALF_N / 4 + m + 1], nb = row[m + 1];
            const float a[4] = {va.x, va.y, va.z, va.w}, b[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
            for (int d = 0; d < 4; d++) y = fmaxf(fa(y, fs(fm(a[d], a[d]), fm(b[d], b[d]))), 1.0f);
            if ((m & 1) == 1) ck[(m + 1) >> 1] = y;  // after 4 (m + 1) steps
            va = na;
            vb = nb;
        }
      }
    }
    {
        // ---- Ph5: two more serial jobs, and the coarse cross-correlation (FMA) ----
        if (warp == YNW && lane < SB) {
            // y_sq_norm of find_best_pitch(xcorr, y_lp4, 240) (src/pitch.rs:379-382, 401-402) over y_lp4[j] = p[2 j]; one
            // checkpoint every second lag: YNK[m] = value seen at lag 2 m (yn4_at replays the odd lags' one step)
            const float4* row = reinterpret_cast<const float4*>(P + ls * P_LD);
            float y = 1.0f;
#pragma unroll 4
            for (int m = 0; m < N4 / 2; m++) {
                const float4 v = row[m];
                y = fa(y, fm(v.x, v.x));
                y = fa(y, fm(v.z, v.z));
            }
            float* out = YNK + ls * YNK_LD;
            out[0] = y;
            float4 va = row[N4 / 2], vb = row[0];
#pragma unroll 2
            for (int m = 0; m < NL4 / 2; m++) {  // two steps per float4, checkpoints up to lag 146
                const float4 na = row[N4 / 2 + m + 1], nb = row[m + 1];
                y = fmaxf(fa(y, fs(fm(va.x, va.x), fm(vb.x, vb.x))), 1.0f);
                y = fmaxf(fa(y, fs(fm(va.z, va.z), fm(vb.z, vb.z))), 1.0f);
                out[m + 1] = y;  // after 2 (m + 1) steps
                va = na;
                vb = nb;
            }
        } else if (warp == YYW) {
            // Four energies, one code path for both half-warps (h = lane >> 4), one pass over the row:
            //   h = 0: p[384..864): xx = inner_prod(x, x, 480) with its four interleaved accumulators (src/pitch.rs:133,
            //          225-244: EXACT, it reaches last_gain) and, from the even samples, sum x_lp4^2
            //   h = 1: p[0..384): sum p^2 and, from the even samples, the rest of sum y_lp4^2   (these three only bound errors)
            const int h = lane >> 4;
            const float4* pr = reinterpret_cast<const float4*>(P + ls * P_LD) + (h ? 0 : HALF_MAX / 4);
            const int np = h ? HALF_MAX / 4 : HALF_N / 4;
            float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f, e0 = 0.0f, e1 = 0.0f;
            unsigned nz = 0;  // does the row hold anything but (signed) zeros?  (a sum of squares may underflow to 0)
            auto step = [&](const float4 x) {
                const float sx = fm(x.x, x.x), sz = fm(x.z, x.z);
                a0 = fa(a0, sx);
                a1 = fa(a1, fm(x.y, x.y));
                a2 = fa(a2, sz);
                a3 = fa(a3, fm(x.w, x.w));
                e0 = fa(e0, sx);
                e1 = fa(e1, sz);
                nz |= __float_as_uint(x.x) | __float_as_uint(x.y) | __float_as_uint(x.z) | __float_as_uint(x.w);
            };
            // the part both half-warps have, then h = 0's tail: no lane-dependent branch inside the unrolled loop
#pragma unroll 4
            for (int m = 0; m < HALF_MAX / 4; m++) step(pr[m]);
#pragma unroll 4
            for (int m = HALF_MAX / 4; m < np; m++) step(pr[m]);
            NZ[h * SB + ls] = (int)(nz & 0x7fffffffu);
            const float sp = fa(fa(fa(a0, a1), a2), a3), sy = fa(e0, e1);
            if (h == 0) {
                XX[ls] = sp;
                BND[0 * SB + ls] = sy;
            } else {
                BND[1 * SB + ls] = sp;
                BND[2 * SB + ls] = sy;
            }
        }
        // coarse xcorr, FMA: lane-task = (stream, group of 16 consecutive lags): 160 tasks = warps 0-4 exactly
        if (warp < CKW) {
            // stream-minor task order: the 8 lanes of a quarter-warp read the SAME columns of 8 DIFFERENT rows (row stride
            // = 4 mod 32 words), so every LDS.128 is conflict-free; a lag-minor order put them 128 bytes apart in one row
            const int L = warp * 32 + lane;
            const int s = L % SB, g = L / SB;
            coarse_group16(P + s * P_LD, g, XC + s * XC_LD);
        }
        PT(9);
        bar_sync(1, G1N);

        // ---- Ph6a (G1): certified coarse selection, one warp per stream, lane = lags lane, lane + 32, ... (src/pitch.rs:83-84) ----
        for (int s = g1idx; s < SB; s += NW) {
            const float* xc = XC + s * XC_LD;
            float cv[NSLOT], yv[NSLOT];
#pragma unroll
            for (int k = 0; k < NSLOT; k++) {
                const int lag = lane + 32 * k;
                cv[k] = lag < NL4 ? xc[lag] : 0.0f;
                yv[k] = lag < NL4 ? yn4_at(s, lag) : 1.0f;
            }
            // approximate top two by score c^2 / y (c > 0): ANY two distinct lags keep the certificate sound, so the scores
            // may be rounded freely (fast division) and the warp maxima taken on their bit patterns (scores >= 0)
            float m1 = 0.0f, m2 = 0.0f;
            int k1 = 0, k2 = 0;
#pragma unroll
            for (int k = 0; k < NSLOT; k++) {
                const float r = cv[k] > 0.0f ? __fdividef(cv[k] * cv[k], yv[k]) : 0.0f;
                if (r > m1) {
                    m2 = m1; k2 = k1;
                    m1 = r; k1 = k;
                } else if (r > m2) {
                    m2 = r; k2 = k;
                }
            }
            const unsigned M1 = __reduce_max_sync(0xffffffffu, __float_as_uint(m1));
            const unsigned w1 = __ballot_sync(0xffffffffu, __float_as_uint(m1) == M1);
            const int L1 = __ffs(w1) - 1;
            int f1 = __shfl_sync(0xffffffffu, lane + 32 * k1, L1);
            if (M1 == 0u) f1 = -1;
            const float c2m = lane == L1 ? m2 : m1;
            const int c2k = lane == L1 ? k2 : k1;
            const unsigned M2 = __reduce_max_sync(0xffffffffu, __float_as_uint(c2m));
            const unsigned w2 = __ballot_sync(0xffffffffu, __float_as_uint(c2m) == M2);
            const int L2 = __ffs(w2) - 1;
            int f2 = __shfl_sync(0xffffffffu, lane + 32 * c2k, L2);
            if (M2 == 0u) f2 = -1;
            const float ex4 = BND[0 * SB + s], y4tot = BND[2 * SB + s] + ex4;
            const float delta = KAPPA4 * sqrtf(ex4 * y4tot) * 1.001f;
            int best = 0, second = 1, nc = 0;
            bool cx = (force_exact & 1) != 0, need = false;
            if (!(delta < 1e30f)) {
                cx = true;  // inf / nan
            } else if ((NZ[s] | NZ[SB + s]) == 0) {
                // the whitened history is exactly zero: every c_i is exactly 0 and the reference keeps its initial (0, 1)
            } else if (!(ex4 > 1e-18f) || !(y4tot > 1e-18f) || !(ex4 * y4tot * (y4tot + 1.0f) < 1e37f)) {
                // Outside the range where find_best_pitch's own products c^2 y (src/pitch.rs:386-388) stay finite and normal
                // (c^2 <= ex4 y4tot by Cauchy-Schwarz, 1 <= y <= y4tot + 1): there the reference selects on signs alone
                // (underflow) or gets stuck on inf > inf (overflow, amplitudes beyond ~2.5x the int16 range it documents).
                // Parity means reproducing that, so those streams take the order-exact path.  Inside the range every
                // score below is a finite, normal quotient.
                cx = true;
            } else if (f1 < 0 || f2 < 0 || f2 == f1) {
                cx = true;
            } else {
                const float c1 = xc[f1], c2 = xc[f2], y1 = yn4_at(s, f1), y2 = yn4_at(s, f2);
                const float a1 = c1 - delta, a2 = c2 - delta;
                if (!(a1 > 0.0f) || !(a2 > 0.0f) || !(a1 * a1 > 1e-20f) || !(a2 * a2 > 1e-20f)) {
                    cx = true;
                } else {
                    // scores as quotients (fast division: its 2 ulp are far inside the slack ETA1 of every comparison)
                    const float lo1 = __fdividef(a1 * a1, y1), lo2 = __fdividef(a2 * a2, y2);
                    const float b1 = c1 + delta, b2 = c2 + delta;
                    const float hi1 = __fdividef(b1 * b1, y1), hi2 = __fdividef(b2 * b2, y2);
                    const float t0s = fminf(lo1, lo2);  // T0 = min(lo_F1, lo_F2)
                    unsigned inmask = 0, masks[NSLOT];
                    float hmax = 0.0f;  // M = max upper bound over the non-candidates
#pragma unroll
                    for (int k = 0; k < NSLOT; k++) {
                        const int lag = lane + 32 * k;
                        const float b = fmaxf(cv[k] + delta, 0.0f);
                        const float hs = __fdividef(b * b, yv[k]);
                        const bool in_c = lag < NL4 && ((lag == f1 || lag == f2) || (hs * ETA1 >= t0s));
                        masks[k] = __ballot_sync(0xffffffffu, in_c);
                        if (in_c) inmask |= 1u << k;
                        if (lag < NL4 && !in_c) hmax = fmaxf(hmax, hs);
                    }
                    const float mbound = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(hmax))) * ETA1;
#pragma unroll
                    for (int k = 0; k < NSLOT; k++) nc += __popc(masks[k]);
                    if (nc > CMAX) {
                        cx = true;
                    } else {
                        int basek = 0;  // candidates in ascending lag order: slot-major, lane-minor
#pragma unroll
                        for (int k = 0; k < NSLOT; k++) {
                            if ((inmask >> k) & 1u) CANDp(s)[basek + __popc(masks[k] & ((1u << lane) - 1u))] = lane + 32 * k;
                            basek += __popc(masks[k]);
                        }
                        if (nc == 2 && lo1 > hi2 * ETA1) {         // lo_F1 > hi_F2 (1 + eta)
                            best = f1;
                            second = f2;
                        } else if (nc == 2 && lo2 > hi1 * ETA1) {  // the rounded scores had them the other way round
                            best = f2;
                            second = f1;
                        } else {
                            need = true;
                        }
                        if (lane == 0) SF[s * SF_LD + SO_MB] = mbound;
                    }
                }
            }
            if (cx) need = false;
            if (lane == 0) {
                SI[0 * SB + s] = best;
                SI[1 * SB + s] = second;
                reinterpret_cast<int*>(SF)[s * SF_LD + SO_NEEDX] = need ? nc : 0;
                if (cx) {
                    FLAG[s] = 1;
                    CXL[atomicAdd(&CTR[2], 1)] = s;
                } else if (need) {
                    const int base = atomicAdd(&CTR[3], nc);
                    for (int i = 0; i < nc; i++) XT[base + i] = (s << 8) | i;
                }
            }
        }
        PT(11);
        bar_sync(1, G1N);

        // ---- Ph6x (G1): exact recomputation where the certificate failed.  Round 0: the candidates of the "need" streams and
        // all 147 lags of the CXL streams; round 1: all lags of streams whose candidates turned out not to dominate. ----
        for (int round = 0; round < 2; round++) {
            const int ncx_lo = CTR[7], ncx = CTR[2], nx = round == 0 ? CTR[3] : 0;
            if (ncx == ncx_lo && nx == 0) break;  // uniform over G1
            for (int L = g1tid; L < nx; L += G1N) {
                const int e = XT[L], s = e >> 8, pos = e & 255;
                const int lag = CANDp(s)[pos];
                const float* prow = P + s * P_LD;
                const float4* xr = reinterpret_cast<const float4*>(prow + HALF_MAX);
                const float* yr = prow + 2 * lag;
                float c = 0.0f;  // src/pitch.rs:296-363: one accumulator per lag, j ascending; x_lp4[j] = p[384 + 2 j], y_lp4[j] = p[2 j]
#pragma unroll 4
                for (int m = 0; m < N4 / 4; m++) {
                    const float4 xa = xr[2 * m], xb = xr[2 * m + 1];
                    c = fa(c, fm(xa.x, yr[8 * m]));
                    c = fa(c, fm(xa.z, yr[8 * m + 2]));
                    c = fa(c, fm(xb.x, yr[8 * m + 4]));
                    c = fa(c, fm(xb.z, yr[8 * m + 6]));
                }
                CEXp(s)[pos] = c;
            }
            for (int L = g1tid; L < (ncx - ncx_lo) * NGRP; L += G1N) {  // stream-minor, like the FMA pass
                const int nst = ncx - ncx_lo, i = L % nst, g = L / nst;
                const int s = CXL[ncx_lo + i];
                coarse_group4_exact(P + s * P_LD, g, XC + s * XC_LD);
            }
            bar_sync(1, G1N);
            if (warp == 0 && lane < SB) {
                const int s = lane;
                const float* xc = XC + s * XC_LD;
                const int fl = FLAG[s];
                const int needx = reinterpret_cast<const int*>(SF)[s * SF_LD + SO_NEEDX];
                if ((fl & 1) && !(fl & 4)) {
                    // the reference's scan over all lags on exact values; its running energy advances with it
                    BestTwo b2;
                    const float* prow = P + s * P_LD;
                    float y = YNK[s * YNK_LD];
                    for (int i = 0; i < NL4; i++) {
                        b2.consider(i, xc[i], y);
                        const float a = prow[2 * (N4 + i)], b = prow[2 * i];
                        y = fmaxf(fa(y, fs(fm(a, a), fm(b, b))), 1.0f);
                    }
                    SI[0 * SB + s] = b2.best;
                    SI[1 * SB + s] = b2.second;
                    FLAG[s] = fl | 4;
                } else if (round == 0 && needx > 0) {
                    const float mbound = SF[s * SF_LD + SO_MB];
                    BestTwo b2;
                    bool ok = true;
                    for (int k = 0; k < needx; k++) {
                        const int lag = CANDp(s)[k];
                        const float c = CEXp(s)[k], ysq = yn4_at(s, lag);
                        // every candidate must beat the upper bound of every non-candidate robustly
                        if (!(c > 0.0f) || !(__fdividef(c * c, ysq) > mbound * ETA1)) ok = false;
                        b2.consider(lag, c, ysq);
                    }
                    if (ok) {
                        SI[0 * SB + s] = b2.best;
                        SI[1 * SB + s] = b2.second;
                    } else {
                        FLAG[s] = fl | 1;
                        CXL[atomicAdd(&CTR[2], 1)] = s;
                    }
                }
            }
            bar_sync(1, G1N);
            if (g1tid == 0) CTR[7] = ncx;
            bar_sync(1, G1N);
        }
        PT(13);

        if (warp == YYW) {
          if (lane < SB) {
            // yy_lookup (src/pitch.rs:135-142): carried unclamped, i = 1..384 walks the rows downwards; one checkpoint every
            // 8 lags (YYK[m] = unclamped value at lag 8 m), the lags the ladder reads are replayed from them in Ph9.
            // Runs beside the fine search (the XC row it writes into is dead after Ph6x).
            const float4* row = reinterpret_cast<const float4*>(P + ls * P_LD);
            float* out = YYKp(ls);
            float y = XX[ls];
            out[0] = y;
#pragma unroll 2
            for (int m = 0; m < HALF_MAX / 4; m++) {
                const float4 va = row[HALF_MAX / 4 - 1 - m];              // p[380-4m .. 383-4m]
                const float4 vb = row[(HALF_MAX + HALF_N) / 4 - 1 - m];   // p[860-4m .. 863-4m]
                const float a[4] = {va.w, va.z, va.y, va.x}, b[4] = {vb.w, vb.z, vb.y, vb.x};
#pragma unroll
                for (int d = 0; d < 4; d++) y = fa(y, fs(fm(a[d], a[d]), fm(b[d], b[d])));
                if ((m & 1) == 1) out[(m + 1) >> 1] = y;  // after 4 (m + 1) steps
            }
          }
        } else {
            // ---- Ph6b (all but YYW): the two 5-lag fine windows of every stream (src/pitch.rs:88-96).  Each window i0c .. i0c+4 (i0c =
            // start clamped into the valid range) lies inside the EVEN-aligned 6 lags a .. a+5, a = i0c & ~1, computed as three 2-lag
            // sliding windows: 96 lane-tasks (stream, window, pair of lags) = warps 0-2, 64-bit reads of the lagged row.
            // Which lags count as candidates is decided in Ph8. ----
            if (warp < 3) {
                const int L = warp * 32 + lane;
                const int s = L / 6, r6 = L - 6 * s, wdw = r6 / 3, qt = r6 - 3 * wdw;
                const int ctr = 2 * SI[wdw * SB + s];
                const int a = min(max(ctr - 2, 0), NL2 - 5) & ~1;
                const float* prow = P + s * P_LD;
                float out[2];
                inner_prod_window2_aligned(reinterpret_cast<const float4*>(prow + HALF_MAX),
                                           reinterpret_cast<const float2*>(prow + a + 2 * qt), out);
                FXp(s)[wdw * 8 + 2 * qt] = fmaxf(out[0], -1.0f);
                FXp(s)[wdw * 8 + 2 * qt + 1] = fmaxf(out[1], -1.0f);
            } else {
                // ---- Ph7 (warps 3-6, beside the fine windows): the fine running energy at the <= 10 lags the fine search reads,
                // one lane-task per (stream, lag), each replayed from the checkpoint at or below it: step i -> i + 1 is
                // y = max(y + p[480 + i]^2 - p[i]^2, 1) (src/pitch.rs:401-402), the chain's operations in its order. ----
                for (int L = tid - 3 * 32; L < SB * 10; L += 4 * 32) {
                    const int s = L % SB, j = L / SB;
                    const FineLags f = fine_lags(s);
                    const int i = j < 5 ? f.lo0 + j : f.lo1 + j - 5;
                    if (i <= (j < 5 ? f.hi0 : f.hi1)) {
                        const float* prow = P + s * P_LD;
                        float y = CK[s * CK_LD + i / CK_STEP];
                        for (int c = i & ~(CK_STEP - 1); c < i; c++) {
                            const float a = prow[HALF_N + c], b = prow[c];
                            y = fmaxf(fa(y, fs(fm(a, a), fm(b, b))), 1.0f);
                        }
                        YNFp(s)[j] = y;
                    }
                }
            }
        }
    }
    if (warp == YNW && lane < SB) {
        // Ph1 of a tile waits on its 110 KB of history from HBM.  Blocks start in index order as resident ones finish, so
        // block blockIdx.x + ahead (ahead = resident blocks of the grid) starts about when this one ends: bring its
        // streams' windows into L2 now, while this block's later phases run.  (Data movement only: no value changes.)
        const int s = s0 + pf_ahead * SB + lane;
        if (pf_ahead > 0 && s < n_streams) {
            const float* h = hist + (size_t)s * HIST_CAP;
            const int n1 = min(PITCH_BUF_SIZE, HIST_CAP - hbase);  // hbase is a multiple of 4: 16-byte aligned pieces
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(h + hbase), "r"(4 * n1) : "memory");
            if (n1 < PITCH_BUF_SIZE) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(h), "r"(4 * (PITCH_BUF_SIZE - n1)) : "memory");
        }
    }
    PT(15);
    if (warp != YYW) bar_sync(2, NT - 32);  // everybody but YYW: FX and YNF complete

    // ---- Ph8: fine best + pseudo-interpolation (src/pitch.rs:97-114), lane = stream ----
    if (warp == 0 && lane < SB) {
        const float* fx = FXp(ls);
        const FineLags f = fine_lags(ls);
        const int cA = f.cA, cB = f.cB;
        const int baseA = min(max(cA - 2, 0), NL2 - 5), baseB = min(max(cB - 2, 0), NL2 - 5);
        // xcorr at fine lag i: computed iff |i - 2 best| <= 2 or |i - 2 second| <= 2 (src/pitch.rs:90-95), else 0
        auto xcf = [&](int i) -> float {
            if (i < 0 || i >= NL2) return 0.0f;
            if (abs(i - cA) <= 2) return fx[i - (baseA & ~1)];
            if (abs(i - cB) <= 2) return fx[8 + i - (baseB & ~1)];
            return 0.0f;
        };
        BestTwo b2;
        // lags outside the windows have xcorr 0 and can never be selected: scan the windows in ascending order
        const float* ynf = YNFp(ls);
        for (int i = f.lo0; i <= f.hi0; i++) b2.consider(i, xcf(i), ynf[i - f.lo0]);
        for (int i = f.lo1; i <= f.hi1; i++) b2.consider(i, xcf(i), ynf[5 + i - f.lo1]);
        const int best = b2.best;
        int offset = 0;
        if (best > 0 && best < NL2 - 1) {
            const float a = xcf(best - 1), b = xcf(best), c = xcf(best + 1);
            if (fs(c, a) > fm(0.7f, fs(b, a))) offset = 1;
            else if (fs(a, c) > fm(0.7f, fs(b, c))) offset = -1;
        }
        const int pitch_idx = PITCH_MAX_PERIOD - (2 * best - offset);  // src/pitch.rs:49,114
        const int t0 = min(pitch_idx / 2, HALF_MAX - 1);                // t0 of remove_doubling
        // The lags remove_doubling needs (src/pitch.rs:134,152-168): t0, then for k = 2.. while t1 >= min_period the
        // pair (t1, t1b); IPR[stream][1 + position] = inner_prod(x, x - lag, 480).
        // (k is a compile-time constant in the unrolled loops below: the divisions by 2k become multiply-shifts)
        {
            SI[2 * SB + ls] = t0;
            int* lg = LAGSp(ls);
            lg[0] = t0;
            int nk = 0;
#pragma unroll
            for (int k = 2; k <= 12; k++) {
                constexpr int sc[16] = {0, 0, 3, 2, 3, 2, 5, 2, 3, 2, 3, 2, 5, 2, 3, 2};  // SECOND_CHECK, src/pitch.rs:489
                const int t1 = (2 * t0 + k) / (2 * k);
                if (nk == k - 2 && t1 >= MIN_PERIOD2) {
                    const int t1b = (k == 2) ? ((t1 + t0 > HALF_MAX) ? t0 : t0 + t1) : (2 * sc[k] * t0 + k) / (2 * k);
                    lg[1 + 2 * nk] = t1;
                    lg[2 + 2 * nk] = t1b;
                    nk++;
                }
            }
            *NLAGp(ls) = 1 + 2 * nk;
        }
    }
    PT(17);
    __syncthreads();  // everybody: LAGS written, yy_lookup complete

    // ---- Ph9: remove_doubling inner products, FMA, one WARP per stream: lane l owns samples 15 l .. 15 l + 14 of x
    // (registers) and of every lagged window (scalar reads at stride 15: conflict-free for any lag); eight lags share
    // one transposed shuffle reduction. ----
    for (;;) {
        int s = 0;
        if (lane == 0) s = atomicAdd(&CTR[1], 1);
        s = __shfl_sync(0xffffffffu, s, 0);
        if (s >= SB) break;
        const float* pl = P + s * P_LD + HALF_MAX + 15 * lane;
        float xr[15];
#pragma unroll
        for (int j = 0; j < 15; j++) xr[j] = pl[j];
        const int n = *NLAGp(s);
        const int* lg = LAGSp(s);
        // yy_lookup at this stream's lags: lane i replays lag lg[i] from the checkpoint at or below it (same operations in the
        // same order as the chain: the same bits); stored clamped at 0 like the reference's table
        if (lane < n) {
            const int L = lg[lane];
            const float* prow = P + s * P_LD;
            float y = YYKp(s)[L / YYK_STEP];
            for (int i = (L / YYK_STEP) * YYK_STEP + 1; i <= L; i++) {
                const float a = prow[HALF_MAX - i], b = prow[HALF_MAX + HALF_N - i];
                y = fa(y, fs(fm(a, a), fm(b, b)));
            }
            YYSp(s)[lane] = fmaxf(y, 0.0f);
        }
        for (int base = 0; base < n; base += 8) {
            float acc[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                acc[i] = 0.0f;
                if (base + i < n) {  // warp-uniform
                    const float* y = pl - lg[base + i];
#pragma unroll
                    for (int j = 0; j < 15; j++) acc[i] = ffma(xr[j], y[j], acc[i]);
                }
            }
            // transposed reduction: after the three exchange steps lane l holds, in acc[0], the sum over the lanes
            // {l ^ 16, l ^ 8, l ^ 4 combinations} of lag index 4 b4 + 2 b3 + b2 (bk = bit k of l)
            const bool h16 = (lane & 16) != 0, h8 = (lane & 8) != 0, h4 = (lane & 4) != 0;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float send = h16 ? acc[i] : acc[i + 4], keep = h16 ? acc[i + 4] : acc[i];
                acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
            }
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const float send = h8 ? acc[i] : acc[i + 2], keep = h8 ? acc[i + 2] : acc[i];
                acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
            {
                const float send = h4 ? acc[0] : acc[1], keep = h4 ? acc[1] : acc[0];
                acc[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], 2);
            acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], 1);
            const int idx = base + (h16 ? 4 : 0) + (h8 ? 2 : 0) + (h4 ? 1 : 0);
            if ((lane & 3) == 0 && idx < n) IPRp(s)[1 + idx] = acc[0];
        }
    }
    PT(19);
    __syncthreads();

    // ---- Ph10g: the gains the sub-harmonic ladder (src/pitch.rs:144-203) compares, one lane-task per (stream, step) on six warps:
    // step 0 = g0 at t0, step k - 1 = g1 of step k = 2..12 (none where t1 < min_period: the ladder stops there), with the
    // certificate's margin dg of each (fast values only).  They go to the stream's (dead) fine running-energy row, with
    // last_gain and the previous period, so the lane-per-stream ladder is a short scan of comparisons. ----
    // yy_lookup values come from YYS: position 0 = lag t0, positions 1 + 2 (k - 2) and 2 + 2 (k - 2) = lags t1, t1b of step k
    constexpr int NGAIN = 12, GO_DG = NGAIN, GO_LG = 2 * NGAIN, GO_PP = 2 * NGAIN + 1;
    static_assert(GO_PP < CK_LD && SB * NGAIN <= NT, "ladder gains: one row per stream, one thread per (stream, step)");
    auto gains = [&](int s, int q, bool exact) {
        float* gk = CK + s * CK_LD;
        const float* ipr = IPRp(s);
        const float* yys = YYSp(s);
        const float xx = XX[s];
        float xy, yy;
        if (q == 0) {
            xy = ipr[1];
            yy = yys[0];
        } else {
            const int k = q + 1, t0 = SI[2 * SB + s];
            if ((2 * t0 + k) / (2 * k) < MIN_PERIOD2) return;
            xy = fm(fa(ipr[2 + 2 * (k - 2)], ipr[3 + 2 * (k - 2)]), 0.5f);
            yy = fm(fa(yys[1 + 2 * (k - 2)], yys[2 + 2 * (k - 2)]), 0.5f);
        }
        gk[q] = pitch_gain(xy, xx, yy);
        if (!exact) {
            const float dip = KAPPA2 * sqrtf(xx * (BND[1 * SB + s] + xx)) * 1.001f;
            gk[GO_DG + q] = __fdiv_rn(dip, __fsqrt_rn(fa(1.0f, fm(xx, yy))));
        }
    };
    if (tid < SB * NGAIN) {
        const int s = tid % SB, q = tid / SB;
        gains(s, q, false);
        if (q == 0) {
            int pp = 0;
            float lgv = 0.0f;
            if (s < ns) {
                pp = last_period[s0 + s] / 2;
                lgv = last_gain[s0 + s];
            }
            CK[s * CK_LD + GO_LG] = lgv;
            reinterpret_cast<int*>(CK + s * CK_LD)[GO_PP] = pp;
        }
    }
    PT(20);
    __syncthreads();

    // ---- Ph10a: the ladder on the fast gains, lane = stream, every decision certified ----
    // exact == false: fast values with margins; exact == true (only for streams in RXL): the same code on exact values.
    auto ladder = [&](bool exact, int& t_out, int& t1b_out, int& pos_out, bool& uncertain) {
        const float* gk = CK + ls * CK_LD;
        const int t0 = SI[2 * SB + ls];
        const float xx = XX[ls];
        const float dip = exact ? 0.0f : KAPPA2 * sqrtf(xx * (BND[1 * SB + ls] + xx)) * 1.001f;
        uncertain = !(dip < 1e30f);
        const int prev_period = reinterpret_cast<const int*>(gk)[GO_PP];
        const float lg = gk[GO_LG];
        const float g0 = gk[0];
        const float dg0 = exact ? 0.0f : gk[GO_DG];
        int t = t0, t1bs = t0, pos = 0;
#pragma unroll
        for (int k = 2; k <= 12; k++) {
            constexpr int sc[16] = {0, 0, 3, 2, 3, 2, 5, 2, 3, 2, 3, 2, 5, 2, 3, 2};  // SECOND_CHECK, src/pitch.rs:489
            const int t1 = (2 * t0 + k) / (2 * k);
            if (t1 < MIN_PERIOD2) break;
            int t1b;
            if (k == 2) t1b = (t1 + t0 > HALF_MAX) ? t0 : t0 + t1;
            else t1b = (2 * sc[k] * t0 + k) / (2 * k);
            const float g1 = gk[k - 1];
            const int d = abs(t1 - prev_period);
            float cont;
            if (d <= 1) cont = lg;
            else if (d <= 2 && 5 * k * k < t0) cont = fm(lg, 0.5f);
            else cont = 0.0f;
            float thresh;
            if (t1 < 3 * MIN_PERIOD2) thresh = fmaxf(fs(fm(0.85f, g0), cont), 0.4f);
            else if (t1 < 2 * MIN_PERIOD2) thresh = fmaxf(fs(fm(0.9f, g0), cont), 0.5f);  // dead branch, as in the reference
            else thresh = fmaxf(fs(fm(0.7f, g0), cont), 0.3f);
            if (!exact) {
                const float dg1 = gk[GO_DG + k - 1];
                if (!(fabsf(g1 - thresh) > dg1 + 0.9f * dg0 + 1e-6f)) uncertain = true;
            }
            if (g1 > thresh) {
                t = t1;
                t1bs = t1b;
                pos = 1 + 2 * (k - 2);
            }
        }
        t_out = t;
        t1b_out = t1bs;
        pos_out = pos;
    };
    if (warp == 0 && lane < SB) {
        int t, t1b, pos;
        bool unc;
        ladder(false, t, t1b, pos, unc);
        if (force_exact & 2) unc = true;
        {
            SI[3 * SB + ls] = t;
            SI[4 * SB + ls] = t1b;
            SI[5 * SB + ls] = pos;
            if (unc) {
                FLAG[ls] |= 2;
                RXL[atomicAdd(&CTR[4], 1)] = ls;
            }
        }
    }
    PT(21);
    __syncthreads();

    // ---- Ph10x: streams whose ladder could not be certified: exact inner products (src/pitch.rs:225-244), exact replay ----
    {
        const int nrx = CTR[4];
        if (nrx > 0) {  // block-uniform
            for (int L = tid; L < nrx * LAG_LD; L += NT) {
                const int i = L / LAG_LD, q = L - i * LAG_LD;
                const int s = RXL[i];
                if (q < *NLAGp(s)) {
                    const float* prow = P + s * P_LD;
                    IPRp(s)[1 + q] = inner_prod_480(reinterpret_cast<const float4*>(prow + HALF_MAX), prow + HALF_MAX - LAGSp(s)[q]);
                }
            }
            __syncthreads();
            for (int L = tid; L < nrx * NGAIN; L += NT) gains(RXL[L / NGAIN], L % NGAIN, true);
            __syncthreads();
            if (warp == 0 && lane < SB && (FLAG[ls] & 2)) {
                int t, t1b, pos;
                bool dummy;
                ladder(true, t, t1b, pos, dummy);
                {
                    SI[3 * SB + ls] = t;
                    SI[4 * SB + ls] = t1b;
                    SI[5 * SB + ls] = pos;
                }
            }
            __syncthreads();
        }
    }
    PT(23);

    // ---- Ph11: what reaches the state and the output is always order-exact: the +-1 refinement (src/pitch.rs:205-218)
    // and last_gain (:199-203).  Four single-lag inner products per stream -- lags t+1, t, t-1 and t1b (the second inner
    // product behind best_xy) -- each split over four lanes, one per accumulator of inner_prod (accumulator u sums
    // x[4m+u] y[4m+u], m ascending), so the tile's 64 products run on all eight warps as 120-step chains; lane u = 0 of
    // the quad adds the four accumulators in the reference's order.  Then one lane per stream finishes. ----
    // (the four results go to the first entries of the dead fine-window row)
    static_assert(NT == SB * 4 * 4, "Ph11: one thread per (stream, lag, accumulator)");
    {
        const int s = tid >> 4, j = (tid >> 2) & 3, u = tid & 3;
        const int t = SI[3 * SB + s], t1b = SI[4 * SB + s];
        const float* x = P + s * P_LD + HALF_MAX + u;
        const float* y = x - (j < 3 ? t + 1 - j : t1b);
        float acc = 0.0f;
#pragma unroll 8
        for (int m = 0; m < HALF_N / 4; m++) acc = fa(acc, fm(x[4 * m], y[4 * m]));
        const float a1 = __shfl_down_sync(0xffffffffu, acc, 1), a2 = __shfl_down_sync(0xffffffffu, acc, 2),
                    a3 = __shfl_down_sync(0xffffffffu, acc, 3);
        if (u == 0) FXp(s)[j] = fa(fa(fa(acc, a1), a2), a3);
    }
    PT(24);
    __syncthreads();
    if (warp == 0 && lane < SB) {
        const int t = SI[3 * SB + ls], t0 = SI[2 * SB + ls];
        const float* yys = YYSp(ls);
        const int pos = SI[5 * SB + ls];
        const float xx = XX[ls];
        const float* xf = FXp(ls);
        const float x_2 = xf[0], x_1 = xf[1], x_0 = xf[2], ipb = xf[3];  // x_k: lag t - 1 + k
        float best_xy, best_yy;
        if (t == t0) {  // no sub-harmonic accepted (an accepted t1 is always < t0)
            best_xy = x_1;
            best_yy = yys[0];
        } else {
            best_xy = fm(fa(x_1, ipb), 0.5f);
            best_yy = fm(fa(yys[pos], yys[pos + 1]), 0.5f);
        }
        const float g = pitch_gain(best_xy, xx, best_yy);
        best_xy = fmaxf(best_xy, 0.0f);
        float pg = (best_yy <= best_xy) ? 1.0f : __fdiv_rn(best_xy, fa(best_yy, 1.0f));
        pg = fminf(pg, g);
        int offset = 0;
        if (fs(x_2, x_0) > fm(0.7f, fs(x_1, x_0))) offset = 1;
        else if (fs(x_0, x_2) > fm(0.7f, fs(x_1, x_2))) offset = -1;
        const int tf = max(2 * t + offset, PITCH_MIN_PERIOD);
        if (lane < ns) {
            pitch_out[s0 + lane] = tf;
            last_period[s0 + lane] = tf;
            last_gain[s0 + lane] = pg;
        }
        if (stats && lane == 0) {
            int n_cx = 0, n_rx = 0;
            for (int i = 0; i < ns; i++) {
                n_cx += FLAG[i] & 1;
                n_rx += (FLAG[i] >> 1) & 1;
            }
            if (n_cx) atomicAdd(&stats[0], (unsigned long long)n_cx);
            if (n_rx) atomicAdd(&stats[1], (unsigned long long)n_rx);
            atomicAdd(&stats[2], (unsigned long long)ns);
        }
    }
    PT(26);
}

}  // namespace

#ifdef PITCH_PROFILE
// trace != nullptr: the following launches write their trace there ([grid][NW][PT_N] int64); nullptr: stop tracing
extern "C" int nnb_pitch_trace_arm(long long* trace) {
    return (int)cudaMemcpyToSymbol(g_pitch_trace, &trace, sizeof trace);
}
#endif

cudaError_t launch_pitch(const BatchBuffers& b, int slot, int force_exact, cudaStream_t st) {
    static std::atomic<unsigned long long> attr_devs{0};  // bit d: attribute set on device d
    static std::atomic<int> resident[64];                 // blocks of pitch_kernel resident at once on device d
    const size_t smem = sizeof(float) * SMEM_FLOATS;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 64 || !((attr_devs.load(std::memory_order_acquire) >> dev) & 1ull)) {
        e = cudaFuncSetAttribute(pitch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        int sms = 0, per_sm = 0;
        e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return e;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pitch_kernel, NT, smem);
        if (e != cudaSuccess) return e;
        if (dev < 64) {
            resident[dev].store(sms * per_sm, std::memory_order_relaxed);
            attr_devs.fetch_or(1ull << dev, std::memory_order_release);
        }
    }
    const int grid = (b.n_streams + SB - 1) / SB;
    const int ahead = dev < 64 ? resident[dev].load(std::memory_order_relaxed) : 0;
    pitch_kernel<<<grid, NT, smem, st>>>(b.hist, b.last_period, b.last_gain, b.pitch, b.n_streams, hist_base(slot), force_exact,
                                         ahead, b.pitch_stats);
    return cudaGetLastError();
}

}  // namespace nnb
