// spectral_warp.cuh -- the warp-per-stream building blocks of the spectral kernels (spectral_warp.cu) that other kernels
// share: the two 480-point FFTs of a warp (fft480_warp) and the Bark-band sums over the spectra in the warp's buffer
// (band_sums_warp), with the warp-buffer layout they assume.  The metrics kernel (metrics.cu) takes its band energies
// from the same two routines, so that they are the analysis kernel's `ex` for the same window.
#pragma once
#include "common.cuh"
#include "fft480.cuh"

namespace nnb {

namespace {

constexpr int WPB = 4;             // warps per block
constexpr int RS = 33;             // transpose row stride in float2: lane L reads row L, 2 * 33 = 2 (mod 32): conflict-free
constexpr int ZP_OFF = 495;        // second spectrum inside the warp buffer; 2 * 495 = 30 (mod 32): X and P lanes interleave
constexpr int WBUF = 30 * RS;      // 990 float2 per warp
constexpr int SC_SR = 0, SC_SG = 32, SC_SN = 64, SC_BAND = 96;  // float offsets in the small per-warp scratch
constexpr int WSC = SC_BAND + 21 * 6 + 2;
static_assert(ZP_OFF + FREQ_SIZE <= WBUF, "two 481-bin spectra must fit the warp buffer");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// forward 480-point FFTs of vx (and vp if TWO) held as z[32 a + lane] -> natural-order spectra in buf[0..480) (and
// buf[ZP_OFF..ZP_OFF+480)).  All 32 lanes must call.
template <bool TWO>
__device__ __forceinline__ void fft480_warp(float2 (&vx)[15], float2 (&vp)[15], float2* __restrict__ buf,
                                            const DeviceTables* __restrict__ tab, int lane) {
    dft15(vx);
    if (TWO) dft15(vp);
#pragma unroll
    for (int k1 = 1; k1 < 15; k1++) {
        const float2 tw = __ldg(&tab->twl[k1][lane]);
        vx[k1] = c_mul(vx[k1], tw);
        if (TWO) vp[k1] = c_mul(vp[k1], tw);
    }
#pragma unroll
    for (int k1 = 0; k1 < 15; k1++) {
        buf[k1 * RS + lane] = vx[k1];
        if (TWO) buf[(15 + k1) * RS + lane] = vp[k1];
    }
    __syncwarp();
    float2 r[32];
    const bool on = lane < (TWO ? 30 : 15);
    // With TWO, lanes 30 and 31 run the column of lane 29 too and store nothing: r is then written on every path.  Left
    // unwritten on some lanes, r reaches its stores through a path that skips the loads, and in the persistent analysis
    // loop the compiler keeps its 64 registers live across the whole loop (DESIGN §8.2).
    if (TWO || on) {
        const int row = TWO ? min(lane, 29) : lane;
#pragma unroll
        for (int b = 0; b < 32; b++) r[b] = buf[row * RS + b];
        fft32_dif(r);
    }
    __syncwarp();
    if (on) {
        const int base = lane < 15 ? lane : ZP_OFF + lane - 15;
#pragma unroll
        for (int k2 = 0; k2 < 32; k2++) buf[base + 15 * k2] = r[bitrev5(k2)];
    }
    __syncwarp();
}

// Band sums (src/lib.rs:65-82) over spectra in the warp buffer: lane l covers bins bp_b0[l] .. +bp_n[l] of segment
// bp_seg[l]; the (1 - frac) parts go to band seg, the frac parts to band seg + 1.  NQ = 3: |X|^2, |P|^2, Re(X conj P);
// NQ = 1: |X|^2 only.  Results: lane b < 22 returns band b in o[0..NQ) (first / last band doubled).  sc: >= 21 * 6 + 2 floats.
template <int NQ>
__device__ __forceinline__ void band_sums_warp(const float2* __restrict__ buf, const DeviceTables* __restrict__ tab, float* __restrict__ sc,
                                               int lane, float (&o)[NQ]) {
    const int sg = tab->bp_seg[lane], b0 = tab->bp_b0[lane], n = tab->bp_n[lane], rot = tab->bp_rot[lane], off0 = tab->bp_off[lane];
    const float inv = tab->bp_inv[lane];  // frac = j / size as j * (1 / size): within an ulp of the reference's quotient
    float a[NQ], b[NQ];
#pragma unroll
    for (int q = 0; q < NQ; q++) a[q] = b[q] = 0.0f;
    // Every lane runs all BP_MAXBINS steps and only steps t < n accumulate: without a branch per step the compiler
    // issues later steps' loads ahead of earlier steps' sums.  For t >= n, i = t + rot - n < 21 and k < 400 + 21: the
    // reads stay inside both spectra.
#pragma unroll
    for (int t = 0; t < BP_MAXBINS; t++) {
        int i = t + rot;  // rotated walk: neighbouring lanes start at different offsets -> different banks
        if (i >= n) i -= n;
        const int k = b0 + i;
        const float f = (float)(off0 + i) * inv, g = 1.0f - f;
        const float2 x = buf[k];
        float e[NQ];
        e[0] = x.x * x.x + x.y * x.y;
        if (NQ == 3) {
            const float2 p = buf[ZP_OFF + k];
            e[1] = p.x * p.x + p.y * p.y;
            e[2] = x.x * p.x + x.y * p.y;
        }
        const bool in = t < n;
#pragma unroll
        for (int q = 0; q < NQ; q++) {
            const float na = fmaf(g, e[q], a[q]), nb = fmaf(f, e[q], b[q]);
            a[q] = in ? na : a[q];
            b[q] = in ? nb : b[q];
        }
    }
    // lanes of one segment are contiguous (at most 4): the first one collects the others' ORIGINAL partial sums in a
    // fixed order (lane + 1, + 2, + 3)
    {
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
    }
    const int psg = __shfl_up_sync(0xffffffffu, sg, 1);
    if (lane == 0 || psg != sg) {
#pragma unroll
        for (int q = 0; q < NQ; q++) {
            sc[SC_BAND + sg * 6 + q] = a[q];
            sc[SC_BAND + sg * 6 + 3 + q] = b[q];
        }
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < NQ; q++) {
        float v = 0.0f;
        if (lane < NB_BANDS) {
            if (lane < NB_BANDS - 1) v = sc[SC_BAND + lane * 6 + q];
            if (lane > 0) v += sc[SC_BAND + (lane - 1) * 6 + 3 + q];
            if (lane == 0 || lane == NB_BANDS - 1) v *= 2.0f;
        }
        o[q] = v;
    }
    __syncwarp();
}

}  // namespace

}  // namespace nnb
