// spectral_warp.cu -- frequency-domain half of the path with ONE WARP PER STREAM and no block barrier:
// windowed 960-point real FFTs of the current and pitch-lagged windows, Bark-band energies / correlations, the 42
// input features (analysis), and after the RNN pitch filtering, band-gain interpolation, inverse FFT, overlap-add
// (synthesis).  Reference: src/features.rs:115-298, src/lib.rs:65-162, src/denoise.rs:95-116.
// f32 with FMA contraction allowed: these stages are compared to the oracle within tolerance.
//
// Mapping (fft480.cuh): the 480-point complex FFT behind each 960-point real transform is 32 lanes x 15 registers --
// a 15-point DFT per lane, a twiddle, a transpose through 7.9 KB of per-warp shared memory, a 32-point FFT per lane.
// The two forward transforms of a frame (X and the pitch-lagged P) share every step: lanes 0-14 finish X while lanes
// 15-29 finish P.  Everything between the transforms works on the warp's own buffer under __syncwarp: the even/odd
// split in place (a lane owns bins k and 480-k), the band sums (every lane stays inside one band segment, <= 22 bins),
// the 22-band feature tail (lane = band).  Round 1 spent a 128-thread block per stream with 12 block barriers.
//
// Analysis is persistent: as many blocks as the GPU holds at once, and warp w of the grid takes streams w, w + G, w + 2G,
// ... (G = warps in the grid).  Lane 0 stages the next stream's history window and cepstral ring in the warp's shared
// memory with cp.async.bulk copies that complete on the warp's mbarrier, issued while the current stream's feature tail
// runs.  Synthesis stays one warp per stream with its loads issued up front.  DESIGN K3 / K5 give the measurements behind
// both layouts.
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

// ---- bulk copies global -> shared memory, completing on an mbarrier (one per warp, one arrival: lane 0) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\tbra WAIT_LOOP;\n\tDONE:\n\t}\n" ::"r"(bar), "r"(parity)
        : "memory");
}
// dst, src and bytes: multiples of 16
__device__ __forceinline__ void bulk_copy(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}
// every lane, then __syncwarp, then the copies: the lanes' plain accesses of a buffer come before a bulk copy into it
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

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

// ================================================================================================
// K3: analysis -- X, P, band energies, features (src/features.rs:115-219)
// ================================================================================================
// Staging.  The next stream's history window is copied into the warp's FFT buffer itself: input_mem[l0 .. 1728), the
// union of the X window [768, 1728) and the P window [768 - pitch, 1728 - pitch), from a multiple of 4 so that the copy
// is whole 16-byte units.  Its cepstral ring goes straight to the feature tail's ring buffer (two, used alternately).
// The copies are issued as soon as the band sums have read the spectra for the last time, so they run under the feature
// tail.  A staging buffer beside the FFT buffer (copies running under the whole round) costs a quarter of the warps and
// measured slower, as did a second stage (half the warps).
__host__ __device__ inline int window_lo(int pitch) { return (PITCH_MAX_PERIOD - pitch) & ~3; }  // 0 <= pitch <= 768
static_assert(PITCH_BUF_SIZE * sizeof(float) <= WBUF * sizeof(float2), "the history window fits the FFT buffer");
constexpr int RING = CEPS_MEM * NB_BANDS;  // 176 floats = 704 B

struct __align__(16) AnalysisWarp {
    float2 buf[WBUF];        // the round's history window, then the FFTs and spectra
    float ceps[2][RING];     // cepstral ring of the streams of even / odd rounds
    float sc[WSC];
    float fsc[CEPS_MEM * CEPS_MEM + NB_FEATURES];  // feature tail: s_dist [8][8] | s_feat [42]
    unsigned long long bar;
    int pitch;               // pitch of the staged stream (written by lane 0 before the copies are issued)
};
constexpr size_t ANALYSIS_SMEM = WINDOW_SIZE * sizeof(float) + WPB * sizeof(AnalysisWarp);  // window table | warps: 43.7 KB
// 4 blocks (16 warps) per SM at 113-114 registers, no spills; the count rests on fft480_warp writing r on every lane.
// B = 65,536 on one H100 80GB HBM3 at 700 W, before the branch-free band sums: 0.414 ms at 3 blocks, 0.401 at 4, 0.411
// at 5 (96 registers; shared memory allows no more).
// NNB_ANALYSIS_BLOCKS overrides the count for a register account (tools/analysis_regs.py); builds leave it alone.
#ifndef NNB_ANALYSIS_BLOCKS
#define NNB_ANALYSIS_BLOCKS 4
#endif
constexpr int ANALYSIS_BLOCKS = NNB_ANALYSIS_BLOCKS;

// lane 0: stream s's inputs -> the warp buffer.  The ring row wraps at most once inside the window: two segments then.
__device__ __forceinline__ void issue_analysis(AnalysisWarp& w, const BatchBuffers& bb, int s, int pitch, int hbase, int ring) {
    const int l0 = window_lo(pitch), n = PITCH_BUF_SIZE - l0;
    int r0 = hbase + l0;  // hbase and l0 are multiples of 4, so are both segments
    if (r0 >= HIST_CAP) r0 -= HIST_CAP;
    const int n1 = min(n, HIST_CAP - r0);
    const float* h = bb.hist + (size_t)s * HIST_CAP;
    const uint32_t bar = smem_u32(&w.bar), dst = smem_u32(w.buf);
    w.pitch = pitch;
    mbar_expect_tx(bar, 4 * (n + RING));
    bulk_copy(dst, h + r0, 4 * n1, bar);
    if (n > n1) bulk_copy(dst + 4 * n1, h, 4 * (n - n1), bar);
    bulk_copy(smem_u32(w.ceps[ring]), bb.ceps_mem + (size_t)s * RING, 4 * RING, bar);
}

// SPLIT (rnnoise_batch_analyze_device): the features of stream s go to feat[s * feat_stride ..] instead of the frame's
// set, and its silence flag also to sil[s] if sil is not NULL.  Everything synthesis reads still goes to the set.
// WINDOW (with SPLIT; rnnoise_batch_analyze_window_device): what synthesis reads (X, P, ex, ep, exp, silence) goes to
// stream s's context record at ctx + s * ctx_stride records instead, with the record's padding zeros; the set is left
// alone.  The stores are the same ones, to other addresses.
template <bool SPLIT, bool WINDOW>
__global__ void __launch_bounds__(WPB * 32, ANALYSIS_BLOCKS)
    analysis_warp_kernel(BatchBuffers bb, const DeviceTables* __restrict__ tab, int hbase, float* __restrict__ feat, long feat_stride,
                         int* __restrict__ sil, float* __restrict__ ctx, long ctx_stride) {
    extern __shared__ __align__(16) unsigned char smem[];
    float* s_win = reinterpret_cast<float*>(smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    AnalysisWarp& w = reinterpret_cast<AnalysisWarp*>(smem + WINDOW_SIZE * sizeof(float))[warp];
    for (int i = threadIdx.x; i < WINDOW_SIZE; i += WPB * 32) s_win[i] = tab->window[i];
    const int n_streams = bb.n_streams, G = gridDim.x * WPB;
    int s = blockIdx.x * WPB + warp;
    int pitch_ahead = 0;  // lane 0: pitch of stream s + G, loaded a round before its copies are issued
    if (lane == 0) {
        mbar_init(smem_u32(&w.bar));
        mbar_init_fence();
        if (s < n_streams) issue_analysis(w, bb, s, bb.pitch[s], hbase, 0);
        if (s + G < n_streams) pitch_ahead = bb.pitch[s + G];
    }
    __syncthreads();  // window table; no block barrier below: a warp may leave
    float2* buf = w.buf;
    float* sc = w.sc;

    for (int it = 0; s < n_streams; it++, s += G) {
        mbar_wait(smem_u32(&w.bar), it & 1);
        const int pitch = w.pitch;
        float* const rec = WINDOW ? ctx + (size_t)s * ctx_stride * CX_FLOATS : nullptr;

        // X = rfft(window * input_mem[768..1728]),  P = rfft(window * input_mem[768-pitch .. 1728-pitch]) (src/features.rs:281-290):
        // lane b takes the complex samples z[32 a + b] = (t[64 a + 2 b], t[64 a + 2 b + 1]), before the FFT overwrites them.
        float2 vx[15], vp[15];
        {
            const float* stg = reinterpret_cast<const float*>(buf);
            const float* xs = stg + (PITCH_BUF_SIZE - WINDOW_SIZE - window_lo(pitch));  // 16-byte aligned
            const float* ps = xs - pitch;
            const bool even = (pitch & 1) == 0;
#pragma unroll
            for (int a = 0; a < 15; a++) {
                const int n2 = 64 * a + 2 * lane;
                const float2 hx = *reinterpret_cast<const float2*>(xs + n2);
                const float2 wv = *reinterpret_cast<const float2*>(s_win + n2);
                float2 hp;
                if (even) hp = *reinterpret_cast<const float2*>(ps + n2);
                else hp = make_float2(ps[n2], ps[n2 + 1]);
                vx[a] = make_float2(hx.x * wv.x, hx.y * wv.y);
                vp[a] = make_float2(hp.x * wv.x, hp.y * wv.y);
            }
        }
        __syncwarp();
        fft480_warp<true>(vx, vp, buf, tab, lane);

        // even/odd split into the 481 bins, in place (a lane owns bins k and 480 - k of both spectra), spectra to HBM
        {
            const float wn = tab->wnorm;
            float2* Xg = WINDOW ? reinterpret_cast<float2*>(rec + CX_X) : bb.X + (size_t)s * FREQ_SIZE;
            float2* Pg = WINDOW ? reinterpret_cast<float2*>(rec + CX_P) : bb.P + (size_t)s * NB_BINS_BANDED;
            if (WINDOW && lane == 0) Xg[FREQ_SIZE] = make_float2(0.f, 0.f);
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const int k = lane + 32 * j;
                if (k <= 240) {
                    const int kc = k == 0 ? 0 : 480 - k;
                    const float2 tw = __ldg(&tab->tw960[k]);
                    float2 x0, x1, p0, p1;
                    rfft_split_pair(buf[k], buf[kc], tw, wn, k == 0, x0, x1);
                    rfft_split_pair(buf[ZP_OFF + k], buf[ZP_OFF + kc], tw, wn, k == 0, p0, p1);
                    buf[k] = x0;
                    buf[ZP_OFF + k] = p0;
                    Xg[k] = x0;
                    Pg[k] = p0;  // k <= 240 < 400
                    if (k != 240) {
                        buf[480 - k] = x1;
                        buf[ZP_OFF + 480 - k] = p1;
                        Xg[480 - k] = x1;
                        if (480 - k < NB_BINS_BANDED) Pg[480 - k] = p1;
                    }
                }
            }
        }
        __syncwarp();

        float bs[3];
        band_sums_warp<3>(buf, tab, sc, lane, bs);

        // the spectra are read for the last time: the buffer takes the next stream's inputs
        fence_proxy_async();
        __syncwarp();
        if (lane == 0 && s + G < n_streams) {
            issue_analysis(w, bb, s + G, pitch_ahead, hbase, (it + 1) & 1);
            if (s + 2 * G < n_streams) pitch_ahead = bb.pitch[s + 2 * G];
        }

        // ---- features (src/features.rs:134-219): 22 bands, lane = band ----
        const bool bl = lane < NB_BANDS;
        const float ex = bs[0], ep = bs[1];
        const float xpn = bl ? bs[2] / sqrtf(0.001f + ex * ep) : 0.0f;
        if (WINDOW) {
            if (lane < CX_BAND_SECTION) {  // lanes 22, 23: ex = ep = xpn = 0, the padding
                rec[CX_EX + lane] = ex;
                rec[CX_EP + lane] = ep;
                rec[CX_EXP + lane] = xpn;
                if (!bl) rec[CX_LASTG + lane] = rec[CX_G + lane] = 0.0f;
            }
        } else if (bl) {
            bb.ex[(size_t)s * NB_BANDS + lane] = ex;
            bb.ep[(size_t)s * NB_BANDS + lane] = ep;
            bb.exp[(size_t)s * NB_BANDS + lane] = xpn;
        }
        float* s_ceps = w.ceps[it & 1];  // the stream's cepstral ring, staged
        float* s_dist = w.fsc;
        float* s_feat = s_dist + CEPS_MEM * CEPS_MEM;
        float* cg = bb.ceps_mem + (size_t)s * RING;
        const int mem_id = bb.ceps_id[s];
        // log band energies with the sequential follower (src/features.rs:147-158) and the silence test (:160)
        const float lg = bl ? log10f(1e-2f + ex) : 0.0f;
        float ly = 0.0f, log_max = -2.0f, follow = -2.0f, e = 0.0f;
#pragma unroll
        for (int k = 0; k < NB_BANDS; k++) {
            const float v = fmaxf(fmaxf(__shfl_sync(0xffffffffu, lg, k), log_max - 7.0f), follow - 1.5f);
            if (lane == k) ly = v;
            log_max = fmaxf(log_max, v);
            follow = fmaxf(follow - 1.5f, v);
            e += __shfl_sync(0xffffffffu, ex, k);
        }
        float* featg = SPLIT ? feat + (size_t)s * feat_stride : bb.features + (size_t)s * NB_FEATURES;
        if (e < 0.04f) {  // silent frame: zero features, cepstral ring untouched (src/features.rs:160-166)
            featg[lane] = 0.0f;
            if (lane + 32 < NB_FEATURES) featg[lane + 32] = 0.0f;
            if (lane == 0) {
                if (WINDOW) *reinterpret_cast<int4*>(rec + CX_SIL) = make_int4(1, 0, 0, 0);
                else bb.silence[s] = 1;
                if (SPLIT && sil) sil[s] = 1;
            }
            continue;
        }
        // both DCTs (src/lib.rs:139-148) share the table: lane i accumulates output i over j in order
        const double dct_scale = 0.30151134457776362265;  // sqrt(2/22), src/lib.rs:146
        float sum_ly = 0.0f, sum_xp = 0.0f;
#pragma unroll
        for (int j = 0; j < NB_BANDS; j++) {
            const float d = bl ? __ldg(&tab->dct[j * NB_BANDS + lane]) : 0.0f;
            sum_ly += __shfl_sync(0xffffffffu, ly, j) * d;
            sum_xp += __shfl_sync(0xffffffffu, xpn, j) * d;
        }
        float ceps = (float)((double)sum_ly * dct_scale);
        float pcor = (float)((double)sum_xp * dct_scale);
        if (lane == 0) {
            ceps -= 12.0f;
            pcor -= 1.3f;
        }
        if (lane == 1) {
            ceps -= 4.0f;
            pcor -= 0.9f;
        }
        // the new row in place
        if (bl) {
            s_ceps[mem_id * NB_BANDS + lane] = ceps;
            cg[mem_id * NB_BANDS + lane] = ceps;
            s_feat[lane] = ceps;
        }
        __syncwarp();
        if (lane < NB_DELTA_CEPS) {
            const int c1 = (mem_id < 1) ? CEPS_MEM + mem_id - 1 : mem_id - 1;
            const int c2 = (mem_id < 2) ? CEPS_MEM + mem_id - 2 : mem_id - 2;
            const float a = s_ceps[mem_id * NB_BANDS + lane], b = s_ceps[c1 * NB_BANDS + lane], c = s_ceps[c2 * NB_BANDS + lane];
            s_feat[lane] = a + b + c;
            s_feat[NB_BANDS + lane] = a - c;
            s_feat[NB_BANDS + NB_DELTA_CEPS + lane] = a - 2.0f * b + c;
            s_feat[NB_BANDS + 2 * NB_DELTA_CEPS + lane] = pcor;
        }
        // spectral variability (src/features.rs:199-216): pairwise squared distances of the 8 ring rows, two pairs per lane
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++) {
            const int pr = lane + 32 * h2, i = pr >> 3, j = pr & 7;
            float dist = 0.0f;
#pragma unroll
            for (int k = 0; k < NB_BANDS; k++) {
                const float t = s_ceps[i * NB_BANDS + k] - s_ceps[j * NB_BANDS + k];
                dist += t * t;
            }
            s_dist[i * CEPS_MEM + j] = dist;
        }
        __syncwarp();
        float md = 1e15f;
        if (lane < CEPS_MEM) {
#pragma unroll
            for (int j = 0; j < CEPS_MEM; j++)
                if (j != lane) md = fminf(md, s_dist[lane * CEPS_MEM + j]);
        }
        float sv = 0.0f;
#pragma unroll
        for (int i = 0; i < CEPS_MEM; i++) sv += __shfl_sync(0xffffffffu, md, i);  // i = 0..7 in order, like the reference
        if (lane == 0) {
            s_feat[NB_BANDS + 3 * NB_DELTA_CEPS] = 0.01f * ((float)pitch - 300.0f);
            s_feat[NB_BANDS + 3 * NB_DELTA_CEPS + 1] = sv / (float)CEPS_MEM - 2.1f;
            bb.ceps_id[s] = (mem_id + 1 == CEPS_MEM) ? 0 : mem_id + 1;
            if (WINDOW) *reinterpret_cast<int4*>(rec + CX_SIL) = make_int4(0, 0, 0, 0);
            else bb.silence[s] = 0;
            if (SPLIT && sil) sil[s] = 0;
        }
        __syncwarp();
        featg[lane] = s_feat[lane];
        if (lane + 32 < NB_FEATURES) featg[lane + 32] = s_feat[lane + 32];
    }
}

// ================================================================================================
// K5: synthesis -- pitch filter, gain floor, band-gain interpolation, inverse FFT, overlap-add
// (src/denoise.rs:102-115, src/features.rs:223-275)
// ================================================================================================
// TOut = float, or short: to_pcm16w (common.cuh).  SPLIT (rnnoise_batch_synthesize_device): the raw gains of stream s
// are gains[s * gain_stride ..] instead of the frame's set, and no vad is read or written.  WINDOW (with SPLIT;
// rnnoise_batch_synthesize_window_device): X, P, ex, ep, exp and the silence flag come from stream s's context record at
// ctx + s * ctx_stride records instead of the set, and lastg before the frame and the raw gains go to the record, from
// the registers that hold them (silent frames load both for it).  CTL (fused frames only): the frame applies the streams'
// controls (rnnoise_batch_set_stream_controls), the attenuation limit on the raw gains and the voice-activity gate on the
// output samples after overlap-add.  Their defaults are identities; the host launches CTL only when some stream of the
// batch has non-default controls, and the kernel without it is the one from before the controls.

template <typename TOut, bool SPLIT, bool WINDOW, bool CTL>
__global__ void __launch_bounds__(WPB * 32, 4) synthesis_warp_kernel(BatchBuffers bb, const DeviceTables* __restrict__ tab,
                                                                  TOut* __restrict__ out, long stream_stride, long sample_stride,
                                                                  float* __restrict__ vad_out, const float* __restrict__ gains,
                                                                  long gain_stride, float* __restrict__ ctx, long ctx_stride) {
    __shared__ __align__(16) float2 sbuf[WPB][WBUF];
    __shared__ float ssc[WPB][WSC];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int s = blockIdx.x * WPB + warp;
    if (s >= bb.n_streams) return;
    float2* buf = sbuf[warp];
    float* sc = ssc[warp];

    // every global load of the stream is issued up front
    float* const rec = WINDOW ? ctx + (size_t)s * ctx_stride * CX_FLOATS : nullptr;
    const float2* Xg = WINDOW ? reinterpret_cast<const float2*>(rec + CX_X) : bb.X + (size_t)s * FREQ_SIZE;
    const float2* Pg = WINDOW ? reinterpret_cast<const float2*>(rec + CX_P) : bb.P + (size_t)s * NB_BINS_BANDED;
    float2 xv[16];
#pragma unroll
    for (int j = 0; j < 16; j++) {
        const int k = lane + 32 * j;
        xv[j] = k <= 480 ? __ldg(Xg + k) : make_float2(0.f, 0.f);
    }
    const float vad_in = SPLIT ? 0.0f : bb.vad[s];
    static_assert(!(CTL && SPLIT), "split and window frames take no controls");
    const StreamCtl ctl = CTL ? bb.ctl[s] : StreamCtl{0.0f, 0.0f, 0.0f, 0};  // every lane reads the same 16 bytes
    const int silent = WINDOW ? reinterpret_cast<const int*>(rec)[CX_SIL] : bb.silence[s];
    float* smem_ola = bb.synth_mem + (size_t)s * FRAME_SIZE;
    float4 ola[4];  // overlap memory, float4 q = lane + 32 j < 120
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int q = lane + 32 * j;
        ola[j] = q < FRAME_SIZE / 4 ? __ldg(reinterpret_cast<const float4*>(smem_ola) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (!silent) {
        float2 pv[13];
#pragma unroll
        for (int j = 0; j < 13; j++) {
            const int k = lane + 32 * j;
            pv[j] = k < NB_BINS_BANDED ? __ldg(Pg + k) : make_float2(0.f, 0.f);
        }
        float b_ex = 0.0f;
        if (lane < NB_BANDS) {
            const float e = WINDOW ? rec[CX_EXP + lane] : bb.exp[(size_t)s * NB_BANDS + lane];
            float g = SPLIT ? gains[(size_t)s * gain_stride + lane] : bb.gains[(size_t)s * NB_BANDS + lane];
            if (CTL && ctl.g_min > 0.0f) g = fmaxf(g, ctl.g_min);  // the attenuation limit
            const float ex = WINDOW ? rec[CX_EX + lane] : bb.ex[(size_t)s * NB_BANDS + lane];
            const float ep = WINDOW ? rec[CX_EP + lane] : bb.ep[(size_t)s * NB_BANDS + lane];
            const float lastg = bb.lastg[(size_t)s * NB_BANDS + lane];
            if (WINDOW) {
                rec[CX_LASTG + lane] = lastg;
                rec[CX_G + lane] = g;
            }
            b_ex = ex;
            // r (src/features.rs:226-235)
            float r;
            if (e > g) {
                r = 1.0f;
            } else {
                const float e2 = e * e, g2 = g * g;
                r = e2 * (1.0f - g2) / (0.001f + g2 * (1.0f - e2));
            }
            r = (r < 0.0f) ? 0.0f : r;
            r = (r > 1.0f) ? 1.0f : r;
            r = sqrtf(r);
            r *= sqrtf(ex / (1e-8f + ep));
            sc[SC_SR + lane] = r;
            // gain floor (src/denoise.rs:106-109)
            const float gg = fmaxf(g, 0.6f * lastg);
            sc[SC_SG + lane] = gg;
            bb.lastg[(size_t)s * NB_BANDS + lane] = gg;
        }
        __syncwarp();
        // x += rf * p  (bin 0 is the real-valued DC offset; its imaginary part stays 0); spectrum to the warp buffer
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int k = lane + 32 * j;
            if (j < 13 && k < NB_BINS_BANDED) {
                const int bi = __ldg(&tab->band_of[k]);
                const float fr = __ldg(&tab->band_frac[k]);
                const float rf = (1.0f - fr) * sc[SC_SR + bi] + fr * sc[SC_SR + bi + 1];
                xv[j].x += pv[j].x * rf;
                if (k > 0) xv[j].y += pv[j].y * rf;
            }
            if (k <= 480) buf[k] = xv[j];
        }
        __syncwarp();
        float ne[1];
        band_sums_warp<1>(buf, tab, sc, lane, ne);
        if (lane < NB_BANDS) sc[SC_SN + lane] = sqrtf(b_ex / (1e-8f + ne[0]));
        __syncwarp();
        // x *= rf2 ; x *= gf   (bins >= 400 are zeroed by both interpolations)
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int k = lane + 32 * j;
            if (k <= 480) {
                float2 x = xv[j];
                if (k < NB_BINS_BANDED) {
                    const int bi = __ldg(&tab->band_of[k]);
                    const float fr = __ldg(&tab->band_frac[k]);
                    const float m1 = (1.0f - fr) * sc[SC_SN + bi] + fr * sc[SC_SN + bi + 1];
                    const float m2 = (1.0f - fr) * sc[SC_SG + bi] + fr * sc[SC_SG + bi + 1];
                    x.x = (x.x * m1) * m2;
                    x.y = (x.y * m1) * m2;
                } else {
                    x = make_float2(0.f, 0.f);
                }
                buf[k] = x;
            }
        }
    } else {
        if (WINDOW && lane < NB_BANDS) {
            rec[CX_LASTG + lane] = bb.lastg[(size_t)s * NB_BANDS + lane];
            rec[CX_G + lane] = gains[(size_t)s * gain_stride + lane];
        }
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const int k = lane + 32 * j;
            if (k <= 480) buf[k] = xv[j];
        }
    }
    __syncwarp();

    // ---- inverse real FFT (unnormalised), src/features.rs:263-275: Z = 2E + i 2O, fed conjugated to the forward FFT;
    // a lane builds Z[k] and Z[480-k] together, in place ----
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int k = lane + 32 * j;
        if (k <= 240) {
            float2 z0, z1;
            irfft_pretwist_pair(buf[k], buf[480 - k], __ldg(&tab->tw960[k]), k == 0, z0, z1);
            buf[k] = z0;
            if (k != 0 && k != 240) buf[480 - k] = z1;
        }
    }
    __syncwarp();
    float2 v[15], dummy[15];
#pragma unroll
    for (int a = 0; a < 15; a++) v[a] = buf[32 * a + lane];
    __syncwarp();  // everybody has its inputs: the buffer becomes the transpose area
    fft480_warp<false>(v, dummy, buf, tab, lane);

    // The voice-activity gate: lane 0 decides from the frame's reported vad and the stream's gate state,
    // and hands out the gain at the frame's start (ell, the previous decision) and at its end (tau).  Output sample i is
    // scaled by ell + (tau - ell) * ramp[i], each operation rounded; both 1 (an open gate, the default) leave it alone.
    float ell = 1.0f, tau = 1.0f;
    if (CTL) {
        if (lane == 0) {
            const int2 g0 = bb.gate[s];
            const float v = silent ? 0.0f : vad_in;
            int hold_left = g0.x, closed = 0;
            if (ctl.threshold == 0.0f || v >= ctl.threshold) hold_left = ctl.hold;
            else if (hold_left > 0) hold_left--;
            else closed = 1;
            if (g0.y) ell = ctl.closed_gain;
            if (closed) tau = ctl.closed_gain;
            if (hold_left != g0.x || closed != g0.y) bb.gate[s] = make_int2(hold_left, closed);
        }
        ell = __shfl_sync(0xffffffffu, ell, 0);
        tau = __shfl_sync(0xffffffffu, tau, 0);
    }
    const bool gated = ell != 1.0f || tau != 1.0f;
    const float dg = __fsub_rn(tau, ell);

    // time samples 4q..4q+3 = (re, -im) of buf[2q], buf[2q+1]; first half -> output (+ overlap memory), second half -> new
    // overlap memory (every lane read its part of the old one at the top).  Vector stores when the caller's rows allow.
    TOut* o = out + (long)s * stream_stride;
    const bool o_vec = sample_stride == 1 && ((reinterpret_cast<uintptr_t>(o) & (4 * sizeof(TOut) - 1)) == 0);
    const long ss = sample_stride;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int q = lane + 32 * j;
        if (q < WINDOW_SIZE / 4) {
            const float4 z = reinterpret_cast<const float4*>(buf)[q];
            const float4 w = __ldg(reinterpret_cast<const float4*>(tab->window) + q);
            const float4 t = make_float4((z.x * 0.5f) * w.x, (-z.y * 0.5f) * w.y, (z.z * 0.5f) * w.z, (-z.w * 0.5f) * w.w);
            if (q < FRAME_SIZE / 4) {
                const float4 m = ola[j < 4 ? j : 0];
                float4 r = make_float4(t.x + m.x, t.y + m.y, t.z + m.z, t.w + m.w);
                if (gated) {
                    const float4 wr = __ldg(reinterpret_cast<const float4*>(tab->ramp) + q);
                    r.x = __fmul_rn(r.x, __fadd_rn(ell, __fmul_rn(dg, wr.x)));
                    r.y = __fmul_rn(r.y, __fadd_rn(ell, __fmul_rn(dg, wr.y)));
                    r.z = __fmul_rn(r.z, __fadd_rn(ell, __fmul_rn(dg, wr.z)));
                    r.w = __fmul_rn(r.w, __fadd_rn(ell, __fmul_rn(dg, wr.w)));
                }
                if (sizeof(TOut) == 4) {
                    float* of = reinterpret_cast<float*>(o);
                    if (o_vec) {
                        reinterpret_cast<float4*>(of)[q] = r;
                    } else {
                        of[(4 * q) * ss] = r.x; of[(4 * q + 1) * ss] = r.y; of[(4 * q + 2) * ss] = r.z; of[(4 * q + 3) * ss] = r.w;
                    }
                } else {
                    short* os = reinterpret_cast<short*>(o);
                    const short p0 = to_pcm16w(r.x), p1 = to_pcm16w(r.y), p2 = to_pcm16w(r.z), p3 = to_pcm16w(r.w);
                    if (o_vec) {
                        reinterpret_cast<uint2*>(os)[q] = make_uint2((unsigned)(unsigned short)p0 | ((unsigned)(unsigned short)p1 << 16),
                                                                     (unsigned)(unsigned short)p2 | ((unsigned)(unsigned short)p3 << 16));
                    } else {
                        os[(4 * q) * ss] = p0; os[(4 * q + 1) * ss] = p1; os[(4 * q + 2) * ss] = p2; os[(4 * q + 3) * ss] = p3;
                    }
                }
            } else {
                reinterpret_cast<float4*>(smem_ola)[q - FRAME_SIZE / 4] = t;
            }
        }
    }
    if (!SPLIT && lane == 0 && vad_out) vad_out[s] = silent ? 0.0f : vad_in;
}

// Blocks of analysis_warp_kernel<SPLIT, WINDOW> resident on device `dev` at once; the shared-memory opt-in and the
// occupancy are looked up once per device.  0 on an error, in *e.
template <bool SPLIT, bool WINDOW>
int analysis_resident(int dev, cudaError_t* e) {
    constexpr int kMaxDevices = 64;
    static int resident[kMaxDevices];
    if (dev >= kMaxDevices) {
        *e = cudaErrorInvalidDevice;
        return 0;
    }
    if (resident[dev] == 0) {
        int sms = 0, per_sm = 0;
        if ((*e = cudaFuncSetAttribute(analysis_warp_kernel<SPLIT, WINDOW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ANALYSIS_SMEM)) !=
            cudaSuccess)
            return 0;
        if ((*e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return 0;
        if ((*e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, analysis_warp_kernel<SPLIT, WINDOW>, WPB * 32, ANALYSIS_SMEM)) != cudaSuccess)
            return 0;
        if (per_sm < 1) {
            *e = cudaErrorInvalidConfiguration;
            return 0;
        }
        resident[dev] = per_sm * sms;
    }
    return resident[dev];
}

}  // namespace

cudaError_t launch_analysis_warp(const BatchBuffers& b, const DeviceTables* tab, int slot, cudaStream_t st, float* features,
                                 long feature_stride, int* silence, void* ctx, long ctx_stride) {
    // persistent grid: min(blocks the streams need, blocks resident on the whole GPU at once)
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const int resident = ctx ? analysis_resident<true, true>(dev, &e)
                             : (features ? analysis_resident<true, false>(dev, &e) : analysis_resident<false, false>(dev, &e));
    if (resident == 0) return e;
    const int grid = min((b.n_streams + WPB - 1) / WPB, resident);
    float* c = static_cast<float*>(ctx);
    if (ctx)
        analysis_warp_kernel<true, true><<<grid, WPB * 32, ANALYSIS_SMEM, st>>>(b, tab, hist_base(slot), features, feature_stride, silence, c,
                                                                                ctx_stride);
    else if (features)
        analysis_warp_kernel<true, false><<<grid, WPB * 32, ANALYSIS_SMEM, st>>>(b, tab, hist_base(slot), features, feature_stride, silence,
                                                                                 nullptr, 0);
    else
        analysis_warp_kernel<false, false><<<grid, WPB * 32, ANALYSIS_SMEM, st>>>(b, tab, hist_base(slot), nullptr, 0, nullptr, nullptr, 0);
    return cudaGetLastError();
}

cudaError_t launch_synthesis_warp(const BatchBuffers& b, const DeviceTables* tab, void* out, bool pcm16, long stream_stride,
                                  long sample_stride, float* vad_out, cudaStream_t st, const float* gains, long gain_stride, void* ctx,
                                  long ctx_stride, bool controls) {
    const int grid = (b.n_streams + WPB - 1) / WPB;
    short* o16 = static_cast<short*>(out);
    float* o32 = static_cast<float*>(out);
    float* c = static_cast<float*>(ctx);
    if (ctx) {
        if (pcm16) synthesis_warp_kernel<short, true, true, false><<<grid, WPB * 32, 0, st>>>(b, tab, o16, stream_stride, sample_stride, nullptr, gains, gain_stride, c, ctx_stride);
        else synthesis_warp_kernel<float, true, true, false><<<grid, WPB * 32, 0, st>>>(b, tab, o32, stream_stride, sample_stride, nullptr, gains, gain_stride, c, ctx_stride);
    } else if (gains) {
        if (pcm16) synthesis_warp_kernel<short, true, false, false><<<grid, WPB * 32, 0, st>>>(b, tab, o16, stream_stride, sample_stride, nullptr, gains, gain_stride, nullptr, 0);
        else synthesis_warp_kernel<float, true, false, false><<<grid, WPB * 32, 0, st>>>(b, tab, o32, stream_stride, sample_stride, nullptr, gains, gain_stride, nullptr, 0);
    } else if (controls) {
        if (pcm16) synthesis_warp_kernel<short, false, false, true><<<grid, WPB * 32, 0, st>>>(b, tab, o16, stream_stride, sample_stride, vad_out, nullptr, 0, nullptr, 0);
        else synthesis_warp_kernel<float, false, false, true><<<grid, WPB * 32, 0, st>>>(b, tab, o32, stream_stride, sample_stride, vad_out, nullptr, 0, nullptr, 0);
    } else {
        if (pcm16) synthesis_warp_kernel<short, false, false, false><<<grid, WPB * 32, 0, st>>>(b, tab, o16, stream_stride, sample_stride, vad_out, nullptr, 0, nullptr, 0);
        else synthesis_warp_kernel<float, false, false, false><<<grid, WPB * 32, 0, st>>>(b, tab, o32, stream_stride, sample_stride, vad_out, nullptr, 0, nullptr, 0);
    }
    return cudaGetLastError();
}

}  // namespace nnb
