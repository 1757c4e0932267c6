// state.cu -- per-stream state records: gather (export) and scatter (import / reset) over a list of streams.
//
// A record holds the persistent fields of the reference's DenoiseState (src/denoise.rs:37-42) in the reference's own
// order and indexing; the layout is documented with rnnoise_batch_get_states in include/rnnoise.h.  input_mem is
// un-rotated from the history ring: after the frame in ring slot s, sample i is at ring position (hist_base(s) + i)
// mod HIST_CAP, a window that is at most two contiguous segments (hist_base and HIST_CAP are multiples of 4, so each
// 128-bit load stays inside one of them).
//
// One warp per record, STATE_WARPS records per block: every section of the record is copied with 128-bit loads and
// stores by consecutive lanes, so a warp moves 512 contiguous bytes per instruction on both sides.
//
// The same copies move the live state of a subset of streams between the batch and a compact work state (subset_*
// kernels, used by rnnoise_batch_process_streams_*): no record format in between, and only the fields the frame kernels
// carry from one frame to the next.
#include "../../include/rnnoise.h"
#include "common.cuh"

namespace nnb {

namespace {

constexpr int STATE_WARPS = 8;
constexpr int IN_Q = PITCH_BUF_SIZE / 4, RING_Q = HIST_CAP / 4, CEPS_Q = CEPS_MEM * NB_BANDS / 4, SYN_Q = FRAME_SIZE / 4;
static_assert(STATE_OFF_INPUT % 16 == 0 && STATE_OFF_CEPS % 16 == 0 && STATE_OFF_SYNTH % 16 == 0 && STATE_OFF_GRU % 16 == 0,
              "record sections must be 16-byte aligned");
static_assert(STATE_OFF_CEPS == STATE_OFF_INPUT + 4 * PITCH_BUF_SIZE && STATE_OFF_SYNTH == STATE_OFF_CEPS + 4 * CEPS_MEM * NB_BANDS &&
                  STATE_OFF_GRU == STATE_OFF_SYNTH + 4 * FRAME_SIZE,
              "record sections must be back to back");
static_assert((CEPS_MEM * NB_BANDS) % 4 == 0 && HIST_CAP % 4 == 0, "sections must be whole float4s");

__device__ __forceinline__ int ring_q(int q0, int j) {
    const int q = q0 + j;
    return q >= RING_Q ? q - RING_Q : q;
}

// rec[r] = state of stream idx[r] (idx NULL: stream r).  hbase = hist_base of the batch's most recent ring slot.
__global__ void __launch_bounds__(STATE_WARPS * 32) state_gather_kernel(BatchBuffers bb, int nv, int nn, int nd, const int* __restrict__ idx,
                                                                        int n, int hbase, int rec_bytes, unsigned char* __restrict__ dst) {
    const int lane = threadIdx.x & 31, r = blockIdx.x * STATE_WARPS + (threadIdx.x >> 5);
    if (r >= n) return;
    const size_t s = idx ? (size_t)idx[r] : (size_t)r;
    const int ss = nv + nn + nd;
    unsigned char* rec = dst + (size_t)r * rec_bytes;

    // words 0..31: magic, version, nv, nn, nd, mem_id, last_period, last_gain, mem_hp_x[2], lastg[22]
    uint32_t w;
    switch (lane) {
        case 0: w = RNNOISE_STATE_MAGIC; break;
        case 1: w = RNNOISE_STATE_VERSION; break;
        case 2: w = (uint32_t)nv; break;
        case 3: w = (uint32_t)nn; break;
        case 4: w = (uint32_t)nd; break;
        case 5: w = (uint32_t)bb.ceps_id[s]; break;
        case 6: w = (uint32_t)bb.last_period[s]; break;
        case 7: w = __float_as_uint(bb.last_gain[s]); break;
        case 8:
        case 9: w = __float_as_uint(bb.hp_mem[2 * s + (lane - 8)]); break;
        default: w = __float_as_uint(bb.lastg[s * NB_BANDS + (lane - 10)]); break;
    }
    reinterpret_cast<uint32_t*>(rec)[lane] = w;

    const float4* h = reinterpret_cast<const float4*>(bb.hist + s * HIST_CAP);
    float4* o = reinterpret_cast<float4*>(rec + STATE_OFF_INPUT);
#pragma unroll 4
    for (int j = lane; j < IN_Q; j += 32) o[j] = __ldg(h + ring_q(hbase / 4, j));
    const float4* c = reinterpret_cast<const float4*>(bb.ceps_mem + s * CEPS_MEM * NB_BANDS);
    o = reinterpret_cast<float4*>(rec + STATE_OFF_CEPS);
    for (int j = lane; j < CEPS_Q; j += 32) o[j] = __ldg(c + j);
    const float4* y = reinterpret_cast<const float4*>(bb.synth_mem + s * FRAME_SIZE);
    o = reinterpret_cast<float4*>(rec + STATE_OFF_SYNTH);
#pragma unroll 4
    for (int j = lane; j < SYN_Q; j += 32) o[j] = __ldg(y + j);

    const float* g = bb.gru_state + s * ss;
    float* og = reinterpret_cast<float*>(rec + STATE_OFF_GRU);
    if ((ss & 3) == 0) {  // rows of gru_state are 16-byte aligned
        for (int j = lane; j < ss / 4; j += 32) reinterpret_cast<float4*>(og)[j] = __ldg(reinterpret_cast<const float4*>(g) + j);
    } else {
        for (int j = lane; j < ss; j += 32) og[j] = __ldg(g + j);
    }
    for (int j = STATE_OFF_GRU / 4 + ss + lane; j < rec_bytes / 4; j += 32) reinterpret_cast<uint32_t*>(rec)[j] = 0u;  // padding
}

// state of stream idx[r] = rec[r]; src NULL: the state of a freshly created stream (all zero).  Records are validated
// on the host before this runs.
__global__ void __launch_bounds__(STATE_WARPS * 32) state_scatter_kernel(BatchBuffers bb, int ss, const int* __restrict__ idx, int n,
                                                                         int hbase, int rec_bytes, const unsigned char* __restrict__ src) {
    const int lane = threadIdx.x & 31, r = blockIdx.x * STATE_WARPS + (threadIdx.x >> 5);
    if (r >= n) return;
    const size_t s = idx ? (size_t)idx[r] : (size_t)r;
    const unsigned char* rec = src ? src + (size_t)r * rec_bytes : nullptr;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);

    const uint32_t w = rec ? __ldg(reinterpret_cast<const uint32_t*>(rec) + lane) : 0u;
    switch (lane) {
        case 5: bb.ceps_id[s] = (int32_t)w; break;
        case 6: bb.last_period[s] = (int32_t)w; break;
        case 7: bb.last_gain[s] = __uint_as_float(w); break;
        case 8:
        case 9: bb.hp_mem[2 * s + (lane - 8)] = __uint_as_float(w); break;
        default:
            if (lane >= 10) bb.lastg[s * NB_BANDS + (lane - 10)] = __uint_as_float(w);
            break;
    }

    float4* h = reinterpret_cast<float4*>(bb.hist + s * HIST_CAP);
    const float4* in = reinterpret_cast<const float4*>(rec + STATE_OFF_INPUT);
#pragma unroll 4
    for (int j = lane; j < IN_Q; j += 32) h[ring_q(hbase / 4, j)] = rec ? __ldg(in + j) : z4;
    float4* c = reinterpret_cast<float4*>(bb.ceps_mem + s * CEPS_MEM * NB_BANDS);
    in = reinterpret_cast<const float4*>(rec + STATE_OFF_CEPS);
    for (int j = lane; j < CEPS_Q; j += 32) c[j] = rec ? __ldg(in + j) : z4;
    float4* y = reinterpret_cast<float4*>(bb.synth_mem + s * FRAME_SIZE);
    in = reinterpret_cast<const float4*>(rec + STATE_OFF_SYNTH);
#pragma unroll 4
    for (int j = lane; j < SYN_Q; j += 32) y[j] = rec ? __ldg(in + j) : z4;

    float* g = bb.gru_state + s * ss;
    const float* ig = reinterpret_cast<const float*>(rec + STATE_OFF_GRU);
    if ((ss & 3) == 0) {
        for (int j = lane; j < ss / 4; j += 32) reinterpret_cast<float4*>(g)[j] = rec ? __ldg(reinterpret_cast<const float4*>(ig) + j) : z4;
    } else {
        for (int j = lane; j < ss; j += 32) g[j] = rec ? __ldg(ig + j) : 0.0f;
    }
}

// *first_bad = min(*first_bad, index of every record whose head fails the checks of rnnoise_batch_set_states)
__global__ void state_check_kernel(const unsigned char* __restrict__ src, int n, int rec_bytes, int nv, int nn, int nd,
                                   int* __restrict__ first_bad) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int4* h = reinterpret_cast<const int4*>(src + (size_t)r * rec_bytes);
    const int4 a = __ldg(h), b = __ldg(h + 1);
    const bool ok = (uint32_t)a.x == RNNOISE_STATE_MAGIC && a.y == RNNOISE_STATE_VERSION && a.z == nv && a.w == nn && b.x == nd &&
                    b.y >= 0 && b.y < CEPS_MEM && b.z >= 0 && b.z <= PITCH_MAX_PERIOD;
    if (!ok) atomicMin(first_bad, r);
}

// Subset calls (rnnoise_batch_process_streams_*): the live state of stream idx[r] of the batch and row r of the work
// state, copied in one direction.  Gather (kScatter false) moves batch -> work; scatter moves work -> batch.  hist_q: the
// ring window as float4 indices, hsrc / hdst its first position on either side (the window is at most two contiguous
// segments on each side, and a float4 never straddles the wrap).
template <bool kScatter>
__device__ __forceinline__ void subset_copy(const BatchBuffers& bat, const BatchBuffers& wk, int ss, const int* __restrict__ idx, int n,
                                            int hsrc, int hdst, int hist_q) {
    const int lane = threadIdx.x & 31, r = blockIdx.x * STATE_WARPS + (threadIdx.x >> 5);
    if (r >= n) return;
    const size_t sb = idx ? (size_t)idx[r] : (size_t)r;
    const BatchBuffers& S = kScatter ? wk : bat;
    const BatchBuffers& D = kScatter ? bat : wk;
    const size_t s = kScatter ? (size_t)r : sb, d = kScatter ? sb : (size_t)r;

    // words: mem_id, last_period, last_gain, mem_hp_x[2], lastg[22]
    switch (lane) {
        case 0: D.ceps_id[d] = S.ceps_id[s]; break;
        case 1: D.last_period[d] = S.last_period[s]; break;
        case 2: D.last_gain[d] = S.last_gain[s]; break;
        case 3:
        case 4: D.hp_mem[2 * d + (lane - 3)] = S.hp_mem[2 * s + (lane - 3)]; break;
        default:
            if (lane < 5 + NB_BANDS) D.lastg[d * NB_BANDS + (lane - 5)] = S.lastg[s * NB_BANDS + (lane - 5)];
            break;
    }

    const float4* h = reinterpret_cast<const float4*>(S.hist + s * HIST_CAP);
    float4* o = reinterpret_cast<float4*>(D.hist + d * HIST_CAP);
#pragma unroll 4
    for (int j = lane; j < hist_q; j += 32) o[ring_q(hdst, j)] = __ldg(h + ring_q(hsrc, j));
    const float4* c = reinterpret_cast<const float4*>(S.ceps_mem + s * CEPS_MEM * NB_BANDS);
    o = reinterpret_cast<float4*>(D.ceps_mem + d * CEPS_MEM * NB_BANDS);
    for (int j = lane; j < CEPS_Q; j += 32) o[j] = __ldg(c + j);
    const float4* y = reinterpret_cast<const float4*>(S.synth_mem + s * FRAME_SIZE);
    o = reinterpret_cast<float4*>(D.synth_mem + d * FRAME_SIZE);
#pragma unroll 4
    for (int j = lane; j < SYN_Q; j += 32) o[j] = __ldg(y + j);

    const float* g = S.gru_state + s * ss;
    float* og = D.gru_state + d * ss;
    if ((ss & 3) == 0) {  // rows of gru_state are 16-byte aligned
        for (int j = lane; j < ss / 4; j += 32) reinterpret_cast<float4*>(og)[j] = __ldg(reinterpret_cast<const float4*>(g) + j);
    } else {
        for (int j = lane; j < ss; j += 32) og[j] = __ldg(g + j);
    }
}

__global__ void __launch_bounds__(STATE_WARPS * 32) subset_gather_kernel(BatchBuffers bat, BatchBuffers wk, int ss, const int* __restrict__ idx,
                                                                         int n, int hq) {
    subset_copy<false>(bat, wk, ss, idx, n, hq, hq, (PITCH_BUF_SIZE - FRAME_SIZE) / 4);
}

__global__ void __launch_bounds__(STATE_WARPS * 32) subset_scatter_kernel(BatchBuffers bat, BatchBuffers wk, int ss, const int* __restrict__ idx,
                                                                          int n, int hq_work, int hq_batch) {
    subset_copy<true>(bat, wk, ss, idx, n, hq_work, hq_batch, IN_Q);
}

}  // namespace

cudaError_t launch_subset_gather(const BatchBuffers& batch, const BatchBuffers& work, int state_size, const int* idx, int n, int slot,
                                 cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    subset_gather_kernel<<<(n + STATE_WARPS - 1) / STATE_WARPS, STATE_WARPS * 32, 0, st>>>(batch, work, state_size, idx, n, hist_base(slot) / 4);
    return cudaGetLastError();
}

cudaError_t launch_subset_scatter(const BatchBuffers& batch, const BatchBuffers& work, int state_size, const int* idx, int n, int work_slot,
                                  int batch_slot, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    subset_scatter_kernel<<<(n + STATE_WARPS - 1) / STATE_WARPS, STATE_WARPS * 32, 0, st>>>(batch, work, state_size, idx, n,
                                                                                         hist_base(work_slot) / 4, hist_base(batch_slot) / 4);
    return cudaGetLastError();
}

cudaError_t launch_state_check(const void* src, int n, const int widths[3], int* first_bad, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    state_check_kernel<<<(n + 255) / 256, 256, 0, st>>>(static_cast<const unsigned char*>(src), n,
                                                        (int)state_record_bytes(widths[0] + widths[1] + widths[2]), widths[0], widths[1],
                                                        widths[2], first_bad);
    return cudaGetLastError();
}

cudaError_t launch_state_gather(const BatchBuffers& b, const int widths[3], const int* idx, int n, int slot, void* dst, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const int rec = (int)state_record_bytes(widths[0] + widths[1] + widths[2]);
    state_gather_kernel<<<(n + STATE_WARPS - 1) / STATE_WARPS, STATE_WARPS * 32, 0, st>>>(b, widths[0], widths[1], widths[2], idx, n, hist_base(slot),
                                                                                       rec, static_cast<unsigned char*>(dst));
    return cudaGetLastError();
}

cudaError_t launch_state_scatter(const BatchBuffers& b, int state_size, const int* idx, int n, int slot, const void* src, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    state_scatter_kernel<<<(n + STATE_WARPS - 1) / STATE_WARPS, STATE_WARPS * 32, 0, st>>>(b, state_size, idx, n, hist_base(slot),
                                                                                        (int)state_record_bytes(state_size),
                                                                                        static_cast<const unsigned char*>(src));
    return cudaGetLastError();
}

}  // namespace nnb
