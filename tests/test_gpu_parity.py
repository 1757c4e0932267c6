"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the C ABI, against
the oracle on the same inputs.  Stated tolerances (f32 path, FFT/GRU summation order differs from the
oracle's): output relative RMS <= 1e-5 (north_star requires 1e-4), VAD |diff| <= 1e-4, pitch period
(integer) bit-exact, golden metric of src/lib.rs:184-194 < 1e-4."""
import ctypes as C

import numpy as np
import pytest

import oracle
import nnnoiseless_b200 as nb
from conftest import golden_metric, synth_streams

pytestmark = pytest.mark.gpu

OUT_REL_RMS = 1e-5
VAD_ATOL = 1e-4


def rel_rms(a, b):
    a = a.astype(np.float64); b = b.astype(np.float64)
    return np.sqrt(((a - b) ** 2).sum() / max((b ** 2).sum(), 1e-30))


def oracle_run(model_bytes, x_bt):
    """x_bt: [B][T][480] -> oracle out/vad/pitch."""
    return oracle.run_batch(oracle.Model(model_bytes), x_bt, n_threads=0)


def check_against_oracle(gout, gvad, gpitch_last, ref, x_bt):
    # gout [T][B][480], gvad [T][B]; ref arrays [B][T]...
    o_ref = ref["out"].transpose(1, 0, 2)
    assert rel_rms(gout, o_ref) <= OUT_REL_RMS
    # per stream too, so one bad stream cannot hide in the batch
    for s in range(gout.shape[1]):
        assert rel_rms(gout[:, s], o_ref[:, s]) <= 5 * OUT_REL_RMS, s
    assert np.abs(gvad - ref["vad"].T).max() <= VAD_ATOL
    dec_g, dec_r = gvad > 0.5, ref["vad"].T > 0.5
    near = np.abs(ref["vad"].T - 0.5) < 1e-5
    assert np.array_equal(dec_g[~near], dec_r[~near])
    if gpitch_last is not None:
        assert np.array_equal(gpitch_last, ref["pitch"][:, -1])


def test_golden_vector_legacy_abi(builtin_bytes, testing_raw, reference_output):
    """rnnoise_create/process_frame exactly as test_data/rnnoise_demo.c drives them (in place)."""
    L = nb.lib()
    st = L.rnnoise_create(None)
    assert st, nb.last_error()
    ost = oracle.State(oracle.Model(builtin_bytes))
    outs, buf = [], np.empty(480, np.float32)
    for f in range(100):
        buf[:] = testing_raw[f]
        vad = L.rnnoise_process_frame(st, buf.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p))
        o_ref, v_ref = ost.process_frame(testing_raw[f])
        assert abs(vad - v_ref) <= VAD_ATOL, f
        assert rel_rms(buf, o_ref) <= 5 * OUT_REL_RMS, f
        if f > 0:
            outs.append(buf.copy())
    L.rnnoise_destroy(st)
    metric, maxdiff = golden_metric(outs, reference_output)
    assert metric < 1e-4
    assert metric < 1e-5 and maxdiff <= 1


def test_pitch_bit_exact_every_frame(builtin_bytes, testing_raw):
    b = nb.DenoiseBatch(1)
    ost = oracle.State(oracle.Model(builtin_bytes))
    for f in range(100):
        b.process_host(testing_raw[f][None, None, :])
        ost.process_frame(testing_raw[f])
        t, g = ost.taps(), b.taps()
        assert g["pitch"][0] == t.pitch and g["silence"][0] == t.silence, f
        assert np.abs(g["features"][0] - np.array(t.features)).max() < 1e-4, f
        if not t.silence:
            assert np.abs(g["gains"][0] - np.array(t.gains)).max() < 1e-4, f


@pytest.mark.parametrize("B,T", [(48, 30), (37, 12), (1, 25)])
def test_batched_synthetic_vs_oracle(builtin_bytes, B, T):
    x = synth_streams(B, T).reshape(B, T, 480)
    ref = oracle_run(builtin_bytes, x)
    b = nb.DenoiseBatch(B)
    pitches = []
    outs, vads = [], []
    for t in range(T):  # frame by frame so the pitch tap of every frame is checked
        o, v = b.process_host(np.ascontiguousarray(x[:, t][None]))
        outs.append(o[0]); vads.append(v[0])
        pitches.append(b.taps()["pitch"].copy())
    assert np.array_equal(np.stack(pitches, 1), ref["pitch"])
    check_against_oracle(np.stack(outs), np.stack(vads), None, ref, x)


def test_multi_frame_call_equals_frame_by_frame(builtin_bytes):
    B, T = 16, 10
    x = synth_streams(B, T, seed=7).reshape(B, T, 480)
    xt = np.ascontiguousarray(x.transpose(1, 0, 2))
    a = nb.DenoiseBatch(B)
    o1, v1 = a.process_host(xt)
    b = nb.DenoiseBatch(B)
    for t in range(T):
        o, v = b.process_host(xt[t:t + 1])
        assert np.array_equal(o[0], o1[t]) and np.array_equal(v[0], v1[t])


def test_custom_model_sh(sh_bytes):
    """BASELINE config 5 model (tanh GRUs): parity vs oracle only -- the reference has no golden for it."""
    B, T = 16, 20
    x = synth_streams(B, T, seed=99).reshape(B, T, 480)
    ref = oracle_run(sh_bytes, x)
    m = nb.RnnModel.from_bytes(sh_bytes)
    b = nb.DenoiseBatch(B, m)
    o, v = b.process_host(np.ascontiguousarray(x.transpose(1, 0, 2)))
    check_against_oracle(o, v, b.taps()["pitch"], ref, x)


def test_batch_position_independence_bitwise(builtin_bytes):
    """4096 copies of one stream: every copy is bit-identical to the B=1 run (no cross-stream leakage)."""
    T = 6
    x1 = synth_streams(1, T, seed=5).reshape(1, T, 480)
    a = nb.DenoiseBatch(1)
    o1, v1 = a.process_host(np.ascontiguousarray(x1.transpose(1, 0, 2)))
    B = 4096
    xb = np.ascontiguousarray(np.broadcast_to(x1.transpose(1, 0, 2), (T, B, 480)))
    b = nb.DenoiseBatch(B)
    ob, vb = b.process_host(xb)
    assert np.array_equal(ob, np.broadcast_to(o1, ob.shape))
    assert np.array_equal(vb, np.broadcast_to(v1, vb.shape))


def test_silence_path_and_recovery(builtin_bytes):
    """Signal -> 45 frames of digital zeros -> signal.  Silent frames: vad exactly 0, state untouched.

    Tolerance (SURVEY H6): in the frames right after the cut-off the window holds only the smooth tail of the high-pass
    filter, every band above ~1 kHz sits at the f32 rounding floor of the FFT and the pitch-correlation features
    (exp / sqrt(ex * ep), src/features.rs:136-137) are ratios of rounding noise; the GRUs remember it.
    tests/test_oracle_golden.py::test_post_silence_is_ill_conditioned_for_any_f32_fft MEASURES this between three correct
    CPU FFTs (two f32 orderings, one f64): ~5e-7 before the cut, 1.2e-4 (batch) / up to 9e-4 (single stream) after it,
    VAD up to 4e-4.  The GPU's FFT is a fourth ordering; it must stay within a small multiple of that spread, measured here
    against the f64-FFT oracle next to the two f32 oracles, not merely within a loose constant.
    Everything well-conditioned stays tight: silence flags, pitch (exact), silent-frame vad, the frames before the cut."""
    B = 64
    sig = synth_streams(B, 8, seed=11).reshape(B, 8, 480)
    x = np.concatenate([sig, np.zeros((B, 45, 480), np.float32), sig], axis=1)
    refs = {}
    try:
        for mode in (0, 1, 2):
            oracle.set_fft_mode(mode)
            refs[mode] = oracle_run(builtin_bytes, x)
    finally:
        oracle.set_fft_mode(0)
    ref = refs[0]
    b = nb.DenoiseBatch(B)
    outs, vads, pitches, sil = [], [], [], []
    for t in range(x.shape[1]):
        o, v = b.process_host(np.ascontiguousarray(x[:, t][None]))
        outs.append(o[0]); vads.append(v[0])
        tp = b.taps()
        pitches.append(tp["pitch"].copy()); sil.append(tp["silence"].copy())
    o, v = np.stack(outs), np.stack(vads)
    assert np.array_equal(np.stack(pitches, 1), ref["pitch"])           # integer output: exact, always
    sil = np.stack(sil, 1)
    assert sil[:, :8].sum() == 0 and sil[:, 30:53].all() and sil[:, 53:].sum() == 0
    assert np.array_equal(v[30:53], np.zeros((23, B), np.float32))      # silent frames return vad == 0.0
    assert np.array_equal(ref["vad"].T[30:53], np.zeros((23, B), np.float32))
    assert np.abs(o[50]).max() < 1e-6                                    # high-pass residue passed straight through
    o_ref = ref["out"].transpose(1, 0, 2)
    assert rel_rms(o[:8], o_ref[:8]) <= OUT_REL_RMS                      # before the cut-off: the usual tolerance
    # after it: distance to the f64-FFT oracle, GPU vs the two f32 CPU FFTs
    o64 = refs[1]["out"].transpose(1, 0, 2)
    v64 = refs[1]["vad"].T
    d_gpu = rel_rms(o[53:], o64[53:])
    d_cpu = max(rel_rms(refs[k]["out"].transpose(1, 0, 2)[53:], o64[53:]) for k in (0, 2))
    per_gpu = max(rel_rms(o[53:, s], o64[53:, s]) for s in range(B))
    per_cpu = max(rel_rms(refs[k]["out"].transpose(1, 0, 2)[53:, s], o64[53:, s]) for k in (0, 2) for s in range(B))
    dv_gpu = np.abs(v - v64).max()
    dv_cpu = max(np.abs(refs[k]["vad"].T - v64).max() for k in (0, 2))
    print("post-silence distance to the f64-FFT oracle: GPU %.3g (worst stream %.3g, vad %.3g); f32 CPU FFTs %.3g (%.3g, vad %.3g)"
          % (d_gpu, per_gpu, dv_gpu, d_cpu, per_cpu, dv_cpu))
    assert d_gpu <= 3 * d_cpu and per_gpu <= 4 * per_cpu and dv_gpu <= 4 * dv_cpu
    assert rel_rms(o, o_ref) <= 6e-4 and np.abs(v - ref["vad"].T).max() <= 2e-3


def test_zero_input_from_start():
    b = nb.DenoiseBatch(3)
    o, v = b.process_host(np.zeros((4, 3, 480), np.float32))
    assert not o.any() and not v.any()
    assert np.array_equal(b.taps()["silence"], np.ones(3, np.int32))


def test_full_scale_and_dc(builtin_bytes):
    """Extreme inputs the reference accepts: int16 full-scale square wave, pure DC."""
    T = 12
    n = np.arange(T * 480)
    sq = np.where((n // 50) % 2 == 0, 32767.0, -32768.0).astype(np.float32)
    dc = np.full(T * 480, 12345.0, np.float32)
    x = np.stack([sq, dc]).reshape(2, T, 480)
    ref = oracle_run(builtin_bytes, x)
    b = nb.DenoiseBatch(2)
    o, v = b.process_host(np.ascontiguousarray(x.transpose(1, 0, 2)))
    assert np.array_equal(b.taps()["pitch"], ref["pitch"][:, -1])
    assert np.abs(v - ref["vad"].T).max() <= VAD_ATOL
    assert np.abs(o - ref["out"].transpose(1, 0, 2)).max() <= 1e-5 * 32768 * 4


def test_reset_equals_fresh(builtin_bytes):
    B, T = 4, 5
    x = np.ascontiguousarray(synth_streams(B, T, seed=3).reshape(B, T, 480).transpose(1, 0, 2))
    b = nb.DenoiseBatch(B)
    o1, v1 = b.process_host(x)
    b.process_host(x)
    b.reset()
    o2, v2 = b.process_host(x)
    assert np.array_equal(o1, o2) and np.array_equal(v1, v2)


def test_pcm16_front_end(builtin_bytes):
    """int16 in, round-to-nearest + clamp out (src/nnnoiseless.rs:152, rnnoise_demo.c:53)."""
    B, T = 6, 10
    x = synth_streams(B, T, seed=21).reshape(B, T, 480)
    ref = oracle_run(builtin_bytes, x)
    b = nb.DenoiseBatch(B)
    o16, v = b.process_pcm16_host(np.ascontiguousarray(x.transpose(1, 0, 2)).astype(np.int16))
    want = np.clip(np.rint(ref["out"].transpose(1, 0, 2)), -32768, 32767).astype(np.int16)  # rint==roundf off ties
    assert np.abs(o16.astype(np.int32) - want.astype(np.int32)).max() <= 1
    assert (o16 != want).mean() < 1e-2  # only samples whose fraction sits within the f32 tolerance of .5


def test_device_pointer_api_stream_major_layout(builtin_bytes):
    """rnnoise_batch_process_device with [B][T][480] (stream-major) torch tensors, in place."""
    import torch
    B, T = 20, 7
    x = synth_streams(B, T, seed=31).reshape(B, T, 480)
    ref = oracle_run(builtin_bytes, x)
    xd = torch.from_numpy(x).cuda()
    vad = torch.empty(T, B, device="cuda")
    b = nb.DenoiseBatch(B)
    b.process_device(xd.data_ptr(), xd.data_ptr(), vad.data_ptr(), T, stream_stride=T * 480, frame_stride=480,
                     cuda_stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    check_against_oracle(xd.cpu().numpy().transpose(1, 0, 2), vad.cpu().numpy(), b.taps()["pitch"], ref, x)


def test_baseline_size_batch_properties(builtin_bytes):
    """BASELINE config 3 size (65,536 streams): 64 distinct streams tiled 1024x.  Every tile must be
    bit-identical (batch-position independence at full size) and tile 0 must match the oracle."""
    import torch
    B, D, T = 65536, 64, 4
    x = synth_streams(D, T, seed=41).reshape(D, T, 480)
    ref = oracle_run(builtin_bytes, x)
    xt = torch.from_numpy(np.ascontiguousarray(x.transpose(1, 0, 2))).cuda()  # [T][D][480]
    xin = xt.repeat(1, B // D, 1).contiguous()                               # [T][B][480]
    out = torch.empty_like(xin)
    vad = torch.empty(T, B, device="cuda")
    b = nb.DenoiseBatch(B)
    b.process_device(out.data_ptr(), xin.data_ptr(), vad.data_ptr(), T, stream_stride=480, frame_stride=B * 480,
                     cuda_stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    tiles = out.view(T, B // D, D, 480)
    assert bool((tiles == tiles[:, :1]).all())
    assert bool((vad.view(T, B // D, D) == vad.view(T, B // D, D)[:, :1]).all())
    check_against_oracle(tiles[:, 0].cpu().numpy(), vad[:, :D].cpu().numpy(), b.taps()["pitch"][:D], ref, x)


def test_frame_pipeline_call_patterns_bitwise(builtin_bytes):
    """The five-stream frame pipeline must be invisible: any split of the same frames into calls (host or device API,
    T = 1 or many), and the serialised reference order (rnnoise_batch_profile_step), alone or mixed with the others on
    one handle, give bit-identical results."""
    import torch
    B, T = 96, 23
    x = np.ascontiguousarray(synth_streams(B, T, seed=77).reshape(B, T, 480).transpose(1, 0, 2))  # [T][B][480]
    a = nb.DenoiseBatch(B)
    o_ref, v_ref = a.process_host(x)
    # irregular call sizes through the host API
    b = nb.DenoiseBatch(B)
    outs, vads, t = [], [], 0
    for n in (1, 5, 2, 9, 1, 5):
        o, v = b.process_host(x[t:t + n]); outs.append(o); vads.append(v); t += n
    assert np.array_equal(np.concatenate(outs), o_ref) and np.array_equal(np.concatenate(vads), v_ref)
    # device API on a torch stream, mixed with host-API calls on the same handle
    c = nb.DenoiseBatch(B)
    xd = torch.from_numpy(x).cuda()
    od = torch.empty_like(xd)
    vd = torch.empty(T, B, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        c.process_device(od[:10].data_ptr(), xd[:10].data_ptr(), vd[:10].data_ptr(), 10, 480, B * 480, st.cuda_stream)
    st.synchronize()
    o_mid, v_mid = c.process_host(x[10:14])
    with torch.cuda.stream(st):
        c.process_device(od[14:].data_ptr(), xd[14:].data_ptr(), vd[14:].data_ptr(), T - 14, 480, B * 480, st.cuda_stream)
    st.synchronize()
    got = np.concatenate([od[:10].cpu().numpy(), o_mid, od[14:].cpu().numpy()])
    assert np.array_equal(got, o_ref)
    assert np.array_equal(np.concatenate([vd[:10].cpu().numpy(), v_mid, vd[14:].cpu().numpy()]), v_ref)
    # two handles interleaved frame by frame do not disturb each other
    d1, d2 = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    for t in range(6):
        o1, _ = d1.process_host(x[t:t + 1])
        o2, _ = d2.process_host(x[t:t + 1])
        assert np.array_equal(o1[0], o_ref[t]) and np.array_equal(o2[0], o_ref[t])
    # serialised single-stream execution (profile_step: every kernel of the frame on one stream) = the same bits
    e = nb.DenoiseBatch(B)
    oe, ve = torch.empty_like(xd), torch.empty(T, B, device="cuda")
    for t in range(T):
        e.profile_step(oe[t].data_ptr(), xd[t].data_ptr(), ve[t].data_ptr(), 480)
    assert np.array_equal(oe.cpu().numpy(), o_ref) and np.array_equal(ve.cpu().numpy(), v_ref)
    # pipelined device frames, profile_step frames (on the batch's stream and on the caller's) and host-API frames on one
    # handle: each kind orders itself after the others (bench.py profiles a batch after its pipelined steps)
    g = nb.DenoiseBatch(B)
    og, vg = torch.empty_like(xd), torch.empty(T, B, device="cuda")
    with torch.cuda.stream(st):
        g.process_device(og[:6].data_ptr(), xd[:6].data_ptr(), vg[:6].data_ptr(), 6, 480, B * 480, st.cuda_stream)
    for t in range(6, 9):
        g.profile_step(og[t].data_ptr(), xd[t].data_ptr(), vg[t].data_ptr(), 480)
    o_mid, v_mid = g.process_host(x[9:13])
    g.profile_step(og[13].data_ptr(), xd[13].data_ptr(), vg[13].data_ptr(), 480, st.cuda_stream)
    with torch.cuda.stream(st):
        g.process_device(og[14:].data_ptr(), xd[14:].data_ptr(), vg[14:].data_ptr(), T - 14, 480, B * 480, st.cuda_stream)
    st.synchronize()
    got_o, got_v = og.cpu().numpy(), vg.cpu().numpy()
    got_o[9:13], got_v[9:13] = o_mid, v_mid
    assert np.array_equal(got_o, o_ref) and np.array_equal(got_v, v_ref)


def test_pcm16_device_api_fused(builtin_bytes):
    """int16 device buffers straight into the first kernel and out of the last one (N1 front-end, fused)."""
    import torch
    B, T = 33, 9
    x = synth_streams(B, T, seed=91).reshape(B, T, 480)
    ref = oracle_run(builtin_bytes, x)
    xi = torch.from_numpy(np.ascontiguousarray(x.transpose(1, 0, 2)).astype(np.int16)).cuda()   # [T][B][480]
    oi = torch.empty_like(xi)
    vad = torch.empty(T, B, device="cuda")
    b = nb.DenoiseBatch(B)
    b.process_device(oi.data_ptr(), xi.data_ptr(), vad.data_ptr(), T, 480, B * 480, torch.cuda.current_stream().cuda_stream, pcm16=True)
    torch.cuda.synchronize()
    want = np.clip(np.rint(ref["out"].transpose(1, 0, 2)), -32768, 32767).astype(np.int16)
    got = oi.cpu().numpy()
    assert np.abs(got.astype(np.int32) - want.astype(np.int32)).max() <= 1 and (got != want).mean() < 1e-2
    assert np.abs(vad.cpu().numpy() - ref["vad"].T).max() <= VAD_ATOL
    # and identical to the host pcm16 entry point
    o16, _ = nb.DenoiseBatch(B).process_pcm16_host(xi.cpu().numpy())
    assert np.array_equal(o16, got)


def test_handles_on_concurrent_host_threads(builtin_bytes):
    """`DenoiseState: Send + Sync` (src/denoise.rs:125) restated: independent states may be driven from different host
    threads at the same time; results equal the single-threaded run bit for bit."""
    import threading
    B, T = 24, 8
    xs = [np.ascontiguousarray(synth_streams(B, T, seed=200 + i).reshape(B, T, 480).transpose(1, 0, 2)) for i in range(4)]
    want = [nb.DenoiseBatch(B).process_host(x) for x in xs]
    got = [None] * 4

    def work(i):
        b = nb.DenoiseBatch(B)
        outs, vads = [], []
        for t in range(T):
            o, v = b.process_host(xs[i][t:t + 1])
            outs.append(o); vads.append(v)
        got[i] = (np.concatenate(outs), np.concatenate(vads))

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th: t.start()
    for t in th: t.join()
    for i in range(4):
        assert np.array_equal(got[i][0], want[i][0]) and np.array_equal(got[i][1], want[i][1])


def test_interleaved_channels_layout(builtin_bytes):
    """Multi-channel interleaved audio, every channel its own stream (src/signal.rs:90-107, src/nnnoiseless.rs:301-330):
    sample (channel c, frame t, i) at [t*480*C + i*C + c].  Same bits as the planar layout, float and int16."""
    import ctypes as C
    import torch
    Cn, T = 6, 7
    x = np.ascontiguousarray(synth_streams(Cn, T, seed=55).reshape(Cn, T, 480).transpose(1, 0, 2))   # planar [T][C][480]
    o_ref, v_ref = nb.DenoiseBatch(Cn).process_host(x)
    xi = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 2, 1))).cuda()                            # [T][480][C]
    oi = torch.empty_like(xi)
    vad = torch.empty(T, Cn, device="cuda")
    b = nb.DenoiseBatch(Cn)
    rc = nb.lib().rnnoise_batch_process_device_strided(b._h, C.c_void_p(oi.data_ptr()), C.c_void_p(xi.data_ptr()), 0,
                                                       C.c_void_p(vad.data_ptr()), T, 1, Cn, 480 * Cn, None)
    assert rc == 0, nb.last_error()
    assert np.array_equal(oi.cpu().numpy().transpose(0, 2, 1), o_ref) and np.array_equal(vad.cpu().numpy(), v_ref)
    # int16, in place
    x16 = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 2, 1)).astype(np.int16)).cuda()
    b2 = nb.DenoiseBatch(Cn)
    rc = nb.lib().rnnoise_batch_process_device_strided(b2._h, C.c_void_p(x16.data_ptr()), C.c_void_p(x16.data_ptr()), 1,
                                                       None, T, 1, Cn, 480 * Cn, None)
    assert rc == 0, nb.last_error()
    want, _ = nb.DenoiseBatch(Cn).process_pcm16_host(x.astype(np.int16))
    assert np.array_equal(x16.cpu().numpy().transpose(0, 2, 1), want)


def test_long_run_no_drift(builtin_bytes):
    """6 s of audio (600 frames) per stream: the recurrent state (GRU, cepstral ring, pitch continuity, overlap-add)
    must not drift away from the oracle over time; the pitch period stays exact on every one of the 2,400 frames."""
    B, T = 4, 600
    x = synth_streams(B, T, seed=123).reshape(B, T, 480)
    ref = oracle_run(builtin_bytes, x)
    b = nb.DenoiseBatch(B)
    xt = np.ascontiguousarray(x.transpose(1, 0, 2))
    outs, vads, pitches = [], [], []
    for t0 in range(0, T, 50):
        for t in range(t0, t0 + 50):
            o, v = b.process_host(xt[t:t + 1])
            outs.append(o[0]); vads.append(v[0]); pitches.append(b.taps()["pitch"].copy())
    o, v = np.stack(outs), np.stack(vads)
    assert np.array_equal(np.stack(pitches, 1), ref["pitch"])
    o_ref = ref["out"].transpose(1, 0, 2)
    assert rel_rms(o, o_ref) <= OUT_REL_RMS
    assert rel_rms(o[-100:], o_ref[-100:]) <= OUT_REL_RMS          # the last second is as good as the first
    assert np.abs(v - ref["vad"].T).max() <= VAD_ATOL


# ---- pitch exactness at scale (the fast pitch kernel certifies its decisions; these sweeps are the evidence) ----------
def _synth_mixed_cuda(B, T, seed, speech):
    """synth_mixed's four families generated on the GPU (the CPU generator would take minutes at 10^6 stream-frames):
    white+sine | harmonic stack with vibrato | looped speech fixture with gain and silence gaps | nearly pure tones."""
    import torch
    dev = torch.device("cuda")
    g = torch.Generator(device=dev); g.manual_seed(seed)
    n = T * 480
    r = torch.rand(10, B, generator=g, device=dev, dtype=torch.float64)
    f0 = 100.0 * torch.pow(torch.tensor(40.0, dtype=torch.float64, device=dev), r[0])
    a, sg, ph = 1000.0 + 11000.0 * r[1], 100.0 + 2900.0 * r[2], 2 * np.pi * r[3]
    vib, vrate, nh, gain = 0.002 + 0.02 * r[4], 3.0 + 5.0 * r[5], 2 + (r[6] * 10).long(), 0.05 + 1.5 * r[7]
    sp = torch.from_numpy(speech.astype(np.float32)).to(dev)
    off = (r[8] * len(speech)).long()
    fam = torch.arange(B, device=dev) % 4
    pure = (torch.arange(B, device=dev) % 8) == 3
    x = torch.empty(B, n, device=dev, dtype=torch.float32)
    CH = 48000
    phase = ph.clone()
    for c0 in range(0, n, CH):
        c1 = min(n, c0 + CH)
        t = torch.arange(c0, c1, device=dev, dtype=torch.float64)[None, :]
        noise = torch.randn(B, c1 - c0, generator=g, device=dev, dtype=torch.float32).double()
        tone = a[:, None] * torch.sin(torch.remainder(2 * np.pi * f0[:, None] * t / 48000.0 + ph[:, None], 2 * np.pi))
        v0 = tone + sg[:, None] * noise
        s3 = torch.where(pure, 1.0 + 20.0 * r[9], 0.1 * sg)
        v3 = tone + s3[:, None] * noise
        fi = torch.clamp(f0[:, None] * 0.25 * (1.0 + vib[:, None] * torch.sin(2 * np.pi * vrate[:, None] * t / 48000.0)), min=60.0)
        pcs = phase[:, None] + 2 * np.pi * torch.cumsum(fi, 1) / 48000.0
        phase = torch.remainder(pcs[:, -1], 2 * np.pi)
        v1 = torch.zeros_like(v0)
        for h in range(1, 12):
            v1 += torch.where((nh >= h)[:, None], a[:, None] / h * torch.sin(torch.remainder(h * pcs, 2 * np.pi)), torch.zeros_like(v0))
        v1 += 0.3 * sg[:, None] * noise
        idx = (off[:, None] + t.long()) % len(speech)
        v2 = gain[:, None] * sp[idx].double() + 0.02 * sg[:, None] * noise
        v2 = torch.where((((t.long() // 480) // 13) % 5) == 4, torch.zeros_like(v2), v2)
        v = torch.where((fam == 0)[:, None], v0, torch.where((fam == 1)[:, None], v1, torch.where((fam == 2)[:, None], v2, v3)))
        x[:, c0:c1] = torch.clamp(torch.round(v), -32768.0, 32767.0).float()
    return x.view(B, T, 480)


def test_pitch_mass_sweep_bit_exact(builtin_bytes):
    """>= 10^6 stream-frames (4,096 streams x 256 frames: harmonic stacks with vibrato, looped speech with silence gaps,
    nearly pure tones, white+sine): the integer pitch period of EVERY frame equals the oracle's.  Also prints how often
    the kernel had to fall back to the order-exact recomputation (rnnoise_batch_pitch_stats)."""
    import torch
    B, T = 4096, 256
    speech = np.fromfile(__import__("os").path.join(__import__("conftest").GOLDEN, "testing.raw"), dtype="<i2")
    xd = _synth_mixed_cuda(B, T, 20260923, speech)                       # [B][T][480] on the device
    x = xd.cpu().numpy()
    ref = oracle.run_batch(oracle.Model(builtin_bytes), x, n_threads=0, want_out=False)   # pitch [B][T]
    xt = xd.permute(1, 0, 2).contiguous()                                 # [T][B][480]
    out = torch.empty(B, 480, device="cuda")
    b = nb.DenoiseBatch(B)
    got = np.empty((B, T), np.int32)
    sp = torch.cuda.current_stream().cuda_stream
    for t in range(T):
        b.process_device(out.data_ptr(), xt[t].data_ptr(), 0, 1, stream_stride=480, frame_stride=B * 480, cuda_stream=sp)
        torch.cuda.synchronize()
        got[:, t] = b.taps()["pitch"]
    st = b.pitch_stats()
    bad = np.argwhere(got != ref["pitch"])
    print("pitch sweep: %d stream-frames, mismatches %d; exact recomputation: coarse %.3f%%, ladder %.4f%%"
          % (B * T, len(bad), 100.0 * st["coarse_exact"] / st["stream_frames"], 100.0 * st["ladder_exact"] / st["stream_frames"]))
    assert st["stream_frames"] == B * T
    assert len(bad) == 0, bad[:10]
    # the certificate must actually certify: the exact recomputation stays the exception
    assert st["coarse_exact"] < 0.05 * B * T and st["ladder_exact"] < 0.02 * B * T


def test_pitch_exact_mode_and_extreme_inputs(builtin_bytes):
    """NNB_PITCH_EXACT=1 routes every stream through the kernel's order-exact recomputation paths (the test reference for
    the certified fast paths): same bits.  Inputs include amplitudes far outside the int16 range the reference documents
    (tiny float audio that nobody scaled, 1e4 x full scale) where the certificate must give up rather than guess."""
    import os
    speech = np.fromfile(os.path.join(__import__("conftest").GOLDEN, "testing.raw"), dtype="<i2")
    from nnnoiseless_b200.synth import synth_mixed
    B, T = 96, 24
    x = synth_mixed(B, T, seed=77, speech=speech).reshape(B, T, 480)
    scale = np.ones(B, np.float32)
    scale[0::12] = 1e-9; scale[1::12] = 3e-5; scale[2::12] = 1e4; scale[3::12] = 1.0 / 32768.0
    x = x * scale[:, None, None]
    ref = oracle_run(builtin_bytes, x)
    xt = np.ascontiguousarray(x.transpose(1, 0, 2))
    fast = nb.DenoiseBatch(B)
    os.environ["NNB_PITCH_EXACT"] = "1"
    try:
        exact = nb.DenoiseBatch(B)
    finally:
        del os.environ["NNB_PITCH_EXACT"]
    for t in range(T):
        of, vf = fast.process_host(xt[t:t + 1])
        oe, ve = exact.process_host(xt[t:t + 1])
        pf, pe = fast.taps()["pitch"], exact.taps()["pitch"]
        assert np.array_equal(pf, ref["pitch"][:, t]), (t, np.argwhere(pf != ref["pitch"][:, t])[:5])
        assert np.array_equal(pe, ref["pitch"][:, t]), t
        assert np.array_equal(of, oe) and np.array_equal(vf, ve)
    se = exact.pitch_stats()
    assert se["coarse_exact"] == B * T and se["ladder_exact"] == B * T
    sf = fast.pitch_stats()
    assert sf["stream_frames"] == B * T and sf["coarse_exact"] < B * T
