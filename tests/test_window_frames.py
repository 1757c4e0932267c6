"""Tests of window frames (rnnoise_batch_analyze_window_device / _synthesize_window_device, DESIGN.md 7j): split frames
of any length whose spectra live in the caller's context records.

- A window run equals the split path with the saving synthesis bit for bit: features, silence flags, output, the state
  records after draining and every byte of the context records, padding included.  Random schedules with the synthesis
  lagging by up to the whole window, windows longer than the pipeline's event ring, batch sizes around the warp tiles.
- Every buffer layout gives the same bits: features, gains and records batch-first or seq-first, int16 samples,
  interleaved stereo.
- Lookahead of 10 frames: gains computed from features t .. t + 10 of the window itself, and a split twin fed them
  gives the same output bits.
- The float32 torch restatement of the built-in network over all of testing.raw, between one analyze_window and one
  synthesize_window, meets the golden metric with the bits of the split path.
- synthesis_grad gives the same gradient bits on window and saving records; a bidirectional GRU trained over whole
  windows lowers a waveform MSE.
- Mixing, ordering and argument refusals change nothing; reset drops owed frames.  The C++ mirror compiles and null
  batches are refused without a GPU.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nnnoiseless_b200 as nb
from test_split_frames import MAXP, TorchDenoiseNet, bits, network_loop, schedule, signals
from test_synth_grad import noisy_clean

F, NBF, NBB, CB = 480, 42, 22, nb.SYNTH_CONTEXT_BYTES
JUNK = 0xA5  # records start as junk: every byte the calls leave must be written by them


def window_schedule(T, rng):
    """A random schedule of ("a" | "s", first frame, frames): analysis chunks of any length, the synthesis lagging by
    anything up to the whole window."""
    ta = ts = 0
    steps = []
    while ts < T:
        if ta < T and (ta == ts or rng.random() < 0.55):
            k = int(rng.integers(1, T - ta + 1))
            steps.append(("a", ta, k))
            ta += k
        else:
            k = int(rng.integers(1, ta - ts + 1))
            steps.append(("s", ts, k))
            ts += k
    return steps


def new_ctx(B, T, seq_first=False):
    import torch
    shape = (T, B, CB) if seq_first else (B, T, CB)
    return torch.full(shape, JUNK, dtype=torch.uint8, device="cuda")


def ctx_at(ctx, t, seq_first=False):
    """(pointer to frame t's records, stream stride, frame stride) in records."""
    if seq_first:
        return ctx[t].data_ptr(), ctx.stride(1) // CB, ctx.stride(0) // CB
    return ctx[:, t].data_ptr(), ctx.stride(0) // CB, ctx.stride(1) // CB


def run(b, steps, xd, gains, window, batch_first=False, seq_first_ctx=False, pcm16=0, sample_stride=1, stream_stride=F,
        frame_stride=None, cuda_stream=0):
    """Frames of xd (frame t at element t * frame_stride of the flat buffer) through `steps`: window calls, or split
    analysis and (float output) saving synthesis.  gains [T][B][22] or (batch_first) [B][T][22].  Returns
    (out like xd, features like gains with 42 columns, silence [T][B], ctx)."""
    import torch
    T, B = (gains.shape[1], gains.shape[0]) if batch_first else (gains.shape[0], gains.shape[1])
    fs = frame_stride if frame_stride is not None else B * F
    out = torch.empty_like(xd)
    feats = torch.full((B, T, NBF) if batch_first else (T, B, NBF), float("nan"), device="cuda")
    sil = torch.full((T, B), -1, dtype=torch.int32, device="cuda")
    ctx = new_ctx(B, T, seq_first_ctx)
    xflat, oflat = xd.reshape(-1), out.reshape(-1)
    for kind, t, k in steps:
        if batch_first:
            fp, fss, ffs = feats[:, t].data_ptr(), feats.stride(0), feats.stride(1)
            gp, gss, gfs = gains[:, t].data_ptr(), gains.stride(0), gains.stride(1)
        else:
            fp, fss, ffs = feats[t].data_ptr(), feats.stride(1), feats.stride(0)
            gp, gss, gfs = gains[t].data_ptr(), gains.stride(1), gains.stride(0)
        cp, css, cfs = ctx_at(ctx, t, seq_first_ctx)
        io = dict(sample_stride=sample_stride, pcm16=pcm16, cuda_stream=cuda_stream)
        if kind == "a" and window:
            before = b.window_frames
            b.analyze_window_device(xflat[t * fs:].data_ptr(), fp, sil[t].data_ptr(), k, stream_stride, fs, fss, ffs, cp, css, cfs, **io)
            assert b.window_frames == before + k
        elif kind == "a":
            b.analyze_device(xflat[t * fs:].data_ptr(), fp, sil[t].data_ptr(), k, stream_stride, fs, fss, ffs, **io)
        elif window:
            before = b.window_frames
            b.synthesize_window_device(oflat[t * fs:].data_ptr(), gp, k, stream_stride, fs, gss, gfs, cp, css, cfs, **io)
            assert b.window_frames == before - k
        elif pcm16:
            b.synthesize_device(oflat[t * fs:].data_ptr(), gp, k, stream_stride, fs, gss, gfs, **io)
        else:
            b.synthesize_saving_device(oflat[t * fs:].data_ptr(), gp, k, stream_stride, fs, gss, gfs, cp, css, cfs, **io)
    torch.cuda.synchronize()
    assert b.window_frames == 0 and b.pending_frames == 0
    return out, feats, sil, ctx


def rand_gains(T, B, seed):
    import torch
    return torch.rand((T, B, NBB), generator=torch.Generator().manual_seed(seed)).cuda()


# ---- 1. window == split + saving, bit for bit ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 5, 17, 40])
@pytest.mark.parametrize("B", [1, 63, 64, 65, 229])
def test_window_equals_split_saving_bitwise(B, T):
    import torch
    x = signals(B, T, seed=500 + B + T)
    xd = torch.from_numpy(x).cuda()
    gains = rand_gains(T, B, B * 100 + T)
    tw = nb.DenoiseBatch(B)
    t_out, t_f, t_s, t_ctx = run(tw, schedule(T, np.random.default_rng(T)), xd, gains, window=False)
    rng = np.random.default_rng(B * 7 + T)
    for i, steps in enumerate([[("a", 0, T), ("s", 0, T)], window_schedule(T, rng)]):
        wb = nb.DenoiseBatch(B)
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            w_out, w_f, w_s, w_ctx = run(wb, steps, xd, gains, window=True, cuda_stream=st.cuda_stream)
        assert np.array_equal(bits(w_f), bits(t_f)), (i, steps)
        assert np.array_equal(w_s.cpu().numpy(), t_s.cpu().numpy()), (i, steps)
        assert np.array_equal(bits(w_out), bits(t_out)), (i, steps)
        assert np.array_equal(w_ctx.cpu().numpy(), t_ctx.cpu().numpy()), (i, steps)
        assert np.array_equal(wb.get_states(), tw.get_states()), (i, steps)
        with pytest.raises(nb.NnnoiselessError, match="split frame"):
            wb.taps()
    if B > 1:
        assert (t_s.cpu().numpy() == 1).any() and (t_s.cpu().numpy() == 0).any()


# ---- 2. layouts ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_layouts_bitwise():
    import torch
    B, T = 65, 21
    x = signals(B, T, seed=17)
    xd = torch.from_numpy(x).cuda()
    g_tb = rand_gains(T, B, 3)
    steps = window_schedule(T, np.random.default_rng(2))
    ref_out, ref_f, ref_s, ref_ctx = run(nb.DenoiseBatch(B), steps, xd, g_tb, window=True)
    # batch-first features and gains, seq-first records
    o, f, s, c = run(nb.DenoiseBatch(B), steps, xd, g_tb.transpose(0, 1).contiguous(), window=True, batch_first=True)
    assert np.array_equal(bits(o), bits(ref_out)) and np.array_equal(bits(f.transpose(0, 1)), bits(ref_f))
    assert np.array_equal(c.cpu().numpy(), ref_ctx.cpu().numpy())
    o, f, s, c = run(nb.DenoiseBatch(B), steps, xd, g_tb, window=True, seq_first_ctx=True)
    assert np.array_equal(bits(o), bits(ref_out)) and np.array_equal(c.transpose(0, 1).cpu().numpy(), ref_ctx.cpu().numpy())
    # int16 in and out: the split path's int16 output and the float run's records
    x16 = torch.from_numpy(x.astype(np.int16)).cuda()
    o16, f16, _, c16 = run(nb.DenoiseBatch(B), steps, x16, g_tb, window=True, pcm16=1)
    t16, _, _, _ = run(nb.DenoiseBatch(B), schedule(T, np.random.default_rng(4)), x16, g_tb, window=False, pcm16=1)
    assert np.array_equal(bits(o16), bits(t16)) and np.array_equal(bits(f16), bits(ref_f))
    assert np.array_equal(c16.cpu().numpy(), ref_ctx.cpu().numpy())
    # interleaved stereo: the same bits as the compact call on those two streams
    Bs = 2
    xs = torch.from_numpy(np.ascontiguousarray(x[:, :Bs].transpose(0, 2, 1))).cuda()  # [T][480][2]
    os_, fs_, _, cs_ = run(nb.DenoiseBatch(Bs), steps, xs, g_tb[:, :Bs].contiguous(), window=True, sample_stride=Bs, stream_stride=1,
                           frame_stride=F * Bs)
    oc, fc, _, cc = run(nb.DenoiseBatch(Bs), steps, xd[:, :Bs].contiguous(), g_tb[:, :Bs].contiguous(), window=True)
    assert np.array_equal(bits(os_.permute(0, 2, 1)), bits(oc)) and np.array_equal(bits(fs_), bits(fc))
    assert np.array_equal(cs_.cpu().numpy(), cc.cpu().numpy())


# ---- 3. lookahead beyond 3 frames ---------------------------------------------------------------------------------------
LOOK = 10


def lookahead_gains(feats, t):
    """Gains of frame t [B][22] from features t .. t + LOOK (clamped to the window's last frame) [T][B][42]."""
    import torch
    T = feats.shape[0]
    idx = torch.tensor([min(t + j, T - 1) for j in range(LOOK + 1)], device=feats.device)
    w = torch.linspace(1.0, 0.2, LOOK + 1, device=feats.device)[:, None, None]
    return torch.sigmoid((feats[idx, :, :NBB] * w).sum(0) * 0.05 + feats[t, :, NBB:NBB + 1])


@pytest.mark.gpu
def test_lookahead_beyond_three_frames():
    import torch
    B, T = 37, 30
    x = signals(B, T, seed=23)
    xd = torch.from_numpy(x).cuda()
    b = nb.DenoiseBatch(B)
    out = torch.empty_like(xd)
    feats = torch.empty((T, B, NBF), device="cuda")
    gains = torch.empty((T, B, NBB), device="cuda")
    ctx = new_ctx(B, T)
    # streaming: analyze one frame, synthesize one frame LOOK behind, then the tail
    for t in range(T + LOOK):
        if t < T:
            b.analyze_window_device(xd[t].data_ptr(), feats[t].data_ptr(), 0, 1, F, B * F, NBF, B * NBF, ctx[:, t].data_ptr(), T, 1)
        s = t - LOOK
        if s >= 0:
            assert b.window_frames == min(t, T - 1) - s + 1
            gains[s] = lookahead_gains(feats[:min(t, T - 1) + 1], s) if t < T else lookahead_gains(feats, s)
            b.synthesize_window_device(out[s].data_ptr(), gains[s].data_ptr(), 1, F, B * F, NBB, B * NBB, ctx[:, s].data_ptr(), T, 1)
    assert b.window_frames == 0
    # the same gains from the whole window at once: the streaming loop saw features t .. t + LOOK in time
    whole = torch.stack([lookahead_gains(feats, t) for t in range(T)])
    assert np.array_equal(bits(whole), bits(gains))
    tw = nb.DenoiseBatch(B)
    t_out, t_f, _, _ = run(tw, schedule(T, np.random.default_rng(9)), xd, gains, window=False)
    assert np.array_equal(bits(t_f), bits(feats))
    assert np.array_equal(bits(t_out), bits(out))
    assert np.array_equal(tw.get_states(), b.get_states())


# ---- 4. golden vector ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_torch_network_over_one_window(builtin_bytes, testing_raw, reference_output):
    import torch
    from conftest import golden_metric
    net = TorchDenoiseNet(builtin_bytes)
    xd = torch.from_numpy(np.ascontiguousarray(testing_raw[:, None, :])).cuda()  # [T][1][480]
    T = xd.shape[0]
    b = nb.DenoiseBatch(1)
    out = torch.empty_like(xd)
    feats = torch.empty((T, 1, NBF), device="cuda")
    sil = torch.empty((T, 1), dtype=torch.int32, device="cuda")
    gains = torch.empty((T, 1, NBB), device="cuda")
    ctx = new_ctx(1, T)
    state = torch.zeros((1, sum(net.widths)), device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        b.analyze_window_device(xd.data_ptr(), feats.data_ptr(), sil.data_ptr(), T, F, F, NBF, NBF, ctx.data_ptr(), T, 1,
                                cuda_stream=st.cuda_stream)
        for t in range(T):
            gains[t], state = net(feats[t], state, sil[t] != 0)
        b.synthesize_window_device(out.data_ptr(), gains.data_ptr(), T, F, F, NBB, NBB, ctx.data_ptr(), T, 1, cuda_stream=st.cuda_stream)
    torch.cuda.synchronize()
    metric, maxdiff = golden_metric(list(out[1:, 0].cpu().numpy()), reference_output)
    print("\ntorch network over one window of %d frames: golden metric %.3g (max %d LSB)" % (T, metric, maxdiff))
    assert metric < 1e-4
    split = network_loop(net, nb.DenoiseBatch(1), xd, MAXP, torch.cuda.Stream())
    assert np.array_equal(bits(out), bits(split))


# ---- 5. training ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gradients_equal_on_window_and_saving_records():
    import torch
    from nnnoiseless_b200.autograd import synthesis_grad
    B, T = 24, 19
    xd = torch.from_numpy(signals(B, T, seed=41)).cuda()
    g = torch.rand((B, T, NBB), generator=torch.Generator().manual_seed(4)).cuda()
    go = torch.randn((B, T, F), generator=torch.Generator().manual_seed(5)).cuda()
    grads = []
    for window in (True, False):
        steps = [("a", 0, T), ("s", 0, T)] if window else schedule(T, np.random.default_rng(3))
        out, _, _, ctx = run(nb.DenoiseBatch(B), steps, xd, g.transpose(0, 1), window=window)
        gl = g.clone().requires_grad_(True)
        synthesis_grad(gl, out.transpose(0, 1).contiguous(), ctx).backward(go)
        grads.append(gl.grad)
    assert np.array_equal(bits(grads[0]), bits(grads[1]))
    assert float(grads[0].abs().max()) > 0


class BiGRUGains:
    """A bidirectional GRU over a whole window of features [B][T][42] -> gains [B][T][22]: a non-causal model."""

    def __init__(self, seed):
        import torch
        torch.manual_seed(seed)
        self.gru = torch.nn.GRU(NBF, 32, batch_first=True, bidirectional=True).cuda()
        self.out = torch.nn.Linear(64, NBB).cuda()

    def parameters(self):
        return list(self.gru.parameters()) + list(self.out.parameters())

    def __call__(self, f):
        import torch
        h, _ = self.gru(f / 10.0)
        return torch.sigmoid(self.out(h))


def train_step(b, net, xd, clean):
    """One whole window: analyze_window -> net -> synthesize_window -> synthesis_grad, MSE of the output against the
    clean signal one frame later, backward."""
    import torch
    from nnnoiseless_b200.autograd import synthesis_grad
    T, B = xd.shape[0], xd.shape[1]
    b.reset()
    feats = torch.empty((B, T, NBF), device="cuda")
    out = torch.empty((B, T, F), device="cuda")
    ctx = torch.empty((B, T, CB), dtype=torch.uint8, device="cuda")
    b.analyze_window_device(xd.data_ptr(), feats.data_ptr(), 0, T, F, B * F, T * NBF, NBF, ctx.data_ptr(), T, 1)
    gains = net(feats)
    gd = gains.detach().contiguous()
    b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1)
    y = synthesis_grad(gains, out, ctx)
    loss = ((y[:, 1:] - clean[:, :-1]) * (1.0 / 32768.0)).pow(2).mean()
    loss.backward()
    return float(loss)


@pytest.mark.gpu
def test_bidirectional_gru_trained_over_whole_windows():
    import torch
    B, T = 16, 32
    clean, noisy = noisy_clean(B, T, 13)
    xd = torch.from_numpy(np.ascontiguousarray(noisy.transpose(1, 0, 2))).cuda()
    cl = torch.from_numpy(clean).cuda()
    b = nb.DenoiseBatch(B)
    net = BiGRUGains(2)
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    losses = []
    for _ in range(40):
        opt.zero_grad()
        losses.append(train_step(b, net, xd, cl))
        opt.step()
    print("\nbidirectional GRU over whole windows: waveform MSE %.4g -> %.4g (40 Adam steps)" % (losses[0], losses[-1]))
    assert np.mean(losses[-3:]) < 0.9 * np.mean(losses[:3])


# ---- 6. refusals change nothing ---------------------------------------------------------------------------------------------
def _rc(rc):
    if rc != 0:
        raise nb.NnnoiselessError(nb.last_error())


def refused_calls(b, B):
    """Every call refused with split frames pending (test_split_frames), by name."""
    import torch
    res = nb.Resampler(B, 16000)
    fr = torch.empty((B, F), device="cuda")
    fr16 = torch.zeros((B, F), dtype=torch.int16, device="cuda")
    vad = torch.empty(B, device="cuda")
    h = np.zeros((1, B, F), np.float32)
    L = nb.lib()
    rec = nb.DenoiseBatch(B).get_states()
    return res, {
        "process_device": lambda: b.process_device(fr.data_ptr(), fr.data_ptr(), 0, 1, F, B * F),
        "process_device_pcm16": lambda: b.process_device(fr16.data_ptr(), fr16.data_ptr(), 0, 1, F, B * F, pcm16=True),
        "process_device_strided": lambda: _rc(L.rnnoise_batch_process_device_strided(b._h, fr.data_ptr(), fr.data_ptr(), 0, None, 1, F, 1,
                                                                                      B * F, None)),
        "process_host": lambda: b.process_host(h),
        "process_pcm16_host": lambda: b.process_pcm16_host(h.astype(np.int16)),
        "process_streams_device": lambda: b.process_streams_device([0, 2], fr.data_ptr(), fr.data_ptr(), 0, 1, F, 2 * F),
        "process_streams_host": lambda: b.process_streams_host([1], h[:, :1]),
        "process_native_device": lambda: b.process_native_device(res, fr.data_ptr(), fr.data_ptr(), 0, 1, F, B * F),
        "process_native_host": lambda: b.process_native_host(res, h),
        "get_states": lambda: b.get_states(),
        "set_states": lambda: b.set_states(rec),
        "reset_streams": lambda: b.reset_streams([0]),
        "set_stream_models": lambda: b.set_stream_models([0], [0]),
        "profile_step": lambda: b.profile_step(fr.data_ptr(), fr.data_ptr(), vad.data_ptr(), F),
        "taps": lambda: b.taps(),
        "rnn_taps": lambda: b.rnn_taps(),
        "spectral_taps": lambda: b.spectral_taps(),
    }


@pytest.mark.gpu
def test_refusals_change_nothing():
    import torch
    B, T = 9, 23
    x = signals(B, T, seed=29)
    xd = torch.from_numpy(x).cuda()
    gains = rand_gains(T, B, 8)
    steps = [("a", 0, 5), ("a", 5, 13), ("s", 0, 3), ("a", 18, 5), ("s", 3, 17), ("s", 20, 3)]
    t_out, t_f, t_s, t_ctx = run(nb.DenoiseBatch(B), steps, xd, gains, window=True)
    b = nb.DenoiseBatch(B)
    res, refused = refused_calls(b, B)
    res_rec = res.get_states()
    out = torch.empty_like(xd)
    feats = torch.empty((T, B, NBF), device="cuda")
    ctx = new_ctx(B, T)
    fb = torch.empty((T, B, NBF), device="cuda")
    for kind, t, k in steps:
        cp = ctx[:, t].data_ptr()
        if kind == "a":
            b.analyze_window_device(xd[t].data_ptr(), feats[t].data_ptr(), 0, k, F, B * F, NBF, B * NBF, cp, T, 1)
        else:
            b.synthesize_window_device(out[t].data_ptr(), gains[t].data_ptr(), k, F, B * F, NBB, B * NBB, cp, T, 1)
        w = b.window_frames
        if w == 0:
            continue
        for name, call in refused.items():
            with pytest.raises(nb.NnnoiselessError, match="%d window frame\\(s\\) owed" % w):
                call()
        # split frames are refused while window frames are owed
        for call in (lambda: b.analyze_device(xd[0].data_ptr(), fb.data_ptr(), 0, 1, F, B * F, NBF, B * NBF),
                     lambda: b.synthesize_device(out[0].data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB),
                     lambda: b.synthesize_saving_device(out[0].data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB, cp, T, 1)):
            with pytest.raises(nb.NnnoiselessError, match="window frame\\(s\\) owed"):
                call()
        with pytest.raises(nb.NnnoiselessError, match="with %d owed" % w):
            b.synthesize_window_device(out[0].data_ptr(), gains.data_ptr(), w + 1, F, B * F, NBB, B * NBB, cp, T, 1)
        a_args = lambda **kw: dict(dict(in_ptr=xd[0].data_ptr(), features_ptr=fb.data_ptr(), silence_ptr=0, n_frames=1, stream_stride=F,  # noqa: E731
                                        frame_stride=B * F, feature_stream_stride=NBF, feature_frame_stride=B * NBF, ctx_ptr=cp,
                                        ctx_stream_stride=T, ctx_frame_stride=1), **kw)
        s_args = lambda **kw: dict(dict(out_ptr=out[0].data_ptr(), gains_ptr=gains.data_ptr(), n_frames=1, stream_stride=F,  # noqa: E731
                                        frame_stride=B * F, gain_stream_stride=NBB, gain_frame_stride=B * NBB, ctx_ptr=cp,
                                        ctx_stream_stride=T, ctx_frame_stride=1), **kw)
        bad = [dict(pcm16=2), dict(in_ptr=0), dict(features_ptr=0), dict(ctx_ptr=0), dict(ctx_ptr=cp + 8), dict(sample_stride=0),
               dict(n_frames=-1), dict(ctx_stream_stride=0), dict(n_frames=2, ctx_frame_stride=0)]
        for kw in bad:
            with pytest.raises(nb.NnnoiselessError):
                b.analyze_window_device(**a_args(**kw))
            skw = {{"in_ptr": "out_ptr", "features_ptr": "gains_ptr"}.get(k, k): v for k, v in kw.items()}
            with pytest.raises(nb.NnnoiselessError):
                b.synthesize_window_device(**s_args(**skw))
        b.analyze_window_device(**a_args(n_frames=0))  # n_frames 0: a no-op
        b.synthesize_window_device(**s_args(n_frames=0))
        assert b.window_frames == w and b.pending_frames == 0
    assert np.array_equal(res.get_states(), res_rec)
    torch.cuda.synchronize()
    assert np.array_equal(bits(out), bits(t_out)) and np.array_equal(bits(feats), bits(t_f))
    assert np.array_equal(ctx.cpu().numpy(), t_ctx.cpu().numpy())
    t_rec = nb.DenoiseBatch(B)
    run(t_rec, steps, xd, gains, window=True)
    assert np.array_equal(b.get_states(), t_rec.get_states())
    # window calls are refused while split frames are pending
    b.analyze_device(xd[0].data_ptr(), fb.data_ptr(), 0, 2, F, B * F, NBF, B * NBF)
    for call in (lambda: b.analyze_window_device(xd[0].data_ptr(), fb.data_ptr(), 0, 1, F, B * F, NBF, B * NBF, ctx.data_ptr(), T, 1),
                 lambda: b.synthesize_window_device(out.data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB, ctx.data_ptr(), T, 1)):
        with pytest.raises(nb.NnnoiselessError, match="2 split frame\\(s\\) pending"):
            call()
    assert b.pending_frames == 2 and b.window_frames == 0
    # reset drops owed frames: the batch then gives a fresh batch's bits, and fused frames again describe the taps
    b.reset()
    b.analyze_window_device(xd[0].data_ptr(), fb.data_ptr(), 0, 7, F, B * F, NBF, B * NBF, ctx.data_ptr(), T, 1)
    assert b.window_frames == 7
    b.reset()
    assert b.window_frames == 0 and b.pending_frames == 0
    o1, o2 = torch.empty_like(xd), torch.empty_like(xd)
    b.process_device(o1.data_ptr(), xd.data_ptr(), 0, T, F, B * F)
    nb.DenoiseBatch(B).process_device(o2.data_ptr(), xd.data_ptr(), 0, T, F, B * F)
    assert np.array_equal(bits(o1), bits(o2))
    b.taps()


# ---- 7. without a GPU: the C++ mirror and null batches ----------------------------------------------------------------------
def test_cpp_mirror_window_methods_compile(tmp_path):
    """nnnoiseless.hpp's DenoiseBatch::window_frames / analyze_window / synthesize_window compile and link."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    inc, libdir = os.path.join(root, "include"), os.path.join(root, "nnnoiseless_b200", "lib")
    src = tmp_path / "t.cpp"
    src.write_text('#include "nnnoiseless.hpp"\n'
                   "void window(nnnoiseless::DenoiseBatch& b, const float* in, float* out, float* feats, const float* gains, void* ctx,\n"
                   "            int T, void* stream) {\n"
                   "    const long B = b.streams();\n"
                   "    b.analyze_window(in, 0, feats, nullptr, T, 480, 1, B * 480, 42, B * 42, ctx, T, 1, stream);\n"
                   "    if (b.window_frames() == T)\n"
                   "        b.synthesize_window(out, 0, gains, T, 480, 1, B * 480, 22, B * 22, ctx, T, 1, stream);\n"
                   "}\n"
                   "int main(int argc, char**) {\n"
                   "    if (argc > 1) { nnnoiseless::DenoiseBatch b(1); window(b, nullptr, nullptr, nullptr, nullptr, nullptr, 1, nullptr); }\n"
                   "    return 0;\n"
                   "}\n")
    exe = tmp_path / "t"
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", inc, str(src), "-o", str(exe), "-L", libdir, "-lnnnoiseless_b200",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0


def test_null_batch_refused_without_device():
    L = nb.lib()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    assert L.rnnoise_batch_window_frames(None) == 0
    assert L.rnnoise_batch_analyze_window_device(None, p, 0, p, None, 1, F, 1, F, NBF, NBF, p, 1, 1, None) != 0
    assert "null batch" in nb.last_error()
    assert L.rnnoise_batch_synthesize_window_device(None, p, 0, p, 1, F, 1, F, NBB, NBB, p, 1, 1, None) != 0
    assert "null batch" in nb.last_error()
