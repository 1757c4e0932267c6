"""GPU tests of split frames (rnnoise_batch_analyze_device / _synthesize_device): the caller's own network between
analysis and synthesis.

- A split frame fed the batch's own raw gains gives the bits of a fused frame: features, silence flags, output and every
  field of the state record but the GRU state, which split frames leave alone.  Any schedule of analyze / synthesize
  chunks with up to 4 frames pending, three models and kernels, batch sizes around the 64-stream tile.
- Every buffer layout gives the same bits: features and gains seq-first or batch-first, int16 samples, interleaved stereo.
- Caller gains are used as given: lastg = max(g, 0.6 lastg) bit for bit, and output and synthesis memory agree with the
  oracle's synthesis statements within the K5 bounds of test_spectral_kernels.
- A float32 torch restatement of the built-in network on a torch stream between the calls meets the reference's golden
  metric on testing.raw, with the same bits as the same loop through synchronous calls.
- Calls that would run between a pending frame's analysis and synthesis, and bad arguments, are refused with no effect.
"""
import contextlib
import os

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle
import rnn_ref
from conftest import golden_metric, synth_streams

F, NBF, NBB = 480, 42, 22
MAXP = 4  # RNNOISE_MAX_PENDING_FRAMES


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def bits(a):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else a
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype.itemsize == 4 else np.uint16)


def signals(B, T, seed):
    """[T][B][480] float32 PCM-valued frames; streams 1 (mod 5) are all zero, 2 (mod 5) near-silent noise, 3 (mod 5) go
    digitally silent for frames 4..6, and a batch's only stream starts with 5 silent frames: silent frames and streams
    leaving silence occur."""
    x = synth_streams(B, T, seed=seed).reshape(B, T, F)
    g = np.random.default_rng(seed)
    if B == 1:
        x[0, :5] = 0.0
    for s in range(B if B > 1 else 0):
        kind = s % 5
        if kind == 1:
            x[s] = 0.0
        elif kind == 2:
            x[s] = np.round(g.normal(0.0, 0.3, (T, F)))
        elif kind == 3:
            x[s, 4:7] = 0.0
    return np.ascontiguousarray(x.transpose(1, 0, 2))


def make_batch(B, model_bytes, mma):
    with env(NNB_RNN_MMA="1" if mma else "0"):
        return nb.DenoiseBatch(B, nb.RnnModel.from_bytes(model_bytes) if model_bytes else None)


def gru_slice(batch):
    return slice(9664, 9664 + 4 * sum(batch.gru_widths))


def twin_frames(batch, xd, spectral=False):
    """Fused frames one at a time on a twin: (out [T][B][480], per-frame dicts of taps)."""
    import torch
    T, B = xd.shape[0], xd.shape[1]
    out = torch.empty_like(xd)
    pcm16 = xd.dtype == torch.int16
    frames = []
    for t in range(T):
        batch.process_device(out[t].data_ptr(), xd[t].data_ptr(), 0, 1, F, B * F, pcm16=pcm16)
        fr = dict(batch.taps())
        fr["raw_gains"] = batch.rnn_taps()["gains"]
        if spectral:
            fr.update(batch.spectral_taps())
        frames.append(fr)
    return out, frames


def schedule(T, rng):
    """A random schedule of ("a" | "s", first frame, frames) with at most MAXP frames pending."""
    ta = ts = 0
    steps = []
    while ts < T:
        can = min(MAXP - (ta - ts), T - ta)
        if can > 0 and (ta == ts or rng.random() < 0.5):
            k = int(rng.integers(1, can + 1))
            steps.append(("a", ta, k))
            ta += k
        else:
            k = int(rng.integers(1, ta - ts + 1))
            steps.append(("s", ts, k))
            ts += k
    return steps


def run_split(batch, steps, xd, out, feats, sil, gains, batch_first=False, sample_stride=1, stream_stride=F, frame_stride=None,
              pcm16=0, cuda_stream=0, t0=0):
    """Runs `steps` (frame numbers relative to t0).  xd / out: frame t at element offset t * frame_stride of the flat
    buffers; feats / gains [T][B][.] or (batch_first) [B][T][.]."""
    B = batch.n_streams
    fs = frame_stride if frame_stride is not None else B * F
    xflat, oflat = xd.reshape(-1), out.reshape(-1)
    for kind, t, k in steps:
        t += t0
        if batch_first:
            fp, fss, ffs = feats[:, t].data_ptr(), feats.stride(0), feats.stride(1)
            gp, gss, gfs = gains[:, t].data_ptr(), gains.stride(0), gains.stride(1)
        else:
            fp, fss, ffs = feats[t].data_ptr(), feats.stride(1), feats.stride(0)
            gp, gss, gfs = gains[t].data_ptr(), gains.stride(1), gains.stride(0)
        before = batch.pending_frames
        if kind == "a":
            batch.analyze_device(xflat[t * fs:].data_ptr(), fp, sil[t].data_ptr() if sil is not None else 0, k, stream_stride, fs, fss,
                                 ffs, sample_stride=sample_stride, pcm16=pcm16, cuda_stream=cuda_stream)
            assert batch.pending_frames == before + k
        else:
            batch.synthesize_device(oflat[t * fs:].data_ptr(), gp, k, stream_stride, fs, gss, gfs, sample_stride=sample_stride,
                                    pcm16=pcm16, cuda_stream=cuda_stream)
            assert batch.pending_frames == before - k


# ---- 1. split == fused, bit for bit ---------------------------------------------------------------------------------
KERNELS = {"builtin": (None, False), "sh": ("sh", False), "builtin-mma": (None, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 63, 64, 65, 229])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_split_equals_fused_bitwise(kernel, B, sh_bytes):
    import torch
    name, mma = KERNELS[kernel]
    model = sh_bytes if name == "sh" else None
    T0, T = 3, 17
    x = signals(B, T, seed=100 + B)
    xd = torch.from_numpy(x).cuda()
    twin, sp = make_batch(B, model, mma), make_batch(B, model, mma)
    tout, tfr = twin_frames(twin, xd)
    assert any(fr["silence"].any() for fr in tfr) and any((~fr["silence"].astype(bool)).any() for fr in tfr)

    out = torch.empty_like(xd)
    sp.process_device(out.data_ptr(), xd.data_ptr(), 0, T0, F, B * F)  # fused frames first: a GRU state to keep
    rec0 = sp.get_states()
    feats = torch.full((T, B, NBF), float("nan"), device="cuda")
    sil = torch.full((T, B), -1, dtype=torch.int32, device="cuda")
    gains = torch.from_numpy(np.stack([fr["raw_gains"] for fr in tfr])).cuda()
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        run_split(sp, schedule(T - T0, np.random.default_rng(B)), xd, out, feats, sil, gains, cuda_stream=st.cuda_stream, t0=T0)
    st.synchronize()
    assert sp.pending_frames == 0
    for t in range(T0, T):
        assert np.array_equal(bits(feats[t]), bits(tfr[t]["features"])), t
        assert np.array_equal(sil[t].cpu().numpy(), tfr[t]["silence"]), t
    assert np.array_equal(bits(out), bits(tout))
    r_sp, r_tw = sp.get_states(), twin.get_states()
    g = gru_slice(sp)
    keep = np.ones(r_sp.shape[1], bool)
    keep[g] = False
    assert np.array_equal(r_sp[:, keep], r_tw[:, keep])
    assert np.array_equal(r_sp[:, g], rec0[:, g])
    with pytest.raises(nb.NnnoiselessError, match="split frame"):
        sp.taps()


# ---- 2. layouts -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_layouts_bitwise():
    import torch
    B, T = 65, 10
    x = signals(B, T, seed=7)
    xd = torch.from_numpy(x).cuda()
    twin = make_batch(B, None, False)
    _, tfr = twin_frames(twin, xd)
    g_tb = torch.from_numpy(np.stack([fr["raw_gains"] for fr in tfr])).cuda()  # [T][B][22]
    steps = schedule(T, np.random.default_rng(1))

    def split(**kw):
        b = make_batch(B, None, False)
        feats = kw.pop("feats", torch.empty((T, B, NBF), device="cuda"))
        out = kw.pop("out", torch.empty_like(xd))
        run_split(b, steps, kw.pop("xd", xd), out, feats, kw.pop("sil", None), kw.pop("gains", g_tb), **kw)
        return out, feats, b.get_states()

    ref_out, ref_f, ref_rec = split()
    for t in range(T):
        assert np.array_equal(bits(ref_f[t]), bits(tfr[t]["features"]))
    # batch-first features and gains
    o, f, r = split(feats=torch.empty((B, T, NBF), device="cuda"), gains=g_tb.transpose(0, 1).contiguous(), batch_first=True)
    assert np.array_equal(bits(o), bits(ref_out)) and np.array_equal(bits(f.transpose(0, 1)), bits(ref_f)) and np.array_equal(r, ref_rec)
    # int16 in and out: the twin's pcm16 fused call
    x16 = torch.from_numpy(x.astype(np.int16)).cuda()
    twin16 = make_batch(B, None, False)
    t16, fr16 = twin_frames(twin16, x16)
    g16 = torch.from_numpy(np.stack([fr["raw_gains"] for fr in fr16])).cuda()
    o, f, r = split(xd=x16, out=torch.empty_like(x16), gains=g16, pcm16=1)
    assert np.array_equal(bits(o), bits(t16)) and np.array_equal(bits(f), bits(ref_f))
    r16, g = twin16.get_states(), gru_slice(twin16)
    assert np.array_equal(r[:, :g.start], r16[:, :g.start]) and np.array_equal(r[:, g.stop:], r16[:, g.stop:])
    # interleaved stereo: streams 2c, 2c + 1 of a frame interleaved; the same bits as the compact call on those streams
    Bs = 2
    xs = torch.from_numpy(np.ascontiguousarray(x[:, :Bs].transpose(0, 2, 1))).cuda()  # [T][480][2]
    b2 = make_batch(Bs, None, False)
    outs = torch.empty_like(xs)
    fs2 = torch.empty((T, Bs, NBF), device="cuda")
    run_split(b2, steps, xs, outs, fs2, None, g_tb[:, :Bs].contiguous(), sample_stride=Bs, stream_stride=1, frame_stride=F * Bs)
    bc = make_batch(Bs, None, False)
    outc = torch.empty((T, Bs, F), device="cuda")
    fc = torch.empty((T, Bs, NBF), device="cuda")
    run_split(bc, steps, xd[:, :Bs].contiguous(), outc, fc, None, g_tb[:, :Bs].contiguous())
    assert np.array_equal(bits(outs.permute(0, 2, 1)), bits(outc)) and np.array_equal(bits(fs2), bits(fc))
    assert np.array_equal(b2.get_states(), bc.get_states())


# ---- 3. caller gains are honoured -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_caller_gains_honoured(builtin_bytes):
    import torch
    import test_spectral_kernels as tsk
    B, T = 40, 12
    x = signals(B, T, seed=3)
    xd = torch.from_numpy(x).cuda()
    twin = make_batch(B, None, False)
    _, tfr = twin_frames(twin, xd, spectral=True)
    b = make_batch(B, None, False)
    dt = nb.state_dtype(b.gru_widths)
    rng = np.random.default_rng(5)
    out = torch.empty_like(xd)
    feats = torch.empty((T, B, NBF), device="cuda")
    sil = torch.empty((T, B), dtype=torch.int32, device="cuda")
    ws, cov = tsk.Worst(), tsk.new_coverage()
    kinds = ["uniform", "zeros", "ones", "exp", "below_floor"]
    prev = b.get_states()
    for t in range(T):
        rb = prev.view(dt).reshape(-1)
        kind = kinds[t % len(kinds)]
        g = {"uniform": lambda: rng.random((B, NBB)), "zeros": lambda: np.zeros((B, NBB)), "ones": lambda: np.ones((B, NBB)),
             "exp": lambda: tfr[t]["exp"], "below_floor": lambda: 0.5 * 0.6 * rb["lastg"]}[kind]().astype(np.float32)
        gd = torch.from_numpy(g).cuda()
        b.analyze_device(xd[t].data_ptr(), feats[t].data_ptr(), sil[t].data_ptr(), 1, F, B * F, NBF, B * NBF)
        b.synthesize_device(out[t].data_ptr(), gd.data_ptr(), 1, F, B * F, NBB, B * NBB)
        rec = b.get_states()
        ra = rec.view(dt).reshape(-1)
        s = sil[t].cpu().numpy() != 0
        assert np.array_equal(s, tfr[t]["silence"] != 0)
        floor = np.maximum(g, np.float32(0.6) * rb["lastg"])
        want = np.where(s[:, None], rb["lastg"], floor)
        assert np.array_equal(ra["lastg"].view(np.uint32), want.view(np.uint32)), (t, kind)
        fr = dict(rb=rb, ra=ra, silence=s.astype(np.int32), X=tfr[t]["X"], P=tfr[t]["P"], ex=tfr[t]["ex"], ep=tfr[t]["ep"],
                  exp=tfr[t]["exp"], gains=g, out=out[t].cpu().numpy(), vad_out=np.zeros(B, np.float32))
        tsk.check_synthesis(fr, ws, cov)
        prev = rec
    assert cov["floor"] and cov["branch_r1"] and cov["branch_ratio"]
    print("\ncaller gains K5: %s" % ws.line())


# ---- 4. a PyTorch network in the loop -------------------------------------------------------------------------------
class TorchDenoiseNet:
    """The reference's network (src/rnn.rs:343-379) in float32 torch on the GPU: weights int8 / 256, tansig from the
    oracle's table with the reference's second-order correction (rnn_ref.tansig)."""

    def __init__(self, model_bytes):
        import torch
        self.torch = torch
        self.table = torch.from_numpy(oracle.tansig_table()).cuda()
        self.layers = []
        for L in rnn_ref.parse(model_bytes):
            d = dict(nn=L["nn"], act=L["act"], w=torch.from_numpy((L["w"] / 256.0).astype(np.float32)).cuda(),
                     b=torch.from_numpy((L["b"] / 256.0).astype(np.float32)).cuda())
            if "r" in L:
                d["r"] = torch.from_numpy((L["r"] / 256.0).astype(np.float32)).cuda()
            self.layers.append(d)
        self.widths = tuple(self.layers[i]["nn"] for i in (1, 2, 3))

    def tansig(self, x):
        torch = self.torch
        ax = torch.clamp(x.abs(), max=8.0)
        fi = torch.floor(0.5 + 25.0 * ax)
        d = ax - 0.04 * fi
        y = self.table[fi.long()]
        y = y + d * (1.0 - y * y) * (1.0 - y * d)
        y = torch.where(x < 0.0, -y, y)
        y = torch.where(x > -8.0, y, torch.full_like(y, -1.0))
        return torch.where(x < 8.0, y, torch.ones_like(y))

    def act(self, a, x):
        if a == rnn_ref.TANH:
            return self.tansig(x)
        if a == rnn_ref.SIGMOID:
            return 0.5 + 0.5 * self.tansig(0.5 * x)
        return self.torch.relu(x)

    def dense(self, L, x):
        return self.act(L["act"], x @ L["w"] + L["b"])

    def gru(self, L, x, h):
        n, W, R, b = L["nn"], L["w"], L["r"], L["b"]
        z = self.act(rnn_ref.SIGMOID, x @ W[:, :n] + h @ R[:, :n] + b[:n])
        r = self.act(rnn_ref.SIGMOID, x @ W[:, n:2 * n] + h @ R[:, n:2 * n] + b[n:2 * n])
        c = self.act(L["act"], x @ W[:, 2 * n:] + (r * h) @ R[:, 2 * n:] + b[2 * n:])
        return z * h + (1.0 - z) * c

    def __call__(self, f, state, silent):
        """features [B][42], state [B][nv + nn + nd], silent [B] -> (gains [B][22], state); a silent frame keeps its
        state, as the reference skips the network on it."""
        torch = self.torch
        dense, vgru, ngru, dgru, out, _ = self.layers
        nv, nn_, _ = self.widths
        hv, hn, hd = state[:, :nv], state[:, nv:nv + nn_], state[:, nv + nn_:]
        d = self.dense(dense, f)
        hv = self.gru(vgru, d, hv)
        hn = self.gru(ngru, torch.cat([d, hv, f], 1), hn)
        hd = self.gru(dgru, torch.cat([hv, hn, f], 1), hd)
        new = torch.cat([hv, hn, hd], 1)
        return self.dense(out, hd), torch.where(silent[:, None], state, new)


def network_loop(net, b, xd, chunk, cuda_stream):
    """testing.raw through analyze -> net -> synthesize in chunks; on cuda_stream (no host synchronisation inside the
    loop), or (cuda_stream None) through synchronous calls with the network on the current stream."""
    torch = net.torch
    T, B = xd.shape[0], xd.shape[1]
    out = torch.empty_like(xd)
    feats = torch.empty((T, B, NBF), device="cuda")
    sil = torch.empty((T, B), dtype=torch.int32, device="cuda")
    gains = torch.empty((T, B, NBB), device="cuda")
    state = torch.zeros((B, sum(net.widths)), device="cuda")
    torch.cuda.synchronize()
    cs = cuda_stream.cuda_stream if cuda_stream is not None else 0
    with torch.cuda.stream(cuda_stream) if cuda_stream is not None else contextlib.nullcontext():
        for t0 in range(0, T, chunk):
            k = min(chunk, T - t0)
            b.analyze_device(xd[t0].data_ptr(), feats[t0].data_ptr(), sil[t0].data_ptr(), k, F, B * F, NBF, B * NBF, cuda_stream=cs)
            for t in range(t0, t0 + k):
                gains[t], state = net(feats[t], state, sil[t] != 0)
            if cuda_stream is None:
                torch.cuda.synchronize()
            b.synthesize_device(out[t0].data_ptr(), gains[t0].data_ptr(), k, F, B * F, NBB, B * NBB, cuda_stream=cs)
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
def test_torch_network_in_the_loop(builtin_bytes, testing_raw, reference_output):
    import torch
    net = TorchDenoiseNet(builtin_bytes)
    xd = torch.from_numpy(np.ascontiguousarray(testing_raw[:, None, :])).cuda()  # [T][1][480]
    out = network_loop(net, nb.DenoiseBatch(1), xd, MAXP, torch.cuda.Stream())
    o = out[:, 0].cpu().numpy()
    metric, maxdiff = golden_metric(list(o[1:]), reference_output)
    fused = torch.empty_like(xd)
    nb.DenoiseBatch(1).process_device(fused.data_ptr(), xd.data_ptr(), 0, xd.shape[0], F, F)
    dmax = float((out - fused).abs().max())
    print("\ntorch network in the loop: golden metric %.3g (max %d LSB), largest difference from the fused path %.3g" % (metric, maxdiff, dmax))
    assert metric < 1e-4
    # the same loop through synchronous calls, with lookahead-sized chunks of 3: the same bits
    out_sync = network_loop(net, nb.DenoiseBatch(1), xd, 3, None)
    assert np.array_equal(bits(out_sync), bits(out))


# ---- 5. refusals change nothing -------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_change_nothing():
    import torch
    B, T = 9, 8
    x = signals(B, T, seed=11)
    xd = torch.from_numpy(x).cuda()
    twin, b = make_batch(B, None, False), make_batch(B, None, False)
    steps = [("a", 0, 3), ("s", 0, 2), ("a", 3, 3), ("s", 2, 4), ("a", 6, 2), ("s", 6, 2)]
    gains = torch.rand((T, B, NBB), generator=torch.Generator().manual_seed(0)).cuda()
    outs = []
    for bb in (twin, b):
        o = torch.empty_like(xd)
        outs.append(o)
        f = torch.empty((T, B, NBF), device="cuda")
        if bb is twin:
            run_split(bb, steps, xd, o, f, None, gains)
            continue
        rec = b.get_states()
        res = nb.Resampler(B, 16000)
        fr = torch.empty((B, F), device="cuda")
        fr16 = torch.zeros((B, F), dtype=torch.int16, device="cuda")
        vad = torch.empty(B, device="cuda")
        h = np.zeros((1, B, F), np.float32)
        L = nb.lib()
        refused = {
            "process_device": lambda: b.process_device(fr.data_ptr(), fr.data_ptr(), 0, 1, F, B * F),
            "process_device_pcm16": lambda: b.process_device(fr16.data_ptr(), fr16.data_ptr(), 0, 1, F, B * F, pcm16=True),
            "process_device_strided": lambda: _rc(L.rnnoise_batch_process_device_strided(b._h, fr.data_ptr(), fr.data_ptr(), 0, None, 1, F,
                                                                                          1, B * F, None)),
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
        res_rec = res.get_states()
        for kind, t, k in steps:
            run_split(b, [(kind, t, k)], xd, o, f, None, gains)
            if b.pending_frames == 0:
                continue
            for name, call in refused.items():
                with pytest.raises(nb.NnnoiselessError, match="%d split frame\\(s\\) pending" % b.pending_frames):
                    call()
            p = b.pending_frames
            with pytest.raises(nb.NnnoiselessError, match="with %d pending" % p):
                b.analyze_device(xd[0].data_ptr(), f.data_ptr(), 0, MAXP - p + 1, F, B * F, NBF, B * NBF)
            with pytest.raises(nb.NnnoiselessError, match="with %d pending" % p):
                b.synthesize_device(o.data_ptr(), gains.data_ptr(), p + 1, F, B * F, NBB, B * NBB)
            bad = [
                lambda: b.analyze_device(xd[0].data_ptr(), f.data_ptr(), 0, 1, F, B * F, NBF, B * NBF, pcm16=2),
                lambda: b.analyze_device(0, f.data_ptr(), 0, 1, F, B * F, NBF, B * NBF),
                lambda: b.analyze_device(xd[0].data_ptr(), 0, 0, 1, F, B * F, NBF, B * NBF),
                lambda: b.analyze_device(xd[0].data_ptr(), f.data_ptr(), 0, 1, F, B * F, NBF, B * NBF, sample_stride=0),
                lambda: b.analyze_device(xd[0].data_ptr(), f.data_ptr(), 0, -1, F, B * F, NBF, B * NBF),
                lambda: b.synthesize_device(o.data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB, pcm16=-1),
                lambda: b.synthesize_device(0, gains.data_ptr(), 1, F, B * F, NBB, B * NBB),
                lambda: b.synthesize_device(o.data_ptr(), 0, 1, F, B * F, NBB, B * NBB),
                lambda: b.synthesize_device(o.data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB, sample_stride=0),
                lambda: b.synthesize_device(o.data_ptr(), gains.data_ptr(), -1, F, B * F, NBB, B * NBB),
            ]
            for call in bad:
                with pytest.raises(nb.NnnoiselessError):
                    call()
            b.analyze_device(xd[0].data_ptr(), f.data_ptr(), 0, 0, F, B * F, NBF, B * NBF)  # n_frames 0: a no-op
            b.synthesize_device(o.data_ptr(), gains.data_ptr(), 0, F, B * F, NBB, B * NBB)
            assert b.pending_frames == p
        assert np.array_equal(res.get_states(), res_rec)
    torch.cuda.synchronize()
    assert np.array_equal(bits(outs[1]), bits(outs[0]))
    assert np.array_equal(b.get_states(), twin.get_states())
    # reset drops the pending frames: the batch then gives a fresh batch's bits
    f = torch.empty((T, B, NBF), device="cuda")
    b.analyze_device(xd[0].data_ptr(), f.data_ptr(), 0, 2, F, B * F, NBF, B * NBF)
    b.reset()
    assert b.pending_frames == 0
    o1, o2 = torch.empty_like(xd), torch.empty_like(xd)
    b.process_device(o1.data_ptr(), xd.data_ptr(), 0, T, F, B * F)
    make_batch(B, None, False).process_device(o2.data_ptr(), xd.data_ptr(), 0, T, F, B * F)
    assert np.array_equal(bits(o1), bits(o2))
    b.taps()  # a fused frame again: taps describe it


def _rc(rc):
    if rc != 0:
        raise nb.NnnoiselessError(nb.last_error())


# ---- 6. the C++ mirror --------------------------------------------------------------------------------------------
def test_cpp_mirror_split_methods_compile(tmp_path):
    """nnnoiseless.hpp's DenoiseBatch::analyze / synthesize / pending_frames compile and link (runs without a GPU)."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    inc, libdir = os.path.join(root, "include"), os.path.join(root, "nnnoiseless_b200", "lib")
    src = tmp_path / "t.cpp"
    src.write_text('#include "nnnoiseless.hpp"\n'
                   "void step(nnnoiseless::DenoiseBatch& b, const float* in, float* out, float* feats, int* sil, const float* gains,\n"
                   "          void* stream) {\n"
                   "    const long B = b.streams();\n"
                   "    b.analyze(in, 0, feats, sil, RNNOISE_MAX_PENDING_FRAMES, 480, 1, B * 480, 42, B * 42, stream);\n"
                   "    if (b.pending_frames() == RNNOISE_MAX_PENDING_FRAMES)\n"
                   "        b.synthesize(out, 0, gains, RNNOISE_MAX_PENDING_FRAMES, 480, 1, B * 480, 22, B * 22, stream);\n"
                   "}\n"
                   "int main(int argc, char**) {\n"
                   "    if (argc > 1) { nnnoiseless::DenoiseBatch b(1); step(b, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr); }\n"
                   "    return 0;\n"
                   "}\n")
    exe = tmp_path / "t"
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", inc, str(src), "-o", str(exe), "-L", libdir, "-lnnnoiseless_b200",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0
