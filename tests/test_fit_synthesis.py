"""GPU tests of training the denoise network on device features (rnnoise_fit_forward_device / _backward_device,
nnnoiseless_b200.autograd.DenoiseNetwork; DESIGN.md §7l): against float64 autograd of the restatement
(tests/fit_synthesis_ref.py) with test_fit_kernels' tolerance scheme; byte identity with the rows path; carried state;
layouts and stream ordering; refusals; the fused path against the trained network; and a fine-tune through synthesis
whose exported model denoises a held-out corpus better on the fused path than the built-in model."""
import numpy as np
import pytest
import torch

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import NnnoiselessError, fit
from nnnoiseless_b200 import training as tr
from nnnoiseless_b200.autograd import DenoiseNetwork, synthesis_grad
from nnnoiseless_b200.synth import synth_streams
import fit_synthesis_ref as fsr
from test_fit_kernels import CASES, _check, _params
from test_training_pool import corpus  # noqa: F401  (the module-scoped WAV fixture)

pytestmark = pytest.mark.gpu
F, NBF, NBB = 480, 42, 22
MASKS = ("none", "random", "first", "last", "all")


def bits(x):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(x).view(np.uint32)


def _mask(kind, S, T, rng):
    m = np.zeros((S, T), bool)
    if kind == "random":
        m = rng.random((S, T)) < 0.2
    elif kind == "first":
        m[:, 0] = True
    elif kind == "last":
        m[:, -1] = True
    elif kind == "all":
        m[:] = True
    return m


class Run:
    """One fit handle driven through raw pointers with batch-first torch tensors."""

    def __init__(self, widths, S, T, params):
        self.f = fit.Fit(widths, S, T, device=0)
        self.S, self.T, self.nw = S, T, sum(widths[1:])
        self.params = torch.as_tensor(np.asarray(params, np.float32)).cuda()

    def forward(self, x, sil=None, state=None, n_seq=None, stream=0, sync=True):
        """x [S][T][42] and sil bool [S][T] (numpy or cuda) -> dict of cuda outputs; silence passed [T][S] as
        analyze_window_device writes it."""
        S = x.shape[0] if n_seq is None else n_seq
        x = torch.as_tensor(x, dtype=torch.float32).cuda()
        s = None if sil is None else torch.as_tensor(np.ascontiguousarray(np.asarray(sil).T), dtype=torch.int32).cuda()
        st = None if state is None else torch.as_tensor(state, dtype=torch.float32).cuda().contiguous()
        out = dict(gains=torch.full((S, self.T, NBB), float("nan"), device="cuda"), vad=torch.full((S, self.T), float("nan"), device="cuda"),
                   state=torch.full((S, self.nw), float("nan"), device="cuda"))
        if sync:
            torch.cuda.synchronize()
        self.f.forward_device(self.params.data_ptr(), S, x.data_ptr(), self.T * NBF, NBF, 0 if s is None else s.data_ptr(), 1, S,
                              0 if st is None else st.data_ptr(), out["state"].data_ptr(), out["gains"].data_ptr(), self.T * NBB, NBB,
                              out["vad"].data_ptr(), self.T, 1, stream)
        out["_keep"] = (x, s, st)
        return out

    def backward(self, gg, gv, stream=0):
        gg = torch.as_tensor(gg, dtype=torch.float32).cuda().contiguous()
        gv = None if gv is None else torch.as_tensor(gv, dtype=torch.float32).cuda().contiguous()
        grad = torch.full_like(self.params, float("nan"))
        self.f.backward_device(self.params.data_ptr(), gg.data_ptr(), gg.stride(0), NBB, 0 if gv is None else gv.data_ptr(), self.T, 1,
                               grad.data_ptr(), stream)
        return grad.cpu().numpy()


# ---- 1. against float64 autograd of the restatement --------------------------------------------------------------------------
@pytest.mark.parametrize("with_state", [False, True])
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("widths,S,T", CASES)
def test_against_float64(widths, S, T, mask, with_state):
    case = "%s S=%d T=%d mask=%s state=%s" % (",".join(map(str, widths)), S, T, mask, with_state)
    rng = np.random.default_rng(S * 1000 + T)
    x = (rng.standard_normal((S, T, NBF)) * 1.5).astype(np.float32)
    p = _params(widths, seed=T)
    sil = _mask(mask, S, T, rng)
    state = rng.uniform(-0.9, 0.9, (S, sum(widths[1:]))).astype(np.float32) if with_state else None
    gg = rng.standard_normal((S, T, NBB)).astype(np.float32)
    # vad_output.bias's gradient is one sum over every frame: with signed terms it can cancel to where that single
    # value's float32 restatement error is no measure of the rounding (seen at S = 3, T = 17), so grad_vad is positive
    gv = rng.uniform(0.0, 1.0, (S, T)).astype(np.float32)
    gg[sil] = np.nan  # ignored on silent frames
    gv[sil] = np.nan
    r = Run(widths, S, T, p)
    out = r.forward(x, sil if mask != "none" else None, state)
    grad = r.backward(gg, gv)
    act = r.f.activations(S)
    g0, v0 = np.where(sil[..., None], 0, gg), np.where(sil, 0, gv)
    fw64, g64 = fsr.forward_and_grad(p, widths, x, g0, v0, sil, state, torch.float64)
    fw32, g32 = fsr.forward_and_grad(p, widths, x, g0, v0, sil, state, torch.float32)
    _check("gains", out["gains"].cpu().numpy(), fw64["gains"], fw32["gains"], case)
    _check("vad", out["vad"].cpu().numpy(), fw64["vad"], fw32["vad"], case)
    _check("gru_state", act["state"], fw64["state"], fw32["state"], case)
    _check("state_out", out["state"].cpu().numpy(), fw64["state"][:, -1], fw32["state"][:, -1], case)
    assert (out["gains"].cpu().numpy()[sil] == 0).all() and (out["vad"].cpu().numpy()[sil] == 0).all()
    off = 0
    for layer, name, shape in fit.layer_shapes(widths):
        k = int(np.prod(shape))
        _check("grad %s.%s" % (layer, name), grad[off:off + k], g64[off:off + k], g32[off:off + k], case)
        off += k


# ---- 2. against the rows path, byte for byte ----------------------------------------------------------------------------------
@pytest.mark.parametrize("widths,S,T", [((24, 24, 48, 96), 5, 40), ((5, 3, 7, 11), 37, 9)])
def test_no_silent_frame_is_the_rows_path(widths, S, T):
    rng = np.random.default_rng(9)
    x = (rng.standard_normal((S, T, NBF)) * 1.5).astype(np.float32)
    rows = np.zeros((S, T, 87), np.float32)
    rows[..., :NBF] = x
    p = _params(widths, seed=2)
    r = Run(widths, S, T, p)
    r.f.set_params(p)
    r.f.evaluate(rows, np.ones((S, T), np.float32))
    ref = r.f.activations(S)
    for sil in (None, np.zeros((S, T), bool)):
        out = r.forward(x, sil)
        got = r.f.activations(S)
        for k in ("gains", "vad", "state"):
            assert np.array_equal(bits(got[k]), bits(ref[k])), k
        assert np.array_equal(bits(out["gains"]), bits(ref["gains"]))
        assert np.array_equal(bits(out["vad"]), bits(ref["vad"]))
        assert np.array_equal(bits(out["state"]), bits(ref["state"][:, -1]))


# ---- 3. two windows with the state carried are one window of twice the length -------------------------------------------------
def test_carried_state_is_one_long_window():
    widths, S, T = (24, 24, 48, 96), 7, 25
    rng = np.random.default_rng(4)
    x = (rng.standard_normal((S, 2 * T, NBF)) * 1.5).astype(np.float32)
    sil = rng.random((S, 2 * T)) < 0.2
    p = _params(widths, seed=4)
    one = Run(widths, S, 2 * T, p).forward(x, sil)
    half = Run(widths, S, T, p)
    a = half.forward(x[:, :T], sil[:, :T])
    b = half.forward(x[:, T:], sil[:, T:], a["state"])
    for k in ("gains", "vad"):
        assert np.array_equal(bits(torch.cat([a[k], b[k]], 1)), bits(one[k])), k
    assert np.array_equal(bits(b["state"]), bits(one["state"]))


# ---- 4. layouts, repeatability and stream ordering ----------------------------------------------------------------------------
def _network_run(net, x, sil, state, gg, gv, batch_first):
    net.params.grad = None
    gains, vad, st = net(x, sil, state, batch_first=batch_first)
    ((gains * gg).sum() + (vad * gv).sum()).backward()
    if not batch_first:
        gains, vad = gains.transpose(0, 1), vad.transpose(0, 1)
    return [bits(gains), bits(vad), bits(st), bits(net.params.grad)]


def test_layouts_repeat_and_streams():
    B, T = 6, 20
    net = DenoiseNetwork.from_model(None, B, T)
    rng = np.random.default_rng(8)
    x = torch.as_tensor(rng.standard_normal((B, T, NBF)) * 3, dtype=torch.float32).cuda()
    sil = torch.as_tensor(rng.random((T, B)) < 0.2, dtype=torch.int32).cuda()
    state = torch.as_tensor(rng.uniform(0, 0.5, (B, net.state_width)), dtype=torch.float32).cuda()
    gg = torch.as_tensor(rng.standard_normal((B, T, NBB)), dtype=torch.float32).cuda()
    gv = torch.as_tensor(rng.standard_normal((B, T)), dtype=torch.float32).cuda()
    ref = _network_run(net, x, sil, state, gg, gv, True)
    again = _network_run(net, x, sil, state, gg, gv, True)
    seq = _network_run(net, x.transpose(0, 1).contiguous(), sil, state, gg.transpose(0, 1), gv.transpose(0, 1), False)
    padded = torch.zeros(B, T + 3, 64, device="cuda")
    padded[:, :T, :NBF] = x
    sil_pad = torch.zeros(T, 2 * B, dtype=torch.int32, device="cuda")
    sil_pad[:, ::2] = sil
    pad = _network_run(net, padded[:, :T, :NBF], sil_pad[:, ::2], state, gg, gv, True)
    for got in (again, seq, pad):
        assert all(np.array_equal(a, b) for a, b in zip(got, ref))
    # a side stream, no host synchronisation between the calls
    st = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(st):
        for _ in range(3):
            xs = x * 1.0  # made on the side stream just before the call
            net.params.grad = None
            gains, vad, so = net(xs, sil, state)
            ((gains * gg).sum() + (vad * gv).sum()).backward()
            outs.append([gains.clone(), vad.clone(), so.clone(), net.params.grad.clone()])
    torch.cuda.synchronize()
    for o in outs:
        assert all(np.array_equal(bits(a), b) for a, b in zip(o, ref))


# ---- 5. refusals change nothing -----------------------------------------------------------------------------------------------
def test_refusals_change_nothing():
    widths, S, T = (24, 24, 48, 96), 4, 12
    rng = np.random.default_rng(12)
    x = (rng.standard_normal((S, T, NBF)) * 1.5).astype(np.float32)
    sil = rng.random((S, T)) < 0.2
    gg = rng.standard_normal((S, T, NBB)).astype(np.float32)
    gv = rng.standard_normal((S, T)).astype(np.float32)
    p = _params(widths, seed=12)
    fresh = Run(widths, S, T, p)
    want = fresh.forward(x, sil)
    want_grad = fresh.backward(gg, gv)

    r = Run(widths, S, T, p)
    with pytest.raises(NnnoiselessError, match="no forward_device"):
        r.backward(gg, gv)
    P, xd = r.params.data_ptr(), torch.as_tensor(x).cuda()
    out = torch.empty(S, T, NBB, device="cuda")
    v = torch.empty(S, T, device="cuda")
    calls = [  # (args of forward_device, error)
        ((P, S + 1, xd.data_ptr(), T * NBF, NBF, 0, 0, 0, 0, 0, out.data_ptr(), T * NBB, NBB, v.data_ptr(), T, 1), "n_seq"),
        ((0, S, xd.data_ptr(), T * NBF, NBF, 0, 0, 0, 0, 0, out.data_ptr(), T * NBB, NBB, v.data_ptr(), T, 1), "null"),
        ((P, S, 0, T * NBF, NBF, 0, 0, 0, 0, 0, out.data_ptr(), T * NBB, NBB, v.data_ptr(), T, 1), "null"),
        ((P, S, xd.data_ptr(), T * NBF, NBF, 0, 0, 0, 0, 0, 0, T * NBB, NBB, v.data_ptr(), T, 1), "null"),
        ((P, S, xd.data_ptr(), T * NBF, NBF, 0, 0, 0, 0, 0, out.data_ptr(), T * NBB, NBB, 0, T, 1), "null"),
        ((P, S, xd.data_ptr(), T * NBF, NBF, 0, 0, 0, 0, 0, out.data_ptr(), T * 21, 21, v.data_ptr(), T, 1), "overlap"),
        ((P, S, xd.data_ptr(), T * NBF, NBF, 0, 0, 0, 0, 0, out.data_ptr(), T * NBB, NBB, v.data_ptr(), 1, 1), "overlap"),
    ]
    got = r.forward(x, sil)
    for args, err in calls:
        with pytest.raises(NnnoiselessError, match=err):
            r.f.forward_device(*args)
    for k in ("gains", "vad", "state"):
        assert np.array_equal(bits(got[k]), bits(want[k])), k
    assert np.array_equal(bits(r.backward(gg, gv)), bits(want_grad))  # the refusals left the forward bound
    other = r.params.clone()
    with pytest.raises(NnnoiselessError, match="not the pointer"):
        r.f.backward_device(other.data_ptr(), torch.as_tensor(gg).cuda().data_ptr(), T * NBB, NBB, 0, 0, 0,
                            torch.empty_like(other).data_ptr())
    with pytest.raises(NnnoiselessError, match="overlaps params"):
        r.f.backward_device(P, torch.as_tensor(gg).cuda().data_ptr(), T * NBB, NBB, 0, 0, 0, P + 4)
    rows = np.zeros((S, T, 87), np.float32)
    rows[..., :NBF] = x
    r.f.set_params(p)
    r.f.step(rows, np.ones((S, T), np.float32))
    with pytest.raises(NnnoiselessError, match="rnnoise_fit_step"):
        r.backward(gg, gv)
    got = r.forward(x, sil)
    for k in ("gains", "vad", "state"):
        assert np.array_equal(bits(got[k]), bits(want[k])), k
    assert np.array_equal(bits(r.backward(gg, gv)), bits(want_grad))


def test_stale_forward_raises():
    B, T = 3, 10
    net = DenoiseNetwork(B, T, seed=1)
    x = torch.randn(B, T, NBF, device="cuda")
    gains, vad, _ = net(x)
    with torch.no_grad():
        net(x * 2)
    with pytest.raises(NnnoiselessError, match="overwritten by a later forward"):
        gains.sum().backward()
    gains, vad, _ = net(x)
    (gains.sum() + vad.sum()).backward()  # a fresh forward differentiates again
    assert torch.isfinite(net.params.grad).all()


# ---- 6. the fused path runs what was trained ----------------------------------------------------------------------------------
# The fused path evaluates the same int8 / 256 weights with table activations (tansig / sigmoid, as src/rnn.rs) and its
# GRUs on f16-split tensor cores; the trained network uses exact f32 activations.  Worst differences measured on an
# H100 over this clip: gains 9.6e-6, vad 1.8e-6, states 1.24e-4 (2.0e-5 on silent frames); the bounds are 4x those.
DEPLOY_TOL = dict(gains=4e-5, vad=8e-6, state=5e-4)


def _clip(B, T, seed):
    """Speech-like streams with silent stretches: [T][B][480]."""
    x = synth_streams(B, T, seed=seed).reshape(B, T, F).copy()
    x[:, 20:35] = 0.0
    x[1::2, 60:64] = 0.0
    return np.ascontiguousarray(x.transpose(1, 0, 2).astype(np.float32))


def _window_features(B, T, x):
    b = nb.DenoiseBatch(B, device=0)
    xd = torch.as_tensor(x).cuda()  # [T][B][480]
    feats = torch.empty(B, T, NBF, device="cuda")
    sil = torch.empty(T, B, dtype=torch.int32, device="cuda")
    ctx = torch.empty(B, T, nb.SYNTH_CONTEXT_BYTES, dtype=torch.uint8, device="cuda")
    b.analyze_window_device(xd.data_ptr(), feats.data_ptr(), sil.data_ptr(), T, F, B * F, T * NBF, NBF, ctx.data_ptr(), T, 1)
    torch.cuda.synchronize()
    return feats, sil


def test_deployed_equals_trained(builtin_bytes):
    B, T = 4, 100
    x = _clip(B, T, seed=31)
    feats, sil = _window_features(B, T, x)
    net = DenoiseNetwork.from_model(None, B, T)
    assert net.export() == builtin_bytes
    with torch.no_grad():
        gains, vad, _ = net(feats, sil)
    state = net._fit.activations(B)["state"]  # [B][T][nw], carried through silent frames
    gains, vad, silent = gains.cpu().numpy(), vad.cpu().numpy(), sil.cpu().numpy().T.astype(bool)
    assert silent.any() and (~silent).any()
    fused = nb.DenoiseBatch(B, device=0)
    worst = dict(gains=0.0, vad=0.0, state=0.0, state_silent=0.0)
    for t in range(T):
        fused.process_host(x[t:t + 1])
        taps = fused.rnn_taps()
        on = ~silent[:, t]
        worst["gains"] = max(worst["gains"], float(np.abs(taps["gains"][on] - gains[on, t]).max(initial=0)))
        worst["vad"] = max(worst["vad"], float(np.abs(taps["vad"][on] - vad[on, t]).max(initial=0)))
        d = np.abs(taps["gru_state"] - state[:, t]).max(axis=1)
        worst["state"] = max(worst["state"], float(d[on].max(initial=0)))
        worst["state_silent"] = max(worst["state_silent"], float(d[~on].max(initial=0)))
    print("\nfused path against the trained network, worst |difference|:", worst)
    assert worst["gains"] <= DEPLOY_TOL["gains"] and worst["vad"] <= DEPLOY_TOL["vad"]
    assert worst["state"] <= DEPLOY_TOL["state"] and worst["state_silent"] <= DEPLOY_TOL["state"]


# ---- 7. fine-tuning through synthesis lowers the fused path's waveform loss ---------------------------------------------------
def _corpus_windows(wc, B, T, n, seed):
    wc.start(B * T * n, seed=seed)
    out = []
    for _ in range(n):
        noisy, clean = torch.empty((B, T, F), device="cuda"), torch.empty((B, T, F), device="cuda")
        assert wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F) == T
        out.append((noisy, clean))
    return out


def _net_loss(b, net, noisy, clean, state, grad):
    """One window through analyze_window -> net -> synthesize_window: the MSE of output frame t + 1 against clean[t].
    -> (loss value, state_out)."""
    B, T = noisy.shape[0], noisy.shape[1]
    feats = torch.empty((B, T, NBF), device="cuda")
    sil = torch.empty((T, B), dtype=torch.int32, device="cuda")
    out = torch.empty((B, T, F), device="cuda")
    ctx = torch.empty((B, T, nb.SYNTH_CONTEXT_BYTES), dtype=torch.uint8, device="cuda")
    b.analyze_window_device(noisy.data_ptr(), feats.data_ptr(), sil.data_ptr(), T, T * F, F, T * NBF, NBF, ctx.data_ptr(), T, 1)
    with torch.set_grad_enabled(grad):
        g, _, state = net(feats, sil, state)
        gd = g.detach().contiguous()
        b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1)
        y = synthesis_grad(g, out, ctx) if grad else out
        loss = ((y[:, 1:] - clean[:, :-1]) * (1.0 / 32768.0)).pow(2).mean()
    if grad:
        loss.backward()
    return float(loss.detach()), state


def _fused_loss(model, wins):
    """The held-out windows, lane after lane, through a fused DenoiseBatch: the MSE of output frame t + 1 against
    clean[t] over every window."""
    B = wins[0][0].shape[0]
    b = nb.DenoiseBatch(B, model=model, device=0)
    total, n = 0.0, 0
    for noisy, clean in wins:
        T = noisy.shape[1]
        out = torch.empty_like(noisy)
        b.process_streams_device(None, out.data_ptr(), noisy.data_ptr(), 0, T, T * F, F, n=B)
        torch.cuda.synchronize()
        total += float((((out[:, 1:] - clean[:, :-1]) / 32768.0) ** 2).sum())
        n += out[:, 1:].numel()
    return total / n


def test_fine_tune_through_synthesis(corpus):  # noqa: F811
    sig_paths, noise_paths = corpus
    B, T, n_win, epochs = 16, 32, 6, 8
    wc = tr.WaveformCorpus(sig_paths, noise_paths, B)
    train = _corpus_windows(wc, B, T, n_win, seed=5)
    held = _corpus_windows(wc, B, T, 3, seed=77)
    net = DenoiseNetwork.from_model(None, B, T)
    opt = torch.optim.Adam([net.params], lr=1e-3)
    b = nb.DenoiseBatch(B, device=0)

    def held_loss():
        b.reset()
        state, total = None, 0.0
        for noisy, clean in held:
            loss, state = _net_loss(b, net, noisy, clean, state, grad=False)
            total += loss
        return total / len(held)

    before = held_loss()
    fused_before = _fused_loss(None, held)
    for _ in range(epochs):
        b.reset()  # the lanes' windows run in order, with the denoiser's and the network's states carried
        state = None
        for noisy, clean in train:
            opt.zero_grad()
            _, state = _net_loss(b, net, noisy, clean, state, grad=True)
            opt.step()
            net.clip_()
    after = held_loss()
    model = net.to_model()
    fused_after = _fused_loss(model, held)
    print("\nheld-out loss of the network %.5g -> %.5g; fused path's waveform MSE, built-in %.5g -> fine-tuned %.5g (%d Adam steps)"
          % (before, after, fused_before, fused_after, epochs * n_win))
    assert after < before
    assert fused_after < fused_before
    assert nb.RnnModel.from_bytes(model.to_bytes()) is not None
    mixed = nb.DenoiseBatch(4, device=0)
    assert mixed.add_model(model) == 1
    mixed.set_stream_models([1, 1], streams=[0, 2])
    x = synth_streams(4, 10, seed=7).reshape(4, 10, F).transpose(1, 0, 2).astype(np.float32)
    out, _ = mixed.process_host(np.ascontiguousarray(x))
    own, _ = nb.DenoiseBatch(4, model=model, device=0).process_host(np.ascontiguousarray(x))
    np.testing.assert_array_equal(out[:, [0, 2]], own[:, [0, 2]])
