"""GPU tests of training through synthesis (DESIGN.md 7i): rnnoise_batch_synthesize_saving_device and
rnnoise_synthesis_backward_device, and the torch wrapper nnnoiseless_b200.autograd.synthesis_grad.

- Saving changes nothing: output and state records equal those of synthesize_device fed the same gains, for batch sizes
  around the warp tiles and chunk schedules of 1 to 4 frames.  The records hold a fused twin's spectral taps bit for bit,
  lastg before the window, and lastg chained as max(g, 0.6f lastg).
- The backward agrees with the float64 restatement (synth_grad_ref) fed the GPU's own contexts, every element within
  its own first-order rounding bound (synth_grad_ref.grad_bounds), over gains at and around every kink, floored runs
  with silent frames inside, exp = 0 bands, random and structured grad_out; and on edge windows built on the CPU
  (test_synth_grad_ref.edge_window): g and exp within ulps of 1, exp == g and one ulp away, q at both clamp edges,
  ep = 0, ex = 0, a cancelling band, floor chains of 40+ frames, grad_out in one half, one band, DC-free or at
  Nyquist, odd shapes, T = 1 and T = 200.
- Same bits on repeated calls, through strided and seq-first layouts, and replayed from a CUDA graph.
- A network trained through analyze -> net -> saving synthesis -> synthesis_grad gets the parameter gradients of the same
  loop through the restatement, and a few dozen Adam steps lower a waveform MSE.
- Bad arguments are refused and change nothing.
"""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import synth_grad_ref as ref
from test_split_frames import bits, schedule, signals
from test_synth_grad_ref import EDGES, edge_window

F, NBF, NBB, CB = 480, 42, 22, nb.SYNTH_CONTEXT_BYTES


def analyze(b, xd, t0, k, feats):
    B = b.n_streams
    b.analyze_device(xd[t0].data_ptr(), feats[t0].data_ptr(), 0, k, F, B * F, NBF, B * NBF)


def run_saving(b, xd, gains, steps=None, saving=True):
    """Frames of xd [T][B][480] through analyze / (saving) synthesize on `steps` (default: chunks of 4).  gains
    [B][T][22] -> (out [B][T][480], ctx uint8 [B][T][CB] or None)."""
    import torch
    T, B = xd.shape[0], xd.shape[1]
    steps = steps or [(kind, t0, min(4, T - t0)) for t0 in range(0, T, 4) for kind in ("a", "s")]
    out = torch.empty((B, T, F), device="cuda")
    ctx = torch.empty((B, T, CB), dtype=torch.uint8, device="cuda") if saving else None
    feats = torch.empty((T, B, NBF), device="cuda")
    for kind, t, k in steps:
        if kind == "a":
            analyze(b, xd, t, k, feats)
        elif saving:
            b.synthesize_saving_device(out[:, t].data_ptr(), gains[:, t].data_ptr(), k, T * F, F, T * NBB, NBB, ctx[:, t].data_ptr(), T, 1)
        else:
            b.synthesize_device(out[:, t].data_ptr(), gains[:, t].data_ptr(), k, T * F, F, T * NBB, NBB)
    torch.cuda.synchronize()
    return out, ctx


# ---- 1. saving changes nothing; the records --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 63, 64, 65, 229])
def test_saving_changes_nothing(B):
    import torch
    T = 13
    x = signals(B, T, seed=300 + B)
    xd = torch.from_numpy(x).cuda()
    gains = torch.rand((B, T, NBB), generator=torch.Generator().manual_seed(B)).cuda()
    steps = schedule(T, np.random.default_rng(B))
    plain, saving = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    rec0 = saving.get_states()
    o1, _ = run_saving(plain, xd, gains, steps, saving=False)
    o2, ctx = run_saving(saving, xd, gains, steps)
    assert np.array_equal(bits(o1), bits(o2))
    assert np.array_equal(plain.get_states(), saving.get_states())
    # the records: a fused twin's spectral taps, the gains, lastg before the window and chained
    twin = nb.DenoiseBatch(B)
    d = ref.parse_ctx(ctx.cpu().numpy())
    tout = torch.empty_like(xd)
    for t in range(T):
        twin.process_device(tout[t].data_ptr(), xd[t].data_ptr(), 0, 1, F, B * F)
        tp = twin.spectral_taps()
        for k in ("ex", "ep", "exp"):
            assert np.array_equal(d[k][:, t].view(np.uint32), tp[k].view(np.uint32)), (k, t)
        assert np.array_equal(d["X"][:, t].astype(np.complex64).view(np.uint32), tp["X"].view(np.uint32)), t
        assert np.array_equal(d["P"][:, t].astype(np.complex64).view(np.uint32), tp["P"].view(np.uint32)), t
        assert np.array_equal(d["silence"][:, t], twin.taps()["silence"] != 0), t
    assert np.array_equal(d["g"].view(np.uint32), gains.cpu().numpy().view(np.uint32))
    r0 = rec0.view(nb.state_dtype(saving.gru_widths)).reshape(-1)
    assert np.array_equal(d["lastg"][:, 0].view(np.uint32), r0["lastg"].view(np.uint32))
    live = ~d["silence"][:, :-1, None]
    nxt = np.maximum(d["g"][:, :-1], np.float32(0.6) * d["lastg"][:, :-1])
    want = np.where(live, nxt, d["lastg"][:, :-1])
    assert np.array_equal(d["lastg"][:, 1:].view(np.uint32), want.view(np.uint32))
    assert d["silence"].any() or B == 1


# ---- 2. gradients against the float64 restatement -------------------------------------------------------------------
N_CASES = 8


def case_gains(B, T, d0, rng):
    """[B][T][22] f32 gains: case (s + t // 12) mod 8 of stream s at frame t -- 0 uniform, 1 near 0, 2 near 1, 3 exactly 1
    and above 1, 4 exp exactly and one ulp above, 5 0.6f lastg exactly, 6 decaying (the floor held for 11 frames), 7
    uniform with exp set to 0 in bands 3..6 (edited into the records).  lastg is chained on the host exactly as K5."""
    g = np.empty((B, T, NBB), np.float32)
    lastg = d0["lastg"][:, 0].copy()
    for t in range(T):
        for s in range(B):
            c = (s + t // 12) % N_CASES
            u = rng.random(NBB).astype(np.float32)
            e = d0["exp"][s, t]
            v = {0: u, 1: u * np.float32(1e-3), 2: np.float32(1) - u * np.float32(1e-3),
                 3: np.where(np.arange(NBB) % 2 == 0, np.float32(1), np.float32(1) + u / 2),
                 4: e if t % 2 == 0 else np.nextafter(e, np.float32(np.inf)),
                 5: np.where(lastg[s] > 0, np.float32(0.6) * lastg[s], u),
                 6: np.full(NBB, 0.9 * 0.35 ** (t % 12)),
                 7: u}[c]
            g[s, t] = np.asarray(v, np.float32)
        nxt = np.maximum(g[:, t], np.float32(0.6) * lastg)
        lastg = np.where(d0["silence"][:, t, None], lastg, nxt)
    return g


def window_case(B, T, seed):
    """(ctx tensor [B][T][CB] with the case-7 edits, grad_out [B][T][480] tensor, parsed records)."""
    import torch
    x = signals(B, T, seed)
    for s in range(B):  # silent frames inside the decaying runs
        for t in range(T):
            if (s + t // 12) % N_CASES == 6 and t % 12 in (4, 5, 6):
                x[t, s] = 0.0
    xd = torch.from_numpy(x).cuda()
    probe = torch.rand((B, T, NBB), generator=torch.Generator().manual_seed(seed)).cuda()
    _, ctx0 = run_saving(nb.DenoiseBatch(B), xd, probe)
    d0 = ref.parse_ctx(ctx0.cpu().numpy())
    g = torch.from_numpy(case_gains(B, T, d0, np.random.default_rng(seed))).cuda()
    out, ctx = run_saving(nb.DenoiseBatch(B), xd, g)
    c = ctx.cpu().numpy()
    cf = c.view(np.float32)
    for s in range(B):
        for t in range(T):
            if (s + t // 12) % N_CASES == 7:
                cf[s, t, 1812 + 3:1812 + 7] = 0.0  # exp of bands 3..6
    rng = np.random.default_rng(seed + 1)
    go = rng.normal(size=(B, T, F)).astype(np.float32)
    n = np.arange(F)
    for s in range(1, B, 3):  # structured: a tone
        go[s] = np.sin(2 * np.pi * (s + 1) * (n[None, :] + F * np.arange(T)[:, None]) / 960.0)
    for s in range(2, B, 3):  # structured: the output itself (the gradient of ||out||^2 / 2)
        go[s] = out[s].cpu().numpy() / 1e4
    return torch.from_numpy(c).cuda(), torch.from_numpy(go).cuda(), ref.parse_ctx(c)


def backward(ctx, go, batch_first=True, grad=None):
    import torch
    B, T = (ctx.shape[0], ctx.shape[1]) if batch_first else (ctx.shape[1], ctx.shape[0])
    grad = grad if grad is not None else torch.full((B, T, NBB) if batch_first else (T, B, NBB), float("nan"), device="cuda")
    ix = (0, 1) if batch_first else (1, 0)
    nbytes = nb.synthesis_backward_workspace_bytes(B, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    nb.synthesis_backward_device(ctx.data_ptr(), ctx.stride(ix[0]) // CB, ctx.stride(ix[1]) // CB, go.data_ptr(), go.stride(ix[0]),
                                 go.stride(ix[1]), grad.data_ptr(), grad.stride(ix[0]), grad.stride(ix[1]), B, T, ws.data_ptr(), nbytes)
    return grad


K_BOUND = 1.0  # grad_bounds bounds the rounding of any correct f32 evaluation to first order: no slack is needed


def check_against_ref(d, go, got):
    """Per element |got - ref64| <= K_BOUND grad_bounds (synth_grad_ref), with no window-relative floor: the only
    absolute floor is the smallest normal f32, for elements whose float64 value lies below it.  Where the float64 q lies
    within its rounding bound of 0 or 1 (masks' ambiguous) either side of the clamp is accepted, each with its own
    bound.  -> (the largest share of the bound used, where, g64)."""
    mk = ref.masks(d)
    g64 = ref.window_grad(d, go, mk=mk)

    def share(m, r64):
        bound = K_BOUND * ref.grad_bounds(d, go, mk=m)
        tol = np.maximum(bound, np.where(np.abs(r64) < ref.TINY, ref.TINY, 0.0))
        with np.errstate(all="ignore"):
            return np.where(got == r64, 0.0, np.abs(got - r64) / tol)

    sh = share(mk, g64)
    if mk["ambiguous"].any():
        alt = dict(mk)
        alt["live"] = mk["live"] ^ mk["ambiguous"]
        alt["one"] = mk["branch"] | (~alt["live"] & mk["ambiguous"] & (ref.q32(d["exp"], d["g"]) > 0.5)) | (mk["one"] & ~mk["ambiguous"])
        sh = np.minimum(sh, share(alt, ref.window_grad(d, go, mk=alt)))
    assert np.all(np.isfinite(got))
    worst = np.unravel_index(np.argmax(sh), sh.shape)
    assert sh[worst] <= 1.0, (worst, got[worst], g64[worst], sh[worst])
    return float(sh[worst]), worst, g64


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(1, 100), (63, 17), (64, 4), (65, 2), (229, 1), (229, 17)])
def test_gradients_against_reference(B, T):
    ctx, go, d = window_case(B, T, seed=B * 1000 + T)
    got = backward(ctx, go).cpu().numpy().astype(np.float64)
    share, worst, _ = check_against_ref(d, go.cpu().numpy().astype(np.float64), got)
    mk = ref.masks(d)
    print("\nB=%d T=%d: largest share of the bound %.3g at %s; floored %d, r = 1 branch %d, clamped %d, silent frames %d"
          % (B, T, share, worst, (~mk["take_g"]).sum(), mk["branch"].sum(), (~mk["live"] & ~mk["branch"]).sum(), d["silence"].sum()))
    if T >= 17 and B > 1:
        assert (~mk["take_g"]).any() and mk["branch"].any() and (~mk["live"] & ~mk["branch"]).any() and d["silence"].any()
        assert np.all(got[d["silence"]] == 0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", EDGES)
def test_edge_windows_against_reference(kind):
    """Records built on the CPU at the edges of the backward's arithmetic (test_synth_grad_ref.edge_window), each
    checked to reach its edge, then held to the bound element by element."""
    import torch
    d, go, reach = edge_window(kind)
    for name, m in reach.items():
        assert m.any(), (kind, name)
    c = ref.make_ctx(d["X"], d["P"], d["ex"], d["ep"], d["exp"], d["lastg"], d["g"], d["silence"])
    go32 = go.astype(np.float32)
    got = backward(torch.from_numpy(c).cuda(), torch.from_numpy(go32).cuda()).cpu().numpy().astype(np.float64)
    share, worst, g64 = check_against_ref(d, go32.astype(np.float64), got)
    print("\n%s (B=%d T=%d): largest share of the bound %.3g at %s" % (kind, d["g"].shape[0], d["g"].shape[1], share, worst))
    assert np.all(got[d["silence"]] == 0.0)
    if kind == "chain":  # carried gradients, far below the window's peak, were held to their own bound
        small = (np.abs(g64) > 0) & (np.abs(g64) < 1e-6 * np.abs(g64).max())
        assert small.sum() >= 20, small.sum()


# ---- 3. determinism, layouts, graph capture ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_determinism_and_layouts():
    import torch
    B, T = 65, 9
    ctx, go, _ = window_case(B, T, seed=77)
    a = backward(ctx, go)
    assert np.array_equal(bits(a), bits(backward(ctx, go)))
    # seq-first copies, and strided views of the batch-first buffers
    b = backward(ctx.transpose(0, 1).contiguous(), go.transpose(0, 1).contiguous(), batch_first=False)
    assert np.array_equal(bits(b.transpose(0, 1)), bits(a))
    wide = torch.zeros((B, T, 2 * NBB), device="cuda")
    backward(ctx.transpose(0, 1), go.transpose(0, 1), batch_first=False, grad=wide[:, :, :NBB].transpose(0, 1))
    assert np.array_equal(bits(wide[:, :, :NBB]), bits(a)) and not wide[:, :, NBB:].any()
    # captured in a CUDA graph (the caller's workspace, no allocation) and replayed
    out = torch.empty_like(a)
    nbytes = nb.synthesis_backward_workspace_bytes(B, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nb.synthesis_backward_device(ctx.data_ptr(), T, 1, go.data_ptr(), T * F, F, out.data_ptr(), T * NBB, NBB, B, T, ws.data_ptr(),
                                     nbytes, cuda_stream=torch.cuda.current_stream().cuda_stream)
    out.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(bits(out), bits(a))


# ---- 4. torch: a network trained through synthesis --------------------------------------------------------------------
def noisy_clean(B, T, seed):
    from nnnoiseless_b200.synth import synth_streams
    clean = synth_streams(B, T, seed=seed).reshape(B, T, F)
    noise = np.random.default_rng(seed).normal(0, 1500, clean.shape).astype(np.float32)
    return clean, np.round(clean + noise).astype(np.float32)


def train_window(b, net, xd, clean, use_ref=False):
    """One window: analyze -> net -> saving synthesis in chunks of 4, synthesis_grad, MSE of the output against the clean
    signal one frame later, backward.  use_ref: the float64 restatement computes dL/dgains instead of the kernel."""
    import torch
    from nnnoiseless_b200.autograd import synthesis_grad
    T, B = xd.shape[0], xd.shape[1]
    b.reset()
    feats = torch.empty((T, B, NBF), device="cuda")
    out = torch.empty((B, T, F), device="cuda")
    ctx = torch.empty((B, T, CB), dtype=torch.uint8, device="cuda")
    chunks = []
    for t0 in range(0, T, 4):
        k = min(4, T - t0)
        analyze(b, xd, t0, k, feats)
        g = net(feats[t0:t0 + k].transpose(0, 1) / 10.0)  # [B][k][22]
        gd = g.detach().contiguous()
        b.synthesize_saving_device(out[:, t0].data_ptr(), gd.data_ptr(), k, T * F, F, k * NBB, NBB, ctx[:, t0].data_ptr(), T, 1)
        chunks.append(g)
    gains = torch.cat(chunks, 1)
    scale = 1.0 / 32768.0
    if not use_ref:
        y = synthesis_grad(gains, out, ctx)
        loss = ((y[:, 1:] - clean[:, :-1]) * scale).pow(2).mean()
        loss.backward()
        return float(loss)
    y = out.clone().requires_grad_(True)
    loss = ((y[:, 1:] - clean[:, :-1]) * scale).pow(2).mean()
    loss.backward()
    d = ref.parse_ctx(ctx.cpu().numpy())
    gref = ref.window_grad(d, y.grad.double().cpu().numpy())
    gains.backward(torch.from_numpy(gref).float().cuda())
    return float(loss)


def small_net(seed):
    import torch
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(NBF, 32), torch.nn.Tanh(), torch.nn.Linear(32, NBB), torch.nn.Sigmoid()).cuda()


@pytest.mark.gpu
def test_torch_gradients_match_reference():
    import torch
    B, T = 12, 10
    clean, noisy = noisy_clean(B, T, 5)
    xd = torch.from_numpy(np.ascontiguousarray(noisy.transpose(1, 0, 2))).cuda()
    cl = torch.from_numpy(clean).cuda()
    b = nb.DenoiseBatch(B)
    net = small_net(0)
    train_window(b, net, xd, cl)
    gk = [p.grad.clone() for p in net.parameters()]
    net.zero_grad()
    train_window(b, net, xd, cl, use_ref=True)
    for p, k in zip(net.parameters(), gk):
        rel = float((k - p.grad).norm() / p.grad.norm())
        print("\nparameter %s: relative gradient difference %.2e" % (tuple(p.shape), rel))
        assert rel <= 1e-3


@pytest.mark.gpu
def test_adam_lowers_waveform_mse():
    import torch
    B, T = 32, 12
    clean, noisy = noisy_clean(B, T, 9)
    xd = torch.from_numpy(np.ascontiguousarray(noisy.transpose(1, 0, 2))).cuda()
    cl = torch.from_numpy(clean).cuda()
    b = nb.DenoiseBatch(B)
    net = small_net(1)
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    losses = []
    for _ in range(40):
        opt.zero_grad()
        losses.append(train_window(b, net, xd, cl))
        opt.step()
    print("\nAdam through synthesis: waveform MSE %.4g -> %.4g (40 steps)" % (losses[0], losses[-1]))
    assert np.mean(losses[-3:]) < 0.9 * np.mean(losses[:3])


# ---- 5. refusals ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_change_nothing():
    import torch
    B, T = 9, 4
    x = signals(B, T, seed=21)
    xd = torch.from_numpy(x).cuda()
    gains = torch.rand((B, T, NBB), generator=torch.Generator().manual_seed(3)).cuda()
    twin, b = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    o_twin, c_twin = run_saving(twin, xd, gains)
    feats = torch.empty((T, B, NBF), device="cuda")
    out = torch.zeros((B, T, F), device="cuda")
    ctx = torch.full((B, T, CB), 0xAB, dtype=torch.uint8, device="cuda")
    with pytest.raises(nb.NnnoiselessError, match="with 0 pending"):
        b.synthesize_saving_device(out.data_ptr(), gains.data_ptr(), 1, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1)
    analyze(b, xd, 0, T, feats)
    sv = lambda **kw: b.synthesize_saving_device(**{**dict(out_ptr=out.data_ptr(), gains_ptr=gains.data_ptr(), n_frames=T,  # noqa: E731
                                                           stream_stride=T * F, frame_stride=F, gain_stream_stride=T * NBB,
                                                           gain_frame_stride=NBB, ctx_ptr=ctx.data_ptr(), ctx_stream_stride=T,
                                                           ctx_frame_stride=1), **kw})
    bad = [dict(ctx_ptr=0), dict(ctx_ptr=ctx.data_ptr() + 8), dict(ctx_stream_stride=1), dict(ctx_frame_stride=0), dict(pcm16=1),
           dict(n_frames=T + 1), dict(out_ptr=0), dict(gains_ptr=0), dict(sample_stride=0), dict(n_frames=-1)]
    for kw in bad:
        with pytest.raises(nb.NnnoiselessError):
            sv(**kw)
        assert b.pending_frames == T, kw
    sv(n_frames=0)
    torch.cuda.synchronize()
    assert not out.any() and bool((ctx == 0xAB).all())
    sv()
    torch.cuda.synchronize()
    assert np.array_equal(bits(out), bits(o_twin)) and torch.equal(ctx, c_twin)
    assert np.array_equal(b.get_states(), twin.get_states())
    # the backward
    go = torch.randn((B, T, F), device="cuda")
    nbytes = nb.synthesis_backward_workspace_bytes(B, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    grad = torch.full((B, T, NBB), 7.0, device="cuda")
    args = dict(ctx_ptr=ctx.data_ptr(), ctx_stream_stride=T, ctx_frame_stride=1, grad_out_ptr=go.data_ptr(), go_stream_stride=T * F,
                go_frame_stride=F, grad_gains_ptr=grad.data_ptr(), gg_stream_stride=T * NBB, gg_frame_stride=NBB, n_streams=B,
                n_frames=T, workspace_ptr=ws.data_ptr(), workspace_bytes=nbytes)
    bad = [dict(ctx_ptr=0), dict(grad_out_ptr=0), dict(grad_gains_ptr=0), dict(workspace_ptr=0), dict(n_frames=0), dict(n_streams=0),
           dict(workspace_bytes=nbytes - 1), dict(gg_frame_stride=NBB - 1), dict(gg_stream_stride=0), dict(ctx_frame_stride=0),
           dict(go_stream_stride=-F), dict(ctx_ptr=ctx.data_ptr() + 4), dict(device=1 << 20)]
    for kw in bad:
        with pytest.raises(nb.NnnoiselessError):
            nb.synthesis_backward_device(**{**args, **kw})
    torch.cuda.synchronize()
    assert bool((grad == 7.0).all())
    assert nb.synthesis_backward_workspace_bytes(0, 1) == 0 and nb.synthesis_backward_workspace_bytes(1, 0) == 0


# ---- 6. the C++ mirror --------------------------------------------------------------------------------------------
def test_cpp_mirror_saving_and_backward_compile(tmp_path):
    """nnnoiseless.hpp's DenoiseBatch::synthesize_saving and synthesis_backward compile and link (runs without a GPU)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    inc, libdir = os.path.join(root, "include"), os.path.join(root, "nnnoiseless_b200", "lib")
    src = tmp_path / "t.cpp"
    src.write_text('#include "nnnoiseless.hpp"\n'
                   "void step(nnnoiseless::DenoiseBatch& b, float* out, const float* gains, void* ctx, const float* go, float* gg,\n"
                   "          void* ws, void* stream) {\n"
                   "    const long B = b.streams(), T = RNNOISE_MAX_PENDING_FRAMES;\n"
                   "    b.synthesize_saving(out, gains, (int)T, T * 480, 1, 480, T * 22, 22, ctx, T, 1, stream);\n"
                   "    const size_t n = nnnoiseless::synthesis_backward_workspace_bytes((int)B, (int)T);\n"
                   "    nnnoiseless::synthesis_backward(ctx, T, 1, go, T * 480, 480, gg, T * 22, 22, (int)B, (int)T, ws, n, -1, stream);\n"
                   "}\n"
                   "int main(int argc, char**) {\n"
                   "    static_assert(RNNOISE_SYNTH_CONTEXT_BYTES == 7552, \"record size\");\n"
                   "    if (argc > 1) { nnnoiseless::DenoiseBatch b(1); step(b, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr); }\n"
                   "    return 0;\n"
                   "}\n")
    exe = tmp_path / "t"
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", inc, str(src), "-o", str(exe), "-L", libdir, "-lnnnoiseless_b200",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0
