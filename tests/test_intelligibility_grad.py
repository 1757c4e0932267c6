"""The STOI / ESTOI backward kernels (rnnoise_intelligibility_backward_device) and autograd.intelligibility on the GPU
(DESIGN.md 7r).

Each stage is checked from the GPU's own inputs to it, read through the forward and backward workspace taps:
- d bands within 1e-12 of the float64 restatement's largest element per pair, from the GPU's float bands;
- d u (the bands backward) within w_i 16 * 9 u (sqrt(512) ||w u_j|| sum_k |d by / by| + 4 sum_k |G(k)|) + 2 u |d u_i| of
  the exact adjoint from the GPU's y10, kept list, bands and d bands: the forward's spectrum bound carried through G and
  the adjoint FFT's own rounding;
- d y10 within gamma_4 sum |terms| of float64 from the GPU's d u, and exactly +0.0 where no STFT frame reads;
- d out within gamma_P sum |h| |d y10| of float64 from the GPU's d y10 (P: the taps an output sums); bit-equal at 10 kHz;
- end to end normwise within 1e-4 of the float64 backward, on clips with no frame within 1e-3 dB of the threshold.
Then directional derivatives, scale invariance, exact zeros, bit-exact invariances, the autograd function and training
through synthesis."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import stoi_grad_ref as gr
import stoi_ref as sr
from test_intelligibility import noisy_pairs, tones
from test_metrics import heldout  # noqa: F401  (the module-scoped corpus fixture)
from test_training_pool import corpus  # noqa: F401

pytestmark = pytest.mark.gpu
F = 480
SHARES = {}


def run(y, x, rate, gs=1.0, ge=1.0, pad=0, gpad=0):
    """Forward then backward on rows y (out) and x (clean) [B][n]; gs, ge scalars, arrays or None.
    -> dict(rec, x10, kept, bands (forward taps), dby, inv, du, dy10 (backward taps), g [B][n])."""
    import torch
    B, n = x.shape
    w = max(n + pad, 1)
    dy = torch.zeros((B, w), dtype=torch.float32)
    dx = torch.zeros((B, w), dtype=torch.float32)
    dy[:, :n] = torch.from_numpy(np.ascontiguousarray(y, np.float32))
    dx[:, :n] = torch.from_numpy(np.ascontiguousarray(x, np.float32))
    dy, dx = dy.cuda(), dx.cuda()
    fb = nb.intelligibility_workspace_bytes(B, n, rate)
    fws = torch.full((fb,), 0x7F, dtype=torch.uint8, device="cuda")
    res = torch.full((B * 32,), 0x7F, dtype=torch.uint8, device="cuda")
    nb.intelligibility_device(dy.data_ptr(), dx.data_ptr(), B, n, w, rate, res.data_ptr(), fws.data_ptr(), fb)
    bb = nb.intelligibility_backward_workspace_bytes(B, n, rate)
    bws = torch.full((bb,), 0x7F, dtype=torch.uint8, device="cuda")
    gw = max(n + gpad, 1)
    g = torch.full((B, gw), float("nan"), dtype=torch.float32, device="cuda")
    grads = [None if v is None else torch.from_numpy(np.broadcast_to(np.asarray(v, np.float64), (B,)).copy()).cuda() for v in (gs, ge)]
    before = nb.kernel_launches()
    nb.intelligibility_backward_device(B, n, rate, res.data_ptr(), fws.data_ptr(), fb, *(0 if t is None else t.data_ptr() for t in grads),
                                       g.data_ptr(), gw, bws.data_ptr(), bb)
    assert nb.kernel_launches() - before == 4
    gh = g.cpu().numpy()
    assert np.isnan(gh[:, n:]).all()  # past n_samples nothing is written
    out = dict(rec=res.cpu().numpy().view(nb.INTELLIGIBILITY_DTYPE).copy(), g=gh[:, :n].copy())
    for k, t in zip(("x10", "kept", "bands"), nb.intelligibility_taps(fws, B, n, rate)):
        out[k] = t.cpu().numpy().copy()
    for k, t in zip(("dby", "inv", "du", "dy10"), nb.intelligibility_backward_taps(bws, B, n, rate)):
        out[k] = t.cpu().numpy().copy()
    return out


def share(name, key, err, bound):
    s = SHARES.setdefault(name, {})
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
    if r.size:
        s[key] = max(s.get(key, 0.0), float(r.max()))


def check_call(name, y, x, rate, gs=1.0, ge=1.0, pad=0, gpad=0, e2e_rows=4):
    """Every backward stage of one call from its own inputs; returns run()'s dict."""
    r = run(y, x, rate, gs, ge, pad, gpad)
    B, n = x.shape
    up, down, half, n10, Fr = sr.sizes(n, rate)
    h = sr.filter_taps(rate)
    P = 1 if h is None else len(h) // down + 2
    u = sr.U32
    gsv = np.broadcast_to(np.asarray(gs if gs is not None else 0.0, np.float64), (B,))
    gev = np.broadcast_to(np.asarray(ge if ge is not None else 0.0, np.float64), (B,))
    for p in range(B):
        S, K = int(r["rec"]["segments"][p]), int(r["rec"]["kept"][p])
        M = max(K - 1, 0)
        kept = r["kept"][p, :K].astype(np.int64)
        if S < 1:
            assert np.array_equal(r["g"][p].view(np.uint32), np.zeros(n, np.uint32)), (name, p)  # +0.0
            continue
        inv = -np.ones(Fr, np.int64)
        inv[kept] = np.arange(K)
        assert np.array_equal(r["inv"][p], inv), (name, p)
        # score backward from the GPU's float bands
        want = gr.score_bwd(r["bands"][0, p][:, :M], r["bands"][1, p][:, :M], None if gs is None else gsv[p], None if ge is None else gev[p])
        got = r["dby"][p][:, :M]
        err = np.abs(got - want)
        bound = 1e-12 * np.abs(want).max()
        assert (err <= bound).all(), (name, p, float(err.max()), bound)
        share(name, "score", err, np.full_like(err, bound))
        # bands backward from the GPU's y10, kept list, bands and d bands
        du64, fnorm, sumsc, sumg = gr.bands_bwd(r["x10"][1, p], kept, r["bands"][1, p][:, :M], got)
        w = sr.window()
        bound = w[None, :] * 16 * 9 * u * (np.sqrt(512) * (fnorm * sumsc)[:, None] + 4 * sumg[:, None]) + 2 * u * np.abs(du64)
        err = np.abs(r["du"][p][:M] - du64)
        assert (err <= bound).all(), (name, p, float((err - bound).max()))
        share(name, "bands", err, bound)
        # overlap-add adjoint from the GPU's d u
        ref = gr.ola_bwd(r["du"][p][:M], kept, n10)
        bound = sr.gamma(4) * gr.ola_bwd(r["du"][p][:M], kept, n10, absolute=True)
        err = np.abs(r["dy10"][p] - ref)
        assert (err <= bound).all(), (name, p, float((err - bound).max()))
        share(name, "ola", err, bound)
        unread = ~gr.read_samples(kept, n10)
        assert np.array_equal(r["dy10"][p][unread].view(np.uint32), np.zeros(int(unread.sum()), np.uint32)), (name, p)
        # resampler adjoint from the GPU's d y10
        if h is None:
            assert np.array_equal(r["g"][p].view(np.uint32), r["dy10"][p][:n].view(np.uint32)), (name, p)
        else:
            ref = gr.resample_bwd(r["dy10"][p], n, rate)
            bound = sr.gamma(P) * gr.resample_bwd(r["dy10"][p], n, rate, absolute=True)
            err = np.abs(r["g"][p] - ref)
            assert (err <= bound).all(), (name, p, float((err - bound).max()))
            share(name, "resample", err, bound)
        # samples whose filter support meets no read 10 kHz sample are +0.0
        sup = gr.resample_bwd((~unread).astype(np.float64), n, rate, absolute=True)
        assert np.array_equal(r["g"][p][sup == 0].view(np.uint32), np.zeros(int((sup == 0).sum()), np.uint32)), (name, p)
        # end to end against the float64 backward
        if p < e2e_rows:
            x64 = sr.resample(x[p], rate, h)
            e = sr.frame_db(x64)
            if np.abs(e - (e.max() - 40.0)).min() >= 1e-3:
                want = gr.intelligibility_grad(y[p], x[p], rate, None if gs is None else gsv[p], None if ge is None else gev[p])
                d = np.linalg.norm(r["g"][p] - want) / max(np.linalg.norm(want), 1e-300)
                assert d <= 1e-4, (name, p, d)
                s = SHARES.setdefault(name, {})
                s["e2e"] = max(s.get("e2e", 0.0), d)
    return r


@pytest.mark.parametrize("B,rate", [(1, 48000), (130, 16000), (33, 44100), (33, 10000)])
def test_speech_like_clips(B, rate):
    rng = np.random.default_rng(B)
    for n in (100, 256 * rate // 10000 + 29 * 128 * rate // 10000, 256 * rate // 10000 + 31 * 128 * rate // 10000,
              rate * (1 if rate == 44100 else 2)):
        y, x = noisy_pairs(B, n, rate, seed=n + B)
        gs, ge = rng.normal(0, 1, B), rng.normal(0, 1, B)
        check_call("speech %d Hz" % rate, y, x, rate, gs, ge, pad=37 if B == 33 else 0, gpad=37 if B == 33 else 0,
                   e2e_rows=2 if B > 1 else 1)
    # one term at a time
    y, x = noisy_pairs(3, rate * 2, rate, seed=5)
    check_call("speech %d Hz" % rate, y, x, rate, 1.0, None, e2e_rows=1)
    check_call("speech %d Hz" % rate, y, x, rate, None, 1.0, e2e_rows=1)


@pytest.mark.parametrize("rate", [48000, 16000, 10000])
def test_tones_and_one_loud_band(rate):
    n = 12 * rate // 10
    rows_x, rows_y = [], []
    for b in range(0, 15, 2):
        lo, hi = sr.EDGES[b], sr.EDGES[b + 1]
        edge = [lo - 0.5, lo, hi - 1, hi - 0.5]
        rows_x.append(tones(n, rate, edge, [3000.0] * 4))
        rows_y.append(tones(n, rate, edge, [3000.0, 1500.0, 700.0, 300.0]))
        others = [(sr.EDGES[c] + sr.EDGES[c + 1]) / 2 for c in range(15) if c != b]
        env = (1.2 + np.sin(2 * np.pi * 2.3 * np.arange(n) / rate)).astype(np.float32)
        loud = tones(n, rate, [(lo + hi) / 2], [10000.0])
        quiet = tones(n, rate, others, [10.0] * len(others))
        rows_x.append(env * (loud + quiet))
        rows_y.append(loud + env * quiet)
    check_call("tones %d Hz" % rate, np.stack(rows_y), np.stack(rows_x), rate, e2e_rows=0)


def test_amplitudes_and_silences():
    n = 2 * 48000
    y, x = noisy_pairs(8, n, 48000, seed=9, scale=1.0)
    scales = np.array([1 / 32768, 1 / 32768, 32767.0, 32767.0, 0.0, 0.0, 1e-12, 1e-9])[:, None]
    x = (x / np.abs(x).max(axis=1, keepdims=True) * scales).astype(np.float32)
    y = (y / np.abs(y).max(axis=1, keepdims=True) * scales[::-1]).astype(np.float32)
    check_call("amplitudes", y, x, 48000, e2e_rows=0)
    # a long leading silence in clean: everything before its filter support is exactly 0
    y, x = noisy_pairs(4, 4 * 48000, 48000, seed=12)
    x[:, :2 * 48000] = 0
    r = check_call("silences", y, x, 48000, e2e_rows=2)
    assert (r["g"][:, :2 * 48000 - 2000] == 0).all() and np.abs(r["g"][:, 2 * 48000:]).max() > 0


def test_short_rows_get_zero_with_nan_gradients():
    rate = 16000
    y, x = noisy_pairs(3, 2 * rate, rate, seed=4)
    x[1, :] = 0  # all frames kept; the other rows are short of 30 frames
    n = 256 * rate // 10000 + 25 * 128 * rate // 10000
    r = run(y[:, :n], x[:, :n], rate, np.full(3, np.nan), np.full(3, np.nan))
    assert (r["rec"]["segments"] == 0).all()
    assert np.array_equal(r["g"].view(np.uint32), np.zeros_like(r["g"]).view(np.uint32))


def test_directional_derivatives_and_scale_invariance():
    for rate in (16000, 48000):
        y, x = noisy_pairs(3, 2 * rate, rate, seed=31)
        for gs, ge in ((1.0, None), (None, 1.0)):
            r = run(y, x, rate, gs, ge)
            k = 0 if gs is not None else 1
            rng = np.random.default_rng(rate + k)
            for p in range(3):
                g = r["g"][p].astype(np.float64)
                kept = sr.kept_frames(sr.resample(x[p], rate))
                d = rng.normal(0, 1, y.shape[1])
                hs = 1e-5 * np.linalg.norm(y[p]) / np.linalg.norm(d)
                fd = (gr.value64(y[p] + hs * d, x[p], rate, kept)[k] - gr.value64(y[p] - hs * d, x[p], rate, kept)[k]) / (2 * hs)
                assert abs(fd - g @ d) <= 1e-3 * abs(fd), (rate, k, p, fd, g @ d)
                # STOI and ESTOI are invariant to a positive scale of out
                assert abs(g @ y[p]) <= 1e-4 * np.linalg.norm(g) * np.linalg.norm(y[p]), (rate, k, p)
            half = run(y * np.float32(0.5), x, rate, gs, ge)["g"]
            for p in range(3):
                d = np.linalg.norm(half[p] - 2 * r["g"][p]) / np.linalg.norm(2 * r["g"][p])
                assert d <= 1e-4, (rate, k, p, d)


def test_repeat_permutation_and_grid():
    import torch
    n = 2 * 48000
    y, x = noisy_pairs(8, n, 48000, seed=21)
    gs, ge = np.linspace(-1, 1, 8), np.linspace(2, -1, 8)
    a = run(y, x, 48000, gs, ge)["g"]
    assert a.tobytes() == run(y, x, 48000, gs, ge)["g"].tobytes()
    perm = np.random.default_rng(2).permutation(8)
    assert run(y[perm], x[perm], 48000, gs[perm], ge[perm])["g"].tobytes() == a[perm].tobytes()
    # 2 x SMs x 64 + 37 pairs of 0.6 s, rows drawn from 37 distinct ones, equal the call on those 37
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    Bb, nn, k = 2 * sms * 64 + 37, 28800, 37
    rng = np.random.default_rng(5)
    xs = (rng.normal(0, 3000, (k, nn)) * (1.0 + 0.5 * np.sin(2 * np.pi * 3.0 * np.arange(nn) / 48000 + rng.uniform(0, 6, (k, 1)))))
    xs = xs.astype(np.float32)
    ys = (xs + rng.normal(0, 2000, xs.shape)).astype(np.float32)
    gk, ek = rng.normal(0, 1, k), rng.normal(0, 1, k)
    small = run(ys, xs, 48000, gk, ek)["g"]
    idx = torch.arange(Bb, device="cuda") % k
    dy, dx = torch.from_numpy(ys).cuda()[idx].contiguous(), torch.from_numpy(xs).cuda()[idx].contiguous()
    fb = nb.intelligibility_workspace_bytes(Bb, nn, 48000)
    fws = torch.empty(fb, dtype=torch.uint8, device="cuda")
    res = torch.empty(Bb * 32, dtype=torch.uint8, device="cuda")
    cs = torch.cuda.current_stream().cuda_stream
    nb.intelligibility_device(dy.data_ptr(), dx.data_ptr(), Bb, nn, nn, 48000, res.data_ptr(), fws.data_ptr(), fb, cuda_stream=cs)
    bb = nb.intelligibility_backward_workspace_bytes(Bb, nn, 48000)
    bws = torch.empty(bb, dtype=torch.uint8, device="cuda")
    g = torch.empty((Bb, nn), device="cuda")
    tg, te = torch.from_numpy(gk).cuda()[idx].contiguous(), torch.from_numpy(ek).cuda()[idx].contiguous()
    nb.intelligibility_backward_device(Bb, nn, 48000, res.data_ptr(), fws.data_ptr(), fb, tg.data_ptr(), te.data_ptr(), g.data_ptr(), nn,
                                       bws.data_ptr(), bb, cuda_stream=cs)
    assert g.cpu().numpy().tobytes() == small[np.arange(Bb) % k].tobytes()


def test_autograd_function_equals_the_hand_call():
    import torch
    from nnnoiseless_b200 import autograd as ag
    y, x = noisy_pairs(5, 2 * 48000, 48000, seed=41)
    gs, ge = np.linspace(-1, 1, 5), np.linspace(0.5, 2, 5)
    hand = run(y, x, 48000, gs, ge)
    out = torch.from_numpy(y).cuda().requires_grad_()
    s, e = ag.intelligibility(out, torch.from_numpy(x).cuda())
    assert s.dtype == torch.float64 and s.shape == (5,)
    assert np.array_equal(s.detach().cpu().numpy(), hand["rec"]["stoi"]) and np.array_equal(e.detach().cpu().numpy(), hand["rec"]["estoi"])
    ((s * torch.from_numpy(gs).cuda()).sum() + (e * torch.from_numpy(ge).cuda()).sum()).backward()
    assert out.grad.cpu().numpy().tobytes() == hand["g"].tobytes()
    # refusals before any device work
    with pytest.raises(ValueError, match="clean requires grad"):
        ag.intelligibility(out, torch.from_numpy(x).cuda().requires_grad_())
    base = torch.zeros(48000 * 3, device="cuda")
    with pytest.raises(ValueError, match="rows must not overlap"):
        ag.intelligibility(base.unfold(0, 96000, 24000), base.unfold(0, 96000, 24000))


def test_training_through_synthesis_raises_estoi(heldout):  # noqa: F811
    import torch
    from nnnoiseless_b200 import training as tr
    from nnnoiseless_b200.autograd import DenoiseNetwork, intelligibility, synthesis_grad
    sig, noise = heldout
    B, T = 4, 300
    wc = tr.WaveformCorpus(sig[-1:], noise, B)  # testing.raw with the pool's noise
    wc.start(B * T, seed=9)
    noisy, clean = torch.empty((B, T, F), device="cuda"), torch.empty((B, T, F), device="cuda")
    assert wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F) == T
    net = DenoiseNetwork.from_model(None, B, T)
    opt = torch.optim.Adam([net.params], lr=3e-3)

    def window(grad):
        b = nb.DenoiseBatch(B, device=0)
        feats = torch.empty((B, T, 42), device="cuda")
        sil = torch.empty((T, B), dtype=torch.int32, device="cuda")
        out = torch.empty((B, T, F), device="cuda")
        ctx = torch.empty((B, T, nb.SYNTH_CONTEXT_BYTES), dtype=torch.uint8, device="cuda")
        b.analyze_window_device(noisy.data_ptr(), feats.data_ptr(), sil.data_ptr(), T, T * F, F, T * 42, 42, ctx.data_ptr(), T, 1)
        with torch.set_grad_enabled(grad):
            g, _, _ = net(feats, sil)
            b.synthesize_window_device(out.data_ptr(), g.detach().contiguous().data_ptr(), T, T * F, F, T * 22, 22, ctx.data_ptr(), T, 1)
            y = synthesis_grad(g, out, ctx) if grad else out
            s, e = intelligibility(y[:, 1:].reshape(B, -1), clean[:, :-1].reshape(B, -1))
        return s, e

    _, e0 = window(False)
    before = float(e0.mean())
    for _ in range(6):
        opt.zero_grad()
        _, e = window(True)
        (1 - e.mean()).backward()
        assert torch.isfinite(net.params.grad).all() and net.params.grad.abs().max() > 0
        opt.step()
        net.clip_()
    _, e1 = window(False)
    after = float(e1.mean())
    print("\nESTOI of one testing.raw window through DenoiseNetwork: %.5f -> %.5f after 6 Adam steps on 1 - ESTOI" % (before, after))
    assert after > before


def test_refusals_change_nothing():
    import torch
    y, x = noisy_pairs(3, 48000, 48000, seed=3)
    dy, dx = torch.from_numpy(y).cuda(), torch.from_numpy(x).cuda()
    fb = nb.intelligibility_workspace_bytes(3, 48000, 48000)
    fws = torch.zeros(fb, dtype=torch.uint8, device="cuda")
    res = torch.zeros(96, dtype=torch.uint8, device="cuda")
    nb.intelligibility_device(dy.data_ptr(), dx.data_ptr(), 3, 48000, 48000, 48000, res.data_ptr(), fws.data_ptr(), fb)
    bb = nb.intelligibility_backward_workspace_bytes(3, 48000, 48000)
    bws = torch.zeros(bb, dtype=torch.uint8, device="cuda")
    g = torch.zeros((3, 48000), device="cuda")
    for kw in (dict(grad_stride=47999), dict(workspace_bytes=bb - 1), dict(fwd_workspace_bytes=fb - 1), dict(rate=48100), dict(n_pairs=0)):
        a = dict(n_pairs=3, n_samples=48000, rate=48000, result_ptr=res.data_ptr(), fwd_workspace_ptr=fws.data_ptr(), fwd_workspace_bytes=fb,
                 grad_stoi_ptr=0, grad_estoi_ptr=0, grad_out_ptr=g.data_ptr(), grad_stride=48000, workspace_ptr=bws.data_ptr(), workspace_bytes=bb)
        a.update(kw)
        with pytest.raises(nb.NnnoiselessError):
            nb.intelligibility_backward_device(**a)
    torch.cuda.synchronize()
    assert not bws.any() and not g.any()


def test_report_shares():
    """Prints the largest share of each bound seen by the stage tests of this module (run after them)."""
    for k, v in SHARES.items():
        print("\n%-16s %s" % (k, "  ".join("%s %.3g" % kv for kv in sorted(v.items()))), end="")
