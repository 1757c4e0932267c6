"""CPU tests of the STOI / ESTOI backward's restatement (tests/stoi_grad_ref.py) against independent derivatives, and
the argument checks rnnoise_intelligibility_backward_device and autograd.intelligibility make before any device work
(DESIGN.md 7r)."""
import ctypes as C

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import stoi_grad_ref as gr
import stoi_ref as sr
from test_intelligibility_cpu import speech_like

RATES = [48000, 44100, 16000, 8000, 10000, 22000]  # the forward tests' rates


def pair(n, rate, seed, snr=5.0):
    x = speech_like(n, seed, 3000.0, rate).astype(np.float64)
    y = x + np.random.default_rng(seed + 1).normal(0, 1, n) * np.sqrt(np.mean(x ** 2) / 10 ** (snr / 10))
    return y.astype(np.float32), x.astype(np.float32)


@pytest.mark.parametrize("rate", [10000, 16000, 48000])
def test_restatement_matches_torch_autograd(rate):
    import torch
    n = int(rate * 1.5)
    y, x = pair(n, rate, seed=rate // 100)
    t = torch.from_numpy(y.astype(np.float64)).requires_grad_()
    s, e = gr.torch_intelligibility(t, x, rate)
    for gs, ge in ((1.0, None), (None, 1.0), (0.3, -1.7)):
        t.grad = None
        ((s * gs if gs is not None else 0) + (e * ge if ge is not None else 0)).backward(retain_graph=True)
        want = t.grad.numpy()
        got = gr.intelligibility_grad(y, x, rate, gs, ge)
        rel = np.linalg.norm(got - want) / np.linalg.norm(want)
        assert rel <= 1e-10, (rate, gs, ge, rel)
    f = sr.intelligibility(y, x, rate)
    assert abs(float(s) - f["stoi"]) < 1e-12 and abs(float(e) - f["estoi"]) < 1e-12


@pytest.mark.parametrize("rate", [10000, 16000])
def test_restatement_matches_central_differences(rate):
    n = int(rate * 1.5)
    y, x = pair(n, rate, seed=7)
    kept = sr.kept_frames(sr.resample(x, rate))
    rng = np.random.default_rng(rate)
    g_s = gr.intelligibility_grad(y, x, rate, 1.0, None)
    g_e = gr.intelligibility_grad(y, x, rate, None, 1.0)
    for _ in range(3):
        d = rng.normal(0, 1, n)
        # a step of 1e-5 of ||y||: small enough that no min(alpha y, c x) changes branch (away from clip ties), large
        # enough that the float64 rounding of the values is far below the difference; the gradient is taken at the
        # float bands, so it differs from the float64 definition's by about 1e-6 relative
        hstep = 1e-5 * np.linalg.norm(y) / np.linalg.norm(d)
        p, m = gr.value64(y + hstep * d, x, rate, kept), gr.value64(y - hstep * d, x, rate, kept)
        for k, g in ((0, g_s), (1, g_e)):
            fd = (p[k] - m[k]) / (2 * hstep)
            an = float(g @ d)
            assert abs(fd - an) <= 1e-4 * abs(an) + 1e-9 * np.linalg.norm(g) * np.linalg.norm(d), (rate, k, fd, an)


@pytest.mark.parametrize("rate", RATES)
def test_resampler_adjoint_identity(rate):
    rng = np.random.default_rng(rate + 3)
    n = 3001
    u = rng.normal(0, 1, n)
    n10 = sr.sizes(n, rate)[3]
    v = rng.normal(0, 1, n10)
    lhs = float(sr.resample(u, rate) @ v)
    rhs = float(u @ gr.resample_bwd(v, n, rate))
    assert abs(lhs - rhs) <= 1e-12 * float(sr.resample(np.abs(u), rate, absolute=True) @ np.abs(v))
    assert np.all(gr.resample_bwd(v, n, rate, absolute=True) >= np.abs(gr.resample_bwd(v, n, rate)))


def test_overlap_add_and_band_spectrum_adjoint_identities():
    rng = np.random.default_rng(1)
    n10 = 256 + 40 * 128
    F = (n10 - 256) // 128 + 1
    for kept in (np.arange(F), np.sort(rng.choice(F, 25, replace=False)), np.array([3, 9]), np.array([5])):
        y = rng.normal(0, 1, n10)
        M = max(len(kept) - 1, 0)
        du = rng.normal(0, 1, (M, 256))
        lhs = float((gr.ola_frames(y, kept) * du).sum())
        rhs = float(y @ gr.ola_bwd(du, kept, n10))
        assert abs(lhs - rhs) <= 1e-12 * (np.abs(y) @ gr.ola_bwd(du, kept, n10, absolute=True) + 1e-300)
        # samples no STFT frame reads get nothing
        assert np.all(gr.ola_bwd(du, kept, n10)[~gr.read_samples(kept, n10)] == 0)
    u = rng.normal(0, 1, (7, 256))
    G = rng.normal(0, 1, (7, 212)) + 1j * rng.normal(0, 1, (7, 212))
    lhs = float(np.real(np.conj(G) * gr.band_spectrum(u)).sum())
    rhs = float((u * gr.band_spectrum_adjoint(G)).sum())
    assert abs(lhs - rhs) <= 1e-12 * np.abs(u).sum() * np.abs(G).sum()


def test_score_backward_zero_rows_and_ties():
    rng = np.random.default_rng(2)
    bx = rng.uniform(1, 2, (15, 29)).astype(np.float32)
    assert not gr.score_bwd(bx, bx, 1.0, 1.0).any()  # S = 0
    bx = rng.uniform(1, 2, (15, 40)).astype(np.float32)
    # a zero out makes ||y|| = 0 and every centred y norm 0: the square roots' zeros contribute 0, the rest stays finite
    assert np.all(np.isfinite(gr.score_bwd(bx, np.zeros_like(bx), 1.0, 1.0)))
    # y = x: alpha = 1, every y' on its y branch; the scores are 1 at their maximum, so the gradient is ~0
    g = gr.score_bwd(bx, bx, 1.0, 1.0)
    assert np.abs(g).max() <= 1e-12 * float(np.abs(gr.score_bwd(bx, bx[:, ::-1].copy(), 1.0, 1.0)).max())


def test_workspace_layout():
    for B, n, rate in ((1, 0, 48000), (3, 48000, 48000), (5, 12345, 44100), (2, 4096, 10000), (7, 300, 8000)):
        _, _, n10, F = nb.intelligibility_sizes(n, rate)
        maxM = max(F - 1, 0)
        r = lambda v: (v + 255) // 256 * 256  # noqa: E731
        regions = r(B * 15 * maxM * 8) + r(B * F * 4) + r(B * maxM * 256 * 4) + r(B * n10 * 4)
        assert nb.intelligibility_backward_workspace_bytes(B, n, rate) == max(regions, 256)
    assert nb.intelligibility_backward_workspace_bytes(1 << 20, 1 << 40, 48000) == 0
    for args in ((0, 100, 48000), (1, -1, 48000), (1, 100, 7999), (1, 100, 10050), (1, 100, 48100)):
        assert nb.intelligibility_backward_workspace_bytes(*args) == 0


def test_refusals_without_a_device():
    L = nb.lib()
    fake = 1 << 20  # never dereferenced: every refusal happens before any CUDA call
    fneed = nb.intelligibility_workspace_bytes(4, 1000, 48000)
    need = nb.intelligibility_backward_workspace_bytes(4, 1000, 48000)
    ok = dict(B=4, n=1000, rate=48000, res=fake, fws=fake, fwsb=fneed, gs=fake, ge=fake, g=fake, stride=1000, ws=fake, wsb=need)

    def call(**kw):
        a = {**ok, **kw}
        p = lambda v: C.c_void_p(v) if v else None  # noqa: E731
        return L.rnnoise_intelligibility_backward_device(a["B"], a["n"], a["rate"], p(a["res"]), p(a["fws"]), a["fwsb"], p(a["gs"]), p(a["ge"]),
                                                         p(a["g"]), a["stride"], p(a["ws"]), a["wsb"], -1, None)

    for kw, msg in ((dict(B=0), "n_pairs must be positive"), (dict(n=-1), "negative n_samples"), (dict(rate=7999), "rate 7999"),
                    (dict(rate=48100), "rate 48100"), (dict(stride=999), "rows overlap"), (dict(wsb=need - 1), "needed"),
                    (dict(fwsb=fneed - 1), "forward workspace"), (dict(res=0), "null argument"), (dict(fws=0), "null argument"),
                    (dict(g=0), "null argument"), (dict(ws=0), "null argument"), (dict(ws=fake + 128), "256-byte aligned"),
                    (dict(fws=fake + 64), "256-byte aligned"), (dict(res=fake + 4), "8-byte"), (dict(gs=fake + 4), "8-byte"),
                    (dict(ge=fake + 2), "8-byte"), (dict(g=fake + 2), "float-aligned")):
        assert call(**kw) == -1, kw
        assert msg in nb.last_error(), (kw, nb.last_error())


def test_autograd_refusals_before_device_work():
    import torch
    from nnnoiseless_b200 import autograd as ag
    sig = torch.arange(10.0)
    for out in (sig.unfold(0, 4, 2), sig[:4].expand(3, 4)):
        with pytest.raises(ValueError, match="rows must not overlap"):
            ag.intelligibility(out, out.clone())
    clean = torch.zeros(2, 4, requires_grad=True)
    with pytest.raises(ValueError, match="clean requires grad"):
        ag.intelligibility(torch.zeros(2, 4), clean)
