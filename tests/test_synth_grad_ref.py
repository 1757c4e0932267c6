"""CPU tests of the float64 restatement of a window of synthesis frames and its gradient (synth_grad_ref).

- Its forward equals spectral_ref.synthesis chained frame by frame (lastg and the overlap memory), to 1e-12.
- Its gradient (autograd through explicit masks) agrees with central finite differences of that chain away from kinks,
  and at each kink with the one-sided difference the contract names.
- The kernel's algorithm restated in numpy (window_grad_manual: the inverse FFT's adjoint as a forward FFT with bins
  1..479 counted twice, the renormalisation term, the reverse-time floor scan) equals autograd.
"""
import numpy as np
import torch

import spectral_ref as sr
import synth_grad_ref as ref

NB = sr.NB_BANDS


def synthetic_window(B, T, seed, silent=()):
    """Contexts of B streams x T frames as analysis would leave them (band energies and correlation from the spectra),
    random raw gains in (0.05, 0.95), lastg chained in f32.  silent: (stream, frame) pairs marked silent."""
    rng = np.random.default_rng(seed)
    W = sr.tables()["W"]
    X = (rng.normal(size=(B, T, 481)) + 1j * rng.normal(size=(B, T, 481))) * 30
    P = (rng.normal(size=(B, T, 481)) + 1j * rng.normal(size=(B, T, 481))) * 30 + 0.5 * X
    X, P = X.astype(np.complex64).astype(complex), P.astype(np.complex64).astype(complex)
    P[..., 400:] = 0
    ex = np.abs(X) ** 2 @ W.T
    ep = np.abs(P) ** 2 @ W.T
    corr = (X.real * P.real + X.imag * P.imag) @ W.T
    exp = (corr / np.sqrt(sr.C_CORR + ex * ep)).astype(np.float32)
    g = rng.uniform(0.05, 0.95, (B, T, NB)).astype(np.float32)
    sil = np.zeros((B, T), bool)
    for s, t in silent:
        sil[s, t] = True
    lastg = np.zeros((B, T, NB), np.float32)
    lastg[:, 0] = rng.uniform(0, 1, (B, NB)).astype(np.float32)
    for t in range(T - 1):
        nxt = np.maximum(g[:, t], np.float32(0.6) * lastg[:, t])
        lastg[:, t + 1] = np.where(sil[:, t, None], lastg[:, t], nxt)
    return dict(X=X, P=P[..., :400], ex=ex.astype(np.float32), ep=ep.astype(np.float32), exp=exp, lastg=lastg, g=g, silence=sil)


def chain(d, g, mem0):
    """spectral_ref.synthesis frame by frame -> out [B][T][480]."""
    B, T = g.shape[:2]
    lg, mem, outs = d["lastg"][:, 0].astype(np.float64), mem0, []
    for t in range(T):
        o = sr.synthesis(d["X"][:, t], d["P"][:, t], d["ex"][:, t], d["ep"][:, t], d["exp"][:, t], g[:, t], lg, mem, d["silence"][:, t])
        outs.append(o["out"])
        lg, mem = o["lastg"], o["synth_mem"]
    return np.stack(outs, 1)


def test_ctx_round_trip():
    d = synthetic_window(2, 3, 0, silent=[(1, 1)])
    e = ref.parse_ctx(ref.make_ctx(d["X"], d["P"], d["ex"], d["ep"], d["exp"], d["lastg"], d["g"], d["silence"]))
    for k in ("ex", "ep", "exp", "lastg", "g", "silence"):
        assert np.array_equal(e[k], d[k]), k
    assert np.array_equal(e["X"], d["X"]) and np.array_equal(e["P"], d["P"])


def test_forward_equals_spectral_ref_chain():
    B, T = 3, 6
    d = synthetic_window(B, T, 1, silent=[(0, 2), (2, 3), (2, 4)])
    mem0 = np.random.default_rng(2).normal(size=(B, 480)) * 100
    g = d["g"].astype(np.float64)
    want = chain(d, g, mem0)
    got = ref.window_out(d, torch.tensor(g), mem0).numpy()
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def _fd(d, go, mem0, idx, h, one_sided=False):
    g = d["g"].astype(np.float64)
    gp = g.copy()
    gp[idx] += h
    lp = (chain(d, gp, mem0) * go).sum()
    if one_sided:
        return (lp - (chain(d, g, mem0) * go).sum()) / h
    gm = g.copy()
    gm[idx] -= h
    return (lp - (chain(d, gm, mem0) * go).sum()) / (2 * h)


def test_gradient_matches_finite_differences():
    B, T = 2, 4
    d = synthetic_window(B, T, 3, silent=[(1, 2)])
    mem0 = np.zeros((B, 480))
    go = np.random.default_rng(4).normal(size=(B, T, 480))
    mk = ref.masks(d)
    grad = ref.window_grad(d, go, mem0)
    scale = np.abs(grad).max()
    checked = 0
    for idx in np.ndindex(B, T, NB):
        g, e, lg = float(d["g"][idx]), float(d["exp"][idx]), float(d["lastg"][idx])
        if abs(g - e) < 1e-3 or abs(g - 0.6 * lg) < 1e-3 or mk["ambiguous"][idx]:
            continue
        fd = _fd(d, go, mem0, idx, 1e-6 * max(g, 1e-3))
        assert abs(fd - grad[idx]) <= 1e-6 * scale + 1e-6 * abs(fd), (idx, fd, grad[idx])
        checked += 1
    assert checked > 0.8 * B * T * NB
    assert np.all(grad[1, 2] == 0.0)  # the silent frame's gains


def test_gradient_at_the_kinks():
    """g == exp (the formula applies), g == 0.6f lastg (the gradient goes to g), g == 1 and g > 1 (q clamped to 0),
    exp == 0 (q == 0): the masked gradient equals the right-sided difference."""
    B, T = 1, 3
    d = synthetic_window(B, T, 5)
    d["exp"][0, 1, 0] = 0.0
    d["g"][0, 1, 1] = d["exp"][0, 1, 1] = np.float32(0.4)
    d["g"][0, 1, 2] = 1.0
    d["g"][0, 1, 3] = 1.5
    # the floor tie: lastg of frame 1 from frame 0, then g = 0.6f lastg exactly
    d["g"][0, 0, 4] = np.float32(0.9)
    d["lastg"][0, 1] = np.maximum(d["g"][0, 0], np.float32(0.6) * d["lastg"][0, 0])
    d["g"][0, 1, 4] = np.float32(0.6) * d["lastg"][0, 1, 4]
    d["lastg"][0, 2] = np.maximum(d["g"][0, 1], np.float32(0.6) * d["lastg"][0, 1])
    mk = ref.masks(d)
    assert mk["take_g"][0, 1, 4] and not mk["branch"][0, 1, 1] and not mk["live"][0, 1, 2] and not mk["live"][0, 1, 0]
    go = np.random.default_rng(6).normal(size=(B, T, 480))
    mem0 = np.zeros((B, 480))
    grad = ref.window_grad(d, go, mem0)
    for band in (0, 1, 2, 3, 4):
        idx = (0, 1, band)
        g = float(d["g"][idx])
        fd = _fd(d, go, mem0, idx, 1e-5 * g, one_sided=True)
        assert abs(fd - grad[idx]) <= 1e-3 * abs(fd) + 1e-7 * np.abs(grad).max(), (band, fd, grad[idx])


def test_manual_adjoint_equals_autograd():
    B, T = 3, 5
    d = synthetic_window(B, T, 7, silent=[(0, 1), (2, 0), (2, 4)])
    # a run of floored frames: decaying gains on stream 1
    d["g"][1] = (0.9 * 0.3 ** np.arange(T))[:, None].astype(np.float32)
    for t in range(T - 1):
        nxt = np.maximum(d["g"][:, t], np.float32(0.6) * d["lastg"][:, t])
        d["lastg"][:, t + 1] = np.where(d["silence"][:, t, None], d["lastg"][:, t], nxt)
    mk = ref.masks(d)
    assert (~mk["take_g"][1, 1:]).all()
    go = np.random.default_rng(8).normal(size=(B, T, 480))
    a = ref.window_grad(d, go)
    m = ref.window_grad_manual(d, go)
    assert np.abs(a - m).max() <= 1e-8 * np.abs(a).max()
