"""CPU tests of the float64 restatement of a window of synthesis frames and its gradient (synth_grad_ref).

- Its forward equals spectral_ref.synthesis chained frame by frame (lastg and the overlap memory), to 1e-12.
- Its gradient (autograd through explicit masks) agrees with central finite differences of that chain away from kinks,
  and at each kink with the one-sided difference the contract names.
- The kernel's algorithm restated in numpy (window_grad_manual: the inverse FFT's adjoint as a forward FFT with bins
  1..479 counted twice, the renormalisation term, the reverse-time floor scan) equals autograd.
- grad_bounds, the first-order rounding bound per element, holds two float32 restatements (torch autograd over BLAS
  matmuls, and the kernel's own order in numpy float32) on synthetic windows and on the edge windows the GPU test
  runs, and is no floor in disguise: its median size relative to the element stays small.
"""
import numpy as np
import pytest
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


# ---- edge windows (the GPU test feeds the same records to the kernel) ------------------------------------------------
def rechain(d):
    """lastg[t + 1] = max(g[t], 0.6f lastg[t]) on non-silent frames, in f32 as K5 stores it."""
    for t in range(d["g"].shape[1] - 1):
        nxt = np.maximum(d["g"][:, t], np.float32(0.6) * d["lastg"][:, t])
        d["lastg"][:, t + 1] = np.where(d["silence"][:, t, None], d["lastg"][:, t], nxt)
    return d


def _tone(B, T, bins, seed):
    """grad_out [B][T][480]: cosines at the given (fractional) bins of the 960-point frame, random phases."""
    rng = np.random.default_rng(seed)
    n = np.arange(T * 480)
    go = np.zeros((B, T * 480))
    for b in bins:
        go += np.cos(2 * np.pi * b * n / 960.0 + rng.uniform(0, 2 * np.pi, (B, 1)))
    return go.reshape(B, T, 480)


EDGES = ("g_near_1", "exp_eq_g", "clamp", "bands", "chain", "halves", "one_band", "dc_free", "nyquist", "odd_shape",
         "t1", "long")


def edge_window(kind, seed=0):
    """(d, grad_out) of one edge window (records built on the CPU, lastg chained as K5 does), and a dict of the edge's
    own checks: name -> boolean array that must be true somewhere."""
    rng = np.random.default_rng(seed)
    B, T = {"chain": (8, 100), "odd_shape": (3, 7), "t1": (5, 1), "long": (1, 200)}.get(kind, (6, 8))
    d = synthetic_window(B, T, 1000 + seed + len(kind))
    go = rng.normal(size=(B, T, 480))
    one = np.float32(1)
    ulp = np.float32(2.0 ** -24)
    reach = {}
    if kind == "g_near_1":
        # g = 1 - k 2^-24, k log-spaced 1 .. 2^14; exp well below, exp = 1 - j 2^-24 a few ulps from 1 (j >= k), or
        # exp a few ulps below g
        k = np.round(np.logspace(0, 14, NB, base=2.0)).astype(np.float32)
        g = one - k * ulp
        d["g"][:] = g
        d["exp"][:, :, :] = np.float32(0.5)
        d["exp"][1::3] = one - (k + np.float32(3)) * ulp            # 1 - exp down to 4 ulps, below g
        d["exp"][2::3] = g - np.float32(2) * ulp * np.maximum(one, k / 64)  # exp a few ulps below g: both near 1
        go = _tone(B, T, [1.5, 3.0, 17.0], seed)
        # streams 0 and 3: band 10 carries bin 48 alone (X = P = 0 on the band's other bins, grad_out a tone at bin 48),
        # so that its dL/dr does not cancel, with k = 2000 .. 3000, where g g loses the most of 1 - g^2
        k10 = np.float32(2000) + np.arange(B * T, dtype=np.float32).reshape(B, T) * np.float32(1000 // (B * T))
        for s in (0, 3):
            d["X"][s, :, 40:64] = d["X"][s, :, 40:64] * (np.arange(40, 64) == 48)
            d["P"][s, :, 40:64] = d["P"][s, :, 40:64] * (np.arange(40, 64) == 48)
            d["g"][s, :, 10] = one - k10[s] * ulp
            d["exp"][s, :, 10] = np.float32(0.5)
            go[s] = _tone(1, T, [48.0], seed + s)[0]
        reach["g within 16 ulps of 1"] = (one - d["g"]) <= 16 * ulp
        reach["exp within 8 ulps of 1"] = (one - d["exp"]) <= 8 * ulp
    elif kind == "exp_eq_g":
        g = rng.uniform(0.05, 0.95, (B, T, NB)).astype(np.float32)
        d["g"][:] = g
        sel = rng.integers(0, 3, (B, T, NB))
        d["exp"][:] = np.where(sel == 0, g, np.where(sel == 1, np.nextafter(g, np.float32(np.inf)), np.nextafter(g, np.float32(-np.inf))))
        reach["exp == g"] = d["exp"] == d["g"]
        reach["exp one ulp above g"] = d["exp"] == np.nextafter(d["g"], np.float32(np.inf))
        reach["exp one ulp below g"] = d["exp"] == np.nextafter(d["g"], np.float32(-np.inf))
    elif kind == "clamp":
        # q near 0: exp^2 subnormal; q near 1: exp = g > 1 large enough that q - 1 = O(u) (den < 0)
        d["exp"][:, :, :6] = np.logspace(-19, -23, 6).astype(np.float32)
        big = np.logspace(np.log10(20.0), np.log10(60.0), 8).astype(np.float32)
        d["exp"][:, :, 6:14] = big
        d["g"][:, :, 6:14] = np.where(np.arange(8) % 2 == 0, big, np.nextafter(big, np.float32(np.inf)))
        q64, dq = ref.q_bound(d["exp"], d["g"])
        reach["q within its bound of 0"] = (np.abs(q64) <= dq) & (q64 > 0)
        reach["q within its bound of 1"] = np.abs(q64 - 1) <= dq
    elif kind == "bands":
        d["ep"][:, :, 2] = 0.0                                     # cb = sqrt(ex / 1e-8)
        d["ex"][:, :, 5] = 0.0                                     # s2 = 0, cb = 0
        # band 9 (bins 32..39): X = -P rf, so that x nearly cancels and new_e is tiny
        o = [sr.synthesis(d["X"][:, t], d["P"][:, t], d["ex"][:, t], d["ep"][:, t], d["exp"][:, t], d["g"][:, t],
                          d["lastg"][:, t], np.zeros((B, 480)), d["silence"][:, t]) for t in range(T)]
        rf = np.stack([x["rf"] for x in o], 1)
        k = np.arange(28, 52)
        P = d["P"][:, :, k]
        d["X"][:, :, k] = (-(P * rf[:, :, k])).astype(np.complex64).astype(complex)
        reach["ep == 0"] = d["ep"] == 0
        reach["ex == 0"] = d["ex"] == 0
    elif kind == "chain":
        # the floor holds from frame 1 for >= 40 frames, with silent frames inside; grad_out only in the chain's last
        # frames, so that the gradient of its first frames is carried alone, down to 0.6^40 of its origin
        d["lastg"][:, 0] = np.float32(0.9)
        d["g"][:, 1:60] = np.float32(1e-12)
        for s in range(B):
            for t in (7 + s, 20, 21, 33 + 2 * s):
                d["silence"][s, t] = True
        go[:, :50] = 0.0
        go[:, 50:56] = _tone(B, 6, [2.5, 9.0], seed)
    elif kind == "halves":
        go[:, 1::2] = 0.0     # frame t's window holds grad_out[t] alone for odd t + 1, grad_out[t + 1] alone for even t
    elif kind == "one_band":
        go = _tone(B, T, list(np.arange(48, 60, 1.0)), seed)  # the bins of band 12 (48 .. 59) and no others
    elif kind == "dc_free":
        go = go - go.mean(axis=2, keepdims=True)
    elif kind == "nyquist":
        go = go * 0.05 + np.cos(np.pi * np.arange(480))[None, None, :] * (1 + 0.1 * rng.normal(size=(B, T, 1)))
    if kind in ("odd_shape", "long"):
        for s in range(B):
            d["silence"][s, rng.integers(0, T, 3)] = True
    rechain(d)
    if kind == "chain":
        mk = ref.masks(d)
        reach["floored >= 40 frames in a row"] = np.stack([(~mk["take_g"][:, t:t + 40] | d["silence"][:, t:t + 40, None]).all(axis=1)
                                                           for t in range(1, T - 40)], 1)
    return d, go, reach


def _window(kind):
    """edge_window(kind), or for "synthetic" a synthetic window with silent frames and noise as grad_out."""
    if kind != "synthetic":
        return edge_window(kind)
    d = synthetic_window(4, 12, 11, silent=[(1, 2), (3, 5), (3, 6)])
    return d, np.random.default_rng(12).normal(size=(4, 12, 480)), {}


def _shares(bound, got, g64):
    """|got - g64| / bound per element (the smallest normal f32 where |g64| is below it)."""
    with np.errstate(all="ignore"):
        tol = np.maximum(bound, np.where(np.abs(g64) < ref.TINY, ref.TINY, 0.0))
        return np.where(got == g64, 0.0, np.abs(got - g64) / tol)


@pytest.mark.parametrize("kind", ("synthetic",) + EDGES)
def test_bounds_hold_f32_restatements(kind):
    """Both float32 restatements lie inside grad_bounds on every element."""
    d, go, reach = _window(kind)
    for name, m in reach.items():
        assert m.any(), name
    mk = ref.masks(d)
    g64 = ref.window_grad(d, go, mk=mk)
    bound = ref.grad_bounds(d, go, mk=mk)
    assert np.all(np.isfinite(bound)) and np.all(bound[d["silence"]] == 0)
    for name, got in (("torch f32", ref.window_grad(d, go, dtype=torch.float32, mk=mk)), ("kernel order f32", ref.window_grad_f32(d, go, mk=mk))):
        share = _shares(bound, got, g64)
        worst = np.unravel_index(np.argmax(share), share.shape)
        print("\n%s %s: largest share of the bound %.3g at %s" % (kind, name, share[worst], worst))
        assert share[worst] <= 1.0, (name, worst, got[worst], g64[worst], bound[worst])


# The FFT's per-bin bound C_FFT u sum|h| is about 30 C_FFT u |H_k| for noise-like grad_out and makes nine tenths of the
# median: without it the median is 8e-5.  A per-bin bound of any FFT is at least u sum|h|, so no first-order bound of
# this kind reaches 1e-5 on such windows.
MEDIAN_LIMIT = 3e-3


def test_bound_is_not_a_floor():
    """Over the windows above, the median of bound / |ref| over non-zero elements stays below MEDIAN_LIMIT: the bound
    follows each element, so that a quiet element is held to its own size (the tolerance it replaces gave every element
    1e-4 of the window's peak: 100 times the element itself for a carried gradient at 1e-6 of the peak)."""
    rel = []
    for kind in ("synthetic",) + EDGES:
        d, go, _ = _window(kind)
        g64 = ref.window_grad(d, go)
        b = ref.grad_bounds(d, go)
        nz = g64 != 0
        rel.append(b[nz] / np.abs(g64[nz]))
        print("\n%s: median bound / |ref| %.3g" % (kind, np.median(rel[-1])))
    med = float(np.median(np.concatenate(rel)))
    print("all: median bound / |ref| %.3g" % med)
    assert med < MEDIAN_LIMIT
