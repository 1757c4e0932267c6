"""Float64 restatement of a window of synthesis frames from saved contexts, and of its gradient (DESIGN.md 7i).

TEST INFRASTRUCTURE.  `window_out` restates T consecutive K5 frames (spectral_ref.synthesis chained through lastg and
the overlap memory) as a torch function of the raw gains, written with explicit masks for the kinks so that the contract
of rnnoise_synthesis_backward_device, not autograd's defaults, defines the gradient:
  - the pitch filter's r = 1 branch (exp > g) and the clamp of q to [0, 1] pass no gradient; q's side is decided in f32
    on the stored values, as the kernel decides it;
  - the floor gg = max(g, 0.6f lastg) takes g when g >= 0.6f lastg (stored f32 values), else 0.6 x the previous gg;
  - a silent frame passes X through and keeps lastg.
The inverse FFT is an explicit matrix (c_k cos, c_k sin), so its adjoint is plain.  `window_grad_manual` is the kernel's
algorithm in float64 numpy (the adjoint of the inverse FFT as a forward real FFT with bins 1..479 counted twice, the
renormalisation term, the reverse-time floor scan), checked against autograd and finite differences on the CPU.
"""
import numpy as np
import torch

import spectral_ref as sr

CTX_BYTES = 7552
NB = sr.NB_BANDS
F = 480
_OFF = dict(X=0, P=964, ex=1764, ep=1788, exp=1812, lastg=1836, g=1860, sil=1884)


def parse_ctx(ctx):
    """uint8 [..][7552] records -> dict of X [..][481], P [..][400] complex128, ex, ep, exp, lastg, g [..][22] float32,
    silence [..] bool."""
    c = np.ascontiguousarray(ctx).view(np.float32)
    lead = c.shape[:-1]
    X = c[..., 0:962].reshape(*lead, 481, 2)
    P = c[..., 964:1764].reshape(*lead, 400, 2)
    d = {}
    for k, v in (("X", X), ("P", P)):  # real and imaginary parts assigned, so that the sign of a zero survives
        z = np.empty(v.shape[:-1], complex)
        z.real, z.imag = v[..., 0], v[..., 1]
        d[k] = z
    for k in ("ex", "ep", "exp", "lastg", "g"):
        d[k] = c[..., _OFF[k]:_OFF[k] + NB].copy()
    d["silence"] = c[..., _OFF["sil"]].view(np.int32) != 0
    return d


def make_ctx(X, P, ex, ep, exp, lastg, g, silence):
    """The inverse of parse_ctx (for contexts built on the CPU)."""
    lead = np.shape(silence)
    c = np.zeros(lead + (CTX_BYTES // 4,), np.float32)
    c[..., 0:962:2], c[..., 1:962:2] = np.real(X), np.imag(X)
    c[..., 964:1764:2], c[..., 965:1764:2] = np.real(P)[..., :400], np.imag(P)[..., :400]
    for k, v in (("ex", ex), ("ep", ep), ("exp", exp), ("lastg", lastg), ("g", g)):
        c[..., _OFF[k]:_OFF[k] + NB] = v
    c[..., _OFF["sil"]] = np.asarray(silence, np.int32).view(np.float32)
    return c.view(np.uint8)


def q32(exp, g):
    """The pitch filter's ratio in f32 from the stored values, as K5 evaluates it (before the clamp)."""
    e, g = np.float32(exp), np.float32(g)
    with np.errstate(all="ignore"):
        e2, g2 = e * e, g * g
        return e2 * (np.float32(1) - g2) / (np.float32(0.001) + g2 * (np.float32(1) - e2))


def masks(d):
    """Kink decisions on the stored f32 values: branch (exp > g), live (0 < q < 1 off the branch), one (r = 1: the
    branch or q >= 1), take_g (g >= 0.6f lastg), ambiguous (the float64 q within f32 rounding of 0 or 1)."""
    exp, g = d["exp"], d["g"]
    branch = exp > g
    q = q32(exp, g)
    live = ~branch & (q > 0) & (q < 1)
    one = branch | (~branch & (q >= 1))
    e, gg = exp.astype(np.float64), g.astype(np.float64)
    with np.errstate(all="ignore"):
        q64 = e * e * (1 - gg * gg) / (sr.C_CORR + gg * gg * (1 - e * e))
    # near 0 only where the other side is a real number (q64 > 0 for the live side)
    amb = ~branch & ((np.abs(q64 - 1) <= 1e-5) | ((np.abs(q64) <= 1e-5) & (live | (q64 > 0))))
    take_g = g >= np.float32(0.6) * d["lastg"]
    return dict(branch=branch, live=live, one=one, take_g=take_g, ambiguous=amb)


_IM = {}


def _imats(dtype):
    """Cr, Ci [481][960]: w_raw = yr @ Cr - yi @ Ci is the unnormalised inverse real FFT (imaginary parts of bins 0 and
    480 unused)."""
    if dtype not in _IM:
        k = np.arange(481)[:, None]
        n = np.arange(960)[None, :]
        c = np.full((481, 1), 2.0)
        c[0] = c[480] = 1.0
        th = 2 * np.pi * k * n / 960.0
        _IM[dtype] = (torch.tensor(c * np.cos(th), dtype=dtype), torch.tensor(c * np.sin(th), dtype=dtype))
    return _IM[dtype]


def window_out(d, gains, synth_mem0=None, dtype=torch.float64, mk=None):
    """Outputs [B][T][480] of a window from contexts d (parse_ctx of [B][T] records) as a torch function of gains
    [B][T][22] (a tensor of `dtype`); synth_mem0 [B][480]: the overlap memory before frame 0 (zeros if None; it is a
    constant).  mk: masks(d) (or an edited copy)."""
    t = sr.tables()
    T = gains.shape[1]
    tt = lambda a: torch.as_tensor(np.asarray(a), dtype=dtype)  # noqa: E731
    W, M, win = tt(t["W"]), tt(t["M"]), tt(t["window"])
    Cr, Ci = (m.to(dtype) for m in _imats(torch.float64))
    mk = mk or masks(d)
    f = lambda v: float(np.float32(v)) if dtype == torch.float64 else v  # noqa: E731
    B = gains.shape[0]
    lg = tt(d["lastg"][:, 0])
    mem = tt(np.zeros((B, F)) if synth_mem0 is None else synth_mem0)
    dc = torch.zeros(481, dtype=torch.bool)
    dc[0] = True
    outs = []
    for ti in range(T):
        Xr, Xi = tt(d["X"][:, ti].real), tt(d["X"][:, ti].imag)
        Pr = torch.zeros((B, 481), dtype=dtype)
        Pi = torch.zeros((B, 481), dtype=dtype)
        Pr[:, :400], Pi[:, :400] = tt(d["P"][:, ti].real), tt(d["P"][:, ti].imag)
        ex, ep, e = tt(d["ex"][:, ti]), tt(d["ep"][:, ti]), tt(d["exp"][:, ti])
        g = gains[:, ti]
        live, one, take = (torch.as_tensor(mk[k][:, ti]) for k in ("live", "one", "take_g"))
        sil = torch.as_tensor(d["silence"][:, ti])[:, None]
        cb = torch.sqrt(ex / (sr.C_EPS + ep))
        e2, g2 = e * e, g * g
        q = e2 * (1.0 - g2) / (sr.C_CORR + g2 * (1.0 - e2))
        r = torch.where(live, torch.sqrt(torch.where(live, q, torch.full_like(q, 0.5))), one.to(dtype)) * cb
        rf = r @ M.T
        xr = Xr + Pr * rf
        xi = torch.where(dc, Xi, Xi + Pi * rf)
        ne = (xr * xr + xi * xi) @ W.T
        s2 = torch.sqrt(ex / (sr.C_EPS + ne))
        gg = torch.where(take, g, f(0.6) * lg)
        a = (s2 @ M.T) * (gg @ M.T)
        yr = torch.where(sil, Xr, xr * a)
        yi = torch.where(sil, Xi, xi * a)
        lg = torch.where(sil, lg, gg)
        w = 0.5 * win * (yr @ Cr - yi @ Ci)
        outs.append(w[:, :F] + mem)
        mem = w[:, F:]
    return torch.stack(outs, 1)


def window_grad(d, grad_out, synth_mem0=None, dtype=torch.float64, mk=None):
    """dL/dg [B][T][22] for L = sum(grad_out * out), by autograd through window_out."""
    g = torch.tensor(d["g"].astype(np.float64), dtype=dtype, requires_grad=True)
    out = window_out(d, g, synth_mem0, dtype, mk)
    out.backward(torch.as_tensor(np.asarray(grad_out), dtype=dtype))
    return g.grad.numpy().astype(np.float64)


def window_grad_manual(d, grad_out, mk=None):
    """The kernel's algorithm in float64 numpy: per frame the adjoint of y -> 0.5 window irfft, the gain interpolation,
    the renormalisation and the pitch filter, then the floor scan backwards in time."""
    t = sr.tables()
    W, M, win = t["W"], t["M"], t["window"]
    mk = mk or masks(d)
    go = np.asarray(grad_out, np.float64)
    B, T = go.shape[:2]
    A = np.zeros((B, T, NB))
    R = np.zeros((B, T, NB))
    ck = np.full(481, 2.0)
    ck[0] = ck[480] = 1.0
    for ti in range(T):
        gw = np.concatenate([go[:, ti], go[:, ti + 1] if ti + 1 < T else np.zeros((B, F))], axis=1)
        H = np.fft.rfft(0.5 * win * gw, axis=1)  # the adjoint of the inverse FFT is a forward FFT ...
        gy = ck * H                               # ... with bins 1..479 counted twice
        gy[:, 0] = gy[:, 0].real
        X, P = d["X"][:, ti], np.zeros((B, 481), complex)
        P[:, :400] = d["P"][:, ti]
        ex, ep, e, g = (d[k][:, ti].astype(np.float64) for k in ("ex", "ep", "exp", "g"))
        lg = d["lastg"][:, ti].astype(np.float64)
        live, one, take = (mk[k][:, ti] for k in ("live", "one", "take_g"))
        cb = np.sqrt(ex / (sr.C_EPS + ep))
        with np.errstate(all="ignore"):
            q = e * e * (1 - g * g) / (sr.C_CORR + g * g * (1 - e * e))
        r = np.where(live, np.sqrt(np.where(live, q, 0.5)), one) * cb
        rf = r @ M.T
        x = X + P * rf
        x[:, 0] = x[:, 0].real + 1j * X[:, 0].imag
        ne = np.abs(x) ** 2 @ W.T
        s2 = np.sqrt(ex / (sr.C_EPS + ne))
        rf2 = s2 @ M.T
        gg = np.where(take, g, sr.C_FLOOR * lg)
        gf = gg @ M.T
        u = gy.real * x.real + gy.imag * x.imag
        A[:, ti] = (rf2 * u) @ M
        dne = ((gf * u) @ M) * (-0.5 * s2 / (sr.C_EPS + ne))  # the renormalisation term
        gx = gy * rf2 * gf + 2 * x * (dne @ W)
        drf = gx.real * P.real + gx.imag * P.imag
        drf[:, 0] = gx[:, 0].real * P[:, 0].real
        dr = drf @ M
        with np.errstate(all="ignore"):
            den = sr.C_CORR + g * g * (1 - e * e)
            dq = -2 * g * (e * e * den + e * e * (1 - g * g) * (1 - e * e)) / den ** 2
            R[:, ti] = np.where(live, dr * cb * 0.5 / np.sqrt(np.where(live, q, 1.0)) * dq, 0.0)
        sil = d["silence"][:, ti][:, None]
        A[:, ti] = np.where(sil, 0.0, A[:, ti])
        R[:, ti] = np.where(sil, 0.0, R[:, ti])
    out = np.zeros((B, T, NB))
    carry = np.zeros((B, NB))
    for ti in range(T - 1, -1, -1):
        sil = d["silence"][:, ti][:, None]
        dgg = A[:, ti] + carry
        take = mk["take_g"][:, ti]
        out[:, ti] = np.where(sil, 0.0, np.where(take, R[:, ti] + dgg, R[:, ti]))
        carry = np.where(sil, carry, np.where(take, 0.0, sr.C_FLOOR * dgg))
    return out
