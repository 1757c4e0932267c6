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
`grad_bounds` is the first-order bound per element of the rounding of any correct float32 evaluation of that gradient,
and `window_grad_f32` evaluates it in float32 in the kernel's summation order.
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


U = sr.U
TINY = 2.0 ** -126  # the smallest normal f32
# Bound of one bin of the 960-point real FFT of the backward (fft480.cuh: 15 = 3 x 5 Good-Thomas, twiddles, a radix-2
# 32-point FFT, the even/odd split), |dH_k| <= C_FFT u sum|h|.  A rounding at any node of the butterfly graph reaches a
# bin with a coefficient of modulus <= 1 before the split (one path per input, unit twiddles) and <= sqrt 2 through it,
# and the nodes of one stage that feed a bin partition the inputs, so a stage whose operations err by at most c u |its
# operands| adds at most c u sum|z| <= c u sum|h| to every bin.  Per stage, as a complex modulus: the 5-point DFT 8.5
# (sqrt 2 gamma_6: five operations deep, constants rounded), the 3-point DFT 5.7 (sqrt 2 gamma_4), the W480 twiddles 4.3
# (sqrt 2 gamma_2 plus the twiddle's rounding), each radix-2 stage 5.3 (the add and its twiddle), five of them 26.5;
# 45 in all, x sqrt 2 through the split, plus 8 for the split's own arithmetic and 1 for rounding 0.5 window grad_out.
C_FFT = 1 + 45 * np.sqrt(2.0) + 8


def _sq_err(v):
    """|fl32(v v) - v^2| for f32 v (the square is exact in float64); where v^2 is below the smallest normal f32, v^2
    itself (a square flushed to zero)."""
    v32 = np.asarray(v, np.float32)
    ex = v32.astype(np.float64) ** 2
    with np.errstate(all="ignore"):
        err = np.abs((v32 * v32).astype(np.float64) - ex)
    return np.where(ex < TINY, np.maximum(err, ex), err)


def q_bound(exp, g):
    """The pitch filter's ratio q = exp^2 (1 - g^2) / (0.001 + g^2 (1 - exp^2)) in float64 from the stored f32 values,
    and the first-order bound of the f32 evaluation K5 and the backward use, with the plain 1 - g2.  g2 = g g is rounded
    once, by a known amount (_sq_err): near g = 1 that rounding, not u |g^2|, is what 1 - g2 loses.  1 - g2 is then exact
    (Sterbenz) or rounded once, or formed by one fused multiply-add: u |1 - g^2| covers each.  -> (q64, dq)."""
    e, gv = np.asarray(exp, np.float64), np.asarray(g, np.float64)
    e2, g2 = e * e, gv * gv
    omg, ome = 1 - g2, 1 - e2
    domg, dome = _sq_err(g) + U * np.abs(omg), _sq_err(exp) + U * np.abs(ome)
    num, den = e2 * omg, sr.C_CORR + g2 * ome
    dnum = np.abs(omg) * _sq_err(exp) + e2 * domg + U * np.abs(num)
    dden = np.abs(ome) * _sq_err(g) + g2 * dome + U * g2 * np.abs(ome) + U * np.abs(den)
    with np.errstate(all="ignore"):
        q = num / den
        dq = dnum / np.abs(den) + np.abs(num) * dden / den ** 2 + U * np.abs(q)
    return q, np.nan_to_num(dq, nan=np.inf)


def masks(d):
    """Kink decisions on the stored f32 values: branch (exp > g), live (0 < q < 1 off the branch), one (r = 1: the
    branch or q >= 1), take_g (g >= 0.6f lastg), ambiguous (the float64 q within its f32 rounding bound, q_bound, of 0
    or 1: an f32 evaluation may take either side of the clamp there)."""
    exp, g = d["exp"], d["g"]
    branch = exp > g
    q = q32(exp, g)
    live = ~branch & (q > 0) & (q < 1)
    one = branch | (~branch & (q >= 1))
    q64, dq = q_bound(exp, g)
    # near 0 only where the other side is a real number (q64 > 0 for the live side)
    amb = ~branch & ((np.abs(q64 - 1) <= dq) | ((np.abs(q64) <= dq) & (live | (q64 > 0))))
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
        # 1 - x^2 as (1 - x)(1 + x) for |x| >= 0.5: the same function, whose float32 evaluation keeps the bits of
        # 1 - g^2 near g = 1 that the backward's derivative relies on (g g rounded would lose them); below 0.5 as
        # 1 - x x, whose derivative autograd forms without the cancellation of (1 - x) - (1 + x)
        omg = torch.where(g.abs() >= 0.5, (1.0 - g) * (1.0 + g), 1.0 - g2)
        ome = torch.where(e.abs() >= 0.5, (1.0 - e) * (1.0 + e), 1.0 - e2)
        q = e2 * omg / (sr.C_CORR + g2 * ome)
        r = torch.where(live, torch.sqrt(torch.where(live, q, torch.full_like(q, 0.5))), one.to(dtype)) * cb
        rf = r @ M.T
        xr = Xr + Pr * rf
        xi = torch.where(dc, Xi, Xi + Pi * rf)
        ne = (xr * xr + xi * xi) @ W.T
        s2 = torch.sqrt(ex) / torch.sqrt(sr.C_EPS + ne)  # not sqrt(ex / ..): finite gradient where ex = 0
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


def _frames(d, go):
    """Per frame t: the float64 K5 intermediates of every stream (spectral_ref.synthesis on the stored lastg) and
    h = 0.5 window (grad_out[t] | grad_out[t+1])."""
    win = sr.tables()["window"]
    B, T = go.shape[:2]
    for ti in range(T):
        o = sr.synthesis(d["X"][:, ti], d["P"][:, ti], d["ex"][:, ti], d["ep"][:, ti], d["exp"][:, ti], d["g"][:, ti],
                         d["lastg"][:, ti], np.zeros((B, F)), d["silence"][:, ti])
        gw = np.concatenate([go[:, ti], go[:, ti + 1] if ti + 1 < T else np.zeros((B, F))], axis=1)
        yield ti, o, 0.5 * win * gw


def grad_bounds(d, grad_out, mk=None):
    """First-order bound [B][T][22] of |g32 - window_grad(d, grad_out)| for a correct f32 implementation of the
    backward with any summation order, on the stored f32 inputs d (parse_ctx) and grad_out [B][T][480].  Step by step:
      - forward: q with the plain 1 - g2 (q_bound), r, rf, x, new_e, s2, rf2 (spectral_ref.spectrum_bounds); gg is
        0.6f lastg after j floored frames, rounded j times from the float64 chain;
      - H = rfft960(h): C_FFT u sum|h| per bin (C_FFT); gy = c_k H;
      - the three band reductions dL/dgg = M^T (rf2 gy.x), dL/ds2 = M^T (gf gy.x), dL/dr = M^T ((dL/dx).P), each
        (gamma_n + 2u) sum|terms| (n <= MAX_BAND_TERMS the band's terms, 2u for the f32 fractions) plus the propagated
        bounds of the terms;
        dL/dx = gy rf2 gf + 2 x W^T (dL/ds2 . -s2 / (2 (1e-8 + new_e))), first and last band doubled;
      - the pitch filter's dL/dg = dL/dr cb 0.5 / sqrt(q) dq with dq from (1 - g)(1 + g) and (1 - exp)(1 + exp): dL/dr's
        bound times that factor, plus the factor's own rounding;
      - the reverse scan: the carry's bound is multiplied by 0.6 with one rounding per floored frame, passes silent
        frames unchanged and is dropped at frames that take g.
    Elements of silent frames get 0 (the kernel stores exact zeros).  mk: masks(d)."""
    t = sr.tables()
    M, Wt = t["M"], t["W"]
    mk = mk or masks(d)
    go = np.asarray(grad_out, np.float64)
    B, T = go.shape[:2]
    nb_terms = (M != 0).sum(axis=0)  # terms of each band sum, at most MAX_BAND_TERMS
    assert nb_terms.max() <= sr.MAX_BAND_TERMS
    gam = nb_terms * U / (1 - nb_terms * U) + 2 * U
    ck = np.full(481, 2.0)
    ck[0] = ck[480] = 1.0
    w2 = np.ones(NB)
    w2[0] = w2[-1] = 2.0
    A, dA, R, dR = (np.zeros((B, T, NB)) for _ in range(4))
    nfl = np.zeros((B, NB))  # floored frames since the last frame that took g: roundings in the stored lastg chain
    for ti, o, h in _frames(d, go):
        live, take = mk["live"][:, ti], mk["take_g"][:, ti]
        e, g = d["exp"][:, ti].astype(np.float64), d["g"][:, ti].astype(np.float64)
        sil = d["silence"][:, ti]
        nfl = np.where(sil[:, None], nfl, np.where(take, 0, nfl + 1))
        q, dq = q_bound(d["exp"][:, ti], d["g"][:, ti])
        with np.errstate(all="ignore"):
            eps_ratio = np.where(live, 0.5 * dq / np.where(live, q, 1.0), 0.0)
        sb =sr.spectrum_bounds(o, eps_ratio, dgg=nfl * U * o["gg"])
        x, ax, dx = o["x"], np.abs(o["x"]), sb["dx"]
        s2, ne, rf2, gf = o["s2"], o["new_e"], o["rf2"], o["gf"]
        # the adjoint of the inverse FFT: H and gy = c_k H
        H = np.fft.rfft(h, axis=1)
        dgy = ck * C_FFT * U * np.abs(h).sum(axis=1, keepdims=True)
        gy = ck * H
        gy[:, 0] = gy[:, 0].real
        agy = np.abs(gy)
        uu = gy.real * x.real + gy.imag * x.imag
        au = np.abs(uu)
        du = agy * dx + ax * dgy + 2 * U * agy * ax
        # dL/dgg and dL/ds2
        A[:, ti] = (rf2 * uu) @ M
        dA[:, ti] = (rf2 * du + au * sb["drf2"] + U * rf2 * au) @ M + gam * ((rf2 * au) @ M)
        D = (gf * uu) @ M
        dD = (gf * du + au * sb["dgf"] + U * gf * au) @ M + gam * ((gf * au) @ M)
        # the renormalisation term: dne = -D s2 / (2 (1e-8 + ne)), first and last band doubled; wd = 2 W^T dne
        kap = 0.5 * s2 / (sr.C_EPS + ne) * w2
        dkap = 0.5 * w2 * (sb["ds2"] + s2 * sb["dne"] / (sr.C_EPS + ne)) / (sr.C_EPS + ne) + 3 * U * kap
        dne = -D * kap
        ddne = np.abs(D) * dkap + kap * dD + U * np.abs(dne)
        wd = 2 * (dne @ M.T)
        dwd = 2 * (ddne @ M.T + 4 * U * (np.abs(dne) @ M.T))
        # dL/dx = gy rf2 gf + wd x, and dL/dr = M^T (dL/dx . P) (bin 0: the real part)
        a = rf2 * gf
        da = gf * sb["drf2"] + rf2 * sb["dgf"] + U * a
        gx = gy * a + wd * x
        dgx = a * dgy + agy * da + U * a * agy + np.abs(wd) * dx + ax * dwd + 2 * U * (a * agy + np.abs(wd) * ax)
        Pb = o["Pb"]
        drfk = gx.real * Pb.real + gx.imag * Pb.imag
        drfk[:, 0] = gx[:, 0].real * Pb[:, 0].real
        aP = np.abs(Pb)
        ddrfk = aP * dgx + 2 * U * np.abs(gx) * aP
        dr = drfk @ M
        ddr = ddrfk @ M + gam * (np.abs(drfk) @ M)
        # the pitch filter's derivative, live elements only
        with np.errstate(all="ignore"):
            e2, g2 = e * e, g * g
            omg, ome = (1 - g) * (1 + g), (1 - e) * (1 + e)
            de2, dg2 = _sq_err(d["exp"][:, ti]), _sq_err(d["g"][:, ti])  # e * e and g * g (subnormal squares too)
            num, den = e2 * omg, sr.C_CORR + g2 * ome
            dnum = np.abs(omg) * de2 + 4 * U * np.abs(num)  # (1 - g)(1 + g): three roundings
            dden = np.abs(ome) * dg2 + 4 * U * g2 * np.abs(ome) + U * np.abs(den)
            T1, T2 = e2 * den, num * ome
            dS = den * de2 + e2 * dden + U * np.abs(T1) + np.abs(ome) * dnum + 4 * U * np.abs(T2) + U * np.abs(T1 + T2)
            dqv = -2 * g * (T1 + T2) / den ** 2
            ddq = 2 * np.abs(g) * (dS / den ** 2 + 2 * np.abs(T1 + T2) * dden / np.abs(den) ** 3) + 3 * U * np.abs(dqv)
            cb = np.sqrt(d["ex"][:, ti] / (sr.C_EPS + d["ep"][:, ti]))
            fac = cb * 0.5 / np.sqrt(num / den)
            rfac = 2 * U + 0.5 * (dnum / np.abs(num) + dden / np.abs(den) + U) + U + 2 * U
            Fp = fac * dqv
            Rv = dr * Fp
            dRv = np.abs(Fp) * ddr + np.abs(dr) * (fac * ddq + np.abs(dqv) * fac * rfac) + 2 * U * np.abs(Rv)
        R[:, ti] = np.where(live, Rv, 0.0)
        dR[:, ti] = np.where(live, dRv, 0.0)
        for v in (A, dA, R, dR):
            v[:, ti] = np.where(sil[:, None], 0.0, v[:, ti])
    out = np.zeros((B, T, NB))
    carry, dcarry = np.zeros((B, NB)), np.zeros((B, NB))
    for ti in range(T - 1, -1, -1):
        sil = d["silence"][:, ti][:, None]
        take = mk["take_g"][:, ti]
        dgg = A[:, ti] + carry
        ddgg = dA[:, ti] + dcarry + U * np.abs(dgg)
        val = np.where(take, R[:, ti] + dgg, R[:, ti])
        out[:, ti] = np.where(sil, 0.0, np.where(take, dR[:, ti] + ddgg + U * np.abs(val), dR[:, ti]))
        ncarry = sr.C_FLOOR * dgg
        carry = np.where(sil, carry, np.where(take, 0.0, ncarry))
        dcarry = np.where(sil, dcarry, np.where(take, 0.0, sr.C_FLOOR * ddgg + U * np.abs(ncarry)))
    return out


# ---- the kernel's algorithm in float32 -----------------------------------------------------------------------------
def _segments():
    """The band segments dealt to 32 lanes as synth_grad.cu's tables do: (segment, first bin, bins, offset, 1 / size)."""
    eb = sr.EBAND_5MS
    segs = []
    for sg in range(NB - 1):
        first, size = eb[sg] * 4, (eb[sg + 1] - eb[sg]) * 4
        nl = 1 if size <= 16 else (2 if size <= 32 else (3 if size <= 48 else 4))
        for q in range(nl):
            lo, hi = first + size * q // nl, first + size * (q + 1) // nl
            segs.append((sg, lo, hi - lo, lo - first, np.float32(1.0) / np.float32(size)))
    assert len(segs) == 32
    return segs


def _fma32(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def band_reduce32(v):
    """band_reduce of synth_grad.cu on f32 per-bin values v [B][400]: per lane a sequential fused sum of its bins with
    weights 1 - f and f (f = offset / size in f32), the lanes of a segment added in lane order, then band b = the (1 - f)
    sum of segment b plus the f sum of segment b - 1.  -> [B][22] f32."""
    B = v.shape[0]
    lo = np.zeros((B, NB - 1), np.float32)
    hi = np.zeros((B, NB - 1), np.float32)
    first = {}
    for sg, b0, n, off, inv in _segments():
        a = np.zeros(B, np.float32)
        b = np.zeros(B, np.float32)
        for i in range(n):
            f = np.float32(off + i) * inv
            gw = np.float32(1) - f
            a = _fma32(np.full(B, gw), v[:, b0 + i], a)
            b = _fma32(np.full(B, f), v[:, b0 + i], b)
        if sg in first:
            lo[:, sg] += a
            hi[:, sg] += b
        else:
            first[sg] = True
            lo[:, sg], hi[:, sg] = a, b
    o = np.zeros((B, NB), np.float32)
    o[:, :NB - 1] = lo
    o[:, 1:] += hi
    return o


def _interp32(vb, fr, bi):
    """[B][22] f32 band values at bins k < 400: (1 - fr) v[bi] + fr v[bi + 1]."""
    return (np.float32(1) - fr) * vb[:, bi] + fr * vb[:, bi + 1]


def window_grad_f32(d, grad_out, mk=None):
    """window_grad_manual in float32 arithmetic in the kernel's order: K5's intermediates from the record, an f32 FFT of
    h (pocketfft's, another summation order than the kernel's), band_reduce32's sums, the pitch filter's derivative with
    (1 - x)(1 + x), and the reverse scan.  -> [B][T][22] float64."""
    import scipy.fft
    f32 = np.float32
    mk = mk or masks(d)
    win = sr.tables()["window"].astype(np.float32)
    go = np.asarray(grad_out, np.float32)
    B, T = go.shape[:2]
    eb = np.array(sr.EBAND_5MS) * 4
    k = np.arange(400)
    bi = np.searchsorted(eb, k, side="right") - 1
    fr = (k - eb[bi]).astype(np.float32) / (eb[bi + 1] - eb[bi]).astype(np.float32)
    A = np.zeros((B, T, NB), np.float32)
    R = np.zeros((B, T, NB), np.float32)
    with np.errstate(all="ignore"):
        for ti in range(T):
            X = d["X"][:, ti].astype(np.complex64)[:, :400]
            P = d["P"][:, ti].astype(np.complex64)
            ex, ep, e, g, lg = (d[n][:, ti].astype(np.float32) for n in ("ex", "ep", "exp", "g", "lastg"))
            live, one = mk["live"][:, ti], mk["one"][:, ti]
            cb = np.sqrt(ex / (f32(1e-8) + ep))
            r = np.where(live, q32(e, g), np.where(one, f32(1), f32(0))).astype(np.float32)
            rb = np.sqrt(r) * cb
            gg = np.maximum(g, f32(0.6) * lg)
            rf = _interp32(rb, fr, bi)
            xr = X.real + P.real * rf
            xi = X.imag + P.imag * rf
            xi[:, 0] = X.imag[:, 0]
            ne = band_reduce32(xr * xr + xi * xi)
            ne[:, 0] *= f32(2)
            ne[:, -1] *= f32(2)
            s2 = np.sqrt(ex / (f32(1e-8) + ne))
            gw = np.concatenate([go[:, ti], go[:, ti + 1] if ti + 1 < T else np.zeros((B, F), np.float32)], axis=1)
            H = scipy.fft.rfft((f32(0.5) * win) * gw, axis=1)[:, :400]
            assert H.dtype == np.complex64
            gyr, gyi = f32(2) * H.real, f32(2) * H.imag
            gyr[:, 0], gyi[:, 0] = H.real[:, 0], f32(0)
            rf2, gf = _interp32(s2, fr, bi), _interp32(gg, fr, bi)
            u = gyr * xr + gyi * xi
            A[:, ti] = band_reduce32(rf2 * u)
            ds2 = band_reduce32(gf * u)
            dne = ds2 * (f32(-0.5) * s2 / (f32(1e-8) + ne))
            dne[:, 0] *= f32(2)
            dne[:, -1] *= f32(2)
            wd = f32(2) * _interp32(dne, fr, bi)
            a = rf2 * gf
            gxr, gxi = gyr * a + wd * xr, gyi * a + wd * xi
            drf = gxr * P.real + gxi * P.imag
            drf[:, 0] = gxr[:, 0] * P.real[:, 0]
            dr = band_reduce32(drf)
            e2, g2 = e * e, g * g
            omg, ome = (f32(1) - g) * (f32(1) + g), (f32(1) - e) * (f32(1) + e)
            num, den = e2 * omg, f32(0.001) + g2 * ome
            dq = f32(-2) * g * (e2 * den + num * ome) / (den * den)
            R[:, ti] = np.where(live, dr * cb * f32(0.5) / np.sqrt(num / den) * dq, f32(0))
            sil = d["silence"][:, ti][:, None]
            A[:, ti] = np.where(sil, f32(0), A[:, ti])
            R[:, ti] = np.where(sil, f32(0), R[:, ti])
    out = np.zeros((B, T, NB), np.float32)
    carry = np.zeros((B, NB), np.float32)
    for ti in range(T - 1, -1, -1):
        sil = d["silence"][:, ti][:, None]
        take = mk["take_g"][:, ti]
        dgg = A[:, ti] + carry
        out[:, ti] = np.where(sil, f32(0), np.where(take, R[:, ti] + dgg, R[:, ti]))
        carry = np.where(sil, carry, np.where(take, f32(0), f32(0.6) * dgg))
    return out.astype(np.float64)
