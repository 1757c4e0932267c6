"""A per-element bound on one step of the GRU network in f32 on tensor cores, and an f32 emulation of the mma.sync
kernel's arithmetic (TEST INFRASTRUCTURE).

`step_bound(layers, state, features)` returns, next to the float64 step of tests/rnn_ref.py, a first-order bound on
|f32 result - float64| for every new state element, every raw gain and the vad of every stream.  It covers any f32
evaluation that

  * splits each activation operand x into f16 halves hi + lo with |hi + lo - x| <= e_split(x) (the tensor-core
    kernels; an evaluation that does not split, like the oracle's, is covered too),
  * accumulates products of int8 weights and operands (exact in f32) with unit roundoff at most U_TC = 2^-23 (round
    to nearest is not assumed for tensor-core accumulation) in any order, the bias included,
  * evaluates the activation tables (src/util.rs:29-53) in f32 with or without FMA contraction, and
  * forms r.h and the update z.h + (1 - z).c from the f32 previous state the stream holds.

It is propagated layer by layer in the network's order: dense -> vad GRU -> vad output -> noise GRU -> denoise GRU ->
denoise output, each pre-activation a = (b + sum w x) / 256 getting

  da = (sum |w| (dx + e_split(|x| + dx)) + gamma_{2n+2}(U_TC) (|b| + sum |w| (|x| + dx)) (1 + 2^-10)) / 256

and each activation |f'| da (the largest |f'| of the table piece over [a - da, a + da]) plus the formula's own f32
rounding (E_TANH, E_SIGMOID, measured by `table_rounding`).  Where a table-index edge (25 |x| = k + 1/2) or the
saturation at |x| = 8 lies within the window (da plus a few f32 ulps of the index arithmetic), the float64 jump between
the two branches is added: the f32 evaluation may take either branch (a tie, counted per quantity).
"""
import numpy as np

import rnn_ref

U = 2.0 ** -24
U_TC = 2.0 ** -23
ETA = 2.0 ** -149  # f32's subnormal spacing: the absolute part of a rounding that underflows
SPLIT_REL, SPLIT_ABS = 2.0 ** -22, 2.0 ** -25
F16_LIMIT = 65520.0  # |x| >= 65520 rounds to inf in f16: the split's hi, and every product with it, is not finite
# the table formulas' own f32 rounding, with and without FMA contraction: `table_rounding` measures 5.9e-8 for both
# (every 61st f32 in [0, 8) and 64 ulps around every edge); the constants leave a factor of 1.5
E_TANH, E_SIGMOID = 9e-8, 9e-8


def gamma(n, u):
    nu = n * u
    return nu / (1.0 - nu)


def e_split(x):
    """Bound on |hi + lo - x| of the two-f16 split of f32 x: relative 2^-22 (the f16 rounding of the remainder) plus
    the absolute 2^-25 where the remainder (|x| < 2^-3) or hi itself (|x| < 2^-14) is an f16 subnormal."""
    return SPLIT_REL * np.abs(x) + SPLIT_ABS


def split16(x):
    """x (f32) -> (hi, lo) as f32, hi = f16(x), lo = f16(x - hi), both rounded to nearest even."""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        hi = x.astype(np.float16).astype(np.float32)
        lo = (x - hi).astype(np.float16).astype(np.float32)
    return hi, lo


# ---- the table formula, piece by piece ----

def _piece(ax, fi):
    T = rnn_ref._table()[np.clip(fi, 0, 200).astype(np.int64)]
    d = ax - 0.04 * fi
    return T + d * (1.0 - T * T) * (1.0 - T * d)


def _dpiece(ax, fi):
    T = rnn_ref._table()[np.clip(fi, 0, 200).astype(np.int64)]
    d = ax - 0.04 * fi
    return (1.0 - T * T) * (1.0 - 2.0 * T * d)


def _tansig_err(x, dx):
    """First-order bound on |tansig(x~) - tansig(x)| over |x~ - x| <= dx (float64 formula), plus the jump of every
    branch edge inside the window.  -> (bound, tie flags)."""
    ax = np.abs(x)
    slack = dx + 8.0 * U * np.maximum(ax, 1.0 / 25)  # the f32 index arithmetic 0.5 + 25 |x| moves the edge
    lo_, hi_ = np.maximum(ax - slack, 0.0), np.minimum(ax + slack, 8.0)
    dmax = np.zeros_like(ax)
    for p in (lo_, ax, hi_):
        pc = np.minimum(p, 8.0)
        fi = np.floor(0.5 + 25.0 * pc)
        dmax = np.maximum(dmax, np.where(p < 8.0, np.abs(_dpiece(pc, fi)), 0.0))
    err = dmax * dx
    # edges k + 1/2 (k = 0 ... 199) of 25 |x| inside [lo_, hi_], and |x| = 8
    k0 = np.floor(25.0 * lo_ - 0.5)
    k1 = np.floor(25.0 * np.minimum(hi_, 8.0) - 0.5)
    tie = k1 > k0
    jump = np.zeros_like(ax)
    for k in np.unique(k1[tie]) if tie.any() else []:
        e = (k + 0.5) / 25.0
        j = abs(float(_piece(np.float64(e), np.float64(k)) - _piece(np.float64(e), np.float64(k + 1))))
        jump = np.where(tie & (k0 < k) & (k <= k1), np.maximum(jump, j), jump)
    sat = (ax + slack >= 8.0) & (ax - slack < 8.0)
    jump = np.where(sat, np.maximum(jump, np.abs(1.0 - _piece(np.float64(8.0), np.float64(200.0)))), jump)
    more = np.where(tie, k1 - k0, 0)  # several edges inside one window: each may add its jump
    return err + jump * np.maximum(more, 1), tie | sat


def act_bound(act, a, da):
    """-> (f(a) in float64, bound on |f32 f(a~) - f(a)| for |a~ - a| <= da, tie flags)."""
    if act == rnn_ref.RELU:
        return np.maximum(a, 0.0), np.where(a + da > 0.0, da, 0.0), np.zeros(a.shape, bool)
    if act == rnn_ref.TANH:
        e, tie = _tansig_err(a, da)
        return rnn_ref.tansig(a), e + E_TANH, tie
    e, tie = _tansig_err(0.5 * a, 0.5 * da)
    return rnn_ref.sigmoid(a), 0.5 * e + E_SIGMOID, tie


def _contract(W, b, x, dx):
    """Pre-activation (b + x W) / 256 of inputs x [B][n] whose f32 values are within dx -> (a, da)."""
    aW = np.abs(W)
    a = (b + x @ W) / 256.0
    n = W.shape[0]
    mag = (np.abs(b) + (np.abs(x) + dx) @ aW) * (1.0 + 2.0 ** -10)
    da = ((dx + e_split(np.abs(x) + dx)) @ aW + gamma(2 * n + 2, U_TC) * mag) / 256.0
    return a, da


class Ties:
    def __init__(self):
        self.count = {}

    def add(self, name, flags):
        self.count[name] = self.count.get(name, 0) + int(np.count_nonzero(flags))


def _gru(L, x, dx, h, ties, name):
    n, W, R, b = L["nn"], L["w"], L["r"], L["b"]
    xh, dxh = np.concatenate([x, h], axis=1), np.concatenate([dx, np.zeros_like(h)], axis=1)
    Wz, Wr = np.concatenate([W[:, :n], R[:, :n]]), np.concatenate([W[:, n:2 * n], R[:, n:2 * n]])
    z, dz, t = act_bound(rnn_ref.SIGMOID, *_contract(Wz, b[:n], xh, dxh))
    ties.add(name + ".z", t)
    r, dr, t = act_bound(rnn_ref.SIGMOID, *_contract(Wr, b[n:2 * n], xh, dxh))
    ties.add(name + ".r", t)
    rh = r * h
    drh = np.abs(h) * dr + U * np.abs(rh) + ETA
    Wc = np.concatenate([W[:, 2 * n:], R[:, 2 * n:]])
    c, dc, t = act_bound(L["act"], *_contract(Wc, b[2 * n:], np.concatenate([x, rh], axis=1), np.concatenate([dx, drh], axis=1)))
    ties.add(name + ".c", t)
    hn = z * h + (1.0 - z) * c
    dh = (np.abs(h) + np.abs(c)) * dz + (1.0 - z) * dc + dz * dc + 4.0 * U * (np.abs(z * h) + np.abs((1.0 - z) * c)) + 4.0 * ETA
    return hn, dh


def step_bound(layers, state, features, given=None):
    """-> dict(state, gains, vad: the float64 step (rnn_ref.step); d_state, d_gains, d_vad: the bounds; ties: {gate:
    count of elements whose window holds a branch edge}).

    given: the evaluation's own new state [B][nv + nn + ndn].  Each GRU's new state is then checked from float64
    inputs as above, but the layers after it read the given f32 state (exact inputs, no upstream bound), as a layer
    of the kernel reads the state the layer before it wrote.  Propagated through four layers, the worst-case sums
    grow some 25-fold per layer (sum |w| / 256); conditioned on the observed states, only the dense layer's bound
    travels (into the vad GRU and the noise GRU)."""
    dense, vgru, ngru, dgru, out, vout = layers
    nv, nn = vgru["nn"], ngru["nn"]
    state = np.asarray(state, np.float64)
    f = np.asarray(features, np.float64)
    df = np.zeros_like(f)
    hv, hn, hd = state[:, :nv], state[:, nv:nv + nn], state[:, nv + nn:]
    ties = Ties()
    d, dd, t = act_bound(dense["act"], *_contract(dense["w"], dense["b"], f, df))
    ties.add("dense", t)
    g_ = None if given is None else np.asarray(given, np.float64)

    def observed(h, dh, lo, hi):  # what the next layers read
        return (h, dh) if g_ is None else (g_[:, lo:hi], np.zeros_like(dh))

    hv, dhv = _gru(vgru, d, dd, hv, ties, "vad_gru")
    xv, dxv = observed(hv, dhv, 0, nv)
    vad, dvad, t = act_bound(vout["act"], *_contract(vout["w"], vout["b"], xv, dxv))
    ties.add("vad_output", t)
    hn, dhn = _gru(ngru, np.concatenate([d, xv, f], axis=1), np.concatenate([dd, dxv, df], axis=1), hn, ties, "noise_gru")
    xn, dxn = observed(hn, dhn, nv, nv + nn)
    hd, dhd = _gru(dgru, np.concatenate([xv, xn, f], axis=1), np.concatenate([dxv, dxn, df], axis=1), hd, ties, "denoise_gru")
    xd, dxd = observed(hd, dhd, nv + nn, None)
    g, dg, t = act_bound(out["act"], *_contract(out["w"], out["b"], xd, dxd))
    ties.add("denoise_output", t)
    return dict(state=np.concatenate([hv, hn, hd], axis=1), gains=g, vad=vad[:, 0],
                d_state=np.concatenate([dhv, dhn, dhd], axis=1), d_gains=dg, d_vad=dvad[:, 0], ties=ties.count)


def preacts(layers, state, features):
    """Every pre-activation of one float64 step: {layer.gate: [B][n]} (layer.c of a GRU is its candidate)."""
    dense, vgru, ngru, dgru, out, vout = layers
    nv, nn = vgru["nn"], ngru["nn"]
    state = np.asarray(state, np.float64)
    f = np.asarray(features, np.float64)
    hv, hn, hd = state[:, :nv], state[:, nv:nv + nn], state[:, nv + nn:]
    P = {}
    P["dense"] = (dense["b"] + f @ dense["w"]) / 256.0
    d = rnn_ref.activate(dense["act"], P["dense"])

    def gru(L, x, h, name):
        n, W, R, b = L["nn"], L["w"], L["r"], L["b"]
        P[name + ".z"] = (b[:n] + x @ W[:, :n] + h @ R[:, :n]) / 256.0
        P[name + ".r"] = (b[n:2 * n] + x @ W[:, n:2 * n] + h @ R[:, n:2 * n]) / 256.0
        z, r = rnn_ref.sigmoid(P[name + ".z"]), rnn_ref.sigmoid(P[name + ".r"])
        P[name + ".c"] = (b[2 * n:] + x @ W[:, 2 * n:] + (r * h) @ R[:, 2 * n:]) / 256.0
        return z * h + (1.0 - z) * rnn_ref.activate(L["act"], P[name + ".c"])

    hv = gru(vgru, d, hv, "vad_gru")
    P["vad_output"] = (vout["b"] + hv @ vout["w"]) / 256.0
    hn = gru(ngru, np.concatenate([d, hv, f], axis=1), hn, "noise_gru")
    hd = gru(dgru, np.concatenate([hv, hn, f], axis=1), hd, "denoise_gru")
    P["denoise_output"] = (out["b"] + hd @ out["w"]) / 256.0
    return P


# ---- f32 evaluations ----

def tansig32(x, fma=False):
    """The table formula in f32 (src/util.rs:29-45), every operation rounded (fma=False) or the four multiply-adds
    fused (fma=True, each emulated as one float64 operation rounded once: the products of two f32 are exact)."""
    x = np.asarray(x, np.float32)
    f32 = np.float32
    tab = rnn_ref._table().astype(np.float32)
    ax = np.fmin(np.abs(x), f32(8.0))  # fminf: NaN -> 8, an index in range; the selects below give NaN -> 1
    if fma:
        fi = np.floor((0.5 + 25.0 * ax.astype(np.float64)).astype(np.float32))
        d = (ax.astype(np.float64) - np.float64(f32(0.04)) * fi).astype(np.float32)
    else:
        fi = np.floor(f32(0.5) + f32(25.0) * ax)
        d = ax - f32(0.04) * fi
    y = tab[fi.astype(np.int64)]
    if fma:
        y64 = y.astype(np.float64)
        dy = (1.0 - y64 * y64).astype(np.float32)
        t = (1.0 - y64 * d).astype(np.float32)
        y = (y64 + (d * dy).astype(np.float64) * t).astype(np.float32)
    else:
        dy = f32(1.0) - y * y
        y = y + d * dy * (f32(1.0) - y * d)
    y = np.where(x < 0, -y, y)
    y = np.where(x > -8.0, y, f32(-1.0))
    return np.where(x < 8.0, y, f32(1.0)).astype(np.float32)


def sigmoid32(x, fma=False):
    return (np.float32(0.5) + np.float32(0.5) * tansig32(np.float32(0.5) * np.asarray(x, np.float32), fma)).astype(np.float32)


def table_rounding(stride=61):
    """Largest |f32 formula - float64 formula on the same table piece| over every `stride`-th f32 in [0, 8) and every
    f32 within 64 ulps of each edge, with and without contraction -> (tanh, sigmoid)."""
    bits = np.arange(0, np.float32(8.0).view(np.uint32), stride, dtype=np.uint32)
    edges = np.float32((np.arange(200) + 0.5) / 25.0).view(np.uint32)
    near = (edges[:, None].astype(np.int64) + np.arange(-64, 65)[None]).reshape(-1).astype(np.uint32)
    x = np.concatenate([bits, near]).view(np.float32)
    worst = [0.0, 0.0]
    for fma in (False, True):
        for i, (f32fn, scale) in enumerate(((tansig32, 1.0), (sigmoid32, 2.0))):
            xs = (x * np.float32(scale)).astype(np.float32)
            y = f32fn(xs, fma).astype(np.float64)
            # the float64 formula on the piece the f32 index took
            t = np.abs(xs.astype(np.float32) / np.float32(scale)).astype(np.float32)
            if fma:
                fi = np.floor((0.5 + 25.0 * t.astype(np.float64)).astype(np.float32)).astype(np.float64)
            else:
                fi = np.floor(np.float32(0.5) + np.float32(25.0) * t).astype(np.float64)
            ref = _piece(t.astype(np.float64), fi)
            ref = np.where(t < 8.0, ref, 1.0)
            if scale != 1.0:
                ref = 0.5 + 0.5 * ref
            worst[i] = max(worst[i], float(np.abs(y - ref).max()))
    return tuple(worst)


def activate32(act, x):
    if act == rnn_ref.TANH:
        return tansig32(x)
    if act == rnn_ref.SIGMOID:
        return sigmoid32(x)
    return np.fmax(np.asarray(x, np.float32), np.float32(0.0))  # fmaxf: NaN -> 0


def _overflow(x):
    """Rows of x with an operand whose f16 split overflows (hi = +-inf): the kernels mark such a stream."""
    return np.isinf(split16(x)[0]).any(axis=1)


def _contract32(W, b, x):
    """The mma.sync kernel's contraction: the accumulator starts at the bias, then adds every int8 weight times the hi
    and the lo half of each operand (exact products) in f32, one input at a time; then the 1/256 scale."""
    hi, lo = split16(x)
    W32 = W.astype(np.float32)
    acc = np.broadcast_to(b.astype(np.float32), (x.shape[0], W.shape[1])).copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(W.shape[0]):
            acc += W32[k] * hi[:, k:k + 1]
            acc += W32[k] * lo[:, k:k + 1]
    return acc * np.float32(1.0 / 256.0)


def _gru32(L, x, h, ovf):
    n, W, R, b = L["nn"], L["w"], L["r"], L["b"]
    xh = np.concatenate([x, h], axis=1)
    z = sigmoid32(_contract32(np.concatenate([W[:, :n], R[:, :n]]), b[:n], xh))
    r = sigmoid32(_contract32(np.concatenate([W[:, n:2 * n], R[:, n:2 * n]]), b[n:2 * n], xh))
    rh = r * h
    ovf |= _overflow(rh)
    c = activate32(L["act"], _contract32(np.concatenate([W[:, 2 * n:], R[:, 2 * n:]]), b[2 * n:], np.concatenate([x, rh], axis=1)))
    with np.errstate(invalid="ignore", over="ignore"):
        hn = z * h + (np.float32(1.0) - z) * c
    ovf |= _overflow(hn)
    return hn


def emulate_mma(layers, state, features):
    """The mma.sync kernel's arithmetic (rnn_mma.cu) in numpy f32: split operands, exact products, f32 sums, the
    tables in f32, r.h and the update from the f32 state.  A stream with an operand at or above the f16 limit (its
    previous state, features, dense outputs, r.h or new states) reports NaN gains, and a NaN vad when the overflow
    comes before the vad output.  -> (new state, gains, vad) as float64 arrays."""
    dense, vgru, ngru, dgru, out, vout = layers
    nv, nn = vgru["nn"], ngru["nn"]
    state = np.asarray(state, np.float32)
    f = np.asarray(features, np.float32)
    ovf = _overflow(state) | _overflow(f)
    hv, hn, hd = state[:, :nv], state[:, nv:nv + nn], state[:, nv + nn:]
    d = activate32(dense["act"], _contract32(dense["w"], dense["b"], f))
    ovf |= _overflow(d)
    hv = _gru32(vgru, d, hv, ovf)
    vad = np.where(ovf, np.float32(np.nan), activate32(vout["act"], _contract32(vout["w"], vout["b"], hv))[:, 0])
    hn = _gru32(ngru, np.concatenate([d, hv, f], axis=1), hn, ovf)
    hd = _gru32(dgru, np.concatenate([hv, hn, f], axis=1), hd, ovf)
    g = np.where(ovf[:, None], np.float32(np.nan), activate32(out["act"], _contract32(out["w"], out["b"], hd)))
    return (np.concatenate([hv, hn, hd], axis=1).astype(np.float64), g.astype(np.float64), vad.astype(np.float64))


def shares(bound, got):
    """{quantity: |got - float64| / bound} for the three outputs; got = (state, gains, vad).  0 where both are 0 (a
    ReLU state that stays exactly 0); inf where the bound is 0 and the error is not."""
    out = {}
    for q, g in zip(("state", "gains", "vad"), got):
        err = np.abs(np.asarray(g, np.float64) - bound[q])
        with np.errstate(divide="ignore", invalid="ignore"):
            out[q] = np.where(err == 0.0, 0.0, err / bound["d_" + q])
    return out


def check(layers, state, features, got, given=True):
    """step_bound conditioned on got's own state (given=True) -> (bound dict, shares); got = (state, gains, vad)."""
    b = step_bound(layers, state, features, got[0] if given else None)
    return b, shares(b, got)
