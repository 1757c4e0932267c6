"""Per-stage references of the fitting kernels (csrc/fit.cu) with a per-element rounding bound, and an f32 emulation of
their arithmetic (TEST INFRASTRUCTURE).

Every stage is written once, over an arithmetic backend:

  * `E`: float64 values with a bound.  Each operation returns the float64 result of its float64 inputs and a bound on
    |f32 result - float64| that holds for any f32 evaluation whose inputs lie within their own bounds: a worst case over
    summation order (gamma_k = k u / (1 - k u) of the sum of magnitudes), FMA contraction or not (a contracted a b + c
    rounds once where the unfused form rounds twice, so the unfused bound covers both), the libdevice ulp errors
    (tanhf, expf 2 ulp; logf 1 ulp) and IEEE sqrtf and division.  Monotone functions propagate an input's bound by
    evaluating at the ends of its window, so no first-order term is dropped there.  ETA, f32's subnormal spacing, is the
    absolute part of a rounding that underflows.
  * `F32`: numpy float32 in the kernels' order, every operation rounded (no contraction): the emulation.

A stage check feeds the stage the GPU's own inputs to it (its taps), so that errors do not compound: exact inputs, and
the bound covers that stage's rounding only.  The kernels' f32 constants (1e-7f, 1 - 2^-23, 0.499f, (float)(1 / R),
the Adam constants, the f32 parameters) are exact inputs here too: the float64 reference uses the same values.

A branch on a computed value may go either way where its input lies within its bound of the branch point: the bound
then covers both sides, and the element is counted as a tie.  The forward's ReLU at 0 and the Adam clip at +-0.499 are
such branches.  ReLU' at 0 and the loss's clamps at eps and 1 - eps read exact inputs (the GPU's h~ or d; the targets),
so they never tie.
"""
import numpy as np

from nnnoiseless_b200.fit import layer_shapes, unflatten

U = 2.0 ** -24        # unit roundoff of f32
ULP = 2.0 ** -23      # the relative spacing of f32 (1 ulp <= ULP |y| for a normal y)
ETA = 2.0 ** -149
ACT_TANH, ACT_SIGMOID, ACT_RELU = 0, 1, 2
SCRIPT_ACTS = (0, 0, 2, 0, 1, 1)
EPS32 = float(np.float32(1e-7))
ONE_M = float(np.float32(1.0) - np.float32(EPS32))  # 1 - 2^-23
CLIP = float(np.float32(0.499))
B1C = float(np.float32(1.0) - np.float32(0.9))      # the kernel's (1.0f - 0.9f), folded in f32
B2C = float(np.float32(1.0) - np.float32(0.999))
L2C = float(np.float32(2e-6))
C01 = float(np.float32(0.01))  # the loss's 0.01f
SPLIT_ROWS, SPLITS_MAX, BK = 2048, 256, 16


def gamma(k):
    k = np.asarray(k, np.float64)
    return k * U / (1.0 - k * U)


def splitk(K):
    """fit.cu launch_gemm's split of a K-long sum -> (kchunk, splits)."""
    if K <= SPLIT_ROWS:
        return K, 1
    s = min(SPLITS_MAX, -(-K // SPLIT_ROWS))
    kc = (-(-K // s) + BK - 1) // BK * BK
    return kc, -(-K // kc)


class Ties:
    def __init__(self):
        self.count = {}

    def add(self, name, flags):
        self.count[name] = self.count.get(name, 0) + int(np.count_nonzero(flags))


class Val:
    """A float64 value v with a bound e on |f32 - v|."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = np.asarray(v, np.float64)
        self.e = np.zeros_like(self.v) if e is None else np.broadcast_to(np.asarray(e, np.float64), self.v.shape)

    def __getitem__(self, k):
        return Val(self.v[k], self.e[k])


def _rnd(v, e):
    """The rounding of a result whose exact value lies within e of v."""
    return U * (np.abs(v) + e) + ETA


def _mono(f, a):
    """A monotone f of a Val: the largest move of f over the input's window."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        y = f(a.v)
        return y, np.maximum(np.abs(f(a.v + a.e) - y), np.abs(y - f(a.v - a.e)))


class E:
    """The float64-with-bound backend."""
    name = "E"

    def __init__(self):
        self.ties = Ties()

    def c(self, x):
        return Val(x)

    def add(self, a, b):
        v, e = a.v + b.v, a.e + b.e
        return Val(v, e + _rnd(v, e))

    def sub(self, a, b):
        v, e = a.v - b.v, a.e + b.e
        return Val(v, e + _rnd(v, e))

    def mul(self, a, b):
        v = a.v * b.v
        e = np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e
        return Val(v, e + _rnd(v, e))

    def neg(self, a):
        return Val(-a.v, a.e)

    def abs(self, a):
        return Val(np.abs(a.v), a.e)

    def div(self, a, b):
        with np.errstate(divide="ignore", invalid="ignore"):
            v = a.v / b.v
            e = (a.e + np.abs(v) * b.e) / (np.abs(b.v) - b.e)
        return Val(v, e + _rnd(v, e))

    def sqrt(self, a):
        y, e = _mono(lambda x: np.sqrt(np.maximum(x, 0.0)), a)
        return Val(y, e + _rnd(y, e))

    def log(self, a):
        y, e = _mono(np.log, a)
        return Val(y, e + ULP * (np.abs(y) + e) + ETA)

    def tanh(self, a):
        y, e = _mono(np.tanh, a)
        return Val(y, e + 2 * ULP * (np.abs(y) + e) + ETA)

    def sigmoid(self, a):  # 1 / (1 + expf(-x)): expf's 2 ulp, the add and the division
        y, e = _mono(lambda x: 1.0 / (1.0 + np.exp(-x)), a)
        return Val(y, e + (2 * ULP + 2 * U) * (y + e) + 2 * ETA)

    def relu(self, a, name=None):
        y = np.maximum(a.v, 0.0)
        e = np.maximum(np.maximum(a.v + a.e, 0.0) - y, y - np.maximum(a.v - a.e, 0.0))
        if name:
            self.ties.add(name, (np.abs(a.v) <= a.e) & (a.e > 0))
        return Val(y, e)

    def clamp(self, a, lo, hi, name=None):
        y = np.clip(a.v, lo, hi)
        e = np.maximum(np.abs(np.clip(a.v + a.e, lo, hi) - y), np.abs(y - np.clip(a.v - a.e, lo, hi)))
        if name:
            self.ties.add(name, ((np.abs(a.v - lo) <= a.e) | (np.abs(a.v - hi) <= a.e)) & (a.e > 0))
        return Val(y, e)

    def fmin(self, a, c):  # exact inputs only (targets)
        return Val(np.minimum(a.v, c), a.e)

    def fmax(self, a, c):
        return Val(np.maximum(a.v, c), a.e)

    def where(self, m, a, b):
        return Val(np.where(m, a.v, b.v), np.where(m, a.e, b.e))

    def select(self, m, a, b):  # exact condition on exact inputs
        return self.where(m, a, b)

    def dot(self, X, W, b=None, extra=0):
        """X [R][K] @ W [K][N] (+ b after the sum, as gemm_store does), one fma chain per element."""
        K = W.shape[0]
        v = X.v @ W
        mag = np.abs(X.v) @ np.abs(W)
        if b is not None:
            v = v + b
            mag = mag + np.abs(b)
        e = X.e @ np.abs(W) + gamma(K + 1 + extra) * mag + (K + 2) * ETA
        return Val(v, e)

    def gru_pre(self, X, W, b, H, Uh):
        """(X W + b) rounded and stored by the projection, then + H U by the recurrence's fma chain."""
        K, n = W.shape[0], Uh.shape[0]
        v = X.v @ W + b + H.v @ Uh
        mag = np.abs(X.v) @ np.abs(W) + np.abs(b) + np.abs(H.v) @ np.abs(Uh)
        e = X.e @ np.abs(W) + H.e @ np.abs(Uh) + gamma(K + n + 2) * mag + (K + n + 2) * ETA
        return Val(v, e)

    def wsum(self, X, G):
        """X^T G over the rows: fit_gemm's split-K partials summed by fit_reduce."""
        kc, s = splitk(X.v.shape[0])
        return Val(X.v.T @ G.v, gamma(kc + s + 1) * (np.abs(X.v).T @ np.abs(G.v)) + (kc + s) * ETA)


class F32:
    """numpy float32 in the kernels' order, unfused."""
    name = "F32"

    def __init__(self):
        self.ties = Ties()

    def c(self, x):
        return np.asarray(x, np.float32)

    def add(self, a, b):
        return (a + b).astype(np.float32)

    def sub(self, a, b):
        return (a - b).astype(np.float32)

    def mul(self, a, b):
        return (a * b).astype(np.float32)

    def neg(self, a):
        return -a

    def abs(self, a):
        return np.abs(a)

    def div(self, a, b):
        with np.errstate(divide="ignore", invalid="ignore"):
            return (a / b).astype(np.float32)

    def sqrt(self, a):
        return np.sqrt(a).astype(np.float32)

    def log(self, a):
        return np.log(a).astype(np.float32)

    def tanh(self, a):
        return np.tanh(a).astype(np.float32)

    def sigmoid(self, a):
        one = np.float32(1.0)
        with np.errstate(over="ignore"):
            return (one / (one + np.exp(-a))).astype(np.float32)

    def relu(self, a, name=None):
        return np.fmax(a, np.float32(0.0))

    def clamp(self, a, lo, hi, name=None):
        return np.fmin(np.fmax(a, np.float32(lo)), np.float32(hi))

    def fmin(self, a, c):
        return np.fmin(a, np.float32(c))

    def fmax(self, a, c):
        return np.fmax(a, np.float32(c))

    def where(self, m, a, b):
        return np.where(m, a, b).astype(np.float32)

    select = where

    def dot(self, X, W, b=None, extra=0):
        W = W.astype(np.float32)
        acc = np.zeros((X.shape[0], W.shape[1]), np.float32)
        for k in range(W.shape[0]):
            acc = (acc + X[:, k:k + 1] * W[k]).astype(np.float32)
        return acc if b is None else (acc + b.astype(np.float32)).astype(np.float32)

    def gru_pre(self, X, W, b, H, Uh):
        acc = self.dot(X, W, b)
        Uh = Uh.astype(np.float32)
        for k in range(Uh.shape[0]):
            acc = (acc + H[:, k:k + 1] * Uh[k]).astype(np.float32)
        return acc

    def wsum(self, X, G):
        kc, s = splitk(X.shape[0])
        tot = np.zeros((X.shape[1], G.shape[1]), np.float32)
        for z in range(s):
            acc = np.zeros_like(tot)
            for k in range(z * kc, min(X.shape[0], (z + 1) * kc)):
                acc = (acc + X[k][:, None] * G[k][None, :]).astype(np.float32)
            tot = (tot + acc).astype(np.float32)
        return tot


def val(A, x):
    """An exact input (a tap, a row, a parameter) in backend A."""
    return Val(np.asarray(x, np.float64)) if A.name == "E" else np.asarray(x, np.float32)


def cat(A, xs):
    if A.name == "E":
        return Val(np.concatenate([x.v for x in xs], -1), np.concatenate([x.e for x in xs], -1))
    return np.concatenate(xs, -1)


def cols(A, x, lo, hi):
    return x[..., lo:hi]


def act(A, code, a, name=None):
    if code == ACT_TANH:
        return A.tanh(a)
    if code == ACT_SIGMOID:
        return A.sigmoid(a)
    return A.relu(a, name)


def dact(A, code, y):
    """fit_dact: through y = act(x); relu' is 0 at 0."""
    if code == ACT_TANH:
        return A.sub(A.c(1.0), A.mul(y, y))
    if code == ACT_SIGMOID:
        return A.mul(y, A.sub(A.c(1.0), y))
    yv = y.v if A.name == "E" else y
    return val(A, (yv > 0).astype(np.float64))


class Net:
    """The network's f32 parameters (as exact float64) and geometry."""

    def __init__(self, params, widths, acts=SCRIPT_ACTS):
        self.widths = tuple(int(w) for w in widths)
        self.acts = tuple(acts)
        self.flat = np.asarray(params, np.float32)
        self.P = {k: np.asarray(v, np.float64) for k, v in unflatten(self.flat, self.widths).items()}
        nd, nv, nn, ndn = self.widths
        self.n = (nv, nn, ndn)
        self.gru = ("vad_gru", "noise_gru", "denoise_gru")

    def W(self, layer, name="kernel"):
        return self.P[(layer, name)]

    def gru_input(self, A, i, x, d, hs):
        """GRU i's input view at the rows: [d] | [d | vad_h | x] | [vad_h | noise_h | x]."""
        if i == 0:
            return d
        if i == 1:
            return cat(A, [d, hs[0], x])
        return cat(A, [hs[0], hs[1], x])


# ---- forward stages ----

def dense(A, net, x):
    return act(A, net.acts[0], A.dot(x, net.W("input_dense"), net.W("input_dense", "bias")))


def gru_zr(A, net, i, X, hp, silent=None):
    n, L = net.n[i], net.gru[i]
    W, Uh, b = net.W(L), net.W(L, "recurrent_kernel"), net.W(L, "bias")
    zr = A.sigmoid(A.gru_pre(X, W[:, :2 * n], b[:2 * n], hp, Uh[:, :2 * n]))
    z, r = cols(A, zr, 0, n), cols(A, zr, n, 2 * n)
    if silent is not None:
        z = A.where(silent[:, None], val(A, np.ones(z.v.shape if A.name == "E" else z.shape)), z)
    return z, r


def gru_cand(A, net, i, X, rh):
    n, L = net.n[i], net.gru[i]
    W, Uh, b = net.W(L), net.W(L, "recurrent_kernel"), net.W(L, "bias")
    return act(A, net.acts[i + 1], A.gru_pre(X, W[:, 2 * n:], b[2 * n:], rh, Uh[:, 2 * n:]), "relu %s" % L)


def gru_state(A, z, hp, hc):
    return A.add(A.mul(z, hp), A.mul(A.sub(A.c(1.0), z), hc))


def outputs(A, net, hd, hv):
    g = act(A, net.acts[4], A.dot(hd, net.W("denoise_output"), net.W("denoise_output", "bias")))
    v = act(A, net.acts[5], A.dot(hv, net.W("vad_output"), net.W("vad_output", "bias")))
    return g, cols(A, v, 0, 1)


# ---- loss and output gradients ----

def loss_terms(A, g, y, w, v, vt, inv_rows, eps=EPS32, one_m=ONE_M, c01=C01):
    """fit_loss_kernel per row: g [R][22] gains, y [R][22] targets, w, v, vt [R][1], inv_rows the f32 1/R ->
    (dzo [R][22], dzv [R][1], (w cost, w xent, msse) each [R][1]).  eps, one_m, c01: the clamp's constants and the
    weight 0.01 (the semantics' 1e-7, 1 - 1e-7 and 0.01 when composing against tests/fit_ref.py; by default the
    kernel's f32 values)."""
    lo, hi = eps, one_m
    one, eps = A.c(1.0), A.c(eps)
    inv = A.c(inv_rows)
    cost = msse = A.c(0.0)
    dzo = []
    for j in range(g.v.shape[1] if A.name == "E" else g.shape[1]):
        gj, t = cols(A, g, j, j + 1), cols(A, y, j, j + 1)
        mask = A.fmin(A.add(t, one), 1.0)
        sg = A.sqrt(A.fmax(gj, 0.0))
        d = A.sub(sg, A.sqrt(A.fmax(t, 0.0)))
        tc = A.fmin(A.fmax(t, lo), hi)
        la, lb = A.log(A.add(tc, eps)), A.log(A.add(A.sub(one, tc), eps))
        bce = A.neg(A.add(A.mul(gj, la), A.mul(A.sub(one, gj), lb)))
        d2 = A.mul(d, d)
        cost = A.add(cost, A.mul(mask, A.add(A.add(A.mul(A.mul(A.c(10.0), d2), d2), d2), A.mul(A.c(c01), bce))))
        msse = A.add(msse, A.mul(mask, d2))
        inner = A.add(A.mul(A.mul(A.c(40.0), d2), d), A.mul(A.c(2.0), d))
        dcost = A.div(A.mul(mask, A.sub(A.mul(inner, A.div(A.c(0.5), sg)), A.mul(A.c(c01), A.sub(la, lb)))), A.c(22.0))
        q = A.mul(A.mul(A.mul(A.mul(w, inv), A.c(10.0)), dcost), gj)
        dzo.append(A.mul(q, A.sub(one, gj)))
    cost, msse = A.div(cost, A.c(22.0)), A.div(msse, A.c(22.0))
    tc = A.fmin(A.fmax(vt, lo), hi)
    la, lb = A.log(A.add(tc, eps)), A.log(A.add(A.sub(one, tc), eps))
    c = A.mul(A.c(2.0), A.abs(A.sub(vt, A.c(0.5))))
    xent = A.mul(c, A.neg(A.add(A.mul(v, la), A.mul(A.sub(one, v), lb))))
    q = A.mul(A.mul(A.mul(A.mul(w, inv), A.c(0.5)), c), A.neg(A.sub(la, lb)))
    dzv = A.mul(A.mul(q, v), A.sub(one, v))
    return cat(A, dzo), dzv, (A.mul(w, cost), A.mul(w, xent), msse)


def grad_in(A, gg, g, gv, v):
    """fit_grad_in_kernel: the caller's output gradients through the sigmoids."""
    one = A.c(1.0)
    return A.mul(A.mul(gg, g), A.sub(one, g)), A.mul(A.mul(gv, v), A.sub(one, v))


# ---- backward stages ----

def bptt_step(A, net, i, dh, z, r, hc, hp, silent=None, dG=None):
    """One step of fit_gru_bwd_kernel at rows: dh the total dL/dh_t it reads.  dG: the GPU's own (daz | dar | dah) at
    these rows, which the step's sums read in place of its own -> (daz, dar, dah, carry = dL/dh_{t-1} less the later
    layers' part)."""
    n, L = net.n[i], net.gru[i]
    Uh = net.W(L, "recurrent_kernel")
    one = A.c(1.0)
    daz = A.mul(A.mul(A.mul(dh, A.sub(hp, hc)), z), A.sub(one, z))
    dah = A.mul(A.mul(dh, A.sub(one, z)), dact(A, net.acts[i + 1], hc))
    carry = A.mul(dh, z)
    dah_in = dah if dG is None else cols(A, dG, 2 * n, 3 * n)
    drh = A.dot(dah_in, Uh[:, 2 * n:].T)
    dar = A.mul(A.mul(A.mul(drh, hp), r), A.sub(one, r))
    if silent is not None:
        dar = A.where(silent[:, None], val(A, np.zeros(dar.v.shape if A.name == "E" else dar.shape)), dar)
    carry = A.add(carry, A.mul(drh, r))
    zr_in = cat(A, [daz, dar]) if dG is None else cols(A, dG, 0, 2 * n)
    carry = _acc_dot(A, carry, zr_in, Uh[:, :2 * n].T)
    return daz, dar, dah, carry


def _acc_dot(A, c, X, W):
    """c + X W as one fma chain that starts at c."""
    if A.name == "E":
        K = W.shape[0]
        v = c.v + X.v @ W
        mag = np.abs(c.v) + np.abs(X.v) @ np.abs(W)
        return Val(v, c.e + X.e @ np.abs(W) + gamma(K + 1) * mag + (K + 1) * ETA)
    W = W.astype(np.float32)
    for k in range(W.shape[0]):
        c = (c + X[:, k:k + 1] * W[k]).astype(np.float32)
    return c


def dx_chain(A, parts):
    """gemm_dx accumulations into one zeroed buffer, in launch order: parts [(dG [R][K], W^T slice [K][N])]."""
    out = None
    for G, Wt in parts:
        v = A.dot(G, Wt)
        out = v if out is None else A.add(out, v)
    return out


def l2_add(A, g, w):
    """fit_adam_kernel's g += 2e-6f w."""
    return A.add(g, A.mul(A.c(L2C), w))


def adam(A, w, g, m, v, lr_t):
    """fit_adam_kernel on the full gradient g (L2 included) -> (w, m, v)."""
    m = A.add(m, A.mul(A.sub(g, m), A.c(B1C)))
    v = A.add(v, A.mul(A.sub(A.mul(g, g), v), A.c(B2C)))
    w = A.sub(w, A.div(A.mul(A.c(lr_t), m), A.add(A.sqrt(v), A.c(EPS32))))
    return A.clamp(w, -CLIP, CLIP, "adam clip"), m, v


def lr_t(step):
    return float(np.float32(1e-3 * np.sqrt(1.0 - 0.999 ** step) / (1.0 - 0.9 ** step)))


def l2_mask(widths):
    """The flat parameters the L2 term covers: the GRUs' kernel and recurrent matrices."""
    out = []
    for layer, name, shape in layer_shapes(widths):
        out.append(np.full(int(np.prod(shape)), layer.endswith("_gru") and name != "bias"))
    return np.concatenate(out)


# ---- the network, composed stage by stage ----

def _rows(a, S, T):
    return a.reshape(S * T, -1)


def forward(A, net, x, silent=None, h0=None):
    """Every forward stage composed in backend A over x [S][T][42] (silent [S][T] bool, h0 [S][nv + nn + ndn]) ->
    taps: d [S][T][nd], gates / rh / hbuf per GRU as fit_get_taps lays them out, gains, vad."""
    S, T, _ = x.shape
    xr = val(A, x.reshape(S * T, -1))
    d = dense(A, net, xr)
    get = (lambda a: a.v) if A.name == "E" else (lambda a: a)
    dS = get(d).reshape(S, T, -1)
    out = dict(d=dS, gates=[], rh=[], hbuf=[])
    hs_t = []  # per GRU, h_t [S][T][n]
    for i in range(3):
        n = net.n[i]
        h = np.zeros((S, n)) if h0 is None else np.asarray(h0, np.float64)[:, sum(net.n[:i]):sum(net.n[:i + 1])]
        hb = [h]
        gates = np.zeros((S, T, 3 * n))
        rhs = np.zeros((S, T, n))
        for t in range(T):
            X = net.gru_input(A, i, val(A, x[:, t]), val(A, dS[:, t]), [val(A, hh[:, t]) for hh in hs_t])
            hp = val(A, hb[-1])
            sil = None if silent is None else silent[:, t]
            z, r = gru_zr(A, net, i, X, hp, sil)
            rh = A.mul(r, hp)
            hc = gru_cand(A, net, i, X, rh)
            hn = gru_state(A, z, hp, hc)
            gates[:, t] = np.concatenate([get(z), get(r), get(hc)], -1)
            rhs[:, t] = get(rh)
            hb.append(get(hn))
        hbuf = np.stack(hb, 1)
        hs_t.append(hbuf[:, 1:])
        out["gates"].append(gates)
        out["rh"].append(rhs)
        out["hbuf"].append(hbuf)
    g, v = outputs(A, net, val(A, _rows(hs_t[2], S, T)), val(A, _rows(hs_t[0], S, T)))
    out["gains"], out["vad"] = get(g).reshape(S, T, -1), get(v).reshape(S, T)
    return out


def backward(A, net, x, tp, dzo, dzv, silent=None):
    """Every backward stage composed in backend A from the forward taps tp and the output gradients dzo [S][T][22],
    dzv [S][T] -> dict(dh, dG, dht per GRU, dd, grad: the flat data gradient, no L2)."""
    S, T, _ = x.shape
    R = S * T
    get = (lambda a: a.v) if A.name == "E" else (lambda a: a)
    nd, nv, nn, ndn = net.widths
    xr = val(A, x.reshape(R, -1))
    d = val(A, tp["d"].reshape(R, -1))
    hs = [val(A, _rows(h[:, 1:], S, T)) for h in tp["hbuf"]]
    hprev = [val(A, _rows(h[:, :-1], S, T)) for h in tp["hbuf"]]
    dzo_, dzv_ = val(A, dzo.reshape(R, -1)), val(A, dzv.reshape(R, 1))
    W3, W2 = net.W("denoise_gru"), net.W("noise_gru")
    dh_ext = [None, None, None]
    dh_ext[2] = dx_chain(A, [(dzo_, net.W("denoise_output").T)])
    dG, dht = [None] * 3, [None] * 3
    pend0 = [(dzv_, net.W("vad_output").T)]
    pend1 = []
    pend_dd = []
    for i in (2, 1, 0):
        n = net.n[i]
        if i == 1:
            dh_ext[1] = dx_chain(A, pend1)
        if i == 0:
            dh_ext[0] = dx_chain(A, pend0)
        ext = get(dh_ext[i]).reshape(S, T, n)
        g = tp["gates"][i]
        carry = np.zeros((S, n))
        dGi = np.zeros((S, T, 3 * n))
        dhti = np.zeros((S, T, n))
        for t in range(T - 1, -1, -1):
            dh = A.add(val(A, carry), val(A, ext[:, t]))
            sil = None if silent is None else silent[:, t]
            daz, dar, dah, c = bptt_step(A, net, i, dh, val(A, g[:, t, :n]), val(A, g[:, t, n:2 * n]), val(A, g[:, t, 2 * n:]),
                                         val(A, tp["hbuf"][i][:, t]), sil)
            dGi[:, t] = np.concatenate([get(daz), get(dar), get(dah)], -1)
            dhti[:, t] = get(dh)
            carry = get(c)
        dG[i], dht[i] = dGi, dhti
        G = val(A, dGi.reshape(R, -1))
        if i == 2:
            pend0.append((G, W3[:nv].T))
            pend1.append((G, W3[nv:nv + nn].T))
        elif i == 1:
            pend_dd.append((G, W2[:nd].T))
            pend0.append((G, W2[nd:nd + nv].T))
        else:
            pend_dd.append((G, net.W("vad_gru")[:nd].T))
    dd = A.mul(dx_chain(A, pend_dd), dact(A, net.acts[0], d))
    taps = dict(dh=[get(a).reshape(S, T, -1) for a in dh_ext], dG=dG, dht=dht, dd=get(dd).reshape(S, T, -1))
    taps["grad"] = get(get_concat(A, wgrads(A, net, xr, hs, hprev, tp, taps, dzo_, dzv_, S, T)))
    return taps


def wgrads(A, net, xr, hs, hprev, tp, bt, dzo, dzv, S, T):
    """Every parameter's data gradient from the backward taps bt, in the flat vector's order -> list of (value) arrays."""
    R = S * T
    d = val(A, tp["d"].reshape(R, -1))
    ones = val(A, np.ones((R, 1)))
    out = []
    dd = val(A, bt["dd"].reshape(R, -1))
    out += [A.wsum(xr, dd), A.wsum(ones, dd)]
    for i in range(3):
        n = net.n[i]
        G = val(A, bt["dG"][i].reshape(R, -1))
        X = net.gru_input(A, i, xr, d, hs)
        rh = val(A, tp["rh"][i].reshape(R, -1))
        out.append(A.wsum(X, G))
        out.append(cat(A, [A.wsum(hprev[i], cols(A, G, 0, 2 * n)), A.wsum(rh, cols(A, G, 2 * n, 3 * n))]))
        out.append(A.wsum(ones, G))
    out += [A.wsum(hs[2], dzo), A.wsum(ones, dzo), A.wsum(hs[0], dzv), A.wsum(ones, dzv)]
    return out


def get_concat(A, parts):
    if A.name == "E":
        return Val(np.concatenate([p.v.reshape(-1) for p in parts]), np.concatenate([p.e.reshape(-1) for p in parts]))
    return np.concatenate([p.reshape(-1) for p in parts])


# ---- per-stage checks from a run's own taps ----

def stage_refs(net, x, tp, rows=None, weights=None, gg=None, gv=None, silent=None, seqs=None, grads=True, l2=False):
    """Every stage's float64 reference and bound, each from the run's own inputs to it: {stage: (got, Val)} over the
    sequences `seqs` (None: all).  tp: the run's taps (fit.Fit.taps plus gains, vad and, for gradients, grad: the data
    gradient).  The rows path passes rows and weights (the loss); the device path gg, gv (fit_grad_in)."""
    A = E()
    S_all, T, _ = x.shape
    sq = np.arange(S_all) if seqs is None else np.asarray(seqs)
    S = len(sq)
    R = S * T
    pick = lambda a: np.asarray(a)[sq]  # noqa: E731
    rw = lambda a: val(A, pick(a).reshape(R, -1))  # noqa: E731
    out = {}
    sil = None if silent is None else pick(silent).reshape(R)
    xr = rw(x)
    out["dense"] = (pick(tp["d"]).reshape(R, -1), dense(A, net, xr))
    d = rw(tp["d"])
    hs = [val(A, pick(h)[:, 1:].reshape(R, -1)) for h in tp["hbuf"]]
    hprev = [val(A, pick(h)[:, :-1].reshape(R, -1)) for h in tp["hbuf"]]
    for i in range(3):
        n, L = net.n[i], net.gru[i]
        g = rw(tp["gates"][i])
        X = net.gru_input(A, i, xr, d, hs)
        z, r = gru_zr(A, net, i, X, hprev[i], sil)
        out[L + ".z"] = (g.v[:, :n], z)
        out[L + ".r"] = (g.v[:, n:2 * n], r)
        rh = rw(tp["rh"][i])
        out[L + ".rh"] = (rh.v, A.mul(g[:, n:2 * n], hprev[i]))
        out[L + ".hc"] = (g.v[:, 2 * n:], gru_cand(A, net, i, X, rh))
        out[L + ".h"] = (hs[i].v, gru_state(A, g[:, :n], hprev[i], g[:, 2 * n:]))
    gains, vad = outputs(A, net, hs[2], hs[0])
    out["gains"] = (pick(tp["gains"]).reshape(R, -1), gains)
    out["vad"] = (pick(tp["vad"]).reshape(R, 1), vad)
    if not grads:
        return out, A.ties.count
    G_ = rw(tp["gains"])
    V_ = rw(tp["vad"])
    if rows is not None:
        rws = pick(rows).reshape(R, -1)
        dzo, dzv, terms = loss_terms(A, G_, val(A, rws[:, 42:64]), rw(weights), V_, val(A, rws[:, 86:87]),
                                     float(np.float32(1.0 / (S_all * T))))
        out["loss rows"] = (None, terms)
    else:
        dzo, dzv = grad_in(A, rw(gg), G_, rw(gv), V_)
        if sil is not None:
            z = val(A, np.zeros(R))
            dzo = A.where(sil[:, None], val(A, np.zeros(dzo.v.shape)), dzo)
            dzv = A.where(sil[:, None], z[:, None], dzv)
    out["dzo"] = (pick(tp["dzo"]).reshape(R, -1), dzo)
    out["dzv"] = (pick(tp["dzv"]).reshape(R, 1), dzv)
    # dX: every gemm_dx from the run's own dzo, dzv and dG, and dd *= act'(d)
    nd, nv, nn, ndn = net.widths
    W3, W2 = net.W("denoise_gru"), net.W("noise_gru")
    dG = [rw(a) for a in tp["dG"]]
    dzo_, dzv_ = rw(tp["dzo"]), rw(tp["dzv"])
    ext = [dx_chain(A, [(dzv_, net.W("vad_output").T), (dG[2], W3[:nv].T), (dG[1], W2[nd:nd + nv].T)]),
           dx_chain(A, [(dG[2], W3[nv:nv + nn].T)]),
           dx_chain(A, [(dzo_, net.W("denoise_output").T)])]
    for i in range(3):
        out[net.gru[i] + ".dh"] = (rw(tp["dh"][i]).v, ext[i])
    out["dd"] = (rw(tp["dd"]).v, A.mul(dx_chain(A, [(dG[1], W2[:nd].T), (dG[0], net.W("vad_gru")[:nd].T)]),
                                      dact(A, net.acts[0], d)))
    # BPTT, one step at a time from the run's own dh_t, gates, states and dG
    for i in range(3):
        n, L = net.n[i], net.gru[i]
        dht = pick(tp["dht"][i])
        g = pick(tp["gates"][i])
        hp = pick(tp["hbuf"][i])[:, :-1]
        dGi = pick(tp["dG"][i])
        ext_i = pick(tp["dh"][i])
        flat = lambda a: val(A, a.reshape(R, -1))  # noqa: E731
        daz, dar, dah, carry = bptt_step(A, net, i, flat(dht), flat(g[..., :n]), flat(g[..., n:2 * n]), flat(g[..., 2 * n:]), flat(hp),
                                         sil, flat(dGi))
        out[L + ".daz"] = (dGi[..., :n].reshape(R, -1), daz)
        out[L + ".dar"] = (dGi[..., n:2 * n].reshape(R, -1), dar)
        out[L + ".dah"] = (dGi[..., 2 * n:].reshape(R, -1), dah)
        # dh_{t-1} = carry_t + the later layers' dh_{t-1}; at t = T - 1 the carry is 0
        c = Val(carry.v.reshape(S, T, n)[:, 1:], carry.e.reshape(S, T, n)[:, 1:])
        prev = A.add(c, val(A, ext_i[:, :-1]))
        first = val(A, ext_i[:, -1:])
        out[L + ".dht"] = (np.concatenate([dht[:, :-1], dht[:, -1:]], 1).reshape(R, -1),
                           Val(np.concatenate([prev.v, first.v], 1).reshape(R, -1), np.concatenate([prev.e, first.e], 1).reshape(R, -1)))
    if seqs is None:
        bt = dict(dd=tp["dd"], dG=tp["dG"])
        g = get_concat(A, wgrads(A, net, xr, hs, hprev, tp, bt, dzo_, dzv_, S, T))
        if l2:  # the rows path reads the gradient back after fit_adam_kernel added the L2 term
            m = l2_mask(net.widths)
            g = A.where(m, l2_add(A, g, val(A, net.flat)), g)
        out["wgrad"] = (tp["grad"], g)
    return out, A.ties.count


def loss_totals(terms, R):
    """fit_finish_kernel's f64 sums of the rows' f32 terms -> {mycost, crossentropy, msse} as Val."""
    out = {}
    for k, t in zip(("mycost", "crossentropy", "msse"), terms):
        s = float(t.v.sum()) / R
        out[k] = Val(s, float(t.e.sum()) / R + 2.0 ** -52 * (len(t.v) + 2) * float(np.abs(t.v).sum() + t.e.sum()) / R)
    return out


def shares(out, K=2.0):
    """{stage: (largest |got - ref| / bound, index of that element, got, ref, bound)}; a stage fails where the share
    exceeds K.  0 where got equals ref; inf where the bound is 0 and the two differ."""
    res = {}
    for k, (got, ref) in out.items():
        if got is None:
            continue
        got = np.asarray(got, np.float64).reshape(ref.v.shape)
        err = np.abs(got - ref.v)
        with np.errstate(divide="ignore", invalid="ignore"):
            s = np.where(err == 0.0, 0.0, err / ref.e)
        s = np.where(np.isnan(s), np.inf, s)
        i = int(np.argmax(s)) if s.size else 0
        res[k] = (float(s.reshape(-1)[i]) if s.size else 0.0, np.unravel_index(i, s.shape) if s.size else (), float(got.reshape(-1)[i]) if s.size else 0.0,
                  float(ref.v.reshape(-1)[i]) if s.size else 0.0, float(ref.e.reshape(-1)[i]) if s.size else 0.0)
    return res


def cancelling_gv(gv, vad, silent):
    """gv [S][T] with its last live (not silent) frame changed so that sum(gv v (1 - v)) over the live frames, the vad
    output bias's gradient, cancels to about its rounding: a sum whose float32 restatement error is no measure of it."""
    gv = np.array(gv, np.float32)
    v = np.asarray(vad, np.float64)
    live = np.ones(gv.shape, bool) if silent is None else ~np.asarray(silent)
    if live.sum() < 2:
        return gv
    s, t = [int(i[-1]) for i in np.nonzero(live)]
    w = v * (1.0 - v)
    rest = float((np.where(live, gv * w, 0.0)).sum() - gv[s, t] * w[s, t])
    gv[s, t] = np.float32(-rest / w[s, t])
    return gv


def run(A, case, semantic=False):
    """A whole fitting pass of `case` (tests/fit_cases.py) composed in backend A -> taps as stage_refs reads them: the
    rows path's loss gradients, or the device path's (silent, h0, gg, gv), and the data gradient.  semantic: the loss
    with the semantics' constants (1 / R, 1e-7, 1 - 1e-7, 0.01) in place of the kernel's f32 ones."""
    net = Net(case["params"], case["widths"])
    x = case["x"]
    S, T, _ = x.shape
    R = S * T
    sil = case.get("silent")
    dev = "gg" in case
    xin = np.where(sil[..., None], 0.0, x).astype(np.float32) if sil is not None else x  # fit_pack zeroes silent rows
    tp = forward(A, net, xin, sil if dev else None, case.get("h0"))
    get = (lambda a: a.v) if A.name == "E" else (lambda a: a)
    G, V = val(A, tp["gains"].reshape(R, -1)), val(A, tp["vad"].reshape(R, 1))
    if dev:
        if case.get("cancel_vad"):
            case["gv"] = cancelling_gv(case["gv"], tp["vad"], sil)
        dzo, dzv = grad_in(A, val(A, case["gg"].reshape(R, -1)), G, val(A, case["gv"].reshape(R, 1)), V)
        dzo, dzv = get(dzo), get(dzv)
        if sil is not None:
            dzo = np.where(sil.reshape(R, 1), 0.0, dzo)
            dzv = np.where(sil.reshape(R, 1), 0.0, dzv)
        terms = None
    else:
        rw = case["rows"].reshape(R, -1)
        consts = (1.0 / R, 1e-7, 1.0 - 1e-7, 0.01) if semantic else (float(np.float32(1.0 / R)), EPS32, ONE_M, C01)
        dzo, dzv, terms = loss_terms(A, G, val(A, rw[:, 42:64]), val(A, case["weights"].reshape(R, 1)), V, val(A, rw[:, 86:87]),
                                     *consts)
        dzo, dzv = get(dzo), get(dzv)
    tp["dzo"], tp["dzv"] = dzo.reshape(S, T, -1), dzv.reshape(S, T)
    bt = backward(A, net, xin, tp, tp["dzo"], tp["dzv"], sil if dev else None)
    tp.update(bt)
    tp["x"], tp["terms"] = xin, terms
    return net, tp


def check_run(net, case, tp, seqs=None, grads=True, l2=False):
    """stage_refs for a run's taps under `case`'s inputs."""
    dev = "gg" in case
    return stage_refs(net, tp["x"], tp, rows=None if dev else case["rows"], weights=None if dev else case["weights"],
                      gg=case.get("gg"), gv=case.get("gv"), silent=case.get("silent") if dev else None, seqs=seqs, grads=grads,
                      l2=l2)
