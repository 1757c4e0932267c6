"""Float64 reference of the GRU network (src/rnn.rs:251-379) and a generator of models of any geometry.

TEST INFRASTRUCTURE.  `step` restates RnnModel::compute in float64, vectorised over streams: dense layers, the three
GRUs (reset gate applied to the state before the recurrent product, src/rnn.rs:292-327) and both output layers.  The
activations are the reference's table formulas (src/util.rs:3-53) evaluated in float64 on the table the oracle
exports; np.tanh differs from them by up to 2e-4, far more than the kernels' rounding.

`make_model` writes the binary model format (src/rnn.rs:116-232) for any layer widths the format admits.
"""
import numpy as np

import oracle

NB_BANDS = 22
NB_FEATURES = 42
TANH, SIGMOID, RELU = 0, 1, 2
_TABLE = None


def _table():
    global _TABLE
    if _TABLE is None:
        _TABLE = oracle.tansig_table().astype(np.float64)
    return _TABLE


def tansig(x):
    """src/util.rs:29-45 in float64: the table entry nearest |x| plus a second-order correction."""
    x = np.asarray(x, np.float64)
    ax = np.fmin(np.abs(x), 8.0)  # NaN -> 8: an index in range; the selects below give the saturated values
    fi = np.floor(0.5 + 25.0 * ax)
    d = ax - 0.04 * fi
    y = _table()[fi.astype(np.int64)]
    y = y + d * (1.0 - y * y) * (1.0 - y * d)
    y = np.where(x < 0.0, -y, y)
    y = np.where(x > -8.0, y, -1.0)
    return np.where(x < 8.0, y, 1.0)  # NaN -> 1, like the reference's !(x < 8)


def sigmoid(x):
    return 0.5 + 0.5 * tansig(0.5 * np.asarray(x, np.float64))


def activate(act, x):
    return tansig(x) if act == TANH else (sigmoid(x) if act == SIGMOID else np.maximum(x, 0.0))


def parse(data: bytes):
    """Model bytes -> six layers (input_dense, vad_gru, noise_gru, denoise_gru, denoise_output, vad_output), each a
    dict(ni, nn, act, w [ni][k nn], r [nn][3 nn] (GRUs), b [k nn]) of float64."""
    raw = np.frombuffer(bytes(data), np.int8)
    p, layers = 0, []
    for gates in (1, 3, 3, 3, 1, 1):
        ni, nn, act = int(raw[p]), int(raw[p + 1]), int(raw[p + 2])
        p += 3
        L = dict(ni=ni, nn=nn, act=act)
        L["w"] = raw[p:p + gates * nn * ni].astype(np.float64).reshape(ni, gates * nn)
        p += gates * nn * ni
        if gates == 3:
            L["r"] = raw[p:p + 3 * nn * nn].astype(np.float64).reshape(nn, 3 * nn)
            p += 3 * nn * nn
        L["b"] = raw[p:p + gates * nn].astype(np.float64)
        p += gates * nn
        layers.append(L)
    assert p == len(raw)
    return layers


def _dense(L, x):
    return activate(L["act"], (L["b"] + x @ L["w"]) / 256.0)


def _gru(L, x, h):
    n, W, R, b = L["nn"], L["w"], L["r"], L["b"]
    z = sigmoid((b[:n] + x @ W[:, :n] + h @ R[:, :n]) / 256.0)
    r = sigmoid((b[n:2 * n] + x @ W[:, n:2 * n] + h @ R[:, n:2 * n]) / 256.0)
    c = activate(L["act"], (b[2 * n:] + x @ W[:, 2 * n:] + (r * h) @ R[:, 2 * n:]) / 256.0)
    return z * h + (1.0 - z) * c


def step(layers, state, features):
    """One step of the network for B streams: state [B][nv + nn + ndn] (vad | noise | denoise), features [B][42] ->
    (new state [B][nv + nn + ndn], gains [B][22], vad [B]), float64."""
    dense, vgru, ngru, dgru, out, vout = layers
    nv, nn = vgru["nn"], ngru["nn"]
    state = np.asarray(state, np.float64)
    f = np.asarray(features, np.float64)
    hv, hn, hd = state[:, :nv], state[:, nv:nv + nn], state[:, nv + nn:]
    d = _dense(dense, f)
    hv = _gru(vgru, d, hv)
    vad = _dense(vout, hv)[:, 0]
    hn = _gru(ngru, np.concatenate([d, hv, f], axis=1), hn)
    hd = _gru(dgru, np.concatenate([hv, hn, f], axis=1), hd)
    return np.concatenate([hv, hn, hd], axis=1), _dense(out, hd), vad


def oracle_step(omodel, widths, state, features):
    """The same step through the oracle's f32 rnn_compute (the reference's arithmetic and summation order), stream by
    stream: -> (new state, gains, vad) as float64 arrays shaped like step's."""
    nv, nn, _ = widths
    B = len(state)
    new = np.empty((B, sum(widths)))
    gains = np.empty((B, NB_BANDS))
    vad = np.empty(B)
    for s in range(B):
        sv, sn, sd, g, v = oracle.rnn_step(omodel, state[s, :nv], state[s, nv:nv + nn], state[s, nv + nn:], features[s])
        new[s] = np.concatenate([sv, sn, sd])
        gains[s] = g
        vad[s] = v
    return new, gains, vad


def make_model(nd, nv, nn, ndn, acts=(TANH, TANH, RELU, TANH, SIGMOID, SIGMOID), seed=0) -> bytes:
    """Model bytes of the given layer widths.  acts: activations of input_dense, vad_gru, noise_gru, denoise_gru,
    denoise_output, vad_output.  Every weight matrix and bias vector of two or more entries holds -128 and 127.  The
    input weights reach +-64 and the recurrent ones +-24, so the pre-activations span the curved part of the tables
    and the recurrences neither die nor blow up: ReLU layers stay in the tens, far below 65504 (the f16 limit the
    tensor-core kernels split activations into)."""
    assert 42 + nd + nv <= 127 and 42 + nv + nn <= 127, "the format stores input counts in one signed byte"
    rng = np.random.default_rng(seed)

    def mat(n, lim):
        m = rng.integers(-lim, lim + 1, size=n)
        if n >= 2:
            i, j = rng.choice(n, size=2, replace=False)
            m[i], m[j] = -128, 127
        return m.astype(np.int8).tobytes()

    def header(ni, nno, act):
        return bytes([ni, nno, act])

    def dense(ni, nno, act):
        return header(ni, nno, act) + mat(ni * nno, 64) + mat(nno, 64)

    def gru(ni, nno, act):
        return header(ni, nno, act) + mat(3 * nno * ni, 64) + mat(3 * nno * nno, 24) + mat(3 * nno, 64)

    return (dense(NB_FEATURES, nd, acts[0]) + gru(nd, nv, acts[1]) + gru(NB_FEATURES + nd + nv, nn, acts[2]) +
            gru(NB_FEATURES + nv + nn, ndn, acts[3]) + dense(ndn, NB_BANDS, acts[4]) + dense(nv, 1, acts[5]))
