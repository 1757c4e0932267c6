"""Constructed GRU states that put one step of the network at the edges where tensor-core arithmetic goes wrong (TEST
INFRASTRUCTURE).

Every case is a previous state for given features: one or two free state elements are solved in float64 so that a
chosen pre-activation (tests/rnn_bounds.preacts) lands where wanted, after the state is rounded to f32.  The features
stay those of the frame they came from, so on the GPU a case is a state record of that frame with its GRU fields
edited (test_rnn_bounds.py), and on the CPU the same state and features go to the oracle and the f32 emulation.

Classes:
  * carry:  the update gate of neuron k driven to a pre-activation of 20 (sigmoid's table saturates at 16: z = 1
            exactly) and h_k set to +-1, 0.3, 1e-2, 1e-4, 1e-6, 1e-8, an f32 subnormal or +-0; the new h_k must equal
            the old one bit for bit (up to the sign of a zero);
  * small:  h_k = 2^-1 ... 2^-30 with the update gate in the curved part (pre-activation 0.7): the split's lo half
            is an f16 subnormal below 2^-3, and hi is too below 2^-14;
  * edge:   a pre-activation at a table-index edge of its activation, 25 |x| = k + 1/2 + m delta (m = -4, -1, 0, 1, 4;
            x = a / 2 for a sigmoid), at |x| = 8 +- delta and at a = 0 +- delta, for the z, r and candidate gates of
            each GRU and both output layers;
  * relu:   a ReLU GRU's state element at 65504, 65519.99, 65520 and 1e5: below 65520 every output is finite and within
            the bound; at 65520 and above the split's hi half is inf, and the kernels report the stream's gains and
            vad as NaN.

The small class holds the update from the f32 state to its bound, but with z in the curved part the new state is
dominated by (1 - z) c, whose bound is larger than the split's 2^-25 floor: an update from the split state would pass
it.  The carry class is the one that catches that (bit for bit).  The dense layer's pre-activations depend on the
features alone, which a state record cannot change: `dense_edges` builds its ladders by editing features, for the
CPU evaluations."""
import numpy as np

import rnn_bounds as rb
import rnn_ref

CARRY_VALUES = [1.0, -1.0, 0.3, 1e-2, 1e-4, 1e-6, 1e-8, float(np.float32(1e-40)), 0.0, -0.0]
SMALL_EXPONENTS = list(range(-1, -31, -1))
LADDER = (-4, -1, 0, 1, 4)
RELU_VALUES = [65504.0, 65519.99, 65520.0, 1e5]
GATES = ["vad_gru.z", "vad_gru.r", "vad_gru.c", "noise_gru.z", "noise_gru.r", "noise_gru.c", "denoise_gru.z",
         "denoise_gru.r", "denoise_gru.c", "vad_output", "denoise_output"]


def _layout(layers):
    nv, nn, nd = layers[1]["nn"], layers[2]["nn"], layers[3]["nn"]
    return {"vad_gru": (0, nv), "noise_gru": (nv, nn), "denoise_gru": (nv + nn, nd), "vad_output": (0, nv),
            "denoise_output": (nv + nn, nd)}


def _act(layers, key):
    name, _, gate = key.partition(".")
    L = layers[["dense", "vad_gru", "noise_gru", "denoise_gru", "denoise_output", "vad_output"].index(name)]
    return rnn_ref.SIGMOID if gate in ("z", "r") else L["act"]


def _solve(layers, state, features, key, j, target, free):
    """Set state[free[0]], then state[free[1]] (a fine correction), so that preacts[key][j] = target after the f32
    rounding of the state; secant steps in float64.  -> the reached pre-activation."""
    s = state.copy()
    f = features[None]

    def pa(v, m):
        t = s.copy()
        t[m] = v
        return float(rb.preacts(layers, t[None].astype(np.float32).astype(np.float64), f)[key][0, j])

    for m in free * 3:  # alternate: the coarse element, then the fine correction, three times
        x0, x1 = float(s[m]), float(s[m]) + 1e-3 * max(1.0, abs(float(s[m])))
        y0, y1 = pa(x0, m) - target, pa(x1, m) - target
        for _ in range(30):
            if y1 == y0 or abs(y1) < 1e-14:
                break
            x0, x1 = x1, x1 - y1 * (x1 - x0) / (y1 - y0)
            y0, y1 = y1, pa(x1, m) - target
        s[m] = np.float32(x1)
    return s.astype(np.float32), pa(float(s[free[-1]]), free[-1])


def _free(layers, key, j, avoid):
    """Two state elements that move preacts[key][j]: the one whose recurrent (or output) weight is largest, and one
    with the smallest nonzero weight for the correction.  None when the layer has no such element."""
    name, _, gate = key.partition(".")
    off, n = _layout(layers)[name]
    if name.endswith("_output"):
        L = layers[4] if name == "denoise_output" else layers[5]
        w = np.abs(L["w"][:, j])
        g = 0
    else:
        L = layers[["vad_gru", "noise_gru", "denoise_gru"].index(name) + 1]
        g = "zrc".index(gate)
        w = np.abs(L["r"][:, g * n + j])
    w = np.where(np.isin(np.arange(n), avoid), 0.0, w)
    if not (w > 0).any():
        return None
    big = int(np.argmax(w))
    w2 = np.where(np.arange(n) == big, 0.0, w)
    nz = np.flatnonzero(w2 > 0)
    small = int(nz[np.argsort(w2[nz])[len(nz) // 4]]) if len(nz) else big  # a lower-quartile weight
    return [off + big, off + small]


def build(layers, state, features, seed=0):
    """-> list of dict(cls, key, j, state (f32 [S]), target, reached, plus class data): cases for one stream's
    (state, features)."""
    rng = np.random.default_rng(seed)
    state = np.asarray(state, np.float32)
    features = np.asarray(features, np.float32)
    cases = []
    for name in ("vad_gru", "noise_gru", "denoise_gru"):
        off, n = _layout(layers)[name]
        if n < 2:
            continue
        key = name + ".z"
        for v in CARRY_VALUES:
            k = int(rng.integers(n))
            s = state.copy()
            s[off + k] = np.float32(v)
            fr = _free(layers, key, k, [k])
            if fr is None:
                continue
            s, reached = _solve(layers, s, features, key, k, 20.0, fr)
            cases.append(dict(cls="carry", key=key, j=k, elem=off + k, value=np.float32(v), state=s, target=20.0,
                              reached=reached, ok=reached >= 16.5))
        for e in SMALL_EXPONENTS[::3] if name != "vad_gru" else SMALL_EXPONENTS:
            k = int(rng.integers(n))
            s = state.copy()
            s[off + k] = np.float32(np.ldexp(1.0, e)) * (1 if e % 2 else -1)
            fr = _free(layers, key, k, [k])
            if fr is None:
                continue
            s, reached = _solve(layers, s, features, key, k, 0.7, fr)
            cases.append(dict(cls="small", key=key, j=k, elem=off + k, state=s, target=0.7, reached=reached,
                              ok=abs(reached - 0.7) < 1e-3))
    for key in GATES:
        name = key.partition(".")[0]
        act = _act(layers, key)
        off, n = _layout(layers)[name]
        nout = layers[4]["nn"] if name == "denoise_output" else (1 if name == "vad_output" else n)
        if n < 2 or nout < 1:
            continue
        j = int(rng.integers(nout))
        fr = _free(layers, key, j, [j] if not name.endswith("_output") else [])
        if fr is None:
            continue
        half = 2.0 if act == rnn_ref.SIGMOID else 1.0  # the table sees a / 2 for a sigmoid
        targets = []
        if act != rnn_ref.RELU:
            kk = int(rng.integers(3, 60))
            sign = 1.0 if rng.random() < 0.5 else -1.0
            edge = sign * half * (kk + 0.5) / 25.0
            targets += [edge * (1.0 + m * 2.0 ** -21) for m in LADDER]
            targets += [sign * half * 8.0 * (1.0 + m * 2.0 ** -21) for m in LADDER]
        targets += [m * 2.0 ** -21 for m in LADDER]
        for t in targets:
            s, reached = _solve(layers, state.copy(), features, key, j, t, fr)
            tol = max(2.0 ** -23 * abs(t), 2.0 ** -23)  # a quarter of the ladder's step near a = 0
            cases.append(dict(cls="edge", key=key, j=j, state=s, target=t, reached=reached,
                              ok=abs(reached - t) <= tol and np.abs(s).max() < 1e3))  # far from the f16 limit
    for name, L in zip(("vad_gru", "noise_gru", "denoise_gru"), layers[1:4]):
        off, n = _layout(layers)[name]
        if L["act"] != rnn_ref.RELU or n < 1:
            continue
        for v in RELU_VALUES:
            k = int(rng.integers(n))
            s = state.copy()
            s[off + k] = np.float32(v)
            cases.append(dict(cls="relu", key=name, j=k, elem=off + k, value=np.float32(v), state=s, target=v,
                              reached=float(s[off + k]), ok=True, overflow=bool(np.float32(v) >= rb.F16_LIMIT)))
    return cases


def dense_edges(layers, features, seed=0):
    """Feature vectors whose dense-layer pre-activation of one neuron sits on the same ladders as the `edge` class
    (table edge, |x| = 8 and 0, for the layer's activation): one feature element solved in float64, a second one
    correcting the f32 rounding.  -> list of dict(target, reached, features, ok)."""
    rng = np.random.default_rng(seed)
    L = layers[0]
    if L["nn"] < 1:
        return []
    j = int(rng.integers(L["nn"]))
    w = np.abs(L["w"][:, j])
    order = np.argsort(w)
    big = int(order[-1])
    nz = order[w[order] > 0]
    small = int(nz[len(nz) // 4])
    half = 2.0 if L["act"] == rnn_ref.SIGMOID else 1.0
    targets = [m * 2.0 ** -21 for m in LADDER]
    if L["act"] != rnn_ref.RELU:
        kk = int(rng.integers(3, 60))
        targets += [half * (kk + 0.5) / 25.0 * (1.0 + m * 2.0 ** -21) for m in LADDER]
        targets += [-half * 8.0 * (1.0 + m * 2.0 ** -21) for m in LADDER]
    out = []
    for t in targets:
        f = np.asarray(features, np.float64).copy()
        for m in (big, small, big, small):
            a = (L["b"][j] + np.float32(f).astype(np.float64) @ L["w"][:, j]) / 256.0
            f[m] = np.float32(f[m] + (t - a) * 256.0 / L["w"][m, j])
        f = f.astype(np.float32)
        reached = float((L["b"][j] + f.astype(np.float64) @ L["w"][:, j]) / 256.0)
        out.append(dict(target=t, reached=reached, features=f,
                        ok=abs(reached - t) <= max(2.0 ** -23 * abs(t), 2.0 ** -23) and np.abs(f).max() < 1e3))
    return out
