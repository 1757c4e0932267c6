"""Constructed inputs for the fitting kernels' per-stage bounds (tests/fit_bounds.py), class by class, each at the edge
where a kernel could go wrong (TEST INFRASTRUCTURE).

A case is dict(widths, params, x [S][T][42], rows [S][T][87], weights [S][T], and for the device path silent, h0,
gg, gv).  Parameters are f32; every array is float32 as the kernels read it.
"""
import numpy as np

from nnnoiseless_b200.fit import init_params, unflatten
import fit_bounds as fb

F32 = np.float32
ULP_EPS = np.spacing(F32(1e-7))


def _rows(rng, S, T, y=None, vt=None):
    rows = np.zeros((S, T, 87), np.float32)
    rows[..., :42] = rng.standard_normal((S, T, 42)) * 1.5
    rows[..., 42:64] = rng.random((S, T, 22)) if y is None else y
    rows[..., 64:86] = rng.standard_normal((S, T, 22))
    rows[..., 86] = rng.choice([0.0, 0.5, 1.0], size=(S, T)) if vt is None else vt
    return rows


def _case(widths, params, rows, weights, **kw):
    c = dict(widths=tuple(widths), params=np.asarray(params, np.float32), rows=np.asarray(rows, np.float32),
             x=np.ascontiguousarray(rows[..., :42]), weights=np.asarray(weights, np.float32))
    c.update(kw)
    return c


def random_case(widths, S, T, seed, device=False, mask=None):
    rng = np.random.default_rng(seed)
    p = init_params(widths, seed)
    P = unflatten(p, widths)
    nn = widths[2]
    P[("noise_gru", "bias")][2 * nn:2 * nn + max(1, nn // 3)] = -0.499  # relu units that go dead
    rows = _rows(rng, S, T)
    y = rows[..., 42:64]
    y[rng.random(y.shape) < 0.2] = -1.0
    w = rng.uniform(0, 2, (S, T)).astype(np.float32)
    w[rng.random((S, T)) < 0.1] = 0.0
    kw = {}
    if device:
        sil = np.zeros((S, T), bool) if mask is None else mask
        kw = dict(silent=sil, h0=rng.uniform(-0.9, 0.9, (S, sum(widths[1:]))).astype(np.float32),
                  gg=rng.standard_normal((S, T, 22)).astype(np.float32), gv=rng.standard_normal((S, T)).astype(np.float32))
    return _case(widths, p, rows, w, **kw)


def gate_cases():
    """z at the sigmoid's f32 saturation (pre-activation 16 .. 17.5, where 1 / (1 + expf(-x)) rounds to 1) and h~ at
    tanhf = +-1 (1 - y^2 -> 0).  Frame 0 has zero features and input_dense a zero bias, so d = 0 and the vad GRU's
    pre-activations at t = 0 are its biases exactly: one ulp below or above each point.  Later frames and GRUs move
    them by the small weights."""
    out = []
    widths = (5, 3, 7, 11)
    for k, z0 in enumerate((16.0, 16.6355, 17.0, 17.5)):
        rng = np.random.default_rng(100 + k)
        p = init_params(widths, k) * F32(0.01)
        P = unflatten(p, widths)
        for layer, n in (("vad_gru", 3), ("noise_gru", 7), ("denoise_gru", 11)):
            b = P[(layer, "bias")]
            b[:n] = np.nextafter(F32(z0), F32(20.0 if k % 2 else 0.0))  # a few ulps off the point
            b[2 * n:] = F32(9.5) * np.where(np.arange(n) % 2, 1, -1)    # tanh saturated (bias unclipped: caller params)
        P[("input_dense", "bias")][:] = 0.0
        rows = _rows(rng, 2, 6)
        rows[:, 0, :42] = 0.0
        out.append(_case(widths, p, rows, np.ones((2, 6), np.float32)))
    return out


def relu_cases():
    """ReLU pre-activations exactly 0 (zero features, bias and state at t = 0), +-m delta around 0, and dead units."""
    out = []
    widths = (4, 3, 6, 5)
    for k, scale in enumerate((0.0, 1e-30, 1e-6)):
        rng = np.random.default_rng(200 + k)
        p = init_params(widths, 10 + k)
        P = unflatten(p, widths)
        P[("noise_gru", "bias")][12:] = 0.0
        P[("noise_gru", "bias")][12:14] = (F32(scale), F32(-scale))
        P[("noise_gru", "bias")][14] = -0.499  # dead
        rows = _rows(rng, 2, 5)
        rows[:, 0, :42] = 0.0
        P[("input_dense", "bias")][:] = 0.0
        out.append(_case(widths, p, rows, np.ones((2, 5), np.float32)))
    return out


def target_cases():
    """Targets -1, in (-1, 0), 0, 1e-7, 1e-7 +- ulp, 1 - 2^-23 and 1; and a third case whose first six bands' targets
    are the f32 emulation's own gains, so that d = sqrt(g) - sqrt(y) is exactly 0 there (within a few ulps on the GPU)."""
    widths = (5, 3, 7, 11)
    vals = np.array([-1.0, -0.5, -0.25, 0.0, 1e-7, F32(1e-7) + ULP_EPS, F32(1e-7) - ULP_EPS, 1.0 - 2.0 ** -23, 1.0, 0.5, 0.3, 0.9,
                     -0.999, 2e-7, 1e-6, 0.999, 0.75, 0.1, 0.01, 1e-3, 0.6, 0.4], np.float32)
    out = []
    for k in range(2):
        rng = np.random.default_rng(300 + k)
        p = init_params(widths, 20 + k)
        y = np.broadcast_to(np.roll(vals, k), (2, 4, 22)).copy()
        out.append(_case(widths, p, _rows(rng, 2, 4, y=y), np.ones((2, 4), np.float32)))
    c = dict(out[0], rows=out[0]["rows"].copy())
    tp = fb.forward(fb.F32(), fb.Net(c["params"], widths), c["x"])
    c["rows"][..., 42:48] = tp["gains"][..., :6]
    out.append(c)
    return out


def small_output_cases():
    """Gains down to about 1e-21: the denoise output's bias far negative (caller parameters are not clipped)."""
    widths = (5, 3, 7, 11)
    out = []
    for k, b in enumerate((-30.0, -48.0)):
        rng = np.random.default_rng(400 + k)
        p = init_params(widths, 30 + k)
        unflatten(p, widths)[("denoise_output", "bias")][:] = b
        out.append(_case(widths, p, _rows(rng, 2, 4), np.ones((2, 4), np.float32)))
    return out


def vad_cases():
    """VAD targets 0.5 (c = 0), 0 and 1, and sample weights of 0."""
    widths = (5, 3, 7, 11)
    rng = np.random.default_rng(500)
    vt = np.tile(np.array([0.5, 0.0, 1.0, 0.25], np.float32), (3, 1))
    w = np.ones((3, 4), np.float32)
    w[1] = 0.0
    return [_case(widths, init_params(widths, 40), _rows(rng, 3, 4, vt=vt), w)]


def device_cases():
    """The device path: silence masks first, last, all and random frames with state_in given, and a signed grad_vad for
    which the vad output bias's gradient, sum(gv v (1 - v)) over the live frames, cancels (fit_bounds.cancelling_gv)."""
    widths = (5, 3, 7, 11)
    out = []
    S, T = 3, 6
    for k, kind in enumerate(("first", "last", "all", "random", "cancel")):
        rng = np.random.default_rng(600 + k)
        m = np.zeros((S, T), bool)
        if kind == "first":
            m[:, 0] = True
        elif kind == "last":
            m[:, -1] = True
        elif kind == "all":
            m[:] = True
        elif kind == "random":
            m = rng.random((S, T)) < 0.3
        c = random_case(widths, S, T, 700 + k, device=True, mask=m)
        if kind == "cancel":  # fit_bounds.run sets the last live frame's gv from the forward's vad
            c["cancel_vad"] = True
        out.append(c)
    return out


CLASSES = {"gates": gate_cases, "relu": relu_cases, "targets": target_cases, "small_outputs": small_output_cases,
           "vad": vad_cases, "device": device_cases}
COUNTS = {"gates": 4, "relu": 3, "targets": 3, "small_outputs": 2, "vad": 1, "device": 5}
