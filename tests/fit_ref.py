"""Torch restatement of what train/rnn_train.py computes under tf.keras 2.x, and of dump_rnn.py's quantiser.

TEST INFRASTRUCTURE, written from the semantics, not from Keras: every function takes a dtype, so the same code gives
the float64 reference and the float32 restatement whose distance from float64 sets the GPU tolerances.

* Network (rnn_train.py:65-77): input_dense 42 -> nd; vad_gru nd -> nv; vad_output nv -> 1; noise_gru
  [dense | vad_h | x] -> nn; denoise_gru [vad_h | noise_h | x] -> ndn; denoise_output ndn -> 22.  GRUs reset_after=False,
  gates z | r | h~: z = sig(x W_z + h U_z + b_z), r likewise, h~ = act(x W_h + (r h) U_h + b_h), h' = z h + (1 - z) h~;
  every sequence from a zero state; exact activations.
* Loss (rnn_train.py:33-43, 79-81): 10 mycost + 0.5 my_crossentropy, each per (sequence, frame) times the sample weight,
  summed and divided by the number of (sequence, frame) pairs; plus 1e-6 sum w^2 over the GRUs' kernel and recurrent
  matrices (rnn_train.py:61, 67-73).  mymask(t) = min(t + 1, 1); K.sqrt clips at 0; K.binary_crossentropy is called
  as (y_pred, y_true), i.e. target = prediction p, output = label t: -(p log(t_c + eps) + (1 - p) log(1 - t_c + eps)),
  t_c = clip(t, eps, 1 - eps), eps = 1e-7.
* Adam (tf.keras defaults lr 1e-3, 0.9, 0.999, eps 1e-7; the update of ResourceApplyAdam) then WeightClip(0.499) on
  every parameter (rnn_train.py:48-62).
* Export (dump_rnn.py:4-48): clip(round_half_even(256 w), -128, 127) per weight, layer header [inputs, neurons, act].
"""
import numpy as np
import torch

from nnnoiseless_b200.fit import LAYERS, layer_shapes, unflatten

EPS = 1e-7
SCRIPT_ACTS = (0, 0, 2, 0, 1, 1)  # input_dense, vad_gru, noise_gru, denoise_gru, denoise_output, vad_output


def act(code, x):
    return torch.tanh(x) if code == 0 else (torch.sigmoid(x) if code == 1 else torch.relu(x))


def params_from_model(data: bytes, widths):
    """A model's int8 weights / 256 as the flat vector (file order, Keras shapes) and its activation codes."""
    raw = np.frombuffer(bytes(data), np.int8)
    parts, acts, p = [], [], 0
    for _, name, shape in layer_shapes(widths):
        if name == "kernel":
            acts.append(int(raw[p + 2]))
            p += 3
        k = int(np.prod(shape))
        parts.append(raw[p:p + k].astype(np.float64) / 256.0)
        p += k
    assert p == len(raw)
    return np.concatenate(parts), tuple(acts)


def gru(x, W, U, b, code):
    """x [S][T][ni] -> h [S][T][n] from a zero state."""
    n = U.shape[0]
    h = torch.zeros(x.shape[0], n, dtype=x.dtype)
    xw = x @ W + b
    out = []
    for t in range(x.shape[1]):
        a = xw[:, t]
        hu = h @ U[:, :2 * n]
        z = torch.sigmoid(a[:, :n] + hu[:, :n])
        r = torch.sigmoid(a[:, n:2 * n] + hu[:, n:])
        hc = act(code, a[:, 2 * n:] + (r * h) @ U[:, 2 * n:])
        h = z * h + (1 - z) * hc
        out.append(h)
    return torch.stack(out, 1)


def forward(P, widths, x, acts=SCRIPT_ACTS):
    """P: {(layer, name): tensor}; x [S][T][42] -> dict(d, hv, hn, hd, gains, vad [S][T])."""
    g = lambda l, n: P[(l, n)]  # noqa: E731
    d = act(acts[0], x @ g("input_dense", "kernel") + g("input_dense", "bias"))
    hv = gru(d, g("vad_gru", "kernel"), g("vad_gru", "recurrent_kernel"), g("vad_gru", "bias"), acts[1])
    vad = act(acts[5], hv @ g("vad_output", "kernel") + g("vad_output", "bias"))[..., 0]
    hn = gru(torch.cat([d, hv, x], -1), g("noise_gru", "kernel"), g("noise_gru", "recurrent_kernel"), g("noise_gru", "bias"), acts[2])
    hd = gru(torch.cat([hv, hn, x], -1), g("denoise_gru", "kernel"), g("denoise_gru", "recurrent_kernel"), g("denoise_gru", "bias"),
             acts[3])
    gains = act(acts[4], hd @ g("denoise_output", "kernel") + g("denoise_output", "bias"))
    return dict(d=d, hv=hv, hn=hn, hd=hd, gains=gains, vad=vad)


def bce(target, output):
    o = torch.clamp(output, EPS, 1 - EPS)
    return -(target * torch.log(o + EPS) + (1 - target) * torch.log(1 - o + EPS))


def frame_terms(gains, vad, y, vt):
    """Per-frame mycost, my_crossentropy and msse (rnn_train.py:33-43): gains [..][22], vad [..], targets y [..][22],
    vt [..]."""
    mask = torch.clamp(y + 1, max=1.0)
    sq = lambda a: torch.sqrt(torch.clamp(a, min=0.0))  # noqa: E731
    d = sq(gains) - sq(y)
    mycost = (mask * (10 * d ** 4 + d ** 2 + 0.01 * bce(gains, y))).mean(-1)
    xent = 2 * torch.abs(vt - 0.5) * bce(vad, vt)
    msse = (mask * d ** 2).mean(-1)
    return mycost, xent, msse


def l2(P):
    return sum((P[(l, n)] ** 2).sum() for l in ("vad_gru", "noise_gru", "denoise_gru") for n in ("kernel", "recurrent_kernel"))


def loss(flat, widths, rows, weights, acts=SCRIPT_ACTS):
    """flat: parameter tensor; rows [S][T][87], weights [S][T] -> (dict(loss, mycost, crossentropy, msse), forward)."""
    P = unflatten(flat, widths)
    rows = torch.as_tensor(rows, dtype=flat.dtype)
    w = torch.as_tensor(weights, dtype=flat.dtype)
    fw = forward(P, widths, rows[..., :42], acts)
    mycost, xent, msse = frame_terms(fw["gains"], fw["vad"], rows[..., 42:64], rows[..., 86])
    R = w.numel()
    c, e = (w * mycost).sum() / R, (w * xent).sum() / R
    return dict(loss=10 * c + 0.5 * e + 1e-6 * l2(P), mycost=c, crossentropy=e, msse=msse.sum() / R), fw


def loss_and_grad(params, widths, rows, weights, dtype=torch.float64, acts=SCRIPT_ACTS):
    flat = torch.tensor(np.asarray(params), dtype=dtype, requires_grad=True)
    terms, fw = loss(flat, widths, rows, weights, acts)
    terms["loss"].backward()
    return {k: float(v.detach()) for k, v in terms.items()}, flat.grad.numpy().copy(), {k: v.detach().numpy() for k, v in fw.items()}


def adam_step(w, g, m, v, t, lr=1e-3, b1=0.9, b2=0.999, eps=1e-7):
    """tf.keras Adam, step t (1-based), then WeightClip(0.499); float64 numpy -> (w, m, v)."""
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    lr_t = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    w = w - lr_t * m / (np.sqrt(v) + eps)
    return np.clip(w, -0.499, 0.499), m, v


def l2_grad(params, widths):
    """d(1e-6 sum w^2)/dw over the GRUs' kernel and recurrent matrices, flat."""
    g, p = np.zeros(len(params)), 0
    for layer, name, shape in layer_shapes(widths):
        k = int(np.prod(shape))
        if layer.endswith("_gru") and name != "bias":
            g[p:p + k] = 2e-6 * np.asarray(params[p:p + k], np.float64)
        p += k
    return g


def quantize(params, widths, acts=SCRIPT_ACTS) -> bytes:
    """dump_rnn.py restated in numpy: per layer [inputs, neurons, act] then each array flattened row-major as
    clip(round_half_even(256 w), -128, 127) in two's complement."""
    out = bytearray()
    P = unflatten(np.asarray(params, np.float32), widths)
    for i, layer in enumerate(LAYERS):
        k = P[(layer, "kernel")]
        n = k.shape[1] // (3 if layer.endswith("_gru") else 1)
        out += bytes([k.shape[0], n, acts[i]])
        for name in ("kernel", "recurrent_kernel", "bias"):
            if (layer, name) in P:
                q = np.clip(np.round(256.0 * P[(layer, name)].astype(np.float64)), -128, 127).astype(np.int8)
                out += q.reshape(-1).tobytes()
    return bytes(out)
