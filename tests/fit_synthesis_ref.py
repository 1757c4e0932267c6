"""Torch restatement of the fitting kernels' device path (rnnoise_fit_forward_device / _backward_device, DESIGN.md §7l),
built on fit_ref's network.

TEST INFRASTRUCTURE, written from the contract in include/rnnoise.h: every function takes a dtype through its inputs,
so the same code gives the float64 reference and the float32 restatement whose distance from float64 sets the GPU
tolerances.

* Silent frames: nothing is evaluated, every GRU state is carried (h_t = h_{t-1}), gains and vad are 0; their output
  gradients are ignored, so they add nothing to any weight gradient and pass dL/dh through unchanged.
* State: sequence s starts from state[s] = [vad | noise | denoise GRU state] (zeros when None); no gradient flows to it.
* Loss: sum(grad_gains * gains) + sum(grad_vad * vad), whose gradient is what the backward returns.
"""
import numpy as np
import torch

from nnnoiseless_b200.fit import unflatten
from fit_ref import SCRIPT_ACTS, act


def gru(x, W, U, b, code, silent, h0):
    """x [S][T][ni], silent bool [S][T], h0 [S][n] -> h [S][T][n]."""
    n = U.shape[0]
    h = h0
    xw = x @ W + b
    out = []
    for t in range(x.shape[1]):
        a = xw[:, t]
        hu = h @ U[:, :2 * n]
        z = torch.sigmoid(a[:, :n] + hu[:, :n])
        r = torch.sigmoid(a[:, n:2 * n] + hu[:, n:])
        hc = act(code, a[:, 2 * n:] + (r * h) @ U[:, 2 * n:])
        h = torch.where(silent[:, t, None], h, z * h + (1 - z) * hc)
        out.append(h)
    return torch.stack(out, 1)


def forward(P, widths, x, silent=None, state=None, acts=SCRIPT_ACTS):
    """P: {(layer, name): tensor}; x [S][T][42]; silent bool [S][T] or None; state [S][nv + nn + ndn] or None ->
    dict(hv, hn, hd, gains [S][T][22], vad [S][T]), gains and vad 0 on silent frames."""
    S, T = x.shape[0], x.shape[1]
    nv, nn, ndn = (int(w) for w in widths[1:])
    sil = torch.zeros((S, T), dtype=torch.bool) if silent is None else torch.as_tensor(np.asarray(silent, bool))
    st = torch.zeros((S, nv + nn + ndn), dtype=x.dtype) if state is None else torch.as_tensor(state, dtype=x.dtype)
    x = torch.where(sil[..., None], torch.zeros((), dtype=x.dtype), x)  # not evaluated: keeps NaN away from the gradients
    g = lambda l, n: P[(l, n)]  # noqa: E731
    d = act(acts[0], x @ g("input_dense", "kernel") + g("input_dense", "bias"))
    hv = gru(d, g("vad_gru", "kernel"), g("vad_gru", "recurrent_kernel"), g("vad_gru", "bias"), acts[1], sil, st[:, :nv])
    vad = act(acts[5], hv @ g("vad_output", "kernel") + g("vad_output", "bias"))[..., 0]
    hn = gru(torch.cat([d, hv, x], -1), g("noise_gru", "kernel"), g("noise_gru", "recurrent_kernel"), g("noise_gru", "bias"), acts[2],
             sil, st[:, nv:nv + nn])
    hd = gru(torch.cat([hv, hn, x], -1), g("denoise_gru", "kernel"), g("denoise_gru", "recurrent_kernel"), g("denoise_gru", "bias"),
             acts[3], sil, st[:, nv + nn:])
    gains = act(acts[4], hd @ g("denoise_output", "kernel") + g("denoise_output", "bias"))
    zero = torch.zeros((), dtype=x.dtype)
    return dict(hv=hv, hn=hn, hd=hd, gains=torch.where(sil[..., None], zero, gains), vad=torch.where(sil, zero, vad))


def forward_and_grad(params, widths, x, grad_gains, grad_vad, silent=None, state=None, dtype=torch.float64, acts=SCRIPT_ACTS):
    """-> (numpy forward dict with `state` [S][T][nv + nn + ndn], flat dL/dparams) for L = sum(grad_gains * gains) +
    sum(grad_vad * vad)."""
    flat = torch.tensor(np.asarray(params), dtype=dtype, requires_grad=True)
    fw = forward(unflatten(flat, widths), widths, torch.as_tensor(np.asarray(x), dtype=dtype), silent, state, acts)
    loss = (torch.as_tensor(np.asarray(grad_gains), dtype=dtype) * fw["gains"]).sum()
    loss = loss + (torch.as_tensor(np.asarray(grad_vad), dtype=dtype) * fw["vad"]).sum()
    loss.backward()
    out = {k: v.detach().numpy() for k, v in fw.items()}
    out["state"] = np.concatenate([out["hv"], out["hn"], out["hd"]], -1)
    return out, flat.grad.numpy().copy()
