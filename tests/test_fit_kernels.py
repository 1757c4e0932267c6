"""GPU tests of the fitting kernels (csrc/fit.cu) against the torch restatement (tests/fit_ref.py): forward activations,
loss and every parameter's gradient against float64 autograd, with a tolerance of K times the float32 restatement's own
distance from float64 (or a floor); Adam and the clip on the GPU's own gradients; bitwise determinism; the export round
trip of the built-in model; and a short end-to-end fit on generated rows."""
import json
import os

import numpy as np
import pytest
import torch

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import fit, training
from nnnoiseless_b200.synth import synth_streams
from fit_ref import adam_step, loss_and_grad

pytestmark = pytest.mark.gpu

K_D32 = 8.0      # GPU error allowed per element, in units of the float32 restatement's error
FLOOR = 2e-5     # ... or this share of the largest magnitude of the array, whichever is larger
STATS = os.environ.get("NNB_FIT_STATS")  # a path: append one JSON line per checked array (the tolerance shares)


def _rows(S, T, seed):
    """Rows with masked bands, one fully masked frame, vad targets 0 / 0.5 / 1 and weights including 0."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((S, T, 87), np.float32)
    rows[..., :42] = rng.standard_normal((S, T, 42)) * 1.5
    y = rng.random((S, T, 22)).astype(np.float32)
    y[rng.random((S, T, 22)) < 0.2] = -1.0
    y[0, T // 2] = -1.0
    rows[..., 42:64] = y
    rows[..., 64:86] = rng.standard_normal((S, T, 22))
    rows[..., 86] = rng.choice([0.0, 0.5, 1.0], size=(S, T))
    w = rng.uniform(0, 2, (S, T)).astype(np.float32)
    w[rng.random((S, T)) < 0.1] = 0.0
    return rows, w


def _params(widths, seed):
    p = fit.init_params(widths, seed)
    P = fit.unflatten(p, widths)
    nn = widths[2]
    P[("noise_gru", "bias")][2 * nn:2 * nn + max(1, nn // 3)] = -0.499  # relu units that go dead
    P[("noise_gru", "kernel")][:, 2 * nn:2 * nn + max(1, nn // 3)] *= 0.01
    return p


def _check(name, got, ref64, ref32, case):
    got, ref64, ref32 = (np.asarray(a, np.float64).ravel() for a in (got, ref64, ref32))
    d32 = np.abs(ref32 - ref64)
    floor = FLOOR * max(np.abs(ref64).max(), 1e-30)
    tol = np.maximum(K_D32 * d32, floor)
    err = np.abs(got - ref64)
    rec = dict(case=case, what=name, n=int(err.size), max_err=float(err.max()), max_d32=float(d32.max()),
               floor=float(floor), share_floor=float(np.mean(K_D32 * d32 < floor)), worst_ratio=float((err / tol).max()))
    if STATS:
        with open(STATS, "a") as fh:
            fh.write(json.dumps(rec) + "\n")
    bad = np.flatnonzero(err > tol)
    assert bad.size == 0, "%s: %d of %d over tolerance, e.g. #%d got %r ref %r tol %r" % (
        name, bad.size, err.size, bad[0], got[bad[0]], ref64[bad[0]], tol[bad[0]])


CASES = [((24, 24, 48, 96), 1, 1), ((24, 24, 48, 96), 3, 17), ((5, 3, 7, 11), 37, 2), ((5, 3, 7, 11), 3, 200),
         ((96, 96, 96, 96), 32, 17), ((24, 24, 48, 96), 32, 200), ((96, 96, 96, 96), 1, 200)]


@pytest.mark.parametrize("widths,S,T", CASES)
def test_forward_loss_and_gradients(widths, S, T):
    case = "%s S=%d T=%d" % (",".join(map(str, widths)), S, T)
    rows, w = _rows(S, T, seed=S * 1000 + T)
    p = _params(widths, seed=T)
    f = fit.Fit(widths, max_sequences=S, window=T, device=0)
    f.set_params(p)
    ev = f.evaluate(rows, w)
    act = f.activations(S)
    loss = f.step(rows, w)
    g = f.grads()
    t64, g64, fw64 = loss_and_grad(p, widths, rows, w, torch.float64)
    t32, g32, fw32 = loss_and_grad(p, widths, rows, w, torch.float32)
    assert loss == ev["loss"]
    for k in ("loss", "mycost", "crossentropy", "msse"):
        _check(k, [ev[k]], [t64[k]], [t32[k]], case)
    _check("gains", act["gains"], fw64["gains"], fw32["gains"], case)
    _check("vad", act["vad"], fw64["vad"], fw32["vad"], case)
    st64 = np.concatenate([fw64["hv"], fw64["hn"], fw64["hd"]], -1)
    st32 = np.concatenate([fw32["hv"], fw32["hn"], fw32["hd"]], -1)
    _check("gru_state", act["state"], st64, st32, case)
    assert (fw64["hn"] == 0).any(), "the case should have dead relu units"
    off = 0
    for layer, name, shape in fit.layer_shapes(widths):
        k = int(np.prod(shape))
        _check("grad %s.%s" % (layer, name), g[off:off + k], g64[off:off + k], g32[off:off + k], case)
        off += k


def test_adam_and_clip_on_gpu_gradients():
    widths, S, T = (24, 24, 48, 96), 4, 30
    rows, w = _rows(S, T, seed=11)
    p = _params(widths, seed=3)
    P = fit.unflatten(p, widths)
    P[("vad_gru", "bias")][:5] = 0.4995  # at the clip
    f = fit.Fit(widths, S, T, device=0)
    f.set_params(p)
    ref = p.astype(np.float64)
    m = np.zeros_like(ref)
    v = np.zeros_like(ref)
    for t in range(1, 5):
        before = f.get_params().astype(np.float64)
        f.step(rows, w)
        g = f.grads().astype(np.float64)
        ref, m, v = adam_step(before, g, m, v, t)
        np.testing.assert_allclose(f.get_params(), ref, rtol=0, atol=2e-7)
    assert np.abs(f.get_params()).max() <= 0.499


def test_five_steps_are_deterministic():
    widths, S, T = (24, 24, 48, 96), 37, 100
    rows, w = _rows(S, T, seed=5)
    out = []
    for _ in range(2):
        f = fit.Fit(widths, S, T, device=0)
        f.set_params(fit.init_params(widths, 1))
        losses = [f.step(rows, w) for _ in range(5)]
        out.append((f.get_params().tobytes(), f.export(), losses))
    assert out[0] == out[1]


def test_builtin_model_round_trip(builtin_bytes):
    f = fit.Fit(fit.WIDTHS, 1, 10, device=0)
    f.set_params_from_model(None)
    assert f.export() == builtin_bytes


def test_fit_end_to_end():
    L, frames, window = 64, 4000, 200
    tb = training.TrainingBatch(L, device=0)
    tb.set_params(training.randomize(L, np.random.default_rng(0)))
    sig = synth_streams(L, frames, seed=101).reshape(L, frames, 480)
    noi = synth_streams(L, frames, seed=202).reshape(L, frames, 480)
    rows = np.concatenate([tb.process_host(np.ascontiguousarray(sig[:, a:a + 500].transpose(1, 0, 2)),
                                           np.ascontiguousarray(noi[:, a:a + 500].transpose(1, 0, 2)))
                           for a in range(0, frames, 500)])
    del sig, noi
    assert rows.shape == (frames, L, 87)
    model, hist = fit.fit(rows, epochs=3, batch_size=32, window=window, seed=0, device=0)
    assert len(hist["loss"]) == 3 and len(hist["val_loss"]) == 3
    assert min(hist["loss"][1:]) < hist["loss"][0]
    assert min(hist["val_loss"][1:]) < hist["val_loss"][0]
    x = synth_streams(4, 20, seed=7).reshape(4, 20, 480).transpose(1, 0, 2)
    out, vad = nb.DenoiseBatch(4, model=model, device=0).process_host(x)
    assert np.isfinite(out).all() and np.isfinite(vad).all()
    batch = nb.DenoiseBatch(4, device=0)
    assert batch.add_model(model) == 1
    batch.set_stream_models([1, 1], streams=[0, 2])
    out2, _ = batch.process_host(x)
    np.testing.assert_array_equal(out2[:, [0, 2]], out[:, [0, 2]])
