"""CPU tests of the fitting semantics (tests/fit_ref.py) and of the host parts of nnnoiseless_b200.fit: the restated
forward pass against the network reference, the loss at each quirk of the script, the sample weights, the Adam step,
and the .rnn export."""
import numpy as np
import pytest
import torch

import nnnoiseless_b200 as nb
import oracle
import rnn_ref
from nnnoiseless_b200 import fit
from fit_ref import SCRIPT_ACTS, adam_step, bce, frame_terms, l2_grad, loss_and_grad, params_from_model, quantize


def _with_acts(data: bytes, acts) -> bytes:
    """The model bytes with the six layers' activation codes replaced."""
    b = bytearray(data)
    p = 0
    for i, gates in enumerate((1, 3, 3, 3, 1, 1)):
        ni, n = b[p], b[p + 1]
        b[p + 2] = acts[i]
        p += 3 + gates * n * ni + (3 * n * n if gates == 3 else 0) + gates * n
    return bytes(b)


def _widths(data: bytes):
    L = rnn_ref.parse(data)
    return (L[0]["nn"], L[1]["nn"], L[2]["nn"], L[3]["nn"])


@pytest.mark.parametrize("which", ["builtin", "sh", "make_5_3_7_11", "make_24_24_48_96"])
def test_forward_matches_rnn_ref(which, builtin_bytes, sh_bytes, monkeypatch):
    data = {"builtin": builtin_bytes, "sh": sh_bytes, "make_5_3_7_11": rnn_ref.make_model(5, 3, 7, 11, seed=3),
            "make_24_24_48_96": rnn_ref.make_model(24, 24, 48, 96, seed=4)}[which]
    data = _with_acts(data, SCRIPT_ACTS)  # the script's topology
    monkeypatch.setattr(rnn_ref, "tansig", np.tanh)  # exact activations instead of the inference tables
    widths = _widths(data)
    params, acts = params_from_model(data, widths)
    assert acts == SCRIPT_ACTS
    rng = np.random.default_rng(7)
    S, T = 3, 12
    x = rng.standard_normal((S, T, 42)) * 2
    rows = np.zeros((S, T, 87))
    rows[..., :42] = x
    _, _, fw = loss_and_grad(params, widths, rows, np.ones((S, T)))
    layers = rnn_ref.parse(data)
    state = np.zeros((S, sum(widths[1:])))
    nv, nn = widths[1], widths[2]
    for t in range(T):
        state, gains, vad = rnn_ref.step(layers, state, x[:, t])
        np.testing.assert_allclose(fw["hv"][:, t], state[:, :nv], rtol=0, atol=1e-12)
        np.testing.assert_allclose(fw["hn"][:, t], state[:, nv:nv + nn], rtol=0, atol=1e-12)
        np.testing.assert_allclose(fw["hd"][:, t], state[:, nv + nn:], rtol=0, atol=1e-12)
        np.testing.assert_allclose(fw["gains"][:, t], gains, rtol=0, atol=1e-12)
        np.testing.assert_allclose(fw["vad"][:, t], vad, rtol=0, atol=1e-12)


def _bce_hand(p, t):
    e = 1e-7
    tc = min(max(t, e), 1 - e)
    return -(p * np.log(tc + e) + (1 - p) * np.log(1 - tc + e))


def test_loss_quirks_by_hand():
    # bands: masked, 0, 0.5, 1, and predictions at eps and 1 - eps
    y = np.array([-1.0, 0.0, 0.5, 1.0, 0.25] + [-1.0] * 17)
    g = np.array([0.3, 1e-7, 0.5, 1 - 1e-7, 0.7] + [0.9] * 17)
    terms = []
    for vt, v in ((0.0, 0.2), (0.5, 0.9), (1.0, 1 - 1e-7)):
        f64 = lambda a: torch.tensor(a, dtype=torch.float64)  # noqa: E731
        mc, xe, ms = frame_terms(f64(g), f64(v), f64(y), f64(vt))
        exp_c = exp_m = 0.0
        for gj, yj in zip(g, y):
            mask = min(yj + 1, 1)
            d = np.sqrt(max(gj, 0)) - np.sqrt(max(yj, 0))  # K.sqrt clips at 0: a masked band reads sqrt(0)
            exp_c += mask * (10 * d ** 4 + d ** 2 + 0.01 * _bce_hand(gj, yj))
            exp_m += mask * d ** 2
        assert float(mc) == pytest.approx(exp_c / 22, rel=1e-13)
        assert float(ms) == pytest.approx(exp_m / 22, rel=1e-13)
        # arguments swapped as in the script: the prediction is the target of K.binary_crossentropy
        assert float(xe) == pytest.approx(2 * abs(vt - 0.5) * _bce_hand(v, vt), rel=1e-13, abs=1e-300)
        terms.append(float(xe))
    assert terms[1] == 0.0  # vad target 0.5 carries no weight
    # a masked band is finite before its mask multiplies it by 0
    assert np.isfinite(float(bce(torch.tensor(0.3, dtype=torch.float64), torch.tensor(-1.0, dtype=torch.float64))))


def test_loss_reduction_and_l2():
    widths = (3, 2, 4, 5)
    rng = np.random.default_rng(1)
    params = fit.init_params(widths, seed=2).astype(np.float64)
    rows = rng.random((2, 4, 87))
    rows[..., 42:50] = -1.0
    w = np.array([[0.0, 1.0, 2.0, 0.5], [3.0, 0.0, 1.0, 1.0]])
    terms, _, fw = loss_and_grad(params, widths, rows, w)
    mc, xe, _ = frame_terms(torch.tensor(fw["gains"]), torch.tensor(fw["vad"]), torch.tensor(rows[..., 42:64]),
                            torch.tensor(rows[..., 86]))
    data = (10 * (w * mc.numpy()).sum() + 0.5 * (w * xe.numpy()).sum()) / 8  # / frames, not / sum of weights
    reg = 1e-6 * 0.5e6 * float(np.dot(l2_grad(params, widths), params))
    assert terms["loss"] == pytest.approx(data + reg, rel=1e-13)


def _row(gains):
    r = np.zeros(87, np.float32)
    r[42:64] = gains
    return r


def test_sample_weights_classes():
    rows = np.stack([_row([0.9] * 22), _row([0.8] * 22), _row([0.5] * 22), _row([0.1] * 22), _row([-1.0] * 22),
                     _row([0.9, 0.0] + [-1.0] * 20)])  # means: hi, hi, med, lo, all masked, 0.45 -> med
    w = fit.sample_weights(rows)
    total = 6
    np.testing.assert_allclose(w, np.array([total / 2, total / 2, total / 2, total / 1, 0.0, total / 2]) / 3, rtol=1e-6)
    # each class carries the same total weight
    assert w[:2].sum() == pytest.approx(w[[2, 5]].sum()) == pytest.approx(w[3])


@pytest.mark.parametrize("missing", ["hi", "med", "lo"])
def test_sample_weights_empty_class_raises(missing):
    rows = {"hi": [_row([0.5] * 22), _row([0.1] * 22)], "med": [_row([0.9] * 22), _row([0.1] * 22)],
            "lo": [_row([0.9] * 22), _row([0.5] * 22)]}[missing]
    with pytest.raises(ValueError, match=missing):
        fit.sample_weights(np.stack(rows))


def test_windows_per_lane():
    frames, lanes = 7, 3
    rows = np.zeros((frames, lanes, 87), np.float32)
    rows[..., 0] = np.arange(frames)[:, None]
    rows[..., 1] = np.arange(lanes)[None, :]
    w = fit.windows(rows, 3)
    assert w.shape == (lanes * 2, 3, 87)
    for i in range(lanes * 2):
        lane, k = divmod(i, 2)
        np.testing.assert_array_equal(w[i, :, 0], np.arange(3 * k, 3 * k + 3))
        assert (w[i, :, 1] == lane).all()


def test_init_params():
    widths = (24, 24, 48, 96)
    p = fit.init_params(widths, seed=5)
    np.testing.assert_array_equal(p, fit.init_params(widths, seed=5))
    P = fit.unflatten(p, widths)
    for (layer, name), a in P.items():
        if name == "bias":
            assert not a.any()
        elif name == "kernel":
            assert np.abs(a).max() <= np.sqrt(6.0 / (a.shape[0] + a.shape[1])) + 1e-7
        else:
            np.testing.assert_allclose(a.astype(np.float64) @ a.T.astype(np.float64), np.eye(a.shape[0]), atol=1e-5)


def test_adam_matches_tf_form():
    rng = np.random.default_rng(3)
    w = rng.uniform(-0.5, 0.5, 50)
    w[:3] = [0.4989, -0.4989, 0.2]
    m, v = np.zeros(50), np.zeros(50)
    hw, hm, hv = w.copy(), m.copy(), v.copy()
    for t in range(1, 6):
        g = rng.standard_normal(50)
        g[:2] = [-50.0, 50.0]  # pushes the first two past the clip
        w, m, v = adam_step(w, g, m, v, t)
        # ResourceApplyAdam as written in TensorFlow's kernel, then the constraint
        lr = 1e-3 * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
        hm = hm + (g - hm) * (1 - 0.9)
        hv = hv + (g * g - hv) * (1 - 0.999)
        hw = np.minimum(np.maximum(hw - lr * hm / (np.sqrt(hv) + 1e-7), -0.499), 0.499)
        np.testing.assert_allclose(w, hw, rtol=1e-13, atol=1e-16)
    assert w[0] == 0.499 and w[1] == -0.499


def test_export_matches_quantiser():
    widths = (24, 24, 48, 96)
    p = fit.init_params(widths, seed=9)
    n = len(p)
    p[:8] = [0.5 / 256, 1.5 / 256, -0.5 / 256, -2.5 / 256, 0.499, -0.499, 127.5 / 256, -128.5 / 256]  # exact ties
    p[8:12] = [0.4990001, 1.0, -1.0, 3.5 / 256]
    b = fit.export_params(p, widths)
    assert b == quantize(p, widths)
    q = np.frombuffer(b, np.int8)
    assert list(q[3:11]) == [0, 2, 0, -2, 127, -128, 127, -128]
    assert nb.RnnModel.from_bytes(b) is not None
    oracle.Model(b)
    assert len(b) == n + 18


def test_export_rejects_wide_inputs():
    p = np.zeros(fit.n_params((96, 96, 96, 96)), np.float32)
    with pytest.raises(nb.NnnoiselessError, match="signed byte"):
        fit.export_params(p, (96, 96, 96, 96))


def test_builtin_round_trip_through_quantiser(builtin_bytes):
    widths = _widths(builtin_bytes)
    params, acts = params_from_model(builtin_bytes, widths)
    assert quantize(params, widths, acts) == builtin_bytes
