"""CPU tests of training the denoise network on device features (DESIGN.md §7l): the restatement of silent frames and
carried state (tests/fit_synthesis_ref.py) against the fitting reference, the checks DenoiseNetwork makes before any
library call, and refusals of the C ABI that need no GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import fit
from nnnoiseless_b200.autograd import check_window
import fit_ref
import fit_synthesis_ref as fsr

WIDTHS = (5, 3, 7, 11)


def _inputs(S, T, seed):
    rng = np.random.default_rng(seed)
    return fit.init_params(WIDTHS, seed), rng.standard_normal((S, T, 42)) * 1.5


def test_no_silent_frame_is_the_fitting_reference():
    p, x = _inputs(3, 9, 1)
    rows = np.zeros((3, 9, 87))
    rows[..., :42] = x
    _, _, ref = fit_ref.loss_and_grad(p, WIDTHS, rows, np.ones((3, 9)))
    got = fsr.forward(fit.unflatten(torch.tensor(p, dtype=torch.float64), WIDTHS), WIDTHS, torch.tensor(x))
    for k in ("hv", "hn", "hd", "gains", "vad"):
        np.testing.assert_allclose(got[k].numpy(), ref[k], rtol=0, atol=1e-12)


def test_silent_frames_carry_the_state_and_output_zeros():
    S, T = 4, 12
    p, x = _inputs(S, T, 2)
    rng = np.random.default_rng(3)
    sil = rng.random((S, T)) < 0.3
    sil[0, 0] = sil[1, -1] = True
    sil[2] = True
    state = rng.uniform(-0.5, 0.5, (S, sum(WIDTHS[1:])))
    x[sil] = np.nan  # what a silent frame holds does not matter
    fw, g = fsr.forward_and_grad(p, WIDTHS, x, rng.standard_normal((S, T, 22)), rng.standard_normal((S, T)), sil, state)
    assert np.isfinite(g).all()
    for s in range(S):
        for t in range(T):
            if sil[s, t]:
                prev = fw["state"][s, t - 1] if t else state[s]
                assert np.array_equal(fw["state"][s, t], prev)
                assert (fw["gains"][s, t] == 0).all() and fw["vad"][s, t] == 0
    assert not np.array_equal(fw["state"][3, 1], fw["state"][3, 0])


def test_silent_window_adds_nothing_to_the_gradient():
    S, T = 3, 8
    p, x = _inputs(S, T, 4)
    rng = np.random.default_rng(5)
    sil = np.zeros((S, T), bool)
    gg, gv = rng.standard_normal((S, T, 22)), rng.standard_normal((S, T))
    _, g_two = fsr.forward_and_grad(p, WIDTHS, x[:2], gg[:2], gv[:2], sil[:2])
    sil[2] = True
    _, g_three = fsr.forward_and_grad(p, WIDTHS, x, gg, gv, sil)
    np.testing.assert_allclose(g_three, g_two, rtol=1e-12, atol=1e-15)


def test_two_windows_with_the_state_carried_are_one_window():
    S, T = 3, 7
    p, x = _inputs(S, 2 * T, 6)
    rng = np.random.default_rng(7)
    sil = rng.random((S, 2 * T)) < 0.25
    P = fit.unflatten(torch.tensor(p, dtype=torch.float64), WIDTHS)
    whole = fsr.forward(P, WIDTHS, torch.tensor(x), sil)
    a = fsr.forward(P, WIDTHS, torch.tensor(x[:, :T]), sil[:, :T])
    carried = torch.cat([a["hv"][:, -1], a["hn"][:, -1], a["hd"][:, -1]], -1)
    b = fsr.forward(P, WIDTHS, torch.tensor(x[:, T:]), sil[:, T:], carried)
    for k in ("hv", "hn", "hd", "gains", "vad"):
        np.testing.assert_allclose(torch.cat([a[k], b[k]], 1).numpy(), whole[k].numpy(), rtol=0, atol=1e-12)


def test_network_inputs_are_checked_before_the_library():
    dev = torch.device("cuda", 0)  # no tensor below lives there: every check fires before any CUDA call
    B, T, W = 4, 6, 10
    f = torch.zeros(B, T, 42)

    def check(features=f, silence=None, state=None, batch_first=True):
        return check_window(features, silence, state, batch_first, T, 8, W, dev)

    bad = [dict(features=f.double()), dict(features=f[..., :41]), dict(features=torch.zeros(B, T, 84)[..., ::2]),
           dict(features=torch.zeros(B, T + 1, 42)), dict(features=torch.zeros(9, T, 42)), dict(features=f, batch_first=False),
           dict(features=f[0]), dict(silence=torch.zeros(T, B)), dict(silence=torch.zeros(B, T, dtype=torch.int32)),
           dict(state=torch.zeros(B, W + 1)), dict(state=torch.zeros(W, B).t()), dict(state=torch.zeros(B, W, dtype=torch.float64))]
    for kw in bad:
        with pytest.raises(ValueError, match="features|silence|state"):
            check(**kw)
    for kw in (dict(), dict(silence=torch.zeros(T, B, dtype=torch.int32)), dict(state=torch.zeros(B, W)),
               dict(features=torch.zeros(T, B, 42), batch_first=False)):
        with pytest.raises(ValueError, match="must be on cuda:0"):
            check(**kw)


def test_null_fit_is_refused_without_a_gpu():
    L = nb.lib()
    x = (C.c_float * 64)()
    assert L.rnnoise_fit_forward_device(None, x, 1, x, 42, 42, None, 0, 0, None, None, x, 22, 22, x, 1, 1, None) == -1
    assert "null argument" in nb.last_error()
    assert L.rnnoise_fit_backward_device(None, x, x, 22, 22, None, 0, 0, x, None) == -1
    assert "null argument" in nb.last_error()
