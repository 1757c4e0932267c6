"""CPU checks of the fitting kernels' per-stage bounds (tests/fit_bounds.py) on the constructed cases of
tests/fit_cases.py: the stages composed in float64 are the semantics (tests/fit_ref.py, tests/fit_synthesis_ref.py) to
1e-12, and an f32 emulation of the kernels' order and the torch f32 restatement lie inside the bound on every element."""
import numpy as np
import pytest
import torch

import fit_bounds as fb
import fit_cases as fc
import fit_synthesis_ref as fsr
from fit_ref import forward as ref_forward, loss_and_grad, l2_grad
from nnnoiseless_b200.fit import unflatten

ALL = [(k, i) for k, n in fc.COUNTS.items() for i in range(n)] + [("random", 0), ("random", 1)]


def _case(cls, i):
    if cls == "random":
        return fc.random_case((24, 24, 48, 96) if i else (5, 3, 7, 11), 2 + i, 5, 900 + i)
    return fc.CLASSES[cls]()[i]


def test_case_counts():
    assert {k: len(f()) for k, f in fc.CLASSES.items()} == fc.COUNTS


@pytest.mark.parametrize("cls,i", ALL)
def test_composed_stages_are_the_semantics(cls, i):
    c = _case(cls, i)
    _, tp = fb.run(fb.E(), c, semantic=True)
    if "gg" in c:
        sil = c["silent"]
        fw, g = fsr.forward_and_grad(c["params"], c["widths"], c["x"], np.where(sil[..., None], 0, c["gg"]),
                                     np.where(sil, 0, c["gv"]), sil, c["h0"], torch.float64)
        want = g
    else:
        _, g, fw = loss_and_grad(c["params"], c["widths"], c["rows"], c["weights"], torch.float64)
        want = g - l2_grad(c["params"], c["widths"])
    scale = max(np.abs(want).max(), 1e-30)
    assert np.abs(tp["grad"] - want).max() <= 1e-12 * scale
    live = ~c["silent"] if "gg" in c else np.ones(c["x"].shape[:2], bool)  # silent frames' gains are written as 0
    assert not live.any() or np.abs(tp["gains"][live] - fw["gains"][live]).max() <= 1e-12 * max(np.abs(fw["gains"][live]).max(), 1e-30)


@pytest.mark.parametrize("cls,i", ALL)
def test_f32_emulation_inside_bound(cls, i):
    c = _case(cls, i)
    net, tp = fb.run(fb.F32(), c)
    out, _ = fb.check_run(net, c, tp)
    worst = {k: v for k, v in fb.shares(out).items() if not v[0] <= 1.0}
    assert not worst, worst
    if tp["terms"] is not None:
        *arrays, inv = _loss_inputs(c, tp)
        _, _, terms = fb.loss_terms(fb.E(), *(fb.Val(a) for a in arrays), inv)
        for (k, ref), got in zip(fb.loss_totals(terms, tp["x"].shape[0] * tp["x"].shape[1]).items(), tp["terms"]):
            assert abs(float(np.asarray(got, np.float64).sum()) / got.shape[0] - ref.v) <= ref.e, k


def _loss_inputs(c, tp):
    R = tp["x"].shape[0] * tp["x"].shape[1]
    rw = c["rows"].reshape(R, -1)
    return (tp["gains"].reshape(R, -1), rw[:, 42:64], c["weights"].reshape(R, 1), tp["vad"].reshape(R, 1), rw[:, 86:87],
            float(np.float32(1.0 / R)))


@pytest.mark.parametrize("cls,i", [a for a in ALL if a[0] != "device"])
def test_torch_f32_restatement_inside_bound(cls, i):
    """The restatement's dense layer from the features, and its output layers from its own GRU states."""
    c = _case(cls, i)
    net = fb.Net(c["params"], c["widths"])
    P = {k: torch.as_tensor(v) for k, v in unflatten(c["params"], c["widths"]).items()}
    fw = {k: v.numpy() for k, v in ref_forward(P, c["widths"], torch.as_tensor(c["x"])).items()}
    R = c["x"].shape[0] * c["x"].shape[1]
    A = fb.E()
    g, v = fb.outputs(A, net, fb.Val(fw["hd"].reshape(R, -1)), fb.Val(fw["hv"].reshape(R, -1)))
    out = {"dense": (fw["d"].reshape(R, -1), fb.dense(A, net, fb.Val(c["x"].reshape(R, -1)))),
           "gains": (fw["gains"].reshape(R, -1), g), "vad": (fw["vad"].reshape(R, 1), v)}
    worst = {k: s for k, s in fb.shares(out).items() if not s[0] <= 1.0}
    assert not worst, worst


def test_adam_emulation_inside_bound():
    rng = np.random.default_rng(3)
    w = rng.uniform(-0.499, 0.499, 4000).astype(np.float32)
    w[:8] = np.float32(0.499)
    g = (rng.standard_normal(4000) * 10.0 ** rng.uniform(-9, 0, 4000)).astype(np.float32)
    m = v = np.zeros(4000, np.float32)
    mE = vE = fb.Val(np.zeros(4000))
    A, F = fb.E(), fb.F32()
    for t in range(1, 4):
        w32, m, v = fb.adam(F, w, g, m, v, fb.lr_t(t))
        ref, mE, vE = fb.adam(A, fb.Val(w), fb.Val(g), mE, vE, fb.lr_t(t))
        assert (np.abs(w32 - ref.v) <= ref.e).all()
        w = w32
