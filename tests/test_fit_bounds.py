"""GPU tests of the fitting kernels (csrc/fit.cu) stage by stage: every element of every stage against the float64
reference of tests/fit_bounds.py evaluated from the GPU's own inputs to that stage (rnnoise_fit_get_taps), within K
times its rounding bound and with no batch-wide floor; at 1 .. 8 windows per recurrence CTA (a full and a partial
last group), exact split-K edges and the 256-split cap, both recurrence instantiations, and a fit of more than
4,194,240 rows (65,535 row tiles of 64).  Taps change no bit and no launch count."""
import numpy as np
import pytest
import torch

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import fit
import fit_bounds as fb
import fit_cases as fc

pytestmark = pytest.mark.gpu
K = 2.0


def _report(case, out, ties):
    sh = fb.shares(out, K)
    worst = max(sh.items(), key=lambda kv: kv[1][0])
    print("%s: worst %s share %.3g at %s (got %r ref %r bound %r); ties %s" % (case, worst[0], worst[1][0], worst[1][1], worst[1][2],
                                                                              worst[1][3], worst[1][4], ties))
    for k, (s, idx, got, ref, e) in sh.items():
        print("  %-18s %.3g" % (k, s))
    bad = {k: v for k, v in sh.items() if not v[0] <= K}
    assert not bad, "%s: over %g x the bound: %s" % (case, K, bad)


def _rows_run(c, taps=True):
    S, T = c["x"].shape[:2]
    f = fit.Fit(c["widths"], S, T, device=0)
    f.set_params(c["params"])
    f.set_taps(taps)
    ev = f.evaluate(c["rows"], c["weights"])
    loss = f.step(c["rows"], c["weights"])
    return f, ev, loss


def _taps(f, S):
    tp = f.taps(S)
    act = f.activations(S)
    tp["gains"], tp["vad"] = act["gains"], act["vad"]
    return tp


SHAPES = [((24, 24, 48, 96), 1, 8), ((24, 24, 48, 96), 37, 4), ((24, 24, 48, 96), 133, 3), ((5, 3, 7, 11), 265, 3),
          ((24, 24, 48, 96), 1056, 2), ((96, 96, 96, 96), 1057, 2), ((1, 1, 1, 1), 7, 5), ((5, 3, 7, 11), 16, 128),
          ((5, 3, 7, 11), 683, 3), ((24, 24, 48, 96), 32, 200), ((1, 1, 1, 1), 4097, 128)]


@pytest.mark.parametrize("widths,S,T", SHAPES)
def test_rows_path_stages(widths, S, T):
    case = "rows %s S=%d T=%d R=%d" % (",".join(map(str, widths)), S, T, S * T)
    c = fc.random_case(widths, S, T, seed=S + T)
    f, ev, loss = _rows_run(c)
    assert loss == ev["loss"]
    tp = _taps(f, S)
    tp["grad"] = f.grads()
    net = fb.Net(c["params"], widths)
    tp["x"] = c["x"]
    out, ties = fb.check_run(net, c, tp, l2=True)
    # the loss: fit_finish's f64 sums of the per-row terms, from the GPU's own gains and vad
    R = S * T
    terms = out.pop("loss rows")[1]
    tot = fb.loss_totals(terms, R)
    for k in ("mycost", "crossentropy", "msse"):
        out["loss " + k] = (np.array([ev[k]]), fb.Val(np.array([float(tot[k].v)]), np.array([float(tot[k].e)])))
    # Adam and the clip, step 1 (m = v = 0), from the GPU's own full gradient
    w, _, _ = fb.adam(fb.E(), fb.Val(c["params"]), fb.Val(tp["grad"]), fb.Val(np.zeros(net.flat.size)), fb.Val(np.zeros(net.flat.size)),
                      fb.lr_t(1))
    out["adam"] = (f.get_params(), w)
    _report(case, out, ties)


@pytest.mark.parametrize("widths,S,T,mask", [((24, 24, 48, 96), 133, 5, "random"), ((5, 3, 7, 11), 1057, 3, "mixed"),
                                             ((96, 96, 96, 96), 3, 40, "random")])
def test_device_path_stages(widths, S, T, mask):
    """The kCarry instantiation: silence, state_in, and a signed grad_vad for which the vad output bias's gradient
    cancels."""
    case = "device %s S=%d T=%d" % (",".join(map(str, widths)), S, T)
    rng = np.random.default_rng(S * T)
    if mask == "random":
        m = rng.random((S, T)) < 0.25
    else:
        m = np.zeros((S, T), bool)
        m[0::4, 0] = True
        m[1::4, -1] = True
        m[2::4] = True
        m[3::4] = rng.random((len(m[3::4]), T)) < 0.3
    c = fc.random_case(widths, S, T, seed=S + 2 * T, device=True, mask=m)
    f = fit.Fit(widths, S, T, device=0)
    f.set_taps(True)
    params = torch.as_tensor(c["params"]).cuda()
    x = torch.as_tensor(c["x"]).cuda()
    sil = torch.as_tensor(np.ascontiguousarray(m.T), dtype=torch.int32).cuda()
    h0 = torch.as_tensor(c["h0"]).cuda()
    gains = torch.empty((S, T, 22), device="cuda")
    vad = torch.empty((S, T), device="cuda")
    f.forward_device(params.data_ptr(), S, x.data_ptr(), T * 42, 42, sil.data_ptr(), 1, S, h0.data_ptr(), 0, gains.data_ptr(), T * 22,
                     22, vad.data_ptr(), T, 1)
    torch.cuda.synchronize()
    gv = fb.cancelling_gv(c["gv"], vad.cpu().numpy(), m)  # the vad output bias's gradient cancels
    gg = torch.as_tensor(np.where(m[..., None], np.nan, c["gg"]).astype(np.float32)).cuda()
    gvt = torch.as_tensor(np.where(m, np.nan, gv).astype(np.float32)).cuda()
    grad = torch.empty_like(params)
    f.backward_device(params.data_ptr(), gg.data_ptr(), T * 22, 22, gvt.data_ptr(), T, 1, grad.data_ptr())
    torch.cuda.synchronize()
    tp = _taps(f, S)
    tp["grad"] = grad.cpu().numpy()
    tp["x"] = np.where(m[..., None], 0.0, c["x"]).astype(np.float32)
    c["gg"], c["gv"] = np.where(m[..., None], 0.0, c["gg"]).astype(np.float32), np.where(m, 0.0, gv).astype(np.float32)
    net = fb.Net(c["params"], widths)
    out, ties = fb.check_run(net, c, tp)
    for i in range(3):  # silent rows: z = 1 and zero gate gradients exactly, dh passed through
        n = net.n[i]
        assert (tp["gates"][i][m][:, :n] == 1.0).all()
        assert (tp["dG"][i][m] == 0.0).all()
    _report(case, out, ties)


def test_taps_change_no_bit_and_no_launch():
    c = fc.random_case((24, 24, 48, 96), 133, 6, seed=3)
    res = []
    for taps in (False, True):
        S, T = c["x"].shape[:2]
        f = fit.Fit(c["widths"], S, T, device=0)
        f.set_params(c["params"])
        f.set_taps(taps)
        n0 = nb.kernel_launches()
        losses = [f.step(c["rows"], c["weights"]) for _ in range(3)]
        res.append((nb.kernel_launches() - n0, losses, f.grads().tobytes(), f.get_params().tobytes(), f.export()))
    assert res[0] == res[1]


def test_more_than_65535_row_tiles():
    """R = 4,097 x 1,024 = 4,195,328 rows, past 65,535 tiles of 64: the step runs, and the per-row stages hold on
    sequences that include the last tile's."""
    widths, S, T = (1, 1, 1, 1), 4097, 1024
    c = fc.random_case(widths, S, T, seed=1)
    f, ev, loss = _rows_run(c)
    assert np.isfinite(loss) and loss == ev["loss"]
    tp = _taps(f, S)
    tp["x"] = c["x"]
    tp["grad"] = f.grads()
    assert np.isfinite(tp["grad"]).all()
    net = fb.Net(c["params"], widths)
    out, ties = fb.check_run(net, c, tp, seqs=[0, 1, 2047, 4095, 4096])
    out.pop("loss rows")
    _report("rows 1,1,1,1 S=4097 T=1024 (sampled)", out, ties)


def test_taps_refusals():
    """A backward's taps are refused after a forward alone, dG / dht after a backward without taps, and every tap for
    another n_seq than the most recent forward's."""
    c = fc.random_case((5, 3, 7, 11), 4, 3, seed=8)
    f = fit.Fit(c["widths"], 4, 3, device=0)
    f.set_params(c["params"])
    f.evaluate(c["rows"], c["weights"])
    assert f.taps(4, backward=False)["gates"][2].shape == (4, 3, 33)
    for call in (lambda: f.taps(4), lambda: f.taps(3, backward=False), lambda: f.taps(5, backward=False)):
        with pytest.raises(nb.NnnoiselessError):
            call()
    f.step(c["rows"], c["weights"])
    with pytest.raises(nb.NnnoiselessError, match="taps on"):
        f.taps(4)
    f.set_taps(True)
    f.step(c["rows"], c["weights"])
    assert np.isfinite(f.taps(4)["dht"][0]).all()
