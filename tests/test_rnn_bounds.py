"""The two GRU kernels (wgmma rnn_tc.cu, mma.sync rnn_mma.cu) element by element against the per-element bound of
tests/rnn_bounds.py, one step at a time from the GPU's own previous state and features: every new state element,
raw gain and vad must lie within K times its own bound (no batch-wide floor), on the natural runs of the model
geometries of test_rnn_kernels, on testing.raw, and on the constructed states of tests/rnn_cases.py (through state
records, each case at three lanes of 64-stream tiles, one of them partial), and on a batch that runs two models of one
geometry on alternating tiles.  A saturated update gate must carry the state bit for bit; a ReLU state at or above
the f16 limit must turn the stream's gains and vad into NaN."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import rnn_bounds as rb
import rnn_cases
import rnn_ref
from test_rnn_kernels import GEOMETRIES, env, KERNELS, model_for, pack_selftest, run_frames, streams

pytestmark = pytest.mark.gpu
K = 2.0


def kernels_for(model):
    """The wgmma kernel when the model fits it (the default), and the mma.sync kernel."""
    return (["default"] if pack_selftest(model) >= 0 else []) + ["mma"]


def check_frames(model, frames, what):
    layers = rnn_ref.parse(model)
    worst = {"state": 0.0, "gains": 0.0, "vad": 0.0}
    for f, fr in enumerate(frames):
        live = np.flatnonzero(fr["silence"] == 0)
        if not len(live):
            continue
        got = (fr["gru_state"][live], fr["gains"][live], fr["vad"][live])
        _, sh = rb.check(layers, fr["prev"][live], fr["features"][live], got)
        for q, v in sh.items():
            if v.size:
                assert np.isfinite(got[("state", "gains", "vad").index(q)]).all(), (what, f, q)
                i = np.unravel_index(int(np.argmax(v)), v.shape)
                assert v.max() <= K, (what, f, q, float(v.max()), "stream", int(live[i[0]]), i)
                worst[q] = max(worst[q], float(v.max()))
    print("%-34s" % (what,), ", ".join("%s %.3f" % kv for kv in worst.items()), "of the bound")
    return worst


@pytest.mark.parametrize("gi", range(len(GEOMETRIES)), ids=["-".join(map(str, g)) for g in GEOMETRIES])
def test_gru_kernels_inside_per_element_bound(gi):
    model = model_for(gi)
    x, _ = streams(229, 6, seed=900 + gi)
    for kernel in kernels_for(model):
        check_frames(model, run_frames(model, x, kernel), (GEOMETRIES[gi], kernel))


def test_gru_kernels_inside_per_element_bound_on_testing_raw(builtin_bytes, sh_bytes, testing_raw):
    """8 streams of testing.raw, each starting 7 frames later than the one before, 40 frames."""
    x = np.ascontiguousarray(np.stack([testing_raw[7 * s:7 * s + 40] for s in range(8)], axis=1))
    for name, model in (("builtin", builtin_bytes), ("sh.rnn", sh_bytes)):
        for kernel in kernels_for(model):
            check_frames(model, run_frames(model, x, kernel), (name, kernel))


def _records_with(rec, dtype, states):
    out = np.repeat(rec[None], len(states), axis=0).view(dtype).reshape(len(states))
    nv, nn = out["vad_gru"].shape[1], out["noise_gru"].shape[1]
    out["vad_gru"] = states[:, :nv]
    out["noise_gru"] = states[:, nv:nv + nn]
    out["denoise_gru"] = states[:, nv + nn:]
    return out


@pytest.mark.parametrize("kernel", ["default", "mma"])
@pytest.mark.parametrize("which", ["builtin", "sh"])
def test_constructed_states_through_records(which, kernel, builtin_bytes, sh_bytes, testing_raw):
    model = builtin_bytes if which == "builtin" else sh_bytes
    assert pack_selftest(model) >= 0  # both models run on the wgmma kernel by default
    layers = rnn_ref.parse(model)
    B, t0 = 3 * 64 + 21, 40  # three whole tiles and a partial one
    with env(**KERNELS[kernel]):
        batch = nb.DenoiseBatch(B, nb.RnnModel.from_bytes(model))
    x = np.ascontiguousarray(np.repeat(testing_raw[:t0 + 1, None], B, axis=1))
    batch.process_host(x[:t0])
    rec = batch.get_states()[0]
    dtype = nb.state_dtype(batch.gru_widths)
    prev = np.concatenate([rec.view(dtype)[0][k] for k in ("vad_gru", "noise_gru", "denoise_gru")]).astype(np.float32)
    batch.process_host(x[t0:t0 + 1])
    F = batch.taps()["features"][0].copy()
    assert not batch.taps()["silence"].any()
    cases = [c for c in rnn_cases.build(layers, prev, F, seed=7) if c["ok"]]
    n = len(cases)
    # the cases laid out three times in a row over as many whole batches as that takes: case i sits at slots i,
    # i + n and i + 2n, three different lanes as long as neither n nor 2n is a multiple of B
    assert n % B and (2 * n) % B
    counts = {}
    worst = {"state": 0.0, "gains": 0.0, "vad": 0.0}
    for rnd in range(-(-3 * n // B)):
        idx = (rnd * B + np.arange(B)) % n
        states = np.array([cases[i]["state"] for i in idx])
        batch.set_states(_records_with(rec, dtype, states))
        batch.process_host(x[t0:t0 + 1])
        t, r = batch.taps(), batch.rnn_taps()
        assert np.array_equal(t["features"].view(np.uint32), np.repeat(F[None], B, axis=0).view(np.uint32)), rnd
        got = (r["gru_state"], r["gains"], r["vad"])
        over = np.array([bool(cases[i].get("overflow")) for i in idx])
        fin = ~over
        _, sh = rb.check(layers, states[fin], np.repeat(F[None], fin.sum(), axis=0), tuple(g[fin] for g in got))
        for q, v in sh.items():
            i = np.unravel_index(int(np.argmax(v)), v.shape)
            c = cases[idx[np.flatnonzero(fin)[i[0]]]]
            assert v.max() <= K, (q, float(v.max()), c["cls"], c["key"], c["target"], "stream", int(np.flatnonzero(fin)[i[0]]))
            worst[q] = max(worst[q], float(v.max()))
        for s, i in enumerate(idx):
            c = cases[i]
            counts[c["cls"]] = counts.get(c["cls"], 0) + 1
            if c["cls"] == "carry":  # z = 1 exactly: the state is carried bit for bit (a zero may change sign)
                g = r["gru_state"][s, c["elem"]]
                assert g == c["value"] and (g == 0 or g.view(np.uint32) == c["value"].view(np.uint32)), \
                    (kernel, c["key"], float(c["value"]), float(g), "stream", s)
            if c.get("overflow"):  # the split's hi half is inf: loud
                assert np.isnan(r["gains"][s]).all() and np.isnan(r["vad"][s]), (kernel, c["key"], float(c["value"]), s)
            else:
                assert np.isfinite(r["gains"][s]).all() and np.isfinite(r["vad"][s]), (kernel, c["cls"], c["key"], s)
    print(which, kernel, counts, ", ".join("%s %.3f" % kv for kv in worst.items()), "of the bound")


@pytest.mark.parametrize("kernel", ["default", "mma"])
def test_two_models_on_alternating_tiles(kernel, builtin_bytes, sh_bytes):
    """The built-in model and sh.rnn (one geometry, different weights and activations) on alternating 64-stream
    blocks of a 229-stream batch (the model-table path of both kernels): every stream is held to its own model's
    bound."""
    B, T = 229, 6
    x, _ = streams(B, T, seed=77)
    models = [builtin_bytes, sh_bytes]
    ids = (np.arange(B) // 64) % 2
    with env(**KERNELS[kernel]):
        batch = nb.DenoiseBatch(B, nb.RnnModel.from_bytes(builtin_bytes))
    assert batch.add_model(nb.RnnModel.from_bytes(sh_bytes)) == 1
    batch.set_stream_models(ids)
    prev = np.zeros((B, sum(batch.gru_widths)), np.float32)
    frames = []
    for f in range(T):
        batch.process_host(x[f:f + 1])
        t, r = batch.taps(), batch.rnn_taps()
        frames.append(dict(prev=prev, features=t["features"], silence=t["silence"], **r))
        prev = r["gru_state"]
    assert not frames[0]["silence"][1::11].any()
    for k, model in enumerate(models):
        sel = ids == k
        check_frames(model, [{q: v[sel] for q, v in fr.items()} for fr in frames], ("model %d of 2" % k, kernel))
