"""GPU tests of per-stream models (rnnoise_batch_add_model / set_stream_models / get_stream_models): a stream on model k
of a batch's model table gives bit for bit what it gives in a batch created with model k -- output, vad, state record
and rnn_taps row -- whatever the other streams run, in full-batch calls, subset calls and with frames in flight."""
import contextlib
import os

import numpy as np
import pytest

import oracle
import nnnoiseless_b200 as nb
import rnn_ref
from conftest import golden_metric, synth_streams

pytestmark = pytest.mark.gpu

TANH, SIGMOID, RELU = rnn_ref.TANH, rnn_ref.SIGMOID, rnn_ref.RELU
BUILTIN_WIDTHS = (24, 24, 48, 96)
ODD_OVER_WGMMA_BUDGET = (43, 41, 43, 127)  # runs on mma.sync


@contextlib.contextmanager
def env(**kv):
    """The kernel selection is read from the environment when a batch is created."""
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def frames(B, T, seed):
    """[T][B][480] synthetic streams (silent and fading ones included)."""
    return np.ascontiguousarray(synth_streams(B, T, seed=seed).reshape(B, T, 480).transpose(1, 0, 2))


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def three_models(sh_bytes):
    """The built-in model, sh.rnn (tanh in two GRUs) and a generated model of that geometry with other activations."""
    gen = rnn_ref.make_model(*BUILTIN_WIDTHS, acts=(RELU, SIGMOID, TANH, RELU, SIGMOID, TANH), seed=11)
    return [None, sh_bytes, gen]


def as_model(mb):
    return nb.RnnModel.from_bytes(mb) if mb is not None else None


def mixed_batch(B, models, ids=None):
    b = nb.DenoiseBatch(B, as_model(models[0]))
    for k, mb in enumerate(models[1:], 1):
        assert b.add_model(as_model(mb)) == k
    if ids is not None:
        b.set_stream_models(ids)
    return b


def run(b, x):
    """Full-batch host frames -> (out, vad, state records, rnn_taps)."""
    o, v = b.process_host(x)
    return o, v, b.get_states(), b.rnn_taps()


def assert_rows_equal(got, ref, rows, what=""):
    o, v, st, taps = got
    o_r, v_r, st_r, taps_r = ref
    assert np.array_equal(bits(o[:, rows]), bits(o_r[:, rows])), ("out", what)
    assert np.array_equal(bits(v[:, rows]), bits(v_r[:, rows])), ("vad", what)
    assert np.array_equal(st[rows], st_r[rows]), ("state", what)
    for key in ("gains", "vad", "gru_state"):
        assert np.array_equal(bits(taps[key][rows]), bits(taps_r[key][rows])), (key, what)


def check_against_singles(models, ids, x, **env_kv):
    B = x.shape[1]
    with env(**env_kv):
        got = run(mixed_batch(B, models, ids), x)
        for k, mb in enumerate(models):
            rows = np.flatnonzero(ids == k)
            if len(rows):
                assert_rows_equal(got, run(nb.DenoiseBatch(B, as_model(mb)), x), rows, "model %d" % k)


@pytest.mark.parametrize("kernel", ["default", "mma"])
def test_mixed_batch_matches_single_model_batches(sh_bytes, kernel):
    models = three_models(sh_bytes)
    B = 229
    ids = np.random.default_rng(5).integers(0, 3, B).astype(np.int32)
    check_against_singles(models, ids, frames(B, 24, seed=501), **({"NNB_RNN_MMA": "1"} if kernel == "mma" else {}))


@pytest.mark.parametrize("layout", ["contiguous", "round_robin"])
def test_tile_boundaries_and_persistent_loop(sh_bytes, layout):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 2 * (2 * sms * 64) + 37  # two passes of the persistent grid of the wgmma kernel, and a partial tile
    models = three_models(sh_bytes)
    sizes = [1, 63, 64, 65, 127, 129]
    if layout == "contiguous":
        ids = np.zeros(B, np.int32)
        at = 0
        for i, n in enumerate(sizes):
            ids[at:at + n] = i % 3
            at += n
        ids[at:] = np.arange(B - at) * 3 // (B - at)  # the rest: three groups
    else:
        ids = (np.arange(B) % 3).astype(np.int32)
    check_against_singles(models, ids, frames(B, 3, seed=502))


def test_switching_with_frames_in_flight(sh_bytes):
    """Pipelined device calls on a side stream; between calls half the streams change model, and one stream on every
    frame.  The reference: one single-model batch per model, a stream's record moved between them when it switches."""
    import torch
    models = three_models(sh_bytes)
    B, K = 229, 3
    rng = np.random.default_rng(9)
    x = frames(B, 12, seed=503)
    a = mixed_batch(B, models)
    refs = [nb.DenoiseBatch(B, as_model(mb)) for mb in models]
    ids = np.zeros(B, np.int32)
    side = torch.cuda.Stream()
    xin = torch.from_numpy(x.transpose(1, 0, 2).copy()).cuda()  # [B][T][480]
    out = torch.empty_like(xin)
    vad = torch.empty((x.shape[0], B), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    t = 0
    for T in (3, 1, 2, 1, 1, 2, 2):
        for f in range(T):
            new = ids.copy()
            if f == 0:
                half = rng.choice(B, B // 2, replace=False)
                new[half] = rng.integers(0, K, len(half))
            new[int(rng.integers(B))] = int(rng.integers(K))
            moved = np.flatnonzero(new != ids)
            for s in moved:
                refs[new[s]].set_states(refs[ids[s]].get_states([s]), [s])
            a.set_stream_models(new[moved], moved)
            ids = new
            with torch.cuda.stream(side):
                a.process_device(out[:, t].data_ptr(), xin[:, t].data_ptr(), vad[t].data_ptr(), 1, x.shape[0] * 480, 480,
                                 cuda_stream=side.cuda_stream)
            o_r = [r.process_host(x[t:t + 1]) for r in refs]
            side.synchronize()
            o = out[:, t].cpu().numpy()
            v = vad[t].cpu().numpy()
            for k in range(K):
                rows = ids == k
                assert np.array_equal(bits(o[rows]), bits(o_r[k][0][0][rows])), (t, k)
                assert np.array_equal(bits(v[rows]), bits(o_r[k][1][0][rows])), (t, k)
            t += 1
    assert np.array_equal(a.stream_models(), ids)
    st = a.get_states()
    for k in range(K):
        assert np.array_equal(st[ids == k], refs[k].get_states()[ids == k])


def test_switching_inside_pipelined_calls(sh_bytes):
    """Multi-frame device calls issued back to back without a host wait, the assignment changed between them."""
    import torch
    models = three_models(sh_bytes)
    B, K = 229, 3
    rng = np.random.default_rng(10)
    x = frames(B, 9, seed=504)
    a = mixed_batch(B, models)
    refs = [nb.DenoiseBatch(B, as_model(mb)) for mb in models]
    side = torch.cuda.Stream()
    xin = torch.from_numpy(x.transpose(1, 0, 2).copy()).cuda()
    out = torch.empty_like(xin)
    vad = torch.empty((x.shape[0], B), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    plan, ids, t = [], np.zeros(B, np.int32), 0
    for T in (3, 2, 4):
        new = ids.copy()
        half = rng.choice(B, B // 2, replace=False)
        new[half] = rng.integers(0, K, len(half))
        a.set_stream_models(new)
        with torch.cuda.stream(side):
            a.process_device(out[:, t].data_ptr(), xin[:, t].data_ptr(), vad[t].data_ptr(), T, x.shape[0] * 480, 480,
                             cuda_stream=side.cuda_stream)
        plan.append((t, T, ids, new))
        ids, t = new, t + T
    side.synchronize()
    o_all, v_all = out.cpu().numpy(), vad.cpu().numpy()
    for t0, T, old, new in plan:
        for s in np.flatnonzero(new != old):
            refs[new[s]].set_states(refs[old[s]].get_states([s]), [s])
        o_r = [r.process_host(x[t0:t0 + T]) for r in refs]
        for k in range(K):
            rows = new == k
            assert np.array_equal(bits(o_all[rows, t0:t0 + T]), bits(o_r[k][0][:, rows].transpose(1, 0, 2))), (t0, k)
            assert np.array_equal(bits(v_all[t0:t0 + T, rows]), bits(o_r[k][1][:, rows])), (t0, k)


@pytest.mark.parametrize("kernel", ["default", "mma"])
def test_growing_the_table_with_frames_in_flight(sh_bytes, kernel):
    """Models added after frames have run: three frames on model 0, then model 1 is added and a third of the streams move
    to it, three more frames, then model 2 and another third, three more.  Last, every stream moves to model 2 for three
    frames: the one-model kernel on an added model.  The frames are pipelined device calls on a side stream, so each
    add_model waits for frames in flight before it copies the table.  The reference: one single-model batch per model, a
    stream's record moved between them when it switches."""
    import torch
    models = three_models(sh_bytes)
    B, K, T = 229, 3, 3
    thirds = np.array_split(np.random.default_rng(15).permutation(B), K)
    plan = [(None, thirds[0][:0], 0), (1, thirds[0], 1), (2, thirds[1], 2), (None, np.concatenate([thirds[0], thirds[2]]), 2)]
    x = frames(B, len(plan) * T, seed=511)
    with env(**({"NNB_RNN_MMA": "1"} if kernel == "mma" else {})):
        a = nb.DenoiseBatch(B, as_model(models[0]))
        refs = [nb.DenoiseBatch(B, as_model(mb)) for mb in models]
    side = torch.cuda.Stream()
    xin = torch.from_numpy(x.transpose(1, 0, 2).copy()).cuda()  # [B][T][480]
    out = torch.empty_like(xin)
    vad = torch.empty((x.shape[0], B), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    for i, (added, moved, k) in enumerate(plan):
        if added is not None:
            assert a.add_model(as_model(models[added])) == added
        if len(moved):
            a.set_stream_models(np.full(len(moved), k, np.int32), moved)
        for t in range(i * T, (i + 1) * T):
            with torch.cuda.stream(side):
                a.process_device(out[:, t].data_ptr(), xin[:, t].data_ptr(), vad[t].data_ptr(), 1, x.shape[0] * 480, 480,
                                 cuda_stream=side.cuda_stream)
    side.synchronize()
    o_all, v_all = out.cpu().numpy(), vad.cpu().numpy()
    ids = np.zeros(B, np.int32)
    for i, (_, moved, k) in enumerate(plan):
        for j in range(K):
            src = moved[ids[moved] == j]
            if len(src) and j != k:
                refs[k].set_states(refs[j].get_states(src), src)
        ids[moved] = k
        t0 = i * T
        o_r = [r.process_host(x[t0:t0 + T]) for r in refs]
        for j in np.unique(ids):
            rows = ids == j
            assert np.array_equal(bits(o_all[rows, t0:t0 + T]), bits(o_r[j][0][:, rows].transpose(1, 0, 2))), (t0, j)
            assert np.array_equal(bits(v_all[t0:t0 + T, rows]), bits(o_r[j][1][:, rows])), (t0, j)
    assert np.array_equal(a.stream_models(), ids)
    st = a.get_states()
    for k in range(K):
        assert np.array_equal(st[ids == k], refs[k].get_states()[ids == k])


@pytest.mark.parametrize("case", ["one_model", "several_models", "single_stream"])
def test_subset_calls_on_mixed_batch(sh_bytes, case):
    models = three_models(sh_bytes)
    B = 229
    rng = np.random.default_rng(12)
    ids = rng.integers(0, 3, B).astype(np.int32)
    a = mixed_batch(B, models, ids)
    ref = mixed_batch(B, models, ids)
    warm = frames(B, 3, seed=505)
    a.process_host(warm)
    ref.process_host(warm)
    if case == "one_model":
        S = rng.permutation(np.flatnonzero(ids == 2))[:40]
    elif case == "several_models":
        S = rng.choice(B, 100, replace=False)
    else:
        S = np.array([int(rng.integers(B))])
    x = frames(len(S), 5, seed=506)
    idle = np.setdiff1d(np.arange(B), S)
    before = a.get_states(idle)
    o, v = a.process_streams_host(S, x)
    assert np.array_equal(a.get_states(idle), before)
    # the same frames as full-batch calls, zeros fed to the idle streams, their records restored
    saved = ref.get_states(idle)
    xf = np.zeros((x.shape[0], B, 480), np.float32)
    xf[:, S] = x
    o_r, v_r = ref.process_host(xf)
    ref.set_states(saved, idle)
    assert np.array_equal(bits(o), bits(o_r[:, S])) and np.array_equal(bits(v), bits(v_r[:, S]))
    assert np.array_equal(a.get_states(), ref.get_states())


def test_every_stream_on_one_added_model(sh_bytes):
    models = three_models(sh_bytes)
    B = 229
    x = frames(B, 10, seed=507)
    for k in (1, 2):
        got = run(mixed_batch(B, models, np.full(B, k, np.int32)), x)
        assert_rows_equal(got, run(nb.DenoiseBatch(B, as_model(models[k])), x), np.arange(B), "model %d" % k)


def test_over_wgmma_budget_runs_on_mma():
    acts = [(TANH, TANH, RELU, TANH, SIGMOID, SIGMOID), (RELU, SIGMOID, TANH, RELU, SIGMOID, TANH),
            (SIGMOID, TANH, TANH, SIGMOID, TANH, SIGMOID)]
    models = [rnn_ref.make_model(*ODD_OVER_WGMMA_BUDGET, acts=a, seed=20 + i) for i, a in enumerate(acts)]
    B = 229
    ids = np.random.default_rng(13).integers(0, 3, B).astype(np.int32)
    check_against_singles(models, ids, frames(B, 12, seed=508))


def test_rejected_calls_change_nothing(sh_bytes):
    models = three_models(sh_bytes)
    B = 229
    ids = np.random.default_rng(14).integers(0, 3, B).astype(np.int32)
    a = mixed_batch(B, models, ids)
    ref = mixed_batch(B, models, ids)
    other = nb.RnnModel.from_bytes(rnn_ref.make_model(24, 25, 48, 96, seed=3))
    with pytest.raises(nb.NnnoiselessError, match=r"layer vad_gru: 24 inputs x 25 neurons, the batch's model has 24 x 24"):
        a.add_model(other)
    with pytest.raises(nb.NnnoiselessError, match=r"model id 3 of stream 5 out of range 0\.\.2"):
        a.set_stream_models([1, 3], [4, 5])
    with pytest.raises(nb.NnnoiselessError, match=r"model id -1 of stream 0 out of range 0\.\.2"):
        a.set_stream_models(np.full(B, -1))
    with pytest.raises(nb.NnnoiselessError, match=r"stream index 4 given twice"):
        a.set_stream_models([1, 2], [4, 4])
    with pytest.raises(nb.NnnoiselessError, match=r"stream index 229 out of range"):
        a.set_stream_models([1], [229])
    assert np.array_equal(a.stream_models(), ids)
    x = frames(B, 6, seed=509)
    assert_rows_equal(run(a, x), run(ref, x), np.arange(B))


def test_oracle_tie_in_mixed_batch(sh_bytes, builtin_bytes, testing_raw, reference_output):
    T = 100
    B = 37
    x = np.zeros((T, B, 480), np.float32)
    x[:, :] = testing_raw[:T][:, None, :]
    x[:, 1::2] += frames(B, T, seed=510)[:, 1::2] * 0.25
    ids = (np.arange(B) % 2).astype(np.int32)  # even streams: the built-in model, odd: sh.rnn
    b = mixed_batch(B, [None, sh_bytes], ids)
    outs, pitch = [], []
    o = np.empty((T, B, 480), np.float32)
    v = np.empty((T, B), np.float32)
    for f in range(T):
        o[f:f + 1], v[f:f + 1] = b.process_host(x[f:f + 1])
        pitch.append(b.taps()["pitch"].copy())
    pitch = np.array(pitch)  # [T][B]
    # a built-in stream fed testing.raw: the golden vector and bit-exact pitch
    metric, _ = golden_metric(list(o[1:, 0]), reference_output)
    assert metric <= 1e-4
    ref = oracle.run_batch(oracle.Model(builtin_bytes), np.ascontiguousarray(x[:, ::2].transpose(1, 0, 2)), n_threads=0)
    assert np.array_equal(pitch[-1, ::2], ref["pitch"][:, -1])
    # sh.rnn streams: the oracle's tolerances for that model
    ref = oracle.run_batch(oracle.Model(sh_bytes), np.ascontiguousarray(x[:, 1::2].transpose(1, 0, 2)), n_threads=0)
    o_r = ref["out"].transpose(1, 0, 2).astype(np.float64)
    rel = np.sqrt(((o[:, 1::2] - o_r) ** 2).sum() / (o_r ** 2).sum())
    assert rel <= 1e-5, rel
    assert np.abs(v[:, 1::2] - ref["vad"].T).max() <= 1e-4
