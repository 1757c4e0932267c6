"""GPU tests of the lifetime of a batch's device buffers, streams and events: a batch whose buffers grow while its earlier
device calls are still queued gives the bits of a batch whose buffers grow with nothing in flight, and destroying a
batch or a trainer waits for the work queued on it."""
import contextlib
import os

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import rnn_ref
from conftest import synth_streams
from nnnoiseless_b200 import training as tr

pytestmark = pytest.mark.gpu

BUILTIN_WIDTHS = (24, 24, 48, 96)


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


def grow_everything(models, synced):
    """One batch taken cold through every growth path: host staging (pcm16, then f32), the work state and work route
    (subset calls of rising n on two models), the state-call indices and record staging (get / set states of rising n
    through host and device buffers), the model table (up to five models) and the route tables.  Before each growing
    call a full-batch device call is queued on a torch side stream; synced: the side stream is synchronised after
    every call, so nothing is in flight when a buffer grows.  Returns every output, vad and state record."""
    import torch
    B, T = 2048, 3
    rng = np.random.default_rng(41)
    subset_n, state_n = (40, 300, 1500), (30, 200, 900)
    # every device input is in place before the first call: the sequence itself never synchronises the device
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    full_in = iter([dev(frames(B, T, 100 + i)) for i in range(2 + 2 * len(subset_n) + 3 * len(state_n) + len(models))])
    subset_in = [dev(frames(n, T, 10 + k)) for k, n in enumerate(subset_n)]
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    cs = st.cuda_stream
    results = []  # numpy arrays, or device tensors read after the side stream has finished

    def after():
        if synced:
            st.synchronize()

    def queue_full_batch():
        x = next(full_in)
        o, v = torch.empty_like(x), torch.empty(T, B, device="cuda")
        with torch.cuda.stream(st):
            b.process_device(o.data_ptr(), x.data_ptr(), v.data_ptr(), T, 480, B * 480, cs)
        results.extend([o, v])
        after()

    b = nb.DenoiseBatch(B)
    assert b.add_model(nb.RnnModel.from_bytes(models[1])) == 1
    b.set_stream_models(rng.integers(0, 2, B))
    # host staging: 16-bit samples, then floats (twice the bytes)
    queue_full_batch()
    results.extend(b.process_pcm16_host(frames(B, T, 1).astype(np.int16)))
    queue_full_batch()
    results.extend(b.process_host(frames(B, T, 2)))
    # the work state and the work route: subset calls of rising n
    for k, n in enumerate(subset_n):
        queue_full_batch()
        x = subset_in[k]
        o, v = torch.empty_like(x), torch.empty(T, n, device="cuda")
        with torch.cuda.stream(st):
            b.process_streams_device(rng.choice(B, n, replace=False), o.data_ptr(), x.data_ptr(), v.data_ptr(), T, 480, n * 480,
                                     cuda_stream=cs)
        results.extend([o, v])
        after()
        queue_full_batch()
        results.extend(b.process_streams_host(rng.choice(B, n + 7, replace=False), frames(n + 7, T, 20 + k)))
    # state-call indices and record staging: get / set states of rising n, host and device buffers
    for n in state_n:
        queue_full_batch()
        results.append(b.get_states(rng.choice(B, n, replace=False)))
        queue_full_batch()
        rec = torch.empty((n + 5, b.state_bytes), dtype=torch.uint8, device="cuda")
        with torch.cuda.stream(st):
            b.get_states_device(rec.data_ptr(), rng.choice(B, n + 5, replace=False), cs)
            b.set_states_device(rec.data_ptr(), rng.choice(B, n + 5, replace=False), cs)
        results.append(rec)
        after()
        queue_full_batch()
        b.set_states(b.get_states(rng.choice(B, n + 9, replace=False)), rng.choice(B, n + 9, replace=False))
    # the model table doubles twice (room for 2 -> 4 -> 8 models), then the streams spread over all five
    for k, mb in enumerate(models[2:], 2):
        queue_full_batch()
        assert b.add_model(nb.RnnModel.from_bytes(mb)) == k
    queue_full_batch()
    b.set_stream_models(rng.integers(0, len(models), B))
    queue_full_batch()
    results.extend(b.process_host(frames(B, T, 3)))
    st.synchronize()
    results.append(b.get_states())
    return [r.cpu().numpy() if isinstance(r, torch.Tensor) else r for r in results]


def test_cold_batch_grows_like_an_idle_one(sh_bytes):
    """Buffers that grow while earlier calls are in flight leave every output, vad and state record as they are when
    nothing is in flight."""
    acts = [(rnn_ref.RELU, rnn_ref.SIGMOID, rnn_ref.TANH, rnn_ref.RELU, rnn_ref.SIGMOID, rnn_ref.TANH),
            (rnn_ref.TANH, rnn_ref.TANH, rnn_ref.RELU, rnn_ref.TANH, rnn_ref.SIGMOID, rnn_ref.SIGMOID),
            (rnn_ref.SIGMOID, rnn_ref.RELU, rnn_ref.TANH, rnn_ref.SIGMOID, rnn_ref.TANH, rnn_ref.RELU)]
    models = [nb.RnnModel().to_bytes(), sh_bytes] + [rnn_ref.make_model(*BUILTIN_WIDTHS, acts=a, seed=60 + i) for i, a in enumerate(acts)]
    cold = grow_everything(models, synced=False)
    idle = grow_everything(models, synced=True)
    assert len(cold) == len(idle)
    for k, (c, i) in enumerate(zip(cold, idle)):
        assert c.shape == i.shape and np.array_equal(c.view(np.uint8), i.view(np.uint8)), k


def destroyed_behind(kind, cuda_stream):
    """A device call queued on cuda_stream (0: a synchronous call), then the batch or trainer destroyed at once; returns
    the call's output tensors."""
    import torch
    if kind == "trainer":
        L, T = 1500, 6
        sig = torch.from_numpy(frames(L, T, seed=72)).cuda()
        noi = torch.from_numpy(frames(L, T, seed=73) * np.float32(0.1)).cuda()
        t = tr.TrainingBatch(L)
        t.set_params(tr.randomize(L, np.random.default_rng(5)))
        rows = torch.empty((T, L, tr.TRAIN_ROW), device="cuda")
        torch.cuda.synchronize()
        t.process_device(rows.data_ptr(), sig.data_ptr(), noi.data_ptr(), T, 480, L * 480, tr.TRAIN_ROW, L * tr.TRAIN_ROW, cuda_stream)
        nb.lib().rnnoise_train_destroy(t._h)
        t._h = None
        return [rows]
    B, T = 4096, 8
    x = torch.from_numpy(frames(B, T, seed=71)).cuda()
    with env(NNB_RNN_MMA="1" if kind == "mma_sync" else "0"):
        b = nb.DenoiseBatch(B)
    o, v = torch.empty_like(x), torch.empty(T, B, device="cuda")
    torch.cuda.synchronize()
    b.process_device(o.data_ptr(), x.data_ptr(), v.data_ptr(), T, 480, B * 480, cuda_stream)
    nb.lib().rnnoise_batch_destroy(b._h)
    b._h = None
    return [o, v]


@pytest.mark.parametrize("kind", ["wgmma", "mma_sync", "trainer"])
def test_destroy_waits_for_queued_work(kind):
    """A batch (either GRU kernel) or a trainer destroyed right after a device call was queued on a torch stream leaves
    that call's output as a synchronous call gives it."""
    import torch
    want = [t.cpu().numpy() for t in destroyed_behind(kind, 0)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        got = destroyed_behind(kind, st.cuda_stream)
    st.synchronize()
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert np.array_equal(bits(g.cpu().numpy()), bits(w))
