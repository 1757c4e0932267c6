"""GPU tests of subset calls (rnnoise_batch_process_streams_device / _host): advancing any subset of a batch's streams
gives every listed stream the bits of a full-batch call and leaves every other stream's state record unchanged.

The reference is what could already be done without subset calls: save the records of the idle streams, run a
full-batch call with zeros fed to them, and restore their records."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest

import oracle
import nnnoiseless_b200 as nb
import rnn_ref
from conftest import golden_metric, synth_streams

pytestmark = pytest.mark.gpu

ODD_OVER_WGMMA_BUDGET = (43, 41, 43, 127)  # (nd, nv, nn, ndn): runs on mma.sync; 211 state floats, rows not 16-byte aligned
N_FRAMES = (1, 2, 3, 5, 8, 9, 17)


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
    """[T][B][480] synthetic streams."""
    return np.ascontiguousarray(synth_streams(B, T, seed=seed).reshape(B, T, 480).transpose(1, 0, 2))


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


class Workaround:
    """A batch driven only by full-batch calls and state records: the reference of a subset call."""

    def __init__(self, B, model=None):
        self.b = nb.DenoiseBatch(B, model)
        self.B = B

    def subset(self, streams, x):
        streams = np.arange(x.shape[1]) if streams is None else np.asarray(streams)
        idle = np.setdiff1d(np.arange(self.B), streams)
        saved = self.b.get_states(idle) if len(idle) else None
        xf = np.zeros((x.shape[0], self.B, 480), np.float32)
        xf[:, streams] = x
        o, v = self.b.process_host(xf)
        if len(idle):
            self.b.set_states(saved, idle)
        return o[:, streams], v[:, streams]


def _random_schedule(model_bytes, seed, **env_kv):
    B, calls = 229, 40
    model = nb.RnnModel.from_bytes(model_bytes) if model_bytes is not None else None
    rng = np.random.default_rng(seed)
    pool = frames(B, 48, seed=seed)  # audio is drawn from here: stream s, frame (cursor + t) mod 48
    with env(**env_kv):
        a = nb.DenoiseBatch(B, model)
        ref = Workaround(B, model)
        donor = nb.DenoiseBatch(11, model)
    donor.process_host(frames(11, 6, seed=seed + 1))
    special = [np.array([int(rng.integers(B))]), np.arange(B), rng.permutation(B)]  # n = 1, n = B in order, permuted
    kinds = ["subset"] * (calls - 9) + ["special"] * 3 + ["full"] * 3 + ["reset"] * 2 + ["set"]
    rng.shuffle(kinds)
    cursor = 0
    for i, kind in enumerate(kinds):
        T = int(rng.choice(N_FRAMES))
        if kind in ("subset", "special"):
            S = special.pop() if kind == "special" else rng.choice(B, int(rng.integers(1, B)), replace=False)
            x = np.ascontiguousarray(pool[(cursor + np.arange(T)) % 48][:, S])
            o, v = a.process_streams_host(S, x)
            o_r, v_r = ref.subset(S, x)
            assert np.array_equal(bits(o), bits(o_r)) and np.array_equal(bits(v), bits(v_r)), (i, kind, len(S), T)
        elif kind == "full":
            x = np.ascontiguousarray(pool[(cursor + np.arange(T)) % 48])
            o, v = a.process_host(x)
            o_r, v_r = ref.b.process_host(x)
            assert np.array_equal(bits(o), bits(o_r)) and np.array_equal(bits(v), bits(v_r)), (i, kind, T)
        elif kind == "reset":
            S = rng.choice(B, 17, replace=False)
            a.reset_streams(S)
            ref.b.reset_streams(S)
        else:
            S = rng.choice(B, 11, replace=False)
            recs = donor.get_states()
            a.set_states(recs, S)
            ref.b.set_states(recs, S)
        cursor += T
    assert np.array_equal(a.get_states(), ref.b.get_states())


def test_random_schedule_bitwise():
    _random_schedule(None, 701)


def test_random_schedule_bitwise_mma():
    _random_schedule(None, 702, NNB_RNN_MMA="1")


def test_random_schedule_bitwise_odd_width_over_wgmma_budget():
    model = rnn_ref.make_model(*ODD_OVER_WGMMA_BUDGET, seed=7)
    assert sum(nb.gru_widths(model)) % 2 == 1
    _random_schedule(model, 703)


@pytest.mark.parametrize("T", [8, 16, 11])
def test_ring_rotation(T):
    """n_frames equal to the ring length, a multiple of it and more than it, from every batch phase."""
    B = 40
    rng = np.random.default_rng(T)
    for phase in range(8):
        a, ref = nb.DenoiseBatch(B), Workaround(B)
        x0 = frames(B, phase, seed=710 + phase)
        if phase:
            a.process_host(x0); ref.b.process_host(x0)
        S = rng.choice(B, 13, replace=False)
        x = frames(13, T, seed=720 + phase)
        o, v = a.process_streams_host(S, x)
        o_r, v_r = ref.subset(S, x)
        assert np.array_equal(bits(o), bits(o_r)) and np.array_equal(bits(v), bits(v_r)), phase
        assert np.array_equal(a.get_states(), ref.b.get_states()), phase
        x1 = frames(B, 3, seed=730 + phase)  # the batch's own ring continues where it was
        assert np.array_equal(bits(a.process_host(x1)[0]), bits(ref.b.process_host(x1)[0])), phase


def test_unlisted_streams_untouched():
    B = 96
    rng = np.random.default_rng(5)
    hist, later = frames(B, 5, seed=741), frames(B, 6, seed=742)
    a, never = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    a.process_host(hist)
    never.process_host(hist)
    pool = rng.choice(B, 60, replace=False)  # only these are ever listed
    rest = np.setdiff1d(np.arange(B), pool)
    before = a.get_states(rest)
    for k in range(25):
        S = rng.choice(pool, int(rng.integers(1, 61)), replace=False)
        T = int(rng.choice(N_FRAMES))
        a.process_streams_host(S, frames(len(S), T, seed=750 + k))
        assert np.array_equal(a.get_states(rest), before), k
    o, v = a.process_host(later)
    o_n, v_n = never.process_host(later)
    assert np.array_equal(bits(o[:, rest]), bits(o_n[:, rest])) and np.array_equal(bits(v[:, rest]), bits(v_n[:, rest]))


def test_golden_through_single_stream_calls(builtin_bytes, testing_raw, reference_output):
    """Stream 5 of 16 gets testing.raw only through n = 1 subset calls; the other streams get other audio at other times."""
    B, me = 16, 5
    F = len(testing_raw)
    rng = np.random.default_rng(9)
    others = np.setdiff1d(np.arange(B), [me])
    a = nb.DenoiseBatch(B)
    ost = oracle.State(oracle.Model(builtin_bytes))
    dt = nb.state_dtype(a.gru_widths)
    outs, f = [], 0
    while f < F:
        if rng.random() < 0.5:
            S = rng.choice(others, int(rng.integers(1, B)), replace=False)
            a.process_streams_host(S, frames(len(S), int(rng.integers(1, 4)), seed=760 + f))
        o, _ = a.process_streams_host([me], np.ascontiguousarray(testing_raw[f][None, None]))
        outs.append(o[0, 0])
        ost.process_frame(testing_raw[f])
        assert a.get_states([me]).view(dt)[0]["last_period"] == ost.taps().pitch, f  # the frame's pitch period
        f += 1
    o_b, _ = nb.DenoiseBatch(1).process_host(np.ascontiguousarray(testing_raw[:, None]))
    assert np.array_equal(bits(np.stack(outs)), bits(o_b[:, 0]))
    metric, maxdiff = golden_metric(outs[1:], reference_output)
    assert metric < 1e-4


def _strided(b, streams, out, inp, pcm16, vad, T, ss, sas, fs):
    idx = np.ascontiguousarray(streams, np.int32)
    return nb.lib().rnnoise_batch_process_streams_device(b._h, idx.ctypes.data_as(C.c_void_p), len(idx), C.c_void_p(out.data_ptr()),
                                                         C.c_void_p(inp.data_ptr()), pcm16, C.c_void_p(vad.data_ptr()) if vad is not None else None,
                                                         T, ss, sas, fs, None)


def test_layouts_pcm16_and_interleaved():
    """Interleaved multi-channel strides (row r of the call = channel r) with every sample format, bitwise against the
    full-batch paths of a fresh batch on the same audio."""
    import torch
    B, n, T = 12, 5, 7
    S = np.array([9, 2, 7, 0, 11])
    x = frames(n, T, seed=771)  # planar [T][n][480]
    x16 = np.ascontiguousarray(np.clip(np.rint(x), -32768, 32767).astype(np.int16))
    o_f, v_f = nb.DenoiseBatch(n).process_host(x16.astype(np.float32))
    o_16, _ = nb.DenoiseBatch(n).process_pcm16_host(x16)
    il = lambda a: torch.from_numpy(np.ascontiguousarray(a.transpose(0, 2, 1))).cuda()  # noqa: E731  [T][480][n]
    back = lambda t: t.cpu().numpy().transpose(0, 2, 1)  # noqa: E731
    for pcm16, xin, want in [(0, il(x16.astype(np.float32)), o_f), (1, il(x16), o_16), (2, il(x16.astype(np.float32)), o_16),
                             (3, il(x16), o_f)]:
        a = nb.DenoiseBatch(B)
        a.process_streams_host([1, 3], frames(2, 4, seed=772))  # other streams have moved on
        out = torch.empty(xin.shape, dtype=torch.int16 if pcm16 in (1, 2) else torch.float32, device="cuda")
        vad = torch.empty(T, n, device="cuda")
        assert _strided(a, S, out, xin, pcm16, vad, T, 1, n, 480 * n) == 0, nb.last_error()
        got = back(out)
        assert got.dtype == want.dtype, pcm16
        assert np.array_equal(got, want) if got.dtype == np.int16 else np.array_equal(bits(got), bits(want)), pcm16
        assert np.array_equal(bits(vad.cpu().numpy()), bits(v_f)), pcm16


def test_host_variant_equals_device_variant():
    """Including a call longer than the 8-frame staging ring, and streams=None (streams 0..n-1)."""
    import torch
    B = 70
    rng = np.random.default_rng(3)
    h, d = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    for k, (S, T) in enumerate([(rng.choice(B, 31, replace=False), 19), (None, 5), (rng.permutation(B), 9), (np.array([69]), 1)]):
        n = 23 if S is None else len(S)
        x = frames(n, T, seed=780 + k)
        o_h, v_h = h.process_streams_host(S, x)
        xd = torch.from_numpy(x).cuda()
        od = torch.empty_like(xd)
        vd = torch.empty(T, n, device="cuda")
        d.process_streams_device(S, od.data_ptr(), xd.data_ptr(), vd.data_ptr(), T, 480, n * 480, n=n)
        assert np.array_equal(bits(od.cpu().numpy()), bits(o_h)) and np.array_equal(bits(vd.cpu().numpy()), bits(v_h)), k
    assert np.array_equal(h.get_states(), d.get_states())


def test_device_calls_ordered_on_a_torch_stream():
    """Full-batch, subset and state calls on one torch side stream with no host synchronisation give the bits of the
    synchronised host sequence."""
    import torch
    B, T1, T2, T3 = 4096, 6, 9, 4
    rng = np.random.default_rng(8)
    S1 = rng.choice(B, 1500, replace=False)
    S2 = rng.choice(B, 700, replace=False)
    P = rng.permutation(B)[:300]
    x1, x2, x3, x4 = frames(B, T1, seed=791), frames(len(S1), T2, seed=792), frames(len(S2), T3, seed=793), frames(B, T1, seed=794)
    r = nb.DenoiseBatch(B)
    want = [r.process_host(x1)]
    want.append(r.process_streams_host(S1, x2))
    r.set_states(r.get_states(S2[:300]), P)
    want.append(r.process_streams_host(S2, x3))
    want.append(r.process_host(x4))
    a = nb.DenoiseBatch(B)
    ins = [torch.from_numpy(x).cuda() for x in (x1, x2, x3, x4)]
    outs = [torch.empty_like(t) for t in ins]
    vads = [torch.empty(t.shape[0], t.shape[1], device="cuda") for t in ins]
    rec = torch.empty((300, a.state_bytes), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        cs = st.cuda_stream
        a.process_device(outs[0].data_ptr(), ins[0].data_ptr(), vads[0].data_ptr(), T1, 480, B * 480, cs)
        a.process_streams_device(S1, outs[1].data_ptr(), ins[1].data_ptr(), vads[1].data_ptr(), T2, 480, len(S1) * 480, cuda_stream=cs)
        a.get_states_device(rec.data_ptr(), S2[:300], cs)
        a.set_states_device(rec.data_ptr(), P, cs)
        a.process_streams_device(S2, outs[2].data_ptr(), ins[2].data_ptr(), vads[2].data_ptr(), T3, 480, len(S2) * 480, cuda_stream=cs)
        a.process_device(outs[3].data_ptr(), ins[3].data_ptr(), vads[3].data_ptr(), T1, 480, B * 480, cs)
    st.synchronize()
    for k, (o, v) in enumerate(want):
        assert np.array_equal(bits(outs[k].cpu().numpy()), bits(o)) and np.array_equal(bits(vads[k].cpu().numpy()), bits(v)), k


def test_rejects_bad_calls_without_side_effects():
    import torch
    B = 40
    b = nb.DenoiseBatch(B)
    b.process_host(frames(B, 4, seed=801))
    before = b.get_states()
    x = torch.from_numpy(frames(5, 2, seed=802)).cuda()
    o = torch.empty_like(x)
    L = nb.lib()
    raw = lambda n, T=2, inp=x, out=o: L.rnnoise_batch_process_streams_device(  # noqa: E731
        b._h, None, n, C.c_void_p(out.data_ptr()) if out is not None else None, C.c_void_p(inp.data_ptr()) if inp is not None else None,
        0, None, T, 480, 1, 5 * 480, None)
    cases = [
        (lambda: b.process_streams_device([1, 2, 3, 4, B], o.data_ptr(), x.data_ptr(), 0, 2, 480, 5 * 480), "out of range"),
        (lambda: b.process_streams_device([1, 2, -1, 4, 5], o.data_ptr(), x.data_ptr(), 0, 2, 480, 5 * 480), "out of range"),
        (lambda: b.process_streams_device([1, 2, 3, 2, 5], o.data_ptr(), x.data_ptr(), 0, 2, 480, 5 * 480), "twice"),
        (lambda: b.process_streams_host([1, 2, 3, 2, 5], frames(5, 2, seed=803)), "twice"),
        (lambda: raw(B + 1), "more streams"),
        (lambda: raw(-1), "negative number"),
        (lambda: raw(5, T=-1), "negative n_frames"),
        (lambda: raw(5, inp=None), "null"),
        (lambda: raw(5, out=None), "null"),
    ]
    for call, text in cases:
        try:
            rc = call()
        except nb.NnnoiselessError as e:  # the wrappers raise
            assert text in str(e), (text, str(e))
        else:  # raw C calls return the code
            assert rc < 0 and text in nb.last_error(), (text, nb.last_error())
        assert np.array_equal(b.get_states(), before), text
    # nothing to do: no-ops, also without buffers
    assert raw(0, inp=None, out=None) == 0 and raw(5, T=0, inp=None, out=None) == 0
    b.process_streams_host([], np.zeros((3, 0, 480), np.float32))
    assert np.array_equal(b.get_states(), before)
    # taps describe full-batch frames only
    b.process_streams_host([3], frames(1, 1, seed=804))
    for taps in (b.taps, b.rnn_taps):
        with pytest.raises(nb.NnnoiselessError, match="subset"):
            taps()
    b.process_host(frames(B, 1, seed=805))
    b.taps(); b.rnn_taps()


def test_size_and_growth():
    """65,536-class batch: n = 4,000, then n = B (the work state grows); 256 streams checked against the reference."""
    import torch
    B = 33829
    rng = np.random.default_rng(11)
    a, ref = nb.DenoiseBatch(B), Workaround(B)
    x0 = frames(B, 2, seed=811)
    a.process_host(x0); ref.b.process_host(x0)
    check = rng.choice(B, 256, replace=False)
    for k, (S, T) in enumerate([(rng.choice(B, 4000, replace=False), 3), (rng.permutation(B), 2)]):
        x = frames(len(S), T, seed=812 + k)
        xd = torch.from_numpy(x).cuda()
        od = torch.empty_like(xd)
        vd = torch.empty(T, len(S), device="cuda")
        a.process_streams_device(S, od.data_ptr(), xd.data_ptr(), vd.data_ptr(), T, 480, len(S) * 480)
        o_r, v_r = ref.subset(S, x)
        rows = np.flatnonzero(np.isin(S, check))
        assert len(rows) or k == 0
        assert np.array_equal(bits(od.cpu().numpy()[:, rows]), bits(o_r[:, rows])), k
        assert np.array_equal(bits(vd.cpu().numpy()[:, rows]), bits(v_r[:, rows])), k
        assert np.array_equal(a.get_states(check), ref.b.get_states(check)), k
