"""GPU tests of per-stream state records (rnnoise_batch_get_states / set_states / reset_streams, rnnoise_clone): the
GPU's records decode to the oracle's state, records move streams between slots, batches and devices bit for bit, the
calls are ordered with the frame pipeline, bad records are rejected without side effects, and a cloned legacy state
continues like the original."""
import contextlib
import os

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle_state as ost
import rnn_ref
from conftest import golden_metric, synth_streams

pytestmark = pytest.mark.gpu

OUT_REL_RMS = 1e-5
VAD_ATOL = 1e-4
TAPS = ("pitch", "silence", "features", "gains")
OVER_WGMMA_BUDGET = (43, 42, 43, 127)  # (nd, nv, nn, ndn): too large for the wgmma kernel, runs on mma.sync


def rel_rms(a, b):
    a = a.astype(np.float64); b = b.astype(np.float64)
    return np.sqrt(((a - b) ** 2).sum() / max((b ** 2).sum(), 1e-30))


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
    """[T][B][480] synthetic streams (no cut to digital silence)."""
    return np.ascontiguousarray(synth_streams(B, T, seed=seed).reshape(B, T, 480).transpose(1, 0, 2))


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def test_state_bytes_matches_dtype(builtin_bytes, sh_bytes):
    for model in (builtin_bytes, sh_bytes, rnn_ref.make_model(5, 13, 37, 45, seed=3)):
        b = nb.DenoiseBatch(3, nb.RnnModel.from_bytes(model))
        w = nb.gru_widths(model)
        assert b.state_bytes == nb.state_dtype(w).itemsize == nb.state_bytes(w) == ost.Model(model).state_bytes
        rec = b.get_states()
        d = rec.view(nb.state_dtype(w))[:, 0]
        assert (d["magic"] == nb.STATE_MAGIC).all() and (d["version"] == 1).all()
        assert (d["nv"] == w[0]).all() and (d["nn"] == w[1]).all() and (d["nd"] == w[2]).all()
        assert not rec[:, 20:].any()  # a fresh stream


def test_gpu_state_matches_oracle_state(builtin_bytes, testing_raw):
    """37 synthetic streams and testing.raw for 25 frames: the decoded records of the GPU and of the oracle agree, the
    order-exact fields bit for bit."""
    T = 25
    x = np.concatenate([frames(37, T, seed=601), testing_raw[:T, None]], axis=1)  # [T][38][480]
    b = nb.DenoiseBatch(x.shape[1])
    b.process_host(x)
    dt = nb.state_dtype(b.gru_widths)
    g = b.get_states().view(dt)[:, 0]
    _, _, _, states = ost.run(ost.Model(builtin_bytes), x.transpose(1, 0, 2))
    o = np.stack([s.export() for s in states]).view(dt)[:, 0]
    for f in ("magic", "version", "nv", "nn", "nd", "mem_id", "last_period"):
        assert np.array_equal(g[f], o[f]), f
    for f in ("input_mem", "mem_hp_x", "last_gain"):
        assert np.array_equal(bits(g[f]), bits(o[f])), f
    assert np.abs(g["cepstral_mem"] - o["cepstral_mem"]).max() <= 1e-4
    assert np.abs(g["lastg"] - o["lastg"]).max() <= 1e-4
    assert rel_rms(g["synthesis_mem"], o["synthesis_mem"]) <= 1e-5
    dev = max(float(np.abs(g[f] - o[f]).max()) for f in ("vad_gru", "noise_gru", "denoise_gru"))
    print("largest GRU state deviation from the oracle after %d frames: %.3g" % (T, dev))
    assert dev <= 1e-3


def test_oracle_records_continue_on_gpu(builtin_bytes, testing_raw):
    """Oracle records after 20 frames, imported into scattered slots of a 64-stream batch whose frame counter differs
    from 20 mod 8, continue 15 frames like the oracle: pitch bit for bit every frame, output and vad within tolerance."""
    T0, K = 20, 15
    x = np.concatenate([frames(37, T0 + K, seed=602), testing_raw[:T0 + K, None]], axis=1)  # [T][38][480]
    m = ost.Model(builtin_bytes)
    _, _, _, states = ost.run(m, x[:T0].transpose(1, 0, 2))
    recs = np.stack([s.export() for s in states])
    o_ref, v_ref, p_ref, _ = ost.run(m, x[T0:].transpose(1, 0, 2), states)
    b = nb.DenoiseBatch(64)
    b.process_host(frames(64, 3, seed=603))
    slots = np.random.default_rng(4).choice(64, x.shape[1], replace=False)
    b.set_states(recs, slots)
    xin = frames(64, K, seed=604)
    xin[:, slots] = x[T0:]
    outs, vads = [], []
    for t in range(K):
        o, v = b.process_host(xin[t:t + 1])
        assert np.array_equal(b.taps()["pitch"][slots], p_ref[:, t]), t
        outs.append(o[0, slots]); vads.append(v[0, slots])
    assert rel_rms(np.stack(outs), o_ref.transpose(1, 0, 2)) <= OUT_REL_RMS
    assert np.abs(np.stack(vads) - v_ref.T).max() <= VAD_ATOL


def _move_clone_checkpoint(model_bytes, **env_kv):
    model = nb.RnnModel.from_bytes(model_bytes) if model_bytes is not None else None
    with env(**env_kv):
        make = lambda n, device=-1: nb.DenoiseBatch(n, model, device)  # noqa: E731
        B, T0, K = 300, 13, 6
        x = frames(B, T0 + K, seed=611)
        ref = make(B)
        o_ref, v_ref = ref.process_host(x)
        t_ref = ref.taps()
        o_ref, v_ref = o_ref[T0:], v_ref[T0:]

        def check(batch, xin, slots, streams):
            o, v = batch.process_host(xin)
            t = batch.taps()
            assert np.array_equal(bits(o[:, slots]), bits(o_ref[:, streams]))
            assert np.array_equal(bits(v[:, slots]), bits(v_ref[:, streams]))
            for k in TAPS:
                assert np.array_equal(t[k][slots], t_ref[k][streams]), k
            return o, v

        rng = np.random.default_rng(12)
        a = make(B)
        a.process_host(x[:T0])
        S = rng.choice(B, 60, replace=False)
        recs = a.get_states(S)
        # another batch of another size and frame counter, other slots
        b = make(77)
        b.process_host(frames(77, 5, seed=612))
        slots = rng.choice(77, len(S), replace=False)
        b.set_states(recs, slots)
        xb = frames(77, K, seed=613)
        xb[:, slots] = x[T0:, S]
        check(b, xb, slots, S)
        # the same batch, the exported streams permuted among their slots
        P = rng.permutation(S)
        a.set_states(recs, P)
        xa = x[T0:].copy()
        xa[:, P] = x[T0:, S]
        rest = np.setdiff1d(np.arange(B), S)
        check(a, xa, np.concatenate([P, rest]), np.concatenate([S, rest]))
        # the whole batch saved to host bytes and restored into a new batch
        c0 = make(B)
        c0.process_host(x[:T0])
        blob = c0.get_states().tobytes()
        del c0
        c = make(B)
        c.process_host(frames(B, 2, seed=614))
        c.set_states(np.frombuffer(blob, np.uint8).reshape(B, -1))
        check(c, x[T0:], np.arange(B), np.arange(B))
        return recs, S, x, (o_ref, v_ref, t_ref), make


def test_move_clone_checkpoint_bitwise(builtin_bytes):
    _move_clone_checkpoint(None)


def test_move_clone_checkpoint_bitwise_mma_model():
    _move_clone_checkpoint(rnn_ref.make_model(*OVER_WGMMA_BUDGET, seed=5), NNB_RNN_MMA="1")


def test_move_clone_checkpoint_bitwise_odd_state_width():
    _move_clone_checkpoint(rnn_ref.make_model(5, 13, 37, 45, seed=6))  # 95 state floats: rows not 16-byte aligned


def test_move_to_second_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device")
    recs, S, x, (o_ref, v_ref, t_ref), make = _move_clone_checkpoint(None)
    d = make(len(S) + 5, device=1)
    slots = np.arange(5, 5 + len(S))
    d.set_states(recs, slots)
    xd = frames(len(S) + 5, len(o_ref), seed=615)
    xd[:, slots] = x[-len(o_ref):, S]
    o, v = d.process_host(xd)
    assert np.array_equal(bits(o[:, slots]), bits(o_ref[:, S])) and np.array_equal(bits(v[:, slots]), bits(v_ref[:, S]))
    for k in TAPS:
        assert np.array_equal(d.taps()[k][slots], t_ref[k][S]), k


def test_other_streams_untouched_and_reset_equals_fresh():
    B, T0, K = 64, 8, 5
    x = frames(B, T0 + K, seed=621)
    ref = nb.DenoiseBatch(B)
    o_ref, v_ref = ref.process_host(x)
    donor = nb.DenoiseBatch(10)
    donor.process_host(frames(10, 11, seed=622))
    a = nb.DenoiseBatch(B)
    a.process_host(x[:T0])
    rng = np.random.default_rng(3)
    pick = rng.choice(B, 20, replace=False)
    moved, reset = pick[:10], pick[10:]
    a.set_states(donor.get_states(), moved)
    a.reset_streams(reset)
    o, v = a.process_host(x[T0:])
    rest = np.setdiff1d(np.arange(B), pick)
    assert np.array_equal(bits(o[:, rest]), bits(o_ref[T0:, rest])) and np.array_equal(bits(v[:, rest]), bits(v_ref[T0:, rest]))
    fresh = nb.DenoiseBatch(len(reset))
    of, vf = fresh.process_host(np.ascontiguousarray(x[T0:, reset]))
    assert np.array_equal(bits(o[:, reset]), bits(of)) and np.array_equal(bits(v[:, reset]), bits(vf))


def test_device_calls_ordered_on_a_torch_stream():
    """process_device -> get_states_device -> set_states_device (other slots) -> process_device on one torch stream
    with no host synchronisation in between gives the bits of the synchronised host sequence."""
    import torch
    B, T1, T2 = 4096, 10, 6
    x = frames(B, T1 + T2, seed=631)
    rng = np.random.default_rng(8)
    S = rng.choice(B, 700, replace=False)
    P = rng.permutation(B)[:700]  # other slots (some overlap S)
    r = nb.DenoiseBatch(B)
    o1, v1 = r.process_host(x[:T1])
    r.set_states(r.get_states(S), P)
    o2, v2 = r.process_host(x[T1:])
    a = nb.DenoiseBatch(B)
    xd = torch.from_numpy(x).cuda()
    out = torch.empty_like(xd)
    vad = torch.empty(T1 + T2, B, device="cuda")
    rec = torch.empty((len(S), a.state_bytes), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        a.process_device(out.data_ptr(), xd.data_ptr(), vad.data_ptr(), T1, 480, B * 480, st.cuda_stream)
        a.get_states_device(rec.data_ptr(), S, st.cuda_stream)
        a.set_states_device(rec.data_ptr(), P, st.cuda_stream)
        a.process_device(out[T1:].data_ptr(), xd[T1:].data_ptr(), vad[T1:].data_ptr(), T2, 480, B * 480, st.cuda_stream)
    st.synchronize()
    assert np.array_equal(bits(out.cpu().numpy()), bits(np.concatenate([o1, o2])))
    assert np.array_equal(bits(vad.cpu().numpy()), bits(np.concatenate([v1, v2])))


def test_set_states_rejects_bad_input_without_side_effects():
    import torch
    B = 40
    b = nb.DenoiseBatch(B)
    b.process_host(frames(B, 4, seed=641))
    donor = nb.DenoiseBatch(5)
    donor.process_host(frames(5, 9, seed=642))
    good = donor.get_states()
    dt = nb.state_dtype(b.gru_widths)
    before = b.get_states()
    slots = np.array([10, 11, 12, 13, 14])
    cases = []
    for field, value, text in [("magic", 0x12345678, "magic"), ("version", 2, "version"), ("nv", 25, "widths"),
                               ("mem_id", 8, "mem_id"), ("last_period", 769, "last_period")]:
        recs = good.copy()
        recs[2:3].view(dt)[0][field] = value  # records before it are valid: nothing may be written
        cases.append((recs, slots, text))
    cases.append((good, np.array([10, 11, 12, 11, 14]), "twice"))
    cases.append((good, np.array([10, 11, 12, 13, B]), "out of range"))
    for where in ("host", "device"):
        for recs, idx, text in cases:
            with pytest.raises(nb.NnnoiselessError, match=text):
                if where == "host":
                    b.set_states(recs, idx)
                else:
                    d = torch.from_numpy(recs).cuda()
                    b.set_states_device(d.data_ptr(), idx, torch.cuda.current_stream().cuda_stream)
            assert np.array_equal(b.get_states(), before), (where, text)
    b.set_states(good, slots)  # the valid records are accepted
    assert np.array_equal(b.get_states(slots), good)


def test_legacy_clone_continues_bitwise(testing_raw, reference_output):
    st = nb.DenoiseState()
    outs = []
    half = len(testing_raw) // 2
    for f in range(half):
        o = np.empty(480, np.float32)
        st.process_frame(o, np.ascontiguousarray(testing_raw[f]))
        outs.append(o)
    c = st.clone()
    for f in range(half, len(testing_raw)):
        x = np.ascontiguousarray(testing_raw[f])
        o1, o2 = np.empty(480, np.float32), np.empty(480, np.float32)
        v1, v2 = st.process_frame(o1, x), c.process_frame(o2, x)
        assert np.array_equal(bits(o1), bits(o2)) and v1 == v2, f
        outs.append(o2)
    metric, maxdiff = golden_metric(outs[1:], reference_output)
    assert metric < 1e-5 and maxdiff <= 1
