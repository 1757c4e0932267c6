"""Per-stream controls (rnnoise_batch_set_stream_controls / _get_): the attenuation limit and the voice-activity gate
applied inside the synthesis kernel.  A limited stream is bit for bit a split frame fed max(g, g_min); a gated stream is
its ungated twin's output times a float32 restatement of the gate's envelope; default controls are today's bits.  The
tests marked gpu run on the device; the others check the restatement, the record layout and the argument checks."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import rnn_ref

F, NBF, NBB = 480, 42, 22
DT = nb.STREAM_CONTROLS_DTYPE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the restatement ---------------------------------------------------------------------------------------------
def gate_envelope(vad, threshold, closed_gain, hold, hold_left=0, closed=0):
    """The gate of include/rnnoise.h in float32 over the reported vad [T] of one stream: (envelope [T][480] float32,
    (hold_left, closed) after the last frame)."""
    w = np.arange(1, F + 1, dtype=np.float32) / np.float32(F)
    th, cg = np.float32(threshold), np.float32(closed_gain)
    env = np.empty((len(vad), F), np.float32)
    for t, v in enumerate(np.asarray(vad, np.float32)):
        if th == 0 or v >= th:
            hold_left, is_open = hold, True
        elif hold_left > 0:
            hold_left, is_open = hold_left - 1, True
        else:
            is_open = False
        tau = np.float32(1) if is_open else cg
        ell = cg if closed else np.float32(1)
        env[t] = ell + (tau - ell) * w
        closed = 0 if is_open else 1
    return env, (hold_left, closed)


def to_pcm16(v):
    """clamp, then round half away from zero (the library's int16 output)"""
    c = np.clip(np.asarray(v, np.float32), -32768.0, 32767.0)
    return (np.sign(c) * np.floor(np.abs(c) + np.float32(0.5))).astype(np.int16)


def g_min_of(lim):
    return np.float32(0.0) if np.isinf(lim) else np.float32(10.0 ** (-float(np.float32(lim)) / 20.0))


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.int16 else np.uint32)


# ---- CPU tests -----------------------------------------------------------------------------------------------------
def test_restatement_hand_worked():
    """theta 0.5, hold 2, closed gain 0.25 over twelve frames, worked out by hand."""
    vad = [0.9, 0.1, 0.1, 0.1, 0.6, 0.5, 0.49, 0.0, 0.0, 0.7, 0.2, 0.2]
    opened = [1, 1, 1, 0, 1, 1, 1, 1, 0, 1, 1, 1]
    holds = [2, 1, 0, 0, 2, 2, 1, 0, 0, 2, 1, 0]
    hl, cl = 0, 0
    for t in range(12):
        env, (hl, cl) = gate_envelope(vad[t:t + 1], 0.5, 0.25, 2, hl, cl)
        assert (hl, cl) == (holds[t], 1 - opened[t]), t
        prev_open = t == 0 or opened[t - 1]
        if prev_open and opened[t]:
            assert np.all(env == 1.0)
        elif prev_open:  # closing: 1 -> 0.25 over the frame
            assert env[0, -1] == np.float32(0.25) and env[0, 0] == np.float32(1) + np.float32(-0.75) * (np.float32(1) / np.float32(480))
        elif opened[t]:  # opening: 0.25 -> 1
            assert env[0, -1] == 1.0 and env[0, 0] == np.float32(0.25) + np.float32(0.75) * (np.float32(1) / np.float32(480))
        assert np.all(np.diff(env[0]) >= 0) if opened[t] else np.all(np.diff(env[0]) <= 0)
    # threshold 0 keeps the gate open whatever the vad, a negative one included; closed gain 1 never changes a sample
    assert np.all(gate_envelope([-0.5, 0.0, 1.0], 0.0, 0.0, 0)[0] == 1.0)
    assert np.all(gate_envelope([0.0, 0.0, 0.9, 0.0], 0.9, 1.0, 0)[0] == 1.0)


def test_dtype_mirrors_the_struct(tmp_path):
    src = tmp_path / "o.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rnnoise.h"\n'
                   "int main(void) {\n"
                   '    printf("%zu %zu %zu %zu %zu %zu %zu %d\\n", sizeof(RNNoiseStreamControls),\n'
                   "           offsetof(RNNoiseStreamControls, atten_lim_db), offsetof(RNNoiseStreamControls, gate_threshold),\n"
                   "           offsetof(RNNoiseStreamControls, gate_closed_gain), offsetof(RNNoiseStreamControls, gate_hold_frames),\n"
                   "           offsetof(RNNoiseStreamControls, gate_hold_left), offsetof(RNNoiseStreamControls, gate_closed),\n"
                   "           RNNOISE_GATE_MAX_HOLD_FRAMES);\n"
                   "    return 0;\n}\n")
    exe = tmp_path / "o"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got[0] == DT.itemsize == 24
    assert got[1:7] == [DT.fields[n][1] for n in DT.names]
    assert got[7] == nb.GATE_MAX_HOLD_FRAMES


def test_python_argument_checks():
    """Checked before the library is called: a batch object without a handle is enough."""
    b = nb.DenoiseBatch.__new__(nb.DenoiseBatch)
    b.n_streams, b._h = 4, None
    bad = [dict(atten_lim_db=np.nan), dict(atten_lim_db=-1.0), dict(gate_threshold=1.5), dict(gate_threshold=np.nan),
           dict(gate_closed_gain=-0.1), dict(gate_closed_gain=np.nan), dict(gate_hold_frames=6001), dict(gate_hold_frames=-1),
           dict(gate_hold_frames=2.5), dict(gate_threshold=[0.1, 0.2]), dict(atten_lim_db=np.zeros((2, 2))),
           # values that the cast to int32 / float32 would wrap or round into range
           dict(gate_hold_frames=2 ** 32), dict(gate_hold_frames=np.full(4, 2 ** 32 + 5, np.int64)),
           dict(gate_hold_frames=np.uint64(2 ** 63)), dict(gate_threshold=1.0 + 1e-12), dict(gate_closed_gain=-1e-300),
           dict(gate_threshold="0.5"), dict(atten_lim_db=2 ** 70)]
    for kw in bad:
        with pytest.raises(ValueError):
            b.set_stream_controls(**kw)
    rec = np.zeros(4, DT)
    rec["atten_lim_db"] = np.inf
    for field, value in (("gate_hold_left", 1), ("gate_closed", 2), ("gate_hold_left", -1)):
        r = rec.copy()
        r[2][field] = value
        with pytest.raises(ValueError, match="record 2"):
            b.set_stream_controls_records(r)
    with pytest.raises(ValueError):
        b.set_stream_controls_records(rec, streams=[0, 1])
    with pytest.raises(ValueError):
        b.set_stream_controls_records(np.zeros(4, np.float32))
    with pytest.raises(ValueError):
        b.set_stream_controls_records(np.zeros(5, DT))
    b._h = None


def test_null_handles():
    L = nb.lib()
    rec = (C.c_byte * 24)()
    assert L.rnnoise_batch_set_stream_controls(None, None, 1, rec) < 0 and "null batch" in nb.last_error()
    assert L.rnnoise_batch_get_stream_controls(None, None, 1, rec) < 0 and "null batch" in nb.last_error()


def test_cpp_mirror_compiles(tmp_path):
    src = tmp_path / "t.cpp"
    src.write_text('#include "nnnoiseless.hpp"\n'
                   "int main(int argc, char**) {\n"
                   "    if (argc > 1) {\n"
                   "        nnnoiseless::DenoiseBatch b(2);\n"
                   "        const int s[1] = {1};\n"
                   "        b.set_stream_controls(s, 1, 12.0f, 0.5f, 0.1f, 50);\n"
                   "        std::vector<RNNoiseStreamControls> c = b.stream_controls(nullptr, 2);\n"
                   "        b.set_stream_controls_records(nullptr, 2, c.data());\n"
                   "        b.set_stream_controls(nullptr, 2);\n"
                   "    }\n"
                   "    return 0;\n}\n")
    exe = tmp_path / "t"
    libdir = os.path.join(ROOT, "nnnoiseless_b200", "lib")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir,
                        "-lnnnoiseless_b200", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0


# ---- GPU helpers ---------------------------------------------------------------------------------------------------
def signals(B, T, seed, speech):
    """[T][B][480] integer-valued float32 (the same values as int16 input): testing.raw speech at offsets per stream plus
    seeded noise at SNRs from clean to 0 dB, digitally silent stretches on every third stream."""
    rng = np.random.default_rng(seed)
    sp = speech.reshape(-1)
    x = np.zeros((B, T * F), np.float64)
    for s in range(B):
        off = (s * 3 * F) % max(len(sp) - T * F, 1)
        seg = sp[off:off + T * F].astype(np.float64)
        seg = np.pad(seg, (0, T * F - len(seg)))
        snr = [np.inf, 20.0, 10.0, 5.0, 0.0][s % 5]
        p = np.mean(seg ** 2) + 1.0
        noise = rng.standard_normal(T * F) * (0.0 if np.isinf(snr) else np.sqrt(p / 10 ** (snr / 10)))
        x[s] = seg * (0.3 + 0.1 * (s % 7)) + noise
        if s % 3 == 0:
            a = (s * 7) % max(T - 12, 1)
            x[s, a * F:(a + 10) * F] = 0.0
    x = np.clip(np.round(x), -32768, 32767).astype(np.float32)
    return np.ascontiguousarray(x.reshape(B, T, F).transpose(1, 0, 2))


def tanh_output_model(layer=4):
    """The built-in model with the activation of layer 4 (the denoise output: negative raw gains occur) or layer 5 (the
    vad output: negative vad occurs) set to tanh."""
    with open(nb.BUILTIN_WEIGHTS_PATH, "rb") as f:
        raw = bytearray(f.read())
    p = 0
    for kind in ("dense", "gru", "gru", "gru", "dense")[:layer]:
        ni, nn = raw[p], raw[p + 1]
        p += 3 + (ni * nn + nn if kind == "dense" else 3 * nn * ni + 3 * nn * nn + 3 * nn)
    assert raw[p + 1] == (NBB if layer == 4 else 1)
    raw[p + 2] = rnn_ref.TANH
    return nb.RnnModel.from_bytes(bytes(raw))


def batch(B, model_ids=None, layer=4):
    b = nb.DenoiseBatch(B)
    if model_ids is not None:
        assert b.add_model(tanh_output_model(layer)) == 1
        b.set_stream_models(np.asarray(model_ids, np.int32))
    return b


def torch():
    import torch as t
    return t


def fused(b, x, per_call=1, pcm16=False, streams=None):
    """x [T][n][480] -> (out [T][n][480], vad [T][n]) through process_device (or process_streams_device when streams is
    given), per_call frames per call."""
    th = torch()
    T, n = x.shape[:2]
    xd = th.from_numpy(np.ascontiguousarray(x.astype(np.int16) if pcm16 else x)).cuda()
    out = th.empty_like(xd)
    vad = th.empty((T, n), device="cuda")
    for t in range(0, T, per_call):
        k = min(per_call, T - t)
        if streams is None:
            b.process_device(out[t].data_ptr(), xd[t].data_ptr(), vad[t].data_ptr(), k, F, n * F, pcm16=pcm16)
        else:
            b.process_streams_device(streams, out[t].data_ptr(), xd[t].data_ptr(), vad[t].data_ptr(), k, F, n * F,
                                     pcm16=1 if pcm16 else 0, n=n)
    return out.cpu().numpy(), vad.cpu().numpy()


def split(b, x, gains, pcm16=False):
    """One split frame per t: analyze x[t], synthesize from gains[t] [B][22]."""
    th = torch()
    T, B = x.shape[:2]
    xd = th.from_numpy(x.astype(np.int16) if pcm16 else x).cuda()
    gd = th.from_numpy(np.ascontiguousarray(gains, np.float32)).cuda()
    out = th.empty_like(xd)
    feats = th.empty((B, NBF), device="cuda")
    for t in range(T):
        b.analyze_device(xd[t].data_ptr(), feats.data_ptr(), 0, 1, F, B * F, NBF, B * NBF, pcm16=int(pcm16))
        b.synthesize_device(out[t].data_ptr(), gd[t].data_ptr(), 1, F, B * F, NBB, B * NBB, pcm16=int(pcm16))
    return out.cpu().numpy()


LIMITS = [np.inf, 0.0, 6.0, 12.0, 20.0, 40.0]


@pytest.fixture(scope="module")
def limit_case(testing_raw):
    """Test 1's three runs.  A: fused without controls, one frame per call, with its raw gains, vad and states per frame.
    S: split frames fed max(g_A, g_min) on the limited streams and g_A elsewhere, float and int16 output."""
    B, T = 16, 100
    x = signals(B, T, seed=1, speech=testing_raw)
    ids = (np.arange(B) % 3 == 0).astype(np.int32)  # tanh output on streams with no limit and with 12 dB
    lims = np.array([LIMITS[s % len(LIMITS)] for s in range(B)], np.float32)
    gmin = np.array([g_min_of(v) for v in lims], np.float32)
    A = batch(B, ids)
    g_a, v_a, st_a, o_a = [], [], [], []
    for t in range(T):
        o, v = fused(A, x[t:t + 1])
        g_a.append(A.rnn_taps()["gains"])
        v_a.append(v[0])
        o_a.append(o[0])
        st_a.append(A.get_states())
    g_a = np.stack(g_a)
    g_s = np.where(gmin[None, :, None] > 0, np.maximum(g_a, gmin[None, :, None]), g_a).astype(np.float32)
    S = batch(B, ids)
    th = torch()
    xd = th.from_numpy(x).cuda()
    gd = th.from_numpy(g_s).cuda()
    o_s = th.empty_like(xd)
    feats = th.empty((B, NBF), device="cuda")
    st_s = []
    for t in range(T):
        S.analyze_device(xd[t].data_ptr(), feats.data_ptr(), 0, 1, F, B * F, NBF, B * NBF)
        S.synthesize_device(o_s[t].data_ptr(), gd[t].data_ptr(), 1, F, B * F, NBB, B * NBB)
        st_s.append(S.get_states())
    o_s16 = split(batch(B, ids), x, g_s, pcm16=True)
    unlimited_tanh = (ids == 1) & np.isinf(lims)
    assert np.any(g_a[:, unlimited_tanh] < 0), "negative raw gains reach the kernel with g_min = 0"
    assert np.any(g_a[:, (ids == 1) & ~np.isinf(lims)] < 0)
    return dict(B=B, T=T, x=x, ids=ids, lims=lims, unlimited_tanh=unlimited_tanh, g_a=g_a, v_a=np.stack(v_a), st_a=st_a, o_a=np.stack(o_a),
                o_s=o_s.cpu().numpy(), o_s16=o_s16, st_s=st_s)


def gru_section(rec):
    return rec[:, 9664:]


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_limit_equals_a_split_frame(limit_case):
    c = limit_case
    B, T, x = c["B"], c["T"], c["x"]
    C_ = batch(B, c["ids"])
    C_.set_stream_controls(atten_lim_db=c["lims"])
    C16 = batch(B, c["ids"])
    C16.set_stream_controls(atten_lim_db=c["lims"])
    for t in range(T):
        o, v = fused(C_, x[t:t + 1])
        assert np.array_equal(bits(o[0]), bits(c["o_s"][t])), t
        # no limit: negative raw gains pass untouched (the g_min > 0 guard), so the output is A's
        assert np.array_equal(bits(o[0][c["unlimited_tanh"]]), bits(c["o_a"][t][c["unlimited_tanh"]])), t
        assert np.array_equal(bits(v[0]), bits(c["v_a"][t])), t
        assert np.array_equal(C_.rnn_taps()["gains"], c["g_a"][t])  # the network's own gains
        rec = C_.get_states()
        assert np.array_equal(rec[:, :9664], c["st_s"][t][:, :9664]), t
        assert np.array_equal(gru_section(rec), gru_section(c["st_a"][t])), t
        o16, _ = fused(C16, x[t:t + 1], pcm16=True)
        assert np.array_equal(o16[0], c["o_s16"][t]), t
    # the limit changes the output: a 0 dB limit always, no limit never (tanh-output streams included), and a 12 dB
    # limit on a tanh-output stream, whose negative gains it raises
    o_a = c["o_a"]
    for s in range(B):
        same = np.array_equal(bits(o_a[:, s]), bits(c["o_s"][:, s]))
        if np.isinf(c["lims"][s]) or c["lims"][s] == 0 or c["ids"][s]:
            assert same == bool(np.isinf(c["lims"][s])), s


@pytest.mark.gpu
def test_gate_equals_its_restatement(testing_raw):
    B, T = 16, 120
    x = signals(B, T, seed=2, speech=testing_raw)
    th = np.array([[0.0, 0.2, 0.5, 0.9][s % 4] for s in range(B)], np.float32)
    hold = np.array([[0, 1, 7, 50][(s // 4) % 4] for s in range(B)], np.int32)
    cg = np.array([[0.0, 0.1, 1.0][s % 3] for s in range(B)], np.float32)
    U, G, G16 = nb.DenoiseBatch(B), nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    for b in (G, G16):
        b.set_stream_controls(gate_threshold=th, gate_closed_gain=cg, gate_hold_frames=hold)
    o_u, v_u = fused(U, x, per_call=7)
    o_g, v_g = fused(G, x, per_call=7)
    o_g16, _ = fused(G16, x, per_call=7, pcm16=True)
    assert np.array_equal(bits(v_g), bits(v_u))
    assert np.array_equal(G.get_states(), U.get_states()) and np.array_equal(G16.get_states(), U.get_states())
    ctl = G.get_stream_controls()
    closed_somewhere = 0
    for s in range(B):
        env, (hl, cl) = gate_envelope(v_u[:, s], th[s], cg[s], hold[s])
        want = o_u[:, s] * env
        assert np.array_equal(bits(o_g[:, s]), bits(want)), s
        assert np.array_equal(o_g16[:, s], to_pcm16(want)), s
        assert (ctl[s]["gate_hold_left"], ctl[s]["gate_closed"]) == (hl, cl), s
        closed_somewhere += int(np.any(env < 1))
    assert closed_somewhere >= 3
    assert np.all(ctl["gate_threshold"] == th) and np.all(ctl["gate_hold_frames"] == hold) and np.all(np.isinf(ctl["atten_lim_db"]))


@pytest.mark.gpu
def test_limit_and_gate_together(limit_case):
    c = limit_case
    B, x = c["B"], c["x"]
    th = np.array([[0.0, 0.3, 0.6][s % 3] for s in range(B)], np.float32)
    hold = np.array([[0, 3, 20][(s // 3) % 3] for s in range(B)], np.int32)
    b = batch(B, c["ids"])
    b.set_stream_controls(atten_lim_db=c["lims"], gate_threshold=th, gate_closed_gain=0.05, gate_hold_frames=hold)
    o, v = fused(b, x, per_call=5)
    assert np.array_equal(bits(v), bits(c["v_a"]))
    for s in range(B):
        env, _ = gate_envelope(c["v_a"][:, s], th[s], 0.05, hold[s])
        assert np.array_equal(bits(o[:, s]), bits(c["o_s"][:, s] * env)), s


@pytest.mark.gpu
def test_defaults_are_todays_bits(testing_raw):
    B, T = 12, 40
    x = signals(B, T, seed=3, speech=testing_raw)
    plain, one, explicit = nb.DenoiseBatch(B), nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    one.set_stream_controls([5], atten_lim_db=6.0, gate_threshold=0.5, gate_closed_gain=0.0, gate_hold_frames=3)
    rec = np.zeros(B, DT)
    rec["atten_lim_db"] = np.inf
    explicit.set_stream_controls_records(rec)
    explicit.set_stream_controls()
    o_p, v_p = fused(plain, x, per_call=4)
    o_1, v_1 = fused(one, x, per_call=4)
    o_e, v_e = fused(explicit, x, per_call=4)
    others = np.arange(B) != 5
    assert np.array_equal(bits(o_1[:, others]), bits(o_p[:, others])) and np.array_equal(bits(v_1), bits(v_p))
    assert not np.array_equal(bits(o_1[:, 5]), bits(o_p[:, 5]))
    assert np.array_equal(one.get_states(np.flatnonzero(others)), plain.get_states(np.flatnonzero(others)))
    assert np.array_equal(bits(o_e), bits(o_p)) and np.array_equal(bits(v_e), bits(v_p))
    assert np.array_equal(explicit.get_states(), plain.get_states())
    assert np.array_equal(explicit.get_stream_controls().view(np.uint8), rec.view(np.uint8))


@pytest.mark.gpu
def test_threshold_zero_keeps_the_gate_open_on_negative_vad(testing_raw):
    """A model whose vad output is tanh reports negative vad.  In a batch whose frames take the controlled kernel, its
    streams on threshold 0 (default or with other inert parameters) give an uncontrolled twin's bits, and a stream on a
    positive threshold follows the restatement."""
    B, T = 8, 60
    x = signals(B, T, seed=14, speech=testing_raw)
    ids = (np.arange(B) % 2 == 1).astype(np.int32)
    plain, ctl = batch(B, ids, layer=5), batch(B, ids, layer=5)
    rec = np.zeros(B, DT)
    rec["atten_lim_db"] = np.inf
    rec["gate_closed_gain"][2:] = 0.3  # threshold 0: never used
    rec["gate_hold_frames"][2:] = 4
    rec[1] = (np.inf, 0.3, 0.1, 2, 0, 0)
    ctl.set_stream_controls_records(rec)
    o_p, v_p = fused(plain, x, per_call=5)
    o_c, v_c = fused(ctl, x, per_call=5)
    assert np.any(v_p[:, ids == 1] < 0), "the tanh vad output goes negative"
    assert np.array_equal(bits(v_c), bits(v_p))
    open_ = np.arange(B) != 1
    assert np.array_equal(bits(o_c[:, open_]), bits(o_p[:, open_]))
    env, (hl, cl) = gate_envelope(v_p[:, 1], 0.3, 0.1, 2)
    assert np.any(env < 1)
    assert np.array_equal(bits(o_c[:, 1]), bits(o_p[:, 1] * env))
    got = ctl.get_stream_controls()
    assert np.all(got["gate_closed"][open_] == 0) and (got[1]["gate_hold_left"], got[1]["gate_closed"]) == (hl, cl)
    assert np.array_equal(ctl.get_states(), plain.get_states())


def mixed_controls(B, seed):
    rng = np.random.default_rng(seed)
    return dict(atten_lim_db=rng.choice(np.array(LIMITS, np.float32), B), gate_threshold=rng.choice([0.0, 0.3, 0.6], B),
                gate_closed_gain=rng.choice([0.0, 0.2], B), gate_hold_frames=rng.choice([0, 2, 9], B))


@pytest.mark.gpu
def test_subsets_are_full_batch_bits(testing_raw):
    B, T = 20, 30
    x = signals(B, T, seed=4, speech=testing_raw)
    kw = mixed_controls(B, 5)
    full, sub = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    for b in (full, sub):
        b.set_stream_controls(**kw)
    o_f, v_f = fused(full, x)
    rng = np.random.default_rng(6)
    for t in range(T):
        perm = rng.permutation(B).astype(np.int32)
        k = int(rng.integers(1, B))
        first, second = perm[:k], perm[k:]
        st_before, ctl_before = sub.get_states(second), sub.get_stream_controls(second)
        o1, v1 = fused(sub, x[t:t + 1, first], streams=first)
        assert np.array_equal(sub.get_states(second), st_before)
        assert np.array_equal(sub.get_stream_controls(second).view(np.uint8), ctl_before.view(np.uint8))
        o2, v2 = fused(sub, x[t:t + 1, second], streams=second)
        assert np.array_equal(bits(o1[0]), bits(o_f[t, first])) and np.array_equal(bits(v1[0]), bits(v_f[t, first])), t
        assert np.array_equal(bits(o2[0]), bits(o_f[t, second])) and np.array_equal(bits(v2[0]), bits(v_f[t, second])), t
    assert np.array_equal(sub.get_states(), full.get_states())
    assert np.array_equal(sub.get_stream_controls().view(np.uint8), full.get_stream_controls().view(np.uint8))


@pytest.mark.gpu
def test_records_move_a_stream_mid_hold_and_reset(testing_raw):
    B, T1, T2 = 8, 40, 30
    x = signals(B, T1 + T2, seed=7, speech=testing_raw)
    X = nb.DenoiseBatch(B)
    X.set_stream_controls(atten_lim_db=12.0, gate_threshold=0.8, gate_closed_gain=0.1, gate_hold_frames=[50, 7] * (B // 2))
    mid = []
    for t in range(T1):  # up to the first frame after which some stream is inside its hold time
        fused(X, x[t:t + 1])
        ctl = X.get_stream_controls()
        mid = np.flatnonzero((ctl["gate_hold_left"] > 0) & (ctl["gate_hold_left"] < ctl["gate_hold_frames"]))
        if t >= 4 and len(mid):
            break
    assert len(mid) > 0, ctl
    T1 = t + 1
    s = int(mid[0])
    rec, c = X.get_states([s]), X.get_stream_controls([s])
    Y = nb.DenoiseBatch(5)
    Y.set_states(rec, [3])  # either order: a state record leaves the controls alone
    Y.set_stream_controls_records(c, [3])
    Y.set_states(rec, [3])
    y_in = np.zeros((T2, 5, F), np.float32)
    y_in[:, 3] = x[T1:T1 + T2, s]
    o_x, v_x = fused(X, x[T1:T1 + T2], per_call=3)
    o_y, v_y = fused(Y, y_in, per_call=3)
    assert np.array_equal(bits(o_y[:, 3]), bits(o_x[:, s])) and np.array_equal(bits(v_y[:, 3]), bits(v_x[:, s]))
    assert np.array_equal(Y.get_stream_controls([3]).view(np.uint8), X.get_stream_controls([s]).view(np.uint8))
    # reset_streams: fresh gate state, parameters kept; the stream then matches a fresh one with the same parameters
    before = X.get_stream_controls()
    X.reset_streams([1, 6])
    after = X.get_stream_controls()
    for r in (1, 6):
        assert after[r]["gate_hold_left"] == 0 and after[r]["gate_closed"] == 0
        for f in ("atten_lim_db", "gate_threshold", "gate_closed_gain", "gate_hold_frames"):
            assert after[r][f] == before[r][f]
    keep = [r for r in range(B) if r not in (1, 6)]
    assert np.array_equal(after[keep].view(np.uint8), before[keep].view(np.uint8))
    Z = nb.DenoiseBatch(B)
    Z.set_stream_controls_records(after)
    o_x, _ = fused(X, x[:T2], per_call=5)
    o_z, _ = fused(Z, x[:T2], per_call=5)
    assert np.array_equal(bits(o_x[:, [1, 6]]), bits(o_z[:, [1, 6]]))
    # the whole-batch reset as well
    X.reset()
    c = X.get_stream_controls()
    assert np.all(c["gate_hold_left"] == 0) and np.all(c["gate_closed"] == 0) and np.all(c["gate_threshold"] == np.float32(0.8))


@pytest.mark.gpu
@pytest.mark.parametrize("pcm16", [0, 1])
def test_native_rate_is_its_parts(pcm16):
    import test_resampler_kernels as trk
    B, T = 24, 12
    rates = np.array([[16000, 8000][s % 2] for s in range(B)], np.int32)
    (b1, r1), (b2, r2) = trk.twins(B, rates)
    kw = mixed_controls(B, 8)
    kw["gate_threshold"] = np.where(np.arange(B) % 3 == 0, 0.0, 0.9)  # the synthetic input rarely reaches a high vad
    for b in (b1, b2):
        b.set_stream_controls(**kw)
    x = trk.native_input(rates, 2 * T, seed=9, pcm16=bool(pcm16))
    o1, v1 = trk.native(b1, r1, x[:, :T], T, pcm16=pcm16)
    o2, v2 = trk.composed(b2, r2, x[:, :T], T, pcm16=pcm16)
    assert np.array_equal(bits(o1), bits(o2)) and np.array_equal(bits(v1), bits(v2))
    S = np.random.default_rng(10).permutation(B)[:15].astype(np.int32)
    o1, v1 = trk.native(b1, r1, x[S, T:], T, streams=S, pcm16=pcm16)
    o2, v2 = trk.composed(b2, r2, x[S, T:], T, streams=S, pcm16=pcm16)
    assert np.array_equal(bits(o1), bits(o2)) and np.array_equal(bits(v1), bits(v2))
    assert np.array_equal(b1.get_stream_controls().view(np.uint8), b2.get_stream_controls().view(np.uint8))
    assert np.any(b1.get_stream_controls()["gate_closed"] == 1) or np.any(b1.get_stream_controls()["gate_hold_left"] > 0)


@pytest.mark.gpu
def test_split_and_window_frames_ignore_the_controls(testing_raw):
    th_ = torch()
    B, T0, T = 10, 25, 6
    x = signals(B, T0 + 2 * T, seed=11, speech=testing_raw)
    K, U = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    K.set_stream_controls(gate_threshold=0.5, gate_closed_gain=0.0, gate_hold_frames=2)
    fused(K, x[:T0], per_call=5)
    fused(U, x[:T0], per_call=5)
    assert np.array_equal(K.get_states(), U.get_states())  # the gate alone leaves the state as the twin's
    K.set_stream_controls_records(np.array([(12.0, r["gate_threshold"], 0.0, 2, r["gate_hold_left"], r["gate_closed"])
                                            for r in K.get_stream_controls()], DT))
    ctl = K.get_stream_controls()
    gains = np.random.default_rng(12).random((2 * T, B, NBB)).astype(np.float32) * 0.5
    o_k, o_u = split(K, x[T0:T0 + T], gains[:T]), split(U, x[T0:T0 + T], gains[:T])
    assert np.array_equal(bits(o_k), bits(o_u))
    for b, o in ((K, "k"), (U, "u")):
        xd = th_.from_numpy(x[T0 + T:]).cuda()
        out = th_.empty_like(xd)
        feats = th_.empty((T, B, NBF), device="cuda")
        ctx = th_.empty((T, B, nb.SYNTH_CONTEXT_BYTES), dtype=th_.uint8, device="cuda")
        gd = th_.from_numpy(gains[T:]).cuda()
        b.analyze_window_device(xd.data_ptr(), feats.data_ptr(), 0, T, F, B * F, NBF, B * NBF, ctx.data_ptr(), 1, B)
        b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, F, B * F, NBB, B * NBB, ctx.data_ptr(), 1, B)
        if o == "k":
            w_k = out.cpu().numpy()
        else:
            w_u = out.cpu().numpy()
    assert np.array_equal(bits(w_k), bits(w_u))
    assert np.array_equal(K.get_states(), U.get_states())
    assert np.array_equal(K.get_stream_controls().view(np.uint8), ctl.view(np.uint8))


@pytest.mark.gpu
def test_refusals_change_nothing(testing_raw):
    B = 6
    x = signals(B, 12, seed=13, speech=testing_raw)
    R, W = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    for b in (R, W):
        b.set_stream_controls(atten_lim_db=6.0, gate_threshold=0.4, gate_closed_gain=0.2, gate_hold_frames=3)
        fused(b, x[:8], per_call=4)
    before = R.get_stream_controls()
    L = nb.lib()

    def raw_set(rec, streams=None):
        rec = np.ascontiguousarray(rec, DT)
        idx = None if streams is None else np.ascontiguousarray(streams, np.int32)
        return L.rnnoise_batch_set_stream_controls(R._h, idx.ctypes.data_as(C.c_void_p) if idx is not None else None, len(rec),
                                                   rec.ctypes.data_as(C.c_void_p))

    good = before.copy()
    cases = [("atten_lim_db", np.nan), ("atten_lim_db", -0.5), ("gate_threshold", np.nan), ("gate_threshold", 1.01),
             ("gate_threshold", -0.1), ("gate_closed_gain", np.nan), ("gate_closed_gain", 1.5), ("gate_hold_frames", 6001),
             ("gate_hold_frames", -1), ("gate_hold_left", 4), ("gate_hold_left", -1), ("gate_closed", 2)]
    for field, value in cases:
        rec = good.copy()
        rec[4][field] = value
        assert raw_set(rec) < 0
        msg = nb.last_error()
        assert "record 4" in msg and field in msg, msg
        assert np.array_equal(R.get_stream_controls().view(np.uint8), before.view(np.uint8))
    assert raw_set(good[:2], [0, 6]) < 0 and "out of range" in nb.last_error()
    assert raw_set(good[:2], [1, 1]) < 0 and "twice" in nb.last_error()
    assert raw_set(good[:2], [-1, 2]) < 0
    # pending split frames: both calls are refused
    th_ = torch()
    xd = th_.from_numpy(x[8:9]).cuda()
    feats = th_.empty((B, NBF), device="cuda")
    R.analyze_device(xd[0].data_ptr(), feats.data_ptr(), 0, 1, F, B * F, NBF, B * NBF)
    assert raw_set(good) < 0 and "pending" in nb.last_error()
    with pytest.raises(nb.NnnoiselessError, match="pending"):
        R.get_stream_controls()
    gains = th_.full((B, NBB), 0.5, device="cuda")
    out = th_.empty_like(xd)
    R.synthesize_device(out[0].data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB)
    W.analyze_device(xd[0].data_ptr(), feats.data_ptr(), 0, 1, F, B * F, NBF, B * NBF)
    W.synthesize_device(out[0].data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB)
    assert np.array_equal(R.get_stream_controls().view(np.uint8), W.get_stream_controls().view(np.uint8))
    o_r, v_r = fused(R, x[9:], per_call=3)
    o_w, v_w = fused(W, x[9:], per_call=3)
    assert np.array_equal(bits(o_r), bits(o_w)) and np.array_equal(bits(v_r), bits(v_w))
    assert np.array_equal(R.get_states(), W.get_states())
