"""Stream links (rnnoise_batch_link_streams / _unlink_streams / _get_stream_links): the members of a group share one band
gain curve, the max or the float32 mean of the non-silent members' raw gains, and a linked stream's gate decides on the
group's vad.  A linked stream is bit for bit a split frame fed the linked gains, so every GPU test runs a linked batch L
next to an unlinked twin A (whose taps give the raw gains, vad and silence) and a split twin C fed the numpy reduction
of A's gains.  The tests not marked gpu check the reduction on a hand-worked case, the linked frame through the CPU
oracle, the argument checks, the C++ mirror and the command line's texts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle
import oracle_state
from nnnoiseless_b200 import files
from test_stream_controls import batch, bits, fused, g_min_of, gate_envelope, signals, split, to_pcm16, torch

F, NBF, NBB = 480, 42, 22
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = {"max": nb.LINK_MODES["max"], "mean": nb.LINK_MODES["mean"]}


# ---- the restatement ---------------------------------------------------------------------------------------------
def link_gains(g, sil, groups):
    """The linked raw gains of include/rnnoise.h: g [B][22] float32 raw gains, sil [B] silence flags, groups a list of
    (mode, members).  A non-silent member's row becomes the reduction over the group's non-silent members in ascending
    stream index (max: fmax; mean: a float32 sum from the first such member's gain, then / n); other rows keep g."""
    g = np.asarray(g, np.float32)
    out = g.copy()
    for mode, members in groups:
        live = [m for m in sorted(members) if not sil[m]]
        if not live:
            continue
        r = g[live[0]].copy()
        for m in live[1:]:
            r = np.fmax(r, g[m]) if mode == "max" else (r + g[m]).astype(np.float32)
        if mode == "mean":
            r = (r / np.float32(len(live))).astype(np.float32)
        out[live] = r
    return out


def group_vad(vad, sil, groups):
    """The vad each stream's gate decides on: its own (0 when silent), or for a linked stream the largest vad of its
    group's non-silent members (0 when every member is silent)."""
    v = np.where(np.asarray(sil) != 0, np.float32(0), np.asarray(vad, np.float32)).astype(np.float32)
    out = v.copy()
    for _, members in groups:
        live = [m for m in members if not sil[m]]
        out[list(members)] = max(v[m] for m in live) if live else np.float32(0)
    return out


# ---- CPU tests -----------------------------------------------------------------------------------------------------
def test_restatement_hand_worked():
    f = np.float32
    g = np.array([[0.1, 0.9], [0.3, 0.2], [0.5, 0.5], [0.7, 0.0]], f)
    sil = np.array([0, 0, 1, 0])
    # max over the non-silent members 0, 1, 3; the silent member 2 keeps its row
    got = link_gains(g, sil, [("max", [3, 0, 2, 1])])
    assert np.array_equal(got[[0, 1, 3]], np.array([[0.7, 0.9]] * 3, f)) and np.array_equal(got[2], g[2])
    # mean: ((g0 + g1) + g3) / 3 in float32, each step rounded, in ascending stream index whatever the listed order
    want = ((f(0.1) + f(0.3)) + f(0.7)) / f(3)
    assert link_gains(g, sil, [("mean", [3, 1, 0, 2])])[0, 0] == want
    # the order matters for a float32 sum: 1e8 + 1 - 1e8 against 1e8 - 1e8 + 1
    h = np.array([[1e8], [1.0], [-1e8]], f)
    assert link_gains(h, [0, 0, 0], [("mean", [0, 1, 2])])[0, 0] == f(0)
    assert link_gains(h[[0, 2, 1]], [0, 0, 0], [("mean", [0, 1, 2])])[0, 0] == f(1) / f(3)
    # every member silent: nothing changes; the group vad is 0
    assert np.array_equal(link_gains(g, [1, 1, 1, 1], [("mean", [0, 1])]), g)
    assert np.array_equal(group_vad([0.2, 0.9, 0.4, 0.1], [1, 1, 0, 0], [("max", [0, 1]), ("mean", [2, 3])]),
                          np.array([0, 0, 0.4, 0.4], f))
    assert np.array_equal(group_vad([0.2, 0.9, 0.4, 0.1], [0, 1, 0, 1], [("max", [0, 1])]), np.array([0.2, 0.2, 0.4, 0], f))


def test_linked_frame_through_the_oracle(testing_raw):
    """Three channels through the CPU oracle: analysis and the network run per channel (a link does not touch them),
    then synthesis_from takes the reduced gains with each channel's own lastg and overlap memory.  With its own gains it
    is the oracle's own frame; with MAX over identical channels the linked frame is the unlinked one."""
    model_bytes = open(nb.BUILTIN_WEIGHTS_PATH, "rb").read()
    om, sm = oracle.Model(model_bytes), oracle_state.Model(model_bytes)
    T, Ch = 24, 3
    rng = np.random.default_rng(21)
    sp = testing_raw[:T].reshape(-1).astype(np.float64)
    x = np.stack([sp * 0.5 + rng.standard_normal(T * F) * 300, sp * 0.2 + rng.standard_normal(T * F) * 1500, sp * 0.5])
    x[1, 4 * F:20 * F] = 0.0  # a silent stretch in one member (the high-pass filter's tail takes a few frames)
    x = np.round(x).astype(np.float32).reshape(Ch, T, F)
    x[2] = x[0]  # channel 2 repeats channel 0
    nv, nn, nd = om_widths = (24, 48, 96)
    states = [oracle_state.State(sm) for _ in range(Ch)]
    lastg = {m: np.zeros((Ch, NBB), np.float32) for m in ("max", "mean")}
    smem = {m: np.zeros((Ch, F), np.float32) for m in ("max", "mean")}
    saw_silent, differs = False, False
    for t in range(T):
        g, vad, sil, spec, own = np.zeros((Ch, NBB), np.float32), np.zeros(Ch, np.float32), np.zeros(Ch, int), [], []
        for c in range(Ch):
            rec = states[c].export()
            a = oracle_state.analysis_frame(sm, rec, x[c, t])
            gru = rec[9664:9664 + 4 * sum(om_widths)].view(np.float32)
            if not a["silence"]:
                _, _, _, g[c], vad[c] = oracle.rnn_step(om, gru[:nv], gru[nv:nv + nn], gru[nv + nn:], a["features"])
            sil[c] = a["silence"]
            spec.append(a)
            lg0, sm0 = rec[40:40 + 88].view(np.float32), rec[7744:7744 + 4 * F].view(np.float32)
            out, _ = states[c].process_frame(x[c, t])
            o2, _, _ = oracle_state.synthesis_from(a["X"], a["P"], a["ex"], a["ep"], a["exp"], g[c], lg0, sm0, a["silence"])
            assert np.array_equal(bits(o2), bits(out)), (t, c)  # the restatement's frame is the oracle's
            own.append(out)
        saw_silent |= bool(sil[1])
        for mode in ("max", "mean"):
            gl = link_gains(g, sil, [(mode, [0, 1, 2])])
            for c in range(Ch):
                a = spec[c]
                o, lastg[mode][c], smem[mode][c] = oracle_state.synthesis_from(a["X"], a["P"], a["ex"], a["ep"], a["exp"], gl[c],
                                                                               lastg[mode][c], smem[mode][c], a["silence"])
                if sil[c]:
                    continue
                if mode == "max" and c == 2:
                    assert np.array_equal(gl[2], gl[0])
                if not np.array_equal(bits(o), bits(own[c])):
                    differs = True
        # MAX over the identical channels 0 and 2 alone gives each its unlinked frame
        gl2 = link_gains(g, sil, [("max", [0, 2])])
        assert np.array_equal(gl2[[0, 2]], g[[0, 0]])
    assert saw_silent and differs


def test_python_argument_checks():
    """Checked before the library is called: a batch object without a handle is enough."""
    b = nb.DenoiseBatch.__new__(nb.DenoiseBatch)
    b.n_streams, b._h = 70, None
    for streams, mode in (([0], "max"), (list(range(65)), "max"), ([0, 0], "max"), ([0, 70], "max"), ([-1, 2], "mean"),
                          ([0, 1], "avg"), ([0, 1], 1), ([0, 1], None), ([0, 2 ** 32 + 1], "max"), ([0.5, 1], "max"),
                          ([[0, 1]], "max")):
        with pytest.raises(ValueError):
            b.link_streams(streams, mode)
    for streams in ([0, 0], [70], [2 ** 32 + 3]):
        with pytest.raises(ValueError):
            b.unlink_streams(streams)
        with pytest.raises(ValueError):
            b.stream_links(streams)
    with pytest.raises(ValueError):
        files.denoise_files([("a.wav", "b.wav")], link_channels="both")


def test_null_handles_and_bad_file_mode(tmp_path):
    L = nb.lib()
    idx = np.array([0, 1], np.int32)
    p = idx.ctypes.data_as(C.c_void_p)
    assert L.rnnoise_batch_link_streams(None, p, 2, 1) < 0 and "null batch" in nb.last_error()
    assert L.rnnoise_batch_unlink_streams(None, p, 2) < 0 and "null batch" in nb.last_error()
    assert L.rnnoise_batch_get_stream_links(None, p, 2, None, None) < 0 and "null batch" in nb.last_error()
    ins, outs = (C.c_char_p * 1)(b"in.wav"), (C.c_char_p * 1)(os.fsencode(str(tmp_path / "o.wav")))
    assert L.rnnoise_denoise_files_linked(1, ins, outs, None, 3) < 0 and "link mode 3" in nb.last_error()
    assert L.rnnoise_denoise_files_linked(-1, None, None, None, 1) < 0 and "bad argument" in nb.last_error()


def test_cpp_mirror_compiles(tmp_path):
    src = tmp_path / "t.cpp"
    src.write_text('#include "nnnoiseless.hpp"\n'
                   "int main(int argc, char**) {\n"
                   "    if (argc > 1) {\n"
                   "        nnnoiseless::DenoiseBatch b(4);\n"
                   "        const int s[3] = {3, 0, 2};\n"
                   "        b.link_streams(s, 3, RNNOISE_LINK_MEAN);\n"
                   "        std::vector<std::pair<int, int>> l = b.stream_links(nullptr, 4);\n"
                   "        b.unlink_streams(s, 1);\n"
                   "        b.unlink_streams();\n"
                   "        nnnoiseless::denoise_files({{\"a.wav\", \"b.wav\"}}, nullptr, RNNOISE_LINK_MAX);\n"
                   "        return l[0].second;\n"
                   "    }\n"
                   "    return 0;\n}\n")
    exe = tmp_path / "t"
    libdir = os.path.join(ROOT, "nnnoiseless_b200", "lib")
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir,
                        "-lnnnoiseless_b200", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0


def test_cli_texts(tmp_path):
    h = subprocess.run([files.CLI_PATH, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--link-channels <MODE>" in h.stdout and "max or mean" in h.stdout
    r = subprocess.run([files.CLI_PATH, "--link-channels", "sum", "a.wav", "b.wav"], capture_output=True, text=True)
    assert r.returncode != 0 and "Invalid value for '--link-channels <MODE>'" in r.stderr and "'sum'" in r.stderr
    r = subprocess.run([files.CLI_PATH, "a.wav", "b.wav", "--link-channels"], capture_output=True, text=True)
    assert r.returncode != 0 and "--link-channels needs a value" in r.stderr
    # a file of 65 channels is refused with the flag, before any GPU work
    wide = tmp_path / "wide.wav"
    files.write_audio(str(wide), np.zeros((2 * F, 65), np.int16), wav=True)
    for mode in ("max", "mean"):
        r = subprocess.run([files.CLI_PATH, "--link-channels=" + mode, str(wide), str(tmp_path / "o.wav")], capture_output=True, text=True)
        assert r.returncode != 0 and "has 65 channels: linked channels are at most 64 per file" in r.stderr, r.stderr
    with pytest.raises(nb.NnnoiselessError, match="65 channels"):
        files.denoise_files([(str(wide), str(tmp_path / "o2.wav"))], link_channels="max")


# ---- GPU helpers ---------------------------------------------------------------------------------------------------
def link_all(b, groups):
    for mode, members in groups:
        b.link_streams(members, mode)


def frame_taps(A):
    r = A.rnn_taps()
    return r["gains"], r["vad"], A.taps()["silence"]


def gru_section(rec):
    return rec[:, 9664:]


def main_groups(flip):
    """Pairs (one of two streams with overlapping silent stretches, one unsorted), a group of 3 that is neither
    contiguous nor sorted, and a group of 64 non-contiguous streams; the modes alternate, flip swaps them."""
    big = [s for s in range(16, 96) if s % 5 != 0]
    assert len(big) == 64
    members = [[0, 1], [5, 2], [12, 3, 7], [6, 9], big]
    return [(("max", "mean")[(i + flip) % 2], m) for i, m in enumerate(members)]


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("flip", [0, 1])
def test_linked_equals_a_split_frame(testing_raw, flip):
    B, T = 96, 40
    x = signals(B, T, seed=31 + flip, speech=testing_raw)
    x[8:30, 6] = 0.0  # both members of the pair {6, 9} silent at once on some frames
    x[10:32, 9] = 0.0
    ids = (np.arange(B) % 4 == 1).astype(np.int32)  # a second model, whose raw gains go negative, on some members
    groups = main_groups(flip)
    A, L, C_, L16, C16 = (batch(B, ids) for _ in range(5))
    for b in (L, L16):
        link_all(b, groups)
    grp, mode = L.stream_links()
    for m, members in groups:
        assert np.all(grp[members] == min(members)) and np.all(mode[members] == MODES[m])
    linked = np.zeros(B, bool)
    for _, members in groups:
        linked[members] = True
    assert np.all(mode[~linked] == 0) and np.array_equal(grp[~linked], np.flatnonzero(~linked))
    changed, all_silent = 0, 0
    for t in range(T):
        o_a, v_a = fused(A, x[t:t + 1])
        g, v, sil = frame_taps(A)
        gl = link_gains(g, sil, groups)
        o_l, v_l = fused(L, x[t:t + 1])
        o_c = split(C_, x[t:t + 1], gl[None])
        assert np.array_equal(bits(o_l[0]), bits(o_c[0])), t
        assert np.array_equal(bits(o_l[0, ~linked]), bits(o_a[0, ~linked])), t
        assert np.array_equal(bits(v_l), bits(v_a)), t  # each stream's own vad
        assert np.array_equal(L.rnn_taps()["gains"], g)  # and its own raw gains
        rec_l = L.get_states()
        assert np.array_equal(rec_l[:, :9664], C_.get_states()[:, :9664]), t
        assert np.array_equal(gru_section(rec_l), gru_section(A.get_states())), t
        o16, _ = fused(L16, x[t:t + 1], pcm16=True)
        assert np.array_equal(o16[0], split(C16, x[t:t + 1], gl[None], pcm16=True)[0]), t
        changed += int(not np.array_equal(bits(o_l[0, linked]), bits(o_a[0, linked])))
        all_silent += int(sil[6] and sil[9])
    assert changed > T // 2 and all_silent > 0


@pytest.mark.gpu
def test_max_of_identical_members_is_the_unlinked_output(testing_raw):
    B, T = 8, 30
    x = signals(B, T, seed=33, speech=testing_raw)
    x[:, 1], x[:, 3], x[:, 7] = x[:, 0], x[:, 2], x[:, 2]
    U, L = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    L.link_streams([1, 0], "max")
    L.link_streams([7, 2, 3], "max")
    o_u, v_u = fused(U, x, per_call=4)
    o_l, v_l = fused(L, x, per_call=4)
    assert np.array_equal(bits(o_l), bits(o_u)) and np.array_equal(bits(v_l), bits(v_u))
    assert np.array_equal(L.get_states(), U.get_states())


@pytest.mark.gpu
def test_limit_and_gate_on_linked_streams(testing_raw):
    """A 12 dB limit on some members applies to the linked gain; a gated group's output is its ungated twin's times the
    gate envelope driven by the group's vad, with the same gate state."""
    B, T = 16, 60
    x = signals(B, T, seed=34, speech=testing_raw)
    groups = [("mean", [0, 3, 5]), ("max", [1, 2]), ("max", [8, 9, 10, 11])]
    lims = np.where(np.isin(np.arange(B), [3, 2, 9, 14]), 12.0, np.inf).astype(np.float32)
    gmin = np.array([g_min_of(v) for v in lims], np.float32)
    gated = np.array([0, 3, 5, 8, 9, 10, 11, 13])
    th = np.zeros(B, np.float32)
    th[gated] = 0.6
    hold = np.zeros(B, np.int32)
    hold[gated] = 2
    A, L0, L1, C_ = (nb.DenoiseBatch(B) for _ in range(4))
    for b in (L0, L1):
        link_all(b, groups)
    for b in (L0, L1, C_):
        b.set_stream_controls(atten_lim_db=lims)
    L1.set_stream_controls(atten_lim_db=lims, gate_threshold=th, gate_closed_gain=0.1, gate_hold_frames=hold)
    o0, o1, vg = [], [], []
    for t in range(T):
        fused(A, x[t:t + 1])
        g, v, sil = frame_taps(A)
        gl = link_gains(g, sil, groups)
        gc = np.where(gmin[:, None] > 0, np.maximum(gl, gmin[:, None]), gl).astype(np.float32)
        a, _ = fused(L0, x[t:t + 1])
        b_, _ = fused(L1, x[t:t + 1])
        assert np.array_equal(bits(a[0]), bits(split(C_, x[t:t + 1], gc[None])[0])), t
        o0.append(a[0])
        o1.append(b_[0])
        vg.append(group_vad(v, sil, groups))
    o0, o1, vg = np.stack(o0), np.stack(o1), np.stack(vg)
    ctl = L1.get_stream_controls()
    closed = 0
    for s in range(B):
        env, (hl, cl) = gate_envelope(vg[:, s], th[s], 0.1, hold[s])
        assert np.array_equal(bits(o1[:, s]), bits(o0[:, s] * env)), s
        assert (ctl[s]["gate_hold_left"], ctl[s]["gate_closed"]) == (hl, cl), s
        closed += int(np.any(env < 1))
    assert closed >= 2
    # members of one group decide together
    for _, members in groups:
        if th[members[0]] > 0:
            assert len({(int(ctl[m]["gate_hold_left"]), int(ctl[m]["gate_closed"])) for m in members}) == 1
    assert np.array_equal(L1.get_states(), L0.get_states())


@pytest.mark.gpu
def test_subsets_are_full_batch_bits_and_split_groups_are_refused(testing_raw):
    B, T = 20, 24
    x = signals(B, T, seed=35, speech=testing_raw)
    groups = [("mean", [0, 7, 13]), ("max", [2, 3]), ("mean", [19, 4]), ("max", [5, 6, 8, 9])]
    full, sub = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    for b in (full, sub):
        link_all(b, groups)
    o_f, v_f = fused(full, x)
    units = [g[1] for g in groups] + [[s] for s in range(B) if not any(s in g[1] for g in groups)]
    rng = np.random.default_rng(36)
    for t in range(T):
        order = rng.permutation(len(units))
        k = int(rng.integers(1, len(units)))
        first = rng.permutation(np.concatenate([units[i] for i in order[:k]])).astype(np.int32)
        second = rng.permutation(np.concatenate([units[i] for i in order[k:]])).astype(np.int32)
        st_before = sub.get_states(second)
        o1, v1 = fused(sub, x[t:t + 1, first], streams=first)
        assert np.array_equal(sub.get_states(second), st_before)
        o2, v2 = fused(sub, x[t:t + 1, second], streams=second)
        assert np.array_equal(bits(o1[0]), bits(o_f[t, first])) and np.array_equal(bits(v1[0]), bits(v_f[t, first])), t
        assert np.array_equal(bits(o2[0]), bits(o_f[t, second])) and np.array_equal(bits(v2[0]), bits(v_f[t, second])), t
    assert np.array_equal(sub.get_states(), full.get_states())
    # a subset that splits a group is refused and changes nothing
    before = sub.get_states()
    th_ = torch()
    xd = th_.from_numpy(x[:1, [0, 7, 1]]).cuda()
    out = th_.empty_like(xd)
    with pytest.raises(nb.NnnoiselessError, match="stream 0 is linked with stream 13"):
        sub.process_streams_device(np.array([0, 7, 1], np.int32), out.data_ptr(), xd.data_ptr(), 0, 1, F, 3 * F, n=3)
    with pytest.raises(nb.NnnoiselessError, match="linked with stream"):
        sub.process_streams_host(np.array([3], np.int32), x[:1, [3]])
    assert np.array_equal(sub.get_states(), before)


@pytest.mark.gpu
def test_relink_unlink_and_resets(testing_raw):
    """Link changes take effect at the next frame; resets keep the links."""
    B, T = 12, 36
    x = signals(B, T, seed=37, speech=testing_raw)
    A, L, C_ = (nb.DenoiseBatch(B) for _ in range(3))
    plan = {0: lambda b: (b.link_streams([0, 1], "max"), b.link_streams([4, 2, 3], "mean")),
            10: lambda b: b.link_streams([2, 1], "mean"),  # {0, 1} dissolves, {3, 4} stays
            18: lambda b: (b.unlink_streams([3]), b.link_streams(list(range(6, 12)), "max")),
            26: lambda b: b.unlink_streams()}
    state = {0: [("max", [0, 1]), ("mean", [2, 3, 4])], 10: [("mean", [1, 2]), ("mean", [3, 4])],
             18: [("mean", [1, 2]), ("max", list(range(6, 12)))], 26: []}
    groups = []
    for t in range(T):
        if t in plan:
            plan[t](L)
            groups = state[t]
            grp, mode = L.stream_links()
            for m, members in groups:
                assert np.all(grp[members] == min(members)) and np.all(mode[members] == MODES[m]), t
            assert int(np.sum(mode > 0)) == sum(len(m) for _, m in groups)
        if t == 22:  # resets, identical on the three batches, keep the links
            before = L.stream_links()
            for b in (A, L, C_):
                b.reset_streams([2, 7])
            assert all(np.array_equal(a, c) for a, c in zip(L.stream_links(), before))
        fused(A, x[t:t + 1])
        g, v, sil = frame_taps(A)
        o_l, _ = fused(L, x[t:t + 1])
        o_c = split(C_, x[t:t + 1], link_gains(g, sil, groups)[None])
        assert np.array_equal(bits(o_l[0]), bits(o_c[0])), t
    L.link_streams([0, 5], "mean")
    before = L.stream_links()
    L.reset()
    assert all(np.array_equal(a, c) for a, c in zip(L.stream_links(), before))


@pytest.mark.gpu
@pytest.mark.parametrize("pcm16", [0, 1])
def test_native_rate_is_its_parts(pcm16):
    import test_resampler_kernels as trk
    B, T = 24, 10
    rates = np.array([[16000, 8000][s % 2] for s in range(B)], np.int32)
    (b1, r1), (b2, r2) = trk.twins(B, rates)
    groups = [("max", [0, 1]), ("mean", [2, 5, 11]), ("mean", [20, 3]), ("max", list(range(12, 20)))]
    for b in (b1, b2):
        link_all(b, groups)
    x = trk.native_input(rates, 2 * T, seed=38, pcm16=bool(pcm16))
    o1, v1 = trk.native(b1, r1, x[:, :T], T, pcm16=pcm16)
    o2, v2 = trk.composed(b2, r2, x[:, :T], T, pcm16=pcm16)
    assert np.array_equal(bits(o1), bits(o2)) and np.array_equal(bits(v1), bits(v2))
    S = np.array([11, 20, 2, 3, 5, 7, 0, 1, 9], np.int32)
    o1, v1 = trk.native(b1, r1, x[S, T:], T, streams=S, pcm16=pcm16)
    o2, v2 = trk.composed(b2, r2, x[S, T:], T, streams=S, pcm16=pcm16)
    assert np.array_equal(bits(o1), bits(o2)) and np.array_equal(bits(v1), bits(v2))
    assert np.array_equal(b1.get_states(), b2.get_states())
    # a native subset that splits a group is refused before anything runs, the resampler included
    rs_before, st_before = r1.get_states(), b1.get_states()
    with pytest.raises(nb.NnnoiselessError, match="stream 2 is linked with stream 11"):
        trk.native(b1, r1, x[[2, 5], :1], 1, streams=np.array([2, 5], np.int32), pcm16=pcm16)
    assert np.array_equal(r1.get_states(), rs_before) and np.array_equal(b1.get_states(), st_before)


@pytest.mark.gpu
def test_split_and_window_frames_ignore_links(testing_raw):
    th_ = torch()
    B, T0, T = 10, 12, 6
    x = signals(B, T0 + 2 * T, seed=39, speech=testing_raw)
    K, U = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    K.link_streams([0, 1, 2], "mean")
    K.link_streams([5, 9], "max")
    fused(K, x[:T0], per_call=4)
    fused(U, x[:T0], per_call=4)
    U.set_states(K.get_states())
    gains = np.random.default_rng(40).random((2 * T, B, NBB)).astype(np.float32) * 0.5
    assert np.array_equal(bits(split(K, x[T0:T0 + T], gains[:T])), bits(split(U, x[T0:T0 + T], gains[:T])))
    outs = []
    for b in (K, U):
        xd = th_.from_numpy(x[T0 + T:]).cuda()
        out = th_.empty_like(xd)
        feats = th_.empty((T, B, NBF), device="cuda")
        ctx = th_.empty((T, B, nb.SYNTH_CONTEXT_BYTES), dtype=th_.uint8, device="cuda")
        gd = th_.from_numpy(gains[T:]).cuda()
        b.analyze_window_device(xd.data_ptr(), feats.data_ptr(), 0, T, F, B * F, NBF, B * NBF, ctx.data_ptr(), 1, B)
        b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, F, B * F, NBB, B * NBB, ctx.data_ptr(), 1, B)
        outs.append(out.cpu().numpy())
    assert np.array_equal(bits(outs[0]), bits(outs[1]))
    assert np.array_equal(K.get_states(), U.get_states())
    assert K.stream_links()[1][[0, 1, 2, 5, 9]].tolist() == [2, 2, 2, 1, 1]


@pytest.mark.gpu
def test_refusals_change_nothing(testing_raw):
    B = 70
    x = signals(B, 10, seed=41, speech=testing_raw)
    R, W = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    for b in (R, W):
        b.link_streams([0, 4], "mean")
        b.link_streams(list(range(10, 20)), "max")
        fused(b, x[:4], per_call=2)
    before = R.stream_links()
    L = nb.lib()

    def raw_link(streams, mode=1):
        idx = np.ascontiguousarray(streams, np.int32)
        return L.rnnoise_batch_link_streams(R._h, idx.ctypes.data_as(C.c_void_p), len(idx), mode)

    def unchanged():
        return all(np.array_equal(a, c) for a, c in zip(R.stream_links(), before))

    for streams, mode, text in (([3], 1, "2..64 streams, not 1"), (list(range(65)), 1, "not 65"), ([1, 1], 1, "twice"),
                                ([1, 70], 1, "out of range"), ([-1, 2], 2, "out of range"), ([1, 2], 0, "link mode 0"),
                                ([1, 2], 3, "link mode 3")):
        assert raw_link(streams, mode) < 0 and text in nb.last_error(), (streams, mode, nb.last_error())
        assert unchanged()
    assert L.rnnoise_batch_link_streams(R._h, None, 2, 1) < 0 and "null argument" in nb.last_error()
    idx = np.array([1, 71], np.int32)
    assert L.rnnoise_batch_unlink_streams(R._h, idx.ctypes.data_as(C.c_void_p), 2) < 0 and "out of range" in nb.last_error()
    # pending split frames: link and unlink are refused
    th_ = torch()
    xd = th_.from_numpy(x[4:5]).cuda()
    feats = th_.empty((B, NBF), device="cuda")
    R.analyze_device(xd[0].data_ptr(), feats.data_ptr(), 0, 1, F, B * F, NBF, B * NBF)
    assert raw_link([1, 2]) < 0 and "pending" in nb.last_error()
    with pytest.raises(nb.NnnoiselessError, match="pending"):
        R.unlink_streams()
    assert unchanged()
    gains = th_.full((B, NBB), 0.5, device="cuda")
    out = th_.empty_like(xd)
    R.synthesize_device(out[0].data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB)
    W.analyze_device(xd[0].data_ptr(), feats.data_ptr(), 0, 1, F, B * F, NBF, B * NBF)
    W.synthesize_device(out[0].data_ptr(), gains.data_ptr(), 1, F, B * F, NBB, B * NBB)
    o_r, v_r = fused(R, x[5:], per_call=3)
    o_w, v_w = fused(W, x[5:], per_call=3)
    assert np.array_equal(bits(o_r), bits(o_w)) and np.array_equal(bits(v_r), bits(v_w))
    assert np.array_equal(R.get_states(), W.get_states())


def wav_input(path, n_ch, seed, speech):
    """A 48 kHz 16-bit WAV of n_ch channels, 15 whole frames and 100 samples: speech at per-channel levels and noise."""
    rng = np.random.default_rng(seed)
    n = 15 * F + 100
    sp = speech.reshape(-1)[:n].astype(np.float64)
    x = np.stack([sp * (0.2 + 0.3 * c) + rng.standard_normal(n) * (200.0 + 900.0 * c) for c in range(n_ch)], axis=1)
    pcm = np.clip(np.round(x), -32768, 32767).astype(np.int16)
    files.write_audio(str(path), pcm, wav=True)
    return pcm


def expected_file(pcm, mode):
    """A DenoiseBatch of the file's channels, linked as one group, frame by frame: int16 in and out, the first frame
    discarded and the trailing partial frame dropped -> [(frames - 1) * 480][channels] int16."""
    n_ch = pcm.shape[1]
    T = pcm.shape[0] // F
    x = np.ascontiguousarray(pcm[:T * F].astype(np.float32).reshape(T, F, n_ch).transpose(0, 2, 1))
    b = nb.DenoiseBatch(n_ch)
    if mode:
        b.link_streams(list(range(n_ch)), mode)
    o, _ = fused(b, x, pcm16=True)
    return np.ascontiguousarray(o[1:].transpose(0, 2, 1).reshape(-1, n_ch))


@pytest.mark.gpu
def test_files_and_cli_link_channels(tmp_path, testing_raw):
    stereo, three = tmp_path / "stereo.wav", tmp_path / "three.wav"
    pcm = {stereo: wav_input(stereo, 2, 42, testing_raw), three: wav_input(three, 3, 43, testing_raw)}
    for mode in ("max", "mean"):
        want = {p: expected_file(a, mode) for p, a in pcm.items()}
        for p in pcm:
            out = tmp_path / ("cli_%s_%s" % (mode, p.name))
            r = subprocess.run([files.CLI_PATH, "--link-channels", mode, str(p), str(out)], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr
            got, rate = files.read_audio(str(out))
            assert rate == 48000.0 and np.array_equal(got.astype(np.int16), want[p]), (mode, p.name)
        # both files in one call: every file's channels are their own group
        pairs = [(str(p), str(tmp_path / ("api_%s_%s" % (mode, p.name)))) for p in pcm]
        files.denoise_files(pairs, link_channels=mode)
        for (src, dst), p in zip(pairs, pcm):
            assert np.array_equal(files.read_audio(dst)[0].astype(np.int16), want[p]), (mode, src)
    # without the flag the channels stay independent, and linking changes the output
    plain = tmp_path / "plain.wav"
    files.denoise_files([(str(stereo), str(plain))])
    unlinked = files.read_audio(str(plain))[0].astype(np.int16)
    assert np.array_equal(unlinked, expected_file(pcm[stereo], None))
    assert not np.array_equal(unlinked, expected_file(pcm[stereo], "mean"))
