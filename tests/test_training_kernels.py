"""train_front_kernel and train_rows_kernel (train.cu) one frame at a time against train_ref.py, on the constructed lanes
of train_cases.py, with the trainer's feature batch read back after every frame (TrainingBatch.feature_batch).

After every frame, for every lane:
- the clean, noise and combined streams' history windows and mem_hp_x (state records) equal the restatement's bits;
- the VAD column equals the restatement's bits;
- the gain columns equal train_ref's float32 row assembly on the GPU's own band energies and silence flags, bit for bit
  (the division and sqrtf are IEEE: the library is built without --use_fast_math);
- the noise levels are within 2 ulp of float64 log10 of the same float32 sum: the CUDA Math API's documented maximum
  error of log10f (single-precision table, 2 ulp over the full range, CUDA 12.x);
- the feature columns equal the combined stream's feature taps, bit for bit;
- feature 40 is 0.01 (period - 300) in float32 for the period the oracle's pitch search finds on the same history with
  the record's carried last_period and last_gain (0 on a silent frame), and the pitch tap and the new record's
  last_period / last_gain are the oracle's.
Layouts: lane counts around the 64-lane front blocks and the 128-thread row blocks, the float4 and the scalar load
path of process_device with padded rows, a multi-frame bitwise comparison of the load paths, and a process_host call
that crosses its 256 MiB staging chunk."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle_state as ost
import train_cases as tc
import train_ref as tr
from nnnoiseless_b200 import training

pytestmark = pytest.mark.gpu
PAD = 96                     # padded row stride of the device layouts
SENTINEL = np.uint32(0x7FC0DEAD)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class HostFrames:
    """One process_host call per frame."""

    def __init__(self, L):
        self.L = L

    def __call__(self, tb, sig, noi):
        return tb.process_host(sig[None], noi[None])[0]


class DeviceFrames:
    """One process_device call per frame: 'vec' (aligned, stream_stride 480: the float4 path), 'off1' (pointer one float
    past an aligned one) or 's481' (stream_stride 481), the two scalar paths; rows PAD floats apart, the padding
    filled with a sentinel that must survive."""

    def __init__(self, L, layout):
        import torch
        self.torch, self.L, self.layout = torch, L, layout
        stride = 481 if layout == "s481" else 480
        self.stride = stride
        self.base = [torch.zeros(L * stride + 1, device="cuda") for _ in range(2)]
        self.off = 1 if layout == "off1" else 0
        self.rows = torch.from_numpy(np.full((L, PAD), SENTINEL, np.uint32).view(np.float32)).cuda()

    def __call__(self, tb, sig, noi):
        torch = self.torch
        ptrs = []
        for buf, x in zip(self.base, (sig, noi)):
            v = buf[self.off:self.off + self.L * self.stride].view(self.L, self.stride)
            v[:, :480].copy_(torch.from_numpy(np.ascontiguousarray(x)))
            ptrs.append(buf.data_ptr() + 4 * self.off)
        tb.process_device(self.rows.data_ptr(), ptrs[0], ptrs[1], 1, self.stride, 0, PAD, 0)
        r = self.rows.cpu().numpy()
        assert np.all(bits(r[:, 87:]) == SENTINEL), "row padding written"
        return r[:, :87]


def run_checked(L, issue, builtin_bytes, shift=0):
    cs = tc.cases()
    lane, sig, noi, table = tc.lay_out(cs, L, shift)
    dt = nb.state_dtype(nb.gru_widths(builtin_bytes))
    tb = training.TrainingBatch(L)
    fb = tb.feature_batch()
    assert fb.state_bytes == dt.itemsize
    ref = tr.FrontRef(L)
    prev = fb.get_states().view(dt)[:, 0]
    bad = []

    def expect(ok, t, what, mask=None):
        if not ok:
            lanes = sorted({lane[l].name for l in np.flatnonzero(mask)}) if mask is not None else []
            bad.append((t, what, lanes[:4]))

    for t in range(tc.T):
        if t in table:
            tb.set_params(table[t])
            ref.set_params(table[t])
        rows = issue(tb, sig[t], noi[t])
        front = ref.frame(sig[t], noi[t])
        rec = fb.get_states().view(dt)[:, 0]
        taps, sp = fb.taps(), fb.spectral_taps()

        h = bits(rec["input_mem"]).reshape(3, L, -1) != bits(ref.hist)
        expect(not h.any(), t, "history", h.any(axis=(0, 2)))
        m = bits(rec["mem_hp_x"]).reshape(3, L, 2) != bits(ref.hp_mem)
        expect(not m.any(), t, "mem_hp_x", m.any(axis=(0, 2)))
        v = bits(rows[:, 86]) != bits(front["vad"])
        expect(not v.any(), t, "vad column", v)

        ex = sp["ex"].reshape(3, L, tr.NB_BANDS)
        sil = taps["silence"].reshape(3, L) != 0
        g = bits(rows[:, 42:64]) != bits(tr.gains_f32(ex[0], ex[2], front["cutoff"], sil[2]))
        expect(not g.any(), t, "gain columns", g.any(axis=1))
        exact = tr.noise_levels_f64(ex[1])
        ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
        n = np.abs(rows[:, 64:86].astype(np.float64) - exact) > 2 * ulp
        expect(not n.any(), t, "noise levels beyond 2 ulp", n.any(axis=1))
        f = bits(rows[:, :42]) != bits(taps["features"][2 * L:])
        expect(not f.any(), t, "feature columns", f.any(axis=1))

        comb = slice(2 * L, 3 * L)
        period, gain = ost.pitch_only(rec["input_mem"][comb], prev["last_period"][comb], prev["last_gain"][comb])
        f40 = np.where(sil[2], np.float32(0.0), np.float32(0.01) * (period.astype(np.float32) - np.float32(300.0)))
        p = (bits(rows[:, 40]) != bits(f40)) | (taps["pitch"][comb] != period) | (rec["last_period"][comb] != period) | \
            (bits(rec["last_gain"][comb]) != bits(gain))
        expect(not p.any(), t, "pitch", p)
        prev = rec
    assert bad == [], bad[:8]


@pytest.mark.parametrize("L", [1, 64, 65, 130])
def test_frames_host_against_restatement(L, builtin_bytes):
    run_checked(L, HostFrames(L), builtin_bytes, shift=L % 7)


@pytest.mark.parametrize("layout", ["vec", "off1", "s481"])
def test_frames_device_layouts_against_restatement(layout, builtin_bytes):
    run_checked(65, DeviceFrames(65, layout), builtin_bytes, shift=3)


def test_load_paths_bitwise_over_multi_frame_calls():
    """The whole case schedule in three multi-frame process_device calls (split where parameters change), lane-major for
    the float4 path and the pointer offset by one float, frame-major with stream_stride 481: rows and every state
    record equal as bits."""
    import torch
    L, T = 65, tc.T
    _, sig, noi, table = tc.lay_out(tc.cases(), L, 5)
    cuts = sorted(table) + [T]
    out = {}
    for layout in ("vec", "off1", "s481"):
        tb = training.TrainingBatch(L)
        if layout == "s481":   # [T][L][481]: sample (l, f, i) at l * 481 + f * L * 481 + i
            host = np.zeros((2, T, L, 481), np.float32)
            host[0, ..., :480], host[1, ..., :480] = sig, noi
            ss, fs = 481, L * 481
        else:                  # [L][T][480]
            host = np.stack([sig.transpose(1, 0, 2), noi.transpose(1, 0, 2)])
            ss, fs = T * 480, 480
        off = 1 if layout == "off1" else 0
        bufs = []
        for k in range(2):
            b = torch.zeros(host[k].size + 1, device="cuda")
            b[off:off + host[k].size].copy_(torch.from_numpy(host[k].reshape(-1)))
            bufs.append(b)
        rows = torch.from_numpy(np.full((L, T, PAD), SENTINEL, np.uint32).view(np.float32)).cuda()
        for t0, t1 in zip(cuts[:-1], cuts[1:]):
            tb.set_params(table[t0])
            tb.process_device(rows.data_ptr() + 4 * t0 * PAD, bufs[0].data_ptr() + 4 * (off + t0 * fs),
                              bufs[1].data_ptr() + 4 * (off + t0 * fs), t1 - t0, ss, fs, T * PAD, PAD)
        r = rows.cpu().numpy()
        assert np.all(bits(r[..., 87:]) == SENTINEL)
        out[layout] = (bits(r[..., :87]), tb.feature_batch().get_states())
    for layout in ("off1", "s481"):
        assert np.array_equal(out[layout][0], out["vec"][0]), layout
        assert np.array_equal(out[layout][1], out["vec"][1]), layout


def test_process_host_crosses_staging_chunk():
    """L = 8192 lanes make process_host stage 17 frames at a time (256 MiB per input); 18 frames cross one chunk boundary.
    The rows and a sample of state records equal one process_device call over the same frames."""
    import torch
    L, T = 8192, 18
    assert (256 << 20) // (L * 480 * 4) == 17
    rng = np.random.default_rng(8)
    p = training.randomize(L, rng)
    sig = np.empty((T, L, 480), np.float32)
    noi = np.empty((T, L, 480), np.float32)
    for t in range(T):
        sig[t] = rng.integers(-6000, 6000, (L, 480), dtype=np.int16)
        noi[t] = rng.integers(-2000, 2000, (L, 480), dtype=np.int16)
    a = training.TrainingBatch(L)
    a.set_params(p)
    got = a.process_host(sig, noi)
    b = training.TrainingBatch(L)
    b.set_params(p)
    ds, dn = torch.from_numpy(sig).cuda(), torch.from_numpy(noi).cuda()
    del sig, noi
    rows = torch.empty((T, L, tr.ROW), device="cuda")
    b.process_device(rows.data_ptr(), ds.data_ptr(), dn.data_ptr(), T, 480, L * 480, tr.ROW, L * tr.ROW)
    assert np.array_equal(bits(rows.cpu().numpy()), bits(got))
    some = np.concatenate([np.arange(0, 3 * L, 193), [L - 1, 2 * L - 1, 3 * L - 1]]).astype(np.int32)
    assert np.array_equal(a.feature_batch().get_states(some), b.feature_batch().get_states(some))
