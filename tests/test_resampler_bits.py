"""GPU tests of the streaming resampler stages (resample_up_kernel / resample_down_kernel, DESIGN.md 7g) bit for bit
against their exact f32 restatement (resample_ref.stages_bits: the fmaf chain in ascending tap index): every one of the
401 stream rates, float and int16 sides, constructed signals, the grid-y split of calls longer than 65,535 frames,
the state records' histories and the int16 conversion's rounding edges."""
import numpy as np
import pytest
from scipy.signal import upfirdn

import nnnoiseless_b200 as nb
from resample_ref import pcm16, stages_bits

pytestmark = pytest.mark.gpu

ALL_RATES = np.arange(8000, 48001, 100, dtype=np.int32)
MAXY = 65535


def torch_cuda():
    import torch
    return torch


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.int16 else np.uint32)


def up(rs, x, calls, fs=480):
    """x: native [n][T][fs] (float32 or int16) -> [T][n][480] float32, in calls of the given frame counts."""
    torch = torch_cuda()
    n, T = x.shape[:2]
    xi = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = torch.empty((T, n, 480), dtype=torch.float32, device="cuda")
    t0 = 0
    for k in calls:
        rs.up_device(out[t0:].data_ptr(), xi[:, t0:].data_ptr(), k, T * fs, fs, pcm16=int(x.dtype == np.int16), n=n)
        t0 += k
    return out.cpu().numpy()


def down(rs, y, calls, pcm16=False):
    """y: [T][n][480] float32 -> native [n][T][480] (float32 or int16; slots past R/100 stay zero)."""
    torch = torch_cuda()
    T, n = y.shape[:2]
    yi = torch.from_numpy(np.ascontiguousarray(y, np.float32)).cuda()
    out = torch.zeros((n, T, 480), dtype=torch.int16 if pcm16 else torch.float32, device="cuda")
    t0 = 0
    for k in calls:
        rs.down_device(out[:, t0:].data_ptr(), yi[t0:].data_ptr(), k, T * 480, 480, pcm16=int(pcm16), n=n)
        t0 += k
    return out.cpu().numpy()


def shuffled_rates(seed=0):
    return ALL_RATES[np.random.default_rng(seed).permutation(len(ALL_RATES))]


def native_kinds(rates, T):
    """Constructed native signals [n][T][480] per kind (the first R/100 samples of each slot); int16-valued kinds
    also run through the int16 input."""
    rng = np.random.default_rng(1)
    out = {}
    for kind in ("random", "dc", "impulses", "alternating", "tiny"):
        x = np.zeros((len(rates), T, 480), np.float32)
        for s, R in enumerate(rates):
            n = R // 100 * T
            if kind == "random":
                v = np.round(rng.standard_normal(n) * 6000.0).clip(-32768, 32767)
            elif kind == "dc":
                v = np.full(n, 12345.0)
            elif kind == "impulses":
                # isolated impulses (23 > 21 taps apart): each output is one product, so every (phase, tap) that meets
                # an impulse shows its own bits; the offsets differ per stream
                v = np.zeros(n)
                v[s % 23:: 23] = rng.integers(-32768, 32768, len(v[s % 23:: 23]))
            elif kind == "alternating":
                v = np.where(np.arange(n) % 2 == 0, 32767.0, -32767.0)
            else:
                v = rng.standard_normal(n) * 1e-38       # products below the normal range: no flush to zero
            x[s, :, : R // 100] = v.reshape(T, R // 100)
        out[kind] = x
    return out


def wide_kinds(n, T):
    """Constructed 48 kHz signals [T][n][480] per kind for the down stage."""
    rng = np.random.default_rng(2)
    out = {"random": rng.standard_normal((T, n, 480)) * 20000.0, "dc": np.full((T, n, 480), -23456.0)}
    imp = np.zeros((n, T * 480))
    for s in range(n):
        imp[s, s % 127:: 127] = rng.integers(-32768, 32768, len(imp[s, s % 127:: 127]))   # 127 > 121 taps apart
    out["impulses"] = imp.reshape(n, T, 480).transpose(1, 0, 2)
    out["alternating"] = np.broadcast_to(np.where(np.arange(T * 480) % 2 == 0, 32767.0, -32767.0).reshape(T, 1, 480), (T, n, 480))
    out["tiny"] = rng.standard_normal((T, n, 480)) * 1e-38
    return {k: np.ascontiguousarray(v, np.float32) for k, v in out.items()}


def test_every_rate_bit_for_bit():
    """One resampler of 401 streams, one per valid rate in a shuffled row order, fed in calls of 2 + 3 frames."""
    rates = shuffled_rates()
    n, T, calls = len(rates), 5, [2, 3]
    for kind, x in native_kinds(rates, T).items():
        got = up(nb.Resampler(n, rates), x, calls)
        want = stages_bits(rates, 0, [x[s, :, : R // 100].reshape(-1) for s, R in enumerate(rates)])
        for s, R in enumerate(rates):
            assert np.array_equal(bits(got[:, s].reshape(-1)), bits(want[s])), ("up", kind, int(R))
        if kind != "tiny":
            got16 = up(nb.Resampler(n, rates), x.astype(np.int16), calls)
            assert np.array_equal(bits(got16), bits(got)), ("up int16", kind)
        if kind == "random":   # the order-free second check, against float64
            for s, R in enumerate(rates):
                h, u, d = nb.resampler_filter(int(R), 0)
                src = x[s, :, : R // 100].reshape(-1).astype(np.float64)
                ref = upfirdn(h.astype(np.float64), src, u, d)[: T * 480]
                tol = 32 * 2.0 ** -24 * upfirdn(np.abs(h.astype(np.float64)), np.abs(src), u, d)[: T * 480]
                assert np.all(np.abs(got[:, s].reshape(-1) - ref) <= tol), ("up f64", int(R))
    for kind, y in wide_kinds(n, T).items():
        got = down(nb.Resampler(n, rates), y, calls)
        got16 = down(nb.Resampler(n, rates), y, calls, pcm16=True)
        want = stages_bits(rates, 1, [y[:, s].reshape(-1) for s in range(n)])
        for s, R in enumerate(rates):
            k = R // 100
            w = want[s].reshape(T, k)
            assert np.array_equal(bits(got[s, :, :k]), bits(w)), ("down", kind, int(R))
            assert np.array_equal(got16[s, :, :k], pcm16(w)), ("down int16", kind, int(R))
            assert not np.any(got[s, :, k:]) and not np.any(got16[s, :, k:])
            if kind == "random":
                h, u, d = nb.resampler_filter(int(R), 1)
                src = y[:, s].reshape(-1).astype(np.float64)
                ref = upfirdn(h.astype(np.float64), src, u, d)[: T * k]
                tol = 32 * 2.0 ** -24 * upfirdn(np.abs(h.astype(np.float64)), np.abs(src), u, d)[: T * k]
                assert np.all(np.abs(w.reshape(-1) - ref) <= tol), ("down f64", int(R))


def records(rs):
    rec = rs.get_states()
    return rec[:, 16:96].copy().view(np.float32), rec[:, 96:576].copy().view(np.float32)


def test_state_records_hold_the_input_tails():
    """After calls of 1, 7 and 40 frames, record bytes 16-95 are the last 20 native samples the up stage read and bytes
    96-575 the last 120 48 kHz samples the down stage read, oldest first, bit for bit."""
    rates = shuffled_rates(seed=3)
    n = len(rates)
    rs = nb.Resampler(n, rates)
    rng = np.random.default_rng(4)
    for T in (1, 7, 40):
        x = (rng.standard_normal((n, T, 480)) * 5000.0).astype(np.float32)
        y = (rng.standard_normal((T, n, 480)) * 5000.0).astype(np.float32)
        up(rs, x, [T])
        down(rs, y, [T])
        hu, hd = records(rs)
        for s, R in enumerate(rates):
            k = R // 100
            assert np.array_equal(bits(hu[s]), bits(x[s, T - 1, k - 20: k])), (T, int(R))
        assert np.array_equal(bits(hd), bits(y[T - 1, :, 360:]))


def frame_bits(rates, direction, src, frames):
    """stages_bits of single frames t of a long call: src(s, t) gives frame t of stream s (zeros before frame 0), each
    emulated after the tail of frame t - 1."""
    hl = 20 if direction == 0 else 120
    rs_, xs, hs, keys = [], [], [], []
    for s, R in enumerate(rates):
        for t in frames:
            f = src(s, t)
            rs_.append(R)
            xs.append(f)
            hs.append(src(s, t - 1)[-hl:] if t > 0 else None)
            keys.append((s, t))
    return dict(zip(keys, stages_bits(rs_, direction, xs, hs)))


@pytest.mark.parametrize("T", [MAXY + 9, 2 * MAXY + 3])
def test_grid_y_split(T):
    """Calls of more than 65,535 frames take several launches (frame = t0 + blockIdx.y).  Bit for bit against the
    restatement at every launch edge and the last frame, equal to the same frames fed in calls of at most 1,000, and
    the records hold the input tails."""
    torch = torch_cuda()
    rates = np.array([8000, 44100, 47900], np.int32)
    n, fs = len(rates), 480
    g = torch.Generator(device="cuda").manual_seed(T)
    x = torch.round(torch.randn((n, T, fs), generator=g, device="cuda") * 5000.0)
    y = torch.randn((T, n, 480), generator=g, device="cuda") * 5000.0
    edges = sorted({0, 1, T - 1} | {e + d for e in range(MAXY, T, MAXY) for d in (-1, 0, 1)})
    whole = [torch.empty((T, n, 480), device="cuda"), torch.zeros((n, T, fs), device="cuda")]
    parts = [torch.empty_like(whole[0]), torch.zeros_like(whole[1])]
    rs_w, rs_p = nb.Resampler(n, rates), nb.Resampler(n, rates)
    for rs, outs, calls in ((rs_w, whole, [T]), (rs_p, parts, [1000] * (T // 1000) + [T % 1000])):
        t0 = 0
        for k in calls:
            rs.up_device(outs[0][t0:].data_ptr(), x[:, t0:].data_ptr(), k, T * fs, fs, n=n)
            rs.down_device(outs[1][:, t0:].data_ptr(), y[t0:].data_ptr(), k, T * fs, fs, n=n)
            t0 += k
    torch.cuda.synchronize()
    assert torch.equal(whole[0].view(torch.int32), parts[0].view(torch.int32))
    assert torch.equal(whole[1].view(torch.int32), parts[1].view(torch.int32))
    et = torch.tensor(edges, device="cuda")
    xe = x[:, (et - 1).clamp(min=0)].cpu().numpy(), x[:, et].cpu().numpy()
    ye = y[(et - 1).clamp(min=0)].cpu().numpy(), y[et].cpu().numpy()
    ue, de = whole[0][et].cpu().numpy(), whole[1][:, et].cpu().numpy()
    at = {t: i for i, t in enumerate(edges)}
    for direction in (0, 1):
        def src(s, t, direction=direction):
            i = at.get(t)
            k = rates[s] // 100
            if i is None:                                   # frame t - 1 of an edge frame
                i = at[t + 1]
                return xe[0][s, i, :k] if direction == 0 else ye[0][i, s]
            return xe[1][s, i, :k] if direction == 0 else ye[1][i, s]
        want = frame_bits(rates, direction, src, edges)
        for (s, t), w in want.items():
            got = ue[at[t], s] if direction == 0 else de[s, at[t], : rates[s] // 100]
            assert np.array_equal(bits(got), bits(w)), (direction, int(rates[s]), t)
    for rs in (rs_w, rs_p):
        hu, hd = records(rs)
        last_x, last_y = x[:, T - 1].cpu().numpy(), y[T - 1].cpu().numpy()
        for s, R in enumerate(rates):
            assert np.array_equal(bits(hu[s]), bits(last_x[s, R // 100 - 20: R // 100]))
        assert np.array_equal(bits(hd), bits(last_y[:, 360:]))
    del x, y, whole, parts


def test_native_device_two_launches_per_stage():
    """One 16 kHz stream for 70,000 frames: one scratch chunk, two launches per stage; the bits of up ->
    process_device -> down."""
    torch = torch_cuda()
    T = 70000
    g = torch.Generator(device="cuda").manual_seed(5)
    xi = (torch.randn((1, T, 480), generator=g, device="cuda") * 3000.0).contiguous()
    xi[:, :, 160:] = 0
    o1, o2 = torch.zeros_like(xi), torch.zeros_like(xi)
    v1, v2 = (torch.empty((T, 1), device="cuda") for _ in range(2))
    b1, r1 = nb.DenoiseBatch(1), nb.Resampler(1, [16000])
    before = nb.kernel_launches()
    b1.process_native_device(r1, o1.data_ptr(), xi.data_ptr(), v1.data_ptr(), T, T * 480, 480)
    launches = nb.kernel_launches() - before
    b2, r2 = nb.DenoiseBatch(1), nb.Resampler(1, [16000])
    w = torch.empty((T, 1, 480), device="cuda")
    before = nb.kernel_launches()
    r2.up_device(w.data_ptr(), xi.data_ptr(), T, T * 480, 480)
    assert nb.kernel_launches() - before == 2
    b2.process_device(w.data_ptr(), w.data_ptr(), v2.data_ptr(), T, 480, 480)
    mid = nb.kernel_launches()
    r2.down_device(o2.data_ptr(), w.data_ptr(), T, T * 480, 480)
    assert nb.kernel_launches() - mid == 2
    assert launches == nb.kernel_launches() - before       # one chunk: the same launches as the three calls
    assert torch.equal(o1.view(torch.int32), o2.view(torch.int32)) and torch.equal(v1.view(torch.int32), v2.view(torch.int32))


EDGES = np.array([0.0, -0.0, 0.49999997, -0.49999997, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 32766.5, -32766.5, 32767.5, -32767.5,
                  32768.0, -32768.5, -32769.0, 1e30, -1e30, np.inf, -np.inf, np.nan], np.float32)


def test_pcm16_conversion_edges():
    """to_pcm16w against `x.max(-32768).min(32767).round() as i16` in float64: at 48 kHz, where the down stage passes
    samples through, and after a 16 kHz down stage against its restatement."""
    T = 2
    y = np.zeros((T, 2, 480), np.float32)
    v = np.tile(EDGES, 480 * T // len(EDGES) + 1)[: 480 * T]
    y[:, 0] = v.reshape(T, 480)
    finite = EDGES[np.abs(EDGES) < 1e5]                     # stream 1: no inf or NaN, which would fill a window
    y[:, 1] = np.tile(finite, 480 * T // len(finite) + 1)[: 480 * T].reshape(T, 480)
    for R in (48000, 16000):
        rates = [R, R]
        got16 = down(nb.Resampler(2, rates), y, [T], pcm16=True)
        gotf = down(nb.Resampler(2, rates), y, [T])
        want = stages_bits(rates, 1, [y[:, s].reshape(-1) for s in range(2)])
        k = R // 100
        for s in range(2):
            w = want[s].reshape(T, k)
            assert np.array_equal(got16[s, :, :k], pcm16(w)), (R, s)
            if R == 48000:
                assert np.array_equal(bits(gotf[s, :, :k]), bits(y[:, s])), s   # passed through, NaN and -0 included
            else:
                assert np.array_equal(np.isnan(gotf[s, :, :k]), np.isnan(w))
                ok = ~np.isnan(w)
                assert np.array_equal(bits(gotf[s, :, :k][ok]), bits(w[ok])), (R, s)
