"""GPU tests of streams at their own sample rate (rnnoise_resampler_*, rnnoise_batch_process_native_*; DESIGN.md 7g):
each stage against scipy's upfirdn in float64, bit-for-bit invariance to call splits, batch layout, subsets and other
streams, 48 kHz streams byte for byte equal to the plain batch calls, process_native equal to its parts called one by
one (per-stream models included), state records, a round trip of tones, and testing.raw end to end at 16 kHz."""
import numpy as np
import pytest
from scipy.signal import resample_poly, upfirdn

import nnnoiseless_b200 as nb
import rnn_ref
from conftest import synth_streams
from resample_ref import Stage, stream

pytestmark = pytest.mark.gpu

MIXED = (8000, 12000, 16000, 24000, 32000, 44100, 48000)


def torch_cuda():
    import torch
    return torch


def rates_for(B, seed=0):
    return np.random.default_rng(seed).choice(MIXED, B).astype(np.int32)


def native_input(rates, T, seed, pcm16=False):
    """[B][T][480] slots, the first R/100 samples of each a stream's frame (random, int16 range), the rest zero."""
    rng = np.random.default_rng(seed)
    x = np.zeros((len(rates), T, 480), np.int16 if pcm16 else np.float32)
    for s, R in enumerate(rates):
        v = rng.standard_normal((T, R // 100)) * 4000.0
        x[s, :, : R // 100] = np.clip(np.round(v), -32768, 32767) if pcm16 else v
    return x


def up(rs, x, streams=None, calls=None):
    """Up stage on device: native [n][T][480] -> [T][n][480]; `calls` splits the frames into calls of those lengths."""
    torch = torch_cuda()
    n, T = x.shape[:2]
    xi = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = torch.empty((T, n, 480), dtype=torch.float32, device="cuda")
    t0 = 0
    for k in calls or [T]:
        rs.up_device(out[t0:].data_ptr(), xi[:, t0:].data_ptr(), k, T * 480, 480, streams=streams, pcm16=int(x.dtype == np.int16), n=n)
        t0 += k
    return out.cpu().numpy()


def down(rs, y, streams=None, calls=None, pcm16=False):
    """Down stage on device: [T][n][480] -> native [n][T][480] (slots past R/100 stay zero)."""
    torch = torch_cuda()
    T, n = y.shape[:2]
    yi = torch.from_numpy(np.ascontiguousarray(y, np.float32)).cuda()
    out = torch.zeros((n, T, 480), dtype=torch.int16 if pcm16 else torch.float32, device="cuda")
    t0 = 0
    for k in calls or [T]:
        rs.down_device(out[:, t0:].data_ptr(), yi[t0:].data_ptr(), k, T * 480, 480, streams=streams, pcm16=int(pcm16), n=n)
        t0 += k
    return out.cpu().numpy()


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint16 if a.dtype == np.int16 else np.uint32)


def test_stages_against_upfirdn_f64():
    rates = np.array([8000, 16000, 24000, 32000, 44100], np.int32)
    T = 12
    rs = nb.Resampler(len(rates), rates)
    x = native_input(rates, T, seed=1)
    y = up(rs, x)
    z48 = np.random.default_rng(2).standard_normal((T, len(rates), 480)).astype(np.float32) * 4000.0
    w = down(rs, z48)
    worst = {}
    for s, R in enumerate(rates):
        n = R // 100
        for direction, src, got in ((0, x[s, :, :n].reshape(-1), y[:, s].reshape(-1)), (1, z48[:, s].reshape(-1), w[s, :, :n].reshape(-1))):
            h, u, d = nb.resampler_filter(R, direction)
            h64, src64 = h.astype(np.float64), src.astype(np.float64)
            ref = upfirdn(h64, src64, u, d)[: len(got)]
            tol = 32 * 2.0 ** -24 * upfirdn(np.abs(h64), np.abs(src64), u, d)[: len(got)]
            share = float(np.max(np.abs(got - ref) / np.maximum(tol, 1e-30)))
            worst["%s %d" % ("up" if direction == 0 else "down", R)] = share
            assert share <= 1.0, (R, direction, share)
    print("worst share of the tolerance 32 * 2^-24 * sum|h x|:", {k: round(v, 4) for k, v in worst.items()})


def test_int16_sides():
    rates = rates_for(19, seed=3)
    T = 5
    xi = native_input(rates, T, seed=4, pcm16=True)
    y_i = up(nb.Resampler(len(rates), rates), xi)
    y_f = up(nb.Resampler(len(rates), rates), xi.astype(np.float32))
    assert np.array_equal(bits(y_i), bits(y_f))
    z = np.random.default_rng(5).standard_normal((T, len(rates), 480)).astype(np.float32) * 20000.0
    w_f = down(nb.Resampler(len(rates), rates), z)
    w_i = down(nb.Resampler(len(rates), rates), z, pcm16=True)
    expect = np.clip(w_f, -32768, 32767)
    expect = (np.sign(expect) * np.floor(np.abs(expect) + 0.5)).astype(np.int16)  # roundf: half away from zero
    assert np.array_equal(w_i, expect)


def test_chunk_invariance_bitwise():
    rates = rates_for(23, seed=6)
    T = 9
    x = native_input(rates, T, seed=7)
    z = np.random.default_rng(8).standard_normal((T, len(rates), 480)).astype(np.float32) * 4000.0
    for calls in ([T], [1, T - 1], [1] * T, [4, 2, 3]):
        yu = up(nb.Resampler(len(rates), rates), x, calls=calls)
        yd = down(nb.Resampler(len(rates), rates), z, calls=calls)
        if calls == [T]:
            ru, rd = yu, yd
        assert np.array_equal(bits(yu), bits(ru)) and np.array_equal(bits(yd), bits(rd)), calls


def test_independence_bitwise():
    """A stream's bits do not depend on the batch size, its row, the other streams' rates or subset membership and order."""
    T = 4
    B_max = 65
    rates = rates_for(B_max, seed=9)
    x = native_input(rates, T, seed=10)
    z = np.random.default_rng(11).standard_normal((T, B_max, 480)).astype(np.float32) * 4000.0
    # the reference: every stream alone in a resampler of one stream
    alone_u = [up(nb.Resampler(1, [R]), x[s: s + 1])[:, 0] for s, R in enumerate(rates)]
    alone_d = [down(nb.Resampler(1, [R]), z[:, s: s + 1])[0] for s, R in enumerate(rates)]
    rng = np.random.default_rng(12)
    for B in (1, 63, 64, 65):
        perm = rng.permutation(B_max)[:B]  # stream perm[r] of the reference sits in row r
        for mode in ("full", "subset"):
            if mode == "full":
                rs = nb.Resampler(B, rates[perm])
                yu, yd = up(rs, x[perm]), down(nb.Resampler(B, rates[perm]), z[:, perm])
            else:  # a resampler of B_max + 7 streams; the rows are a shuffled subset of its streams
                N = B_max + 7
                slots = rng.permutation(N)[:B].astype(np.int32)
                all_rates = np.full(N, 16000, np.int32)
                all_rates[slots] = rates[perm]
                yu = up(nb.Resampler(N, all_rates), x[perm], streams=slots)
                yd = down(nb.Resampler(N, all_rates), z[:, perm], streams=slots)
            for r, s in enumerate(perm):
                assert np.array_equal(bits(yu[:, r]), bits(alone_u[s])), (B, mode, r)
                assert np.array_equal(bits(yd[r]), bits(alone_d[s])), (B, mode, r)


@pytest.mark.parametrize("pcm16", [0, 1])
def test_48k_streams_are_the_batch_path(pcm16):
    torch = torch_cuda()
    B, T = 11, 6
    x = np.ascontiguousarray(synth_streams(B, T, seed=13).reshape(B, T, 480))
    if pcm16:
        x = np.clip(np.round(x), -32768, 32767).astype(np.int16)
    xi = torch.from_numpy(x).cuda()
    dt = torch.int16 if pcm16 else torch.float32
    o_nat, o_ref = torch.empty((B, T, 480), dtype=dt, device="cuda"), torch.empty((B, T, 480), dtype=dt, device="cuda")
    v_nat, v_ref = (torch.empty((T, B), dtype=torch.float32, device="cuda") for _ in range(2))
    b1, b2 = nb.DenoiseBatch(B), nb.DenoiseBatch(B)
    b1.process_native_device(nb.Resampler(B), o_nat.data_ptr(), xi.data_ptr(), v_nat.data_ptr(), T, T * 480, 480, pcm16=pcm16)
    b2.process_device(o_ref.data_ptr(), xi.data_ptr(), v_ref.data_ptr(), T, T * 480, 480, pcm16=bool(pcm16))
    assert o_nat.cpu().numpy().tobytes() == o_ref.cpu().numpy().tobytes()
    assert v_nat.cpu().numpy().tobytes() == v_ref.cpu().numpy().tobytes()
    # host slots, frame-major
    xh = np.ascontiguousarray(x.transpose(1, 0, 2))
    o_h, v_h = nb.DenoiseBatch(B).process_native_host(nb.Resampler(B), xh)
    assert o_h.tobytes() == np.ascontiguousarray(o_ref.cpu().numpy().transpose(1, 0, 2)).tobytes()
    assert v_h.tobytes() == v_ref.cpu().numpy().tobytes()


def composed(batch, rs, x, T, streams=None, pcm16=0):
    """up -> process_device / process_streams_device -> down, three calls."""
    torch = torch_cuda()
    n = x.shape[0]
    xi = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    w = torch.empty((T, n, 480), dtype=torch.float32, device="cuda")
    out = torch.zeros_like(xi)
    vad = torch.empty((T, n), dtype=torch.float32, device="cuda")
    rs.up_device(w.data_ptr(), xi.data_ptr(), T, T * 480, 480, streams=streams, pcm16=pcm16, n=n)
    if streams is None and n == batch.n_streams:
        batch.process_device(w.data_ptr(), w.data_ptr(), vad.data_ptr(), T, 480, n * 480)
    else:
        batch.process_streams_device(streams, w.data_ptr(), w.data_ptr(), vad.data_ptr(), T, 480, n * 480, n=n)
    rs.down_device(out.data_ptr(), w.data_ptr(), T, T * 480, 480, streams=streams, pcm16=pcm16, n=n)
    return out.cpu().numpy(), vad.cpu().numpy()


def native(batch, rs, x, T, streams=None, pcm16=0):
    torch = torch_cuda()
    n = x.shape[0]
    xi = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = torch.zeros_like(xi)
    vad = torch.empty((T, n), dtype=torch.float32, device="cuda")
    batch.process_native_device(rs, out.data_ptr(), xi.data_ptr(), vad.data_ptr(), T, T * 480, 480, streams=streams, pcm16=pcm16, n=n)
    return out.cpu().numpy(), vad.cpu().numpy()


def twins(B, rates, models=None):
    """Two identical (batch, resampler) pairs; models: per-stream model ids over the built-in model and one more."""
    pairs = []
    for _ in range(2):
        b = nb.DenoiseBatch(B)
        if models is not None:
            b.add_model(nb.RnnModel.from_bytes(rnn_ref.make_model(24, 24, 48, 96, seed=77)))
            b.set_stream_models(models)
        pairs.append((b, nb.Resampler(B, rates)))
    return pairs


@pytest.mark.parametrize("pcm16", [0, 1])
def test_native_is_its_parts(pcm16):
    B, T = 37, 5
    rates = rates_for(B, seed=14)
    models = (np.arange(B) % 3 == 0).astype(np.int32)
    (b1, r1), (b2, r2) = twins(B, rates, models)
    x = native_input(rates, 2 * T, seed=15, pcm16=bool(pcm16))
    o1, v1 = native(b1, r1, x[:, :T], T, pcm16=pcm16)
    o2, v2 = composed(b2, r2, x[:, :T], T, pcm16=pcm16)
    assert np.array_equal(bits(o1), bits(o2)) and np.array_equal(bits(v1), bits(v2))
    # then a subset call, rows in shuffled order
    S = np.random.default_rng(16).permutation(B)[:20].astype(np.int32)
    o1, v1 = native(b1, r1, x[S, T:], T, streams=S, pcm16=pcm16)
    o2, v2 = composed(b2, r2, x[S, T:], T, streams=S, pcm16=pcm16)
    assert np.array_equal(bits(o1), bits(o2)) and np.array_equal(bits(v1), bits(v2))
    assert np.array_equal(b1.get_states(), b2.get_states()) and np.array_equal(r1.get_states(), r2.get_states())


def test_native_across_the_scratch_chunk():
    """B = 65,536: the 256 MiB scratch holds two frames, so three frames take two chunks; the bits are those of the parts
    called once over all three frames."""
    torch = torch_cuda()
    B, T = 65536, 3
    rates = rates_for(B, seed=17).astype(np.int32)
    (b1, r1), (b2, r2) = twins(B, rates)
    rng = torch.Generator(device="cuda").manual_seed(18)
    xi = (torch.randn((B, T, 480), generator=rng, device="cuda") * 3000.0).contiguous()
    o1, o2 = torch.zeros_like(xi), torch.zeros_like(xi)
    v1, v2 = (torch.empty((T, B), device="cuda") for _ in range(2))
    b1.process_native_device(r1, o1.data_ptr(), xi.data_ptr(), v1.data_ptr(), T, T * 480, 480)
    w = torch.empty((T, B, 480), device="cuda")
    r2.up_device(w.data_ptr(), xi.data_ptr(), T, T * 480, 480)
    b2.process_device(w.data_ptr(), w.data_ptr(), v2.data_ptr(), T, 480, B * 480)
    r2.down_device(o2.data_ptr(), w.data_ptr(), T, T * 480, 480)
    assert torch.equal(o1.view(torch.int32), o2.view(torch.int32)) and torch.equal(v1.view(torch.int32), v2.view(torch.int32))
    del w, xi, o1, o2


def test_records_continue_a_stream_bit_for_bit():
    B, T = 29, 4
    rates = rates_for(B, seed=19)
    x = native_input(rates, 2 * T, seed=20)
    b1, r1 = nb.DenoiseBatch(B), nb.Resampler(B, rates)
    o_all, v_all = native(b1, r1, x, 2 * T)
    b2, r2 = nb.DenoiseBatch(B), nb.Resampler(B, rates)
    native(b2, r2, x[:, :T], T)
    rec_b, rec_r = b2.get_states(), r2.get_states()
    assert np.array_equal(r2.stream_rates(), rates)
    hdr = rec_r[:, :16].copy().view("<i4")
    assert np.all(hdr[:, 0] == nb.RESAMPLER_STATE_MAGIC) and np.all(hdr[:, 1] == 1) and np.array_equal(hdr[:, 2], rates)
    # moved to fresh handles of another layout: stream s goes to slot perm[s]
    perm = np.random.default_rng(21).permutation(B).astype(np.int32)
    b3, r3 = nb.DenoiseBatch(B), nb.Resampler(B)
    b3.set_states(rec_b, perm)
    r3.set_states(rec_r, perm)
    assert np.array_equal(r3.stream_rates(perm), rates)
    inv = np.argsort(perm)
    o3, v3 = native(b3, r3, x[inv, T:], T)
    assert np.array_equal(bits(o3[perm]), bits(o_all[:, T:])) and np.array_equal(bits(v3[:, perm]), bits(v_all[T:]))
    # malformed records are refused and change nothing
    before = r3.get_states()
    for field, value in ((0, 0x12345678), (1, 2), (2, 7900), (2, 8050), (2, 48100)):
        bad = rec_r.copy()
        bad[5, 4 * field: 4 * field + 4] = np.frombuffer(np.int32(value).tobytes(), np.uint8)
        with pytest.raises(nb.NnnoiselessError, match="resampler state record 5"):
            r3.set_states(bad, perm)
        assert np.array_equal(r3.get_states(), before)
    with pytest.raises(nb.NnnoiselessError, match="stream 3: rate 7900"):
        r3.set_stream_rates([16000, 16000, 16000, 7900])
    with pytest.raises(nb.NnnoiselessError, match="given twice"):
        r3.set_stream_rates([16000, 16000], streams=[1, 1])
    assert np.array_equal(r3.get_states(), before)
    # set_stream_rates resets, even to the same rate
    r3.set_stream_rates(rates[inv][:1], streams=[0])
    assert not np.any(r3.get_states([0])[0, 16:]) and r3.stream_rates([0])[0] == rates[inv][0]


def test_native_argument_checks():
    b, rs = nb.DenoiseBatch(4), nb.Resampler(5)
    with pytest.raises(nb.NnnoiselessError, match="the batch has 4 streams, the resampler 5"):
        b.process_native_host(rs, np.zeros((1, 4, 480), np.float32))
    with pytest.raises(nb.NnnoiselessError, match="out of range"):
        b.process_native_host(nb.Resampler(4), np.zeros((1, 1, 480), np.float32), streams=[4])


@pytest.mark.parametrize("rate", [8000, 12000, 16000, 24000, 32000])
def test_round_trip_of_tones(rate):
    """down(up(x)) without the denoiser: the tones come back, shifted by the reported delay (20 native samples)."""
    n, T = rate // 100, 40
    t = np.arange(T * n) / rate
    x = sum(np.sin(2 * np.pi * f * rate * t + k) for k, f in enumerate((0.05, 0.13, 0.22, 0.31, 0.38))) * 3000.0
    rs = nb.Resampler(1, [rate])
    slots = np.zeros((1, T, 480), np.float32)
    slots[0, :, :n] = x.reshape(T, n)
    y = down(rs, up(rs, slots))[0, :, :n].reshape(-1).astype(np.float64)
    d = nb.resampler_delay(rate) * rate / 48000.0
    assert d == int(d)
    d = int(d)
    a, b = x[4 * n: len(x) - d], y[4 * n + d:]
    snr = 10 * np.log10((a ** 2).sum() / ((a - b) ** 2).sum())
    print("rate %d: round trip %.1f dB" % (rate, snr))
    assert snr >= 40.0


def test_testing_raw_end_to_end(testing_raw):
    """testing.raw at 16 kHz through process_native_host, against the float64 restatement of the stages around the 48 kHz
    GPU path.  The two differ where float and double resampling differ, amplified by the denoiser."""
    x48 = testing_raw.reshape(-1).astype(np.float64)
    x16 = resample_poly(x48, 1, 3)
    T = len(x16) // 160
    x16 = x16[: T * 160].astype(np.float32)
    slots = np.zeros((T, 1, 480), np.float32)
    slots[:, 0, :160] = x16.reshape(T, 160)
    out, vad = nb.DenoiseBatch(1).process_native_host(nb.Resampler(1, [16000]), slots)
    assert not np.any(out[:, 0, 160:])
    got = out[:, 0, :160].reshape(-1).astype(np.float64)
    assert np.all(np.isfinite(got)) and np.abs(got).max() <= 32768.0
    assert np.all((vad >= 0) & (vad <= 1))
    y48 = stream(16000, 0, x16).astype(np.float32).reshape(T, 1, 480)
    d48, _ = nb.DenoiseBatch(1).process_host(y48)
    ref = stream(16000, 1, d48.reshape(-1))
    rel = float(np.sqrt(((got - ref) ** 2).sum() / (ref ** 2).sum()))
    print("testing.raw at 16 kHz: rel rms %.3g against the float64 stages, %d frames" % (rel, T))
    assert rel <= 2e-2
