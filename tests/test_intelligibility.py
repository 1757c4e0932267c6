"""The STOI / ESTOI kernels (intelligibility.cu) and evaluate's intelligibility option on the GPU (DESIGN.md 7q).

Each stage is checked from the GPU's own inputs to it, read through the workspace taps:
- 10 kHz samples within gamma_P sum |h| |x| of float64 (P: the taps of a phase); bit-equal at 10 kHz;
- the kept list equal to the float64 decision on the GPU's own clean x10;
- every band within 16 * 9 * u32 * sqrt(512) * ||frame|| + gamma_45 B + u B of float64 from the GPU's x10 and kept list;
- STOI and ESTOI within 1e-12 of the float64 tail from the GPU's own bands;
- end to end within 1e-4 of the float64 definition, on clips with no frame within 1e-3 dB of the threshold.
Then invariances (power-of-two scaling, row permutation, a grid of 2 x SMs x 64 + 37 pairs), alignment with the
denoiser, and evaluate against a hand-written loop."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import stoi_ref as sr
from nnnoiseless_b200 import evaluate as ev
from nnnoiseless_b200 import training as tr
from test_intelligibility_cpu import speech_like
from test_metrics import _aligned_windows, calls_of, heldout  # noqa: F401  (heldout: the module-scoped corpus fixture)
from test_training_pool import corpus  # noqa: F401

pytestmark = pytest.mark.gpu
F = 480
SHARES = {}


def run(y, x, rate, pad=0):
    """One call on rows y (out) and x (clean) [B][n] -> (records, x10 [2][B][n10], kept [B][F], bands [2][B][15][maxM])."""
    import torch
    B, n = x.shape
    w = max(n + pad, 1)  # an empty tensor has no data pointer, and a null one is refused
    dy = torch.zeros((B, w), dtype=torch.float32)
    dx = torch.zeros((B, w), dtype=torch.float32)
    dy[:, :n] = torch.from_numpy(np.ascontiguousarray(y, np.float32))
    dx[:, :n] = torch.from_numpy(np.ascontiguousarray(x, np.float32))
    dy, dx = dy.cuda(), dx.cuda()
    nbytes = nb.intelligibility_workspace_bytes(B, n, rate)
    ws = torch.full((nbytes,), 0x7F, dtype=torch.uint8, device="cuda")
    res = torch.full((B * 32,), 0x7F, dtype=torch.uint8, device="cuda")
    before = nb.kernel_launches()
    nb.intelligibility_device(dy.data_ptr(), dx.data_ptr(), B, n, w, rate, res.data_ptr(), ws.data_ptr(), nbytes)
    assert nb.kernel_launches() - before == 4
    rec = res.cpu().numpy().view(nb.INTELLIGIBILITY_DTYPE).copy()
    return (rec,) + tuple(t.cpu().numpy().copy() for t in nb.intelligibility_taps(ws, B, n, rate))


def check_call(name, y, x, rate, pad=0, e2e=True):
    """Every stage of one call from its own inputs; returns the records."""
    rec, x10, kept, bands = run(y, x, rate, pad)
    B, n = x.shape
    up, down, half, n10, Fr = sr.sizes(n, rate)
    h = sr.filter_taps(rate)
    P = 1 if h is None else -(-len(h) // up)
    u = sr.U32
    share = SHARES.setdefault(name, dict(x10=0.0, bands=0.0, e2e=0.0, near_db=np.inf))
    assert (rec["reserved"] == 0).all() and (rec["frames"] == Fr).all()
    for p in range(B):
        r64 = []
        for s, sig in enumerate((x[p], y[p])):
            g = x10[s, p]
            r64.append(sr.resample(sig, rate, h))
            if h is None:
                assert np.array_equal(g.view(np.uint32), np.asarray(sig, np.float32).view(np.uint32)), (name, p)
                continue
            ref = r64[-1]
            bound = sr.gamma(P) * sr.resample(sig, rate, h, absolute=True)
            err = np.abs(g - ref)
            assert (err <= bound).all(), (name, p, s, float((err - bound).max()))
            if bound.size and bound.max() > 0:
                share["x10"] = max(share["x10"], float((err / np.where(bound > 0, bound, np.inf)).max()))
        # the kept list from the GPU's own clean x10
        want = sr.kept_frames(x10[0, p].astype(np.float64))
        K = len(want)
        assert rec["kept"][p] == K and np.array_equal(kept[p, :K], want) and (kept[p, K:] == -1).all(), (name, p)
        e = sr.frame_db(x10[0, p].astype(np.float64))
        if len(e):
            share["near_db"] = min(share["near_db"], float(np.abs(e - (e.max() - 40.0)).min()))
        M = max(K - 1, 0)
        assert rec["segments"][p] == max(M - 29, 0)
        # bands from the GPU's own x10 and kept list
        for s in range(2):
            fr = sr.stft_frames(x10[s, p].astype(np.float64), want)
            ref = sr.bands_of_frames(fr)
            got = bands[s, p][:, :M].astype(np.float64)
            bound = 16 * 9 * u * np.sqrt(512) * np.sqrt((fr * fr).sum(axis=1))[None, :] + (sr.gamma(45) + u) * ref
            err = np.abs(got - ref)
            assert (err <= bound).all(), (name, p, s, float((err - bound).max()))
            if M:
                share["bands"] = max(share["bands"], float((err / np.where(bound > 0, bound, np.inf)).max()))
        # the double tail from the GPU's own bands
        st, es, S = sr.score(bands[0, p][:, :M], bands[1, p][:, :M])
        assert S == rec["segments"][p]
        if S:
            assert abs(rec["stoi"][p] - st) <= 1e-12 and abs(rec["estoi"][p] - es) <= 1e-12, (name, p, rec[p], st, es)
        else:
            assert np.isnan(rec["stoi"][p]) and np.isnan(rec["estoi"][p])
        if e2e and S:
            # the whole definition in float64 (bands rounded to float, as specified)
            e64 = sr.frame_db(r64[0])
            if np.abs(e64 - (e64.max() - 40.0)).min() >= 1e-3:
                k64 = sr.kept_frames(r64[0])
                st64, es64, _ = sr.score(sr.bands(r64[0], k64).astype(np.float32), sr.bands(r64[1], k64).astype(np.float32))
                d = max(abs(rec["stoi"][p] - st64), abs(rec["estoi"][p] - es64))
                assert d <= 1e-4, (name, p, d)
                share["e2e"] = max(share["e2e"], d)
    return rec


def noisy_pairs(B, n, rate, seed, scale=3000.0):
    rng = np.random.default_rng(seed)
    x = np.stack([speech_like(n, seed * 1000 + p, scale, rate) for p in range(B)])
    snr = rng.uniform(-10, 20, (B, 1))
    px = np.mean(x.astype(np.float64) ** 2, axis=1, keepdims=True) + 1e-30
    y = (x + rng.normal(0, 1, x.shape) * np.sqrt(px / 10 ** (snr / 10))).astype(np.float32)
    return y, x


@pytest.mark.parametrize("B,rate", [(1, 48000), (130, 16000), (33, 44100), (33, 10000)])
def test_speech_like_clips(B, rate):
    # n from empty through the 29 / 30 STFT-frame edge to 3 s (2 s at 44.1 kHz, whose float64 resampling is slow)
    for n in (0, 100, rate * 3 // 10, 256 * rate // 10000 + 31 * 128 * rate // 10000, rate * (2 if rate == 44100 else 3)):
        y, x = noisy_pairs(B, n, rate, seed=n + B)
        check_call("speech %d Hz" % rate, y, x, rate, pad=37 if B == 33 else 0)


def tones(n, rate, bins, levels):
    t = np.arange(n) / rate
    return sum(a * np.sin(2 * np.pi * k * 10000.0 / 512 * t + k) for k, a in zip(bins, levels)).astype(np.float32)


@pytest.mark.parametrize("rate", [48000, 44100, 16000, 10000])
def test_tones_on_band_edges_and_one_loud_band(rate):
    n = 12 * rate // 10
    rows_x, rows_y = [], []
    for b in range(15):
        lo, hi = sr.EDGES[b], sr.EDGES[b + 1]
        edge = [lo - 0.5, lo, hi - 1, hi - 0.5]  # on and between the band's edge bins
        rows_x.append(tones(n, rate, edge, [3000.0] * 4))
        rows_y.append(tones(n, rate, edge, [3000.0, 1500.0, 700.0, 300.0]))
        # one band loud, every other band 60 dB down, with a slow envelope so the correlations are not rounding noise
        others = [(sr.EDGES[c] + sr.EDGES[c + 1]) / 2 for c in range(15) if c != b]
        env = (1.2 + np.sin(2 * np.pi * 2.3 * np.arange(n) / rate)).astype(np.float32)
        loud = tones(n, rate, [(lo + hi) / 2], [10000.0])
        quiet = tones(n, rate, others, [10.0] * len(others))
        rows_x.append(env * (loud + quiet))
        rows_y.append(loud + env * quiet)
    check_call("tones %d Hz" % rate, np.stack(rows_y), np.stack(rows_x), rate, e2e=False)


def near_threshold_clip(n, deltas, seed):
    """10 kHz rows (x10 = x exactly): a loud noise burst, silence, and copies of the burst scaled by 10^((-40 + d) / 20),
    so the copy's loudest frame lies d dB from the 40 dB threshold (up to the float rounding of the scaled samples)."""
    rng = np.random.default_rng(seed)
    rows = []
    burst = rng.normal(0, 8000, 2048)
    for d in deltas:
        x = np.zeros(n)
        x[1024:1024 + 2048] = burst
        for k, start in enumerate(range(8192, n - 2048, 6144)):
            x[start:start + 2048] = burst * 10 ** ((-40.0 + d * (k + 1)) / 20.0)
        rows.append(x.astype(np.float32))
    return np.stack(rows)


def test_silences_and_the_threshold():
    n = 60000
    x = near_threshold_clip(n, [1e-6, -1e-6, 3e-7, -3e-7, 0.0], seed=4)
    y = (x + np.random.default_rng(1).normal(0, 50, x.shape)).astype(np.float32)
    check_call("threshold 10 kHz", y, x, 10000, e2e=False)
    print("\nnearest frame to the threshold: %.3g dB" % SHARES["threshold 10 kHz"]["near_db"])
    # the same clips at 48 kHz: long silences between bursts
    x48 = np.repeat(x, 5, axis=1)[:, :48000 * 5]
    y48 = np.repeat(y, 5, axis=1)[:, :48000 * 5]
    check_call("silences 48 kHz", y48, x48, 48000, e2e=False)


def test_amplitudes():
    n = 3 * 48000
    y, x = noisy_pairs(8, n, 48000, seed=9, scale=1.0)
    # 1e-9 and 1e-12 put the band rows' and segments' norms under EPS, where EPS is added matters
    scales = np.array([1 / 32768, 1 / 32768, 32767.0, 32767.0, 0.0, 0.0, 1e-12, 1e-9])[:, None]
    x = (x / np.abs(x).max(axis=1, keepdims=True) * scales).astype(np.float32)
    y = (y / np.abs(y).max(axis=1, keepdims=True) * scales[::-1]).astype(np.float32)
    rec = check_call("amplitudes", y, x, 48000, e2e=False)
    assert (rec["kept"][4:6] == rec["frames"][4:6]).all()  # an all-zero clean signal keeps every frame


def test_power_of_two_scaling_permutation_and_grid():
    import torch
    n = 3 * 48000
    y, x = noisy_pairs(8, n, 48000, seed=21)
    a = run(y, x, 48000)[0]
    assert run(y * np.float32(0.5), x, 48000)[0].tobytes() == a.tobytes()
    assert run(x * np.float32(0.5), x, 48000)[0].tobytes() == run(x, x, 48000)[0].tobytes()
    perm = np.random.default_rng(2).permutation(8)
    assert run(y[perm], x[perm], 48000)[0].tobytes() == a[perm].tobytes()
    # 2 x SMs x 64 + 37 pairs of 0.6 s, rows drawn from 37 distinct ones, equal the call on those 37
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    Bb, nn, k = 2 * sms * 64 + 37, 28800, 37
    rng = np.random.default_rng(5)  # steady noise under a shallow envelope: every frame is kept, so S = 15
    xs = (rng.normal(0, 3000, (k, nn)) * (1.0 + 0.5 * np.sin(2 * np.pi * 3.0 * np.arange(nn) / 48000 + rng.uniform(0, 6, (k, 1)))))
    xs = xs.astype(np.float32)
    ys = (xs + rng.normal(0, 2000, xs.shape)).astype(np.float32)
    small = run(ys, xs, 48000)[0]
    assert (small["segments"] > 0).all()
    idx = torch.arange(Bb, device="cuda") % k
    dy, dx = torch.from_numpy(ys).cuda()[idx].contiguous(), torch.from_numpy(xs).cuda()[idx].contiguous()
    nbytes = nb.intelligibility_workspace_bytes(Bb, nn, 48000)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    res = torch.empty(Bb * 32, dtype=torch.uint8, device="cuda")
    nb.intelligibility_device(dy.data_ptr(), dx.data_ptr(), Bb, nn, nn, 48000, res.data_ptr(), ws.data_ptr(), nbytes,
                              cuda_stream=torch.cuda.current_stream().cuda_stream)
    big = res.cpu().numpy().view(nb.INTELLIGIBILITY_DTYPE)
    assert big.tobytes() == small[np.arange(Bb) % k].tobytes()
    assert nb.intelligibility(dy[:k], dx[:k]).tobytes() == small.tobytes()


def test_alignment_with_the_denoiser():
    import torch
    noisy, clean = _aligned_windows()
    L, T = noisy.shape[:2]
    b = nb.DenoiseBatch(L)
    b.set_stream_controls(atten_lim_db=0.0)
    dn = torch.from_numpy(noisy).cuda()
    out = torch.empty_like(dn)
    b.process_device(out.data_ptr(), dn.data_ptr(), 0, T, T * F, F)
    torch.cuda.synchronize()
    dc = torch.from_numpy(clean).cuda()
    aligned = nb.intelligibility(out[:, 1:].reshape(L, -1).contiguous(), dc[:, :-1].reshape(L, -1).contiguous())
    shifted = nb.intelligibility(out[:, 2:].reshape(L, -1).contiguous(), dc[:, :-2].reshape(L, -1).contiguous())
    print("\naligned STOI %s ESTOI %s; one frame late: STOI %s" % (np.round(aligned["stoi"], 5), np.round(aligned["estoi"], 5),
                                                                   np.round(shifted["stoi"], 4)))
    assert (aligned["segments"] > 0).all() and (aligned["stoi"] >= 0.999).all()


def _hand_stoi(sig, noise, L, T, frames_, warmup, seed, limits):
    """evaluate's intelligibility scoring written out for the built-in model at the given limits: -> [V][windows][L]."""
    import torch
    wc = tr.WaveformCorpus(sig, noise, L)
    wc.start(L * (warmup + frames_), seed)
    lims = [0.0] + list(limits)
    V = len(lims)
    b = nb.DenoiseBatch(V * L)
    b.set_stream_controls(atten_lim_db=np.repeat(lims, L).astype(np.float32))
    noisy, clean = (torch.empty((L, T, F), device="cuda") for _ in range(2))
    vt = torch.empty((L, T), device="cuda")
    rep, out = (torch.empty((V, L, T, F), device="cuda") for _ in range(2))
    vad = torch.empty((T, V * L), device="cuda")
    nbytes = nb.intelligibility_workspace_bytes(V * L, (T - 1) * F, 48000)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    recs = []
    for k, n in enumerate([warmup] + calls_of(T, frames_)):
        wc.next(n, noisy.data_ptr(), clean.data_ptr(), T * F, F, vad_ptr=vt.data_ptr(), vad_stream_stride=T, vad_frame_stride=1)
        rep.copy_(noisy.unsqueeze(0).expand(V, L, T, F))
        b.process_device(out.data_ptr(), rep.data_ptr(), vad.data_ptr(), n, T * F, F)
        torch.cuda.synchronize()
        rep.copy_(clean.unsqueeze(0).expand(V, L, T, F))
        torch.cuda.synchronize()
        if k > 0 and n > 1:
            res = torch.empty(V * L * 32, dtype=torch.uint8, device="cuda")
            nb.intelligibility_device(out.data_ptr() + 4 * F, rep.data_ptr(), V * L, (n - 1) * F, T * F, 48000, res.data_ptr(), ws.data_ptr(),
                                      nbytes)
            recs.append(res.cpu().numpy().view(nb.INTELLIGIBILITY_DTYPE).reshape(V, L))
    return np.stack(recs, axis=1)


def test_evaluate_with_intelligibility(heldout):  # noqa: F811
    sig, noise = heldout
    L, T, frames_, warmup, seed = 8, 100, 250, 40, 3
    rep = ev.evaluate(sig, noise, ["builtin"], [np.inf, 12.0], L, frames_, seed=seed, window=T, warmup_frames=warmup, intelligibility=True)
    hand = _hand_stoi(sig, noise, L, T, frames_, warmup, seed, [np.inf, 12.0])
    plain = ev.evaluate(sig, noise, ["builtin"], [np.inf, 12.0], L, frames_, seed=seed, window=T, warmup_frames=warmup)
    for v, var in enumerate(rep["variants"]):
        assert var["intelligibility"].tobytes() == hand[v].tobytes(), var["name"]
        assert var["records"].tobytes() == plain["variants"][v]["records"].tobytes()
        assert "intelligibility" not in plain["variants"][v] and "stoi" not in plain["variants"][v]["figures"]
        for k in ("stoi", "estoi"):
            x = hand[v][k].astype(np.float64)
            ok = np.isfinite(x)
            lane = np.array([x[ok[:, l], l].mean() if ok[:, l].any() else np.nan for l in range(L)])
            xb = hand[0][k].astype(np.float64)
            okb = np.isfinite(xb)
            lane_b = np.array([xb[okb[:, l], l].mean() if okb[:, l].any() else np.nan for l in range(L)])
            f, d = var["figures"][k], var["figures"]["delta_" + k]
            good = np.isfinite(lane)
            assert f["lanes"] == good.sum() and f["windows"] == ok.sum() and f["nan_windows"] == (~ok).sum()
            assert np.isclose(f["mean"], lane[good].mean(), rtol=0, atol=1e-14)
            assert np.isclose(d["mean"], np.nanmean(lane - lane_b), rtol=0, atol=1e-14)
    assert "stoi" in ev.format_table(rep) and "stoi" not in ev.format_table(plain)
    print("\n" + ev.format_table(rep))
    # the golden speech (testing.raw) with the pool fixture's noise: the built-in model against the unprocessed mix
    g = ev.evaluate(sig[-1:], noise, ["builtin"], [np.inf], L, frames_, seed=seed, window=T, warmup_frames=warmup, intelligibility=True)
    f = g["variants"][1]["figures"]
    print("built-in model on testing.raw against the unprocessed mix: delta STOI %.4f +- %.4f, delta ESTOI %.4f +- %.4f "
          "(%d windows scored, %d NaN)" % (f["delta_stoi"]["mean"], f["delta_stoi"]["ci95"], f["delta_estoi"]["mean"],
                                          f["delta_estoi"]["ci95"], f["stoi"]["windows"], f["stoi"]["nan_windows"]))


def test_refusals_change_nothing():
    import torch
    y, x = noisy_pairs(3, 48000, 48000, seed=3)
    dy, dx = torch.from_numpy(y).cuda(), torch.from_numpy(x).cuda()
    nbytes = nb.intelligibility_workspace_bytes(3, 48000, 48000)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    res = torch.zeros(96, dtype=torch.uint8, device="cuda")
    for kw in (dict(stream_stride=47999), dict(workspace_bytes=nbytes - 1), dict(rate=48100), dict(n_pairs=0)):
        a = dict(out_ptr=dy.data_ptr(), clean_ptr=dx.data_ptr(), n_pairs=3, n_samples=48000, stream_stride=48000, rate=48000,
                 result_ptr=res.data_ptr(), workspace_ptr=ws.data_ptr(), workspace_bytes=nbytes)
        a.update(kw)
        with pytest.raises(nb.NnnoiselessError):
            nb.intelligibility_device(**a)
    torch.cuda.synchronize()
    assert not ws.any() and not res.any()


def test_report_shares():
    """Prints the largest share of each bound seen by the stage tests of this module (run after them)."""
    for k, v in SHARES.items():
        print("\n%-20s x10 %.3f  bands %.3f  end to end %.2g  nearest frame to the threshold %.3g dB" % (k, v["x10"], v["bands"], v["e2e"],
                                                                                                        v["near_db"]), end="")
