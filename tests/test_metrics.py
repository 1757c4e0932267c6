"""The metrics kernel (metrics.cu) and the evaluation driver on the GPU (DESIGN.md 7p).

- From the kernel's own inputs: per-frame band energies (read after one-frame calls) lie within the per-band bound of
  float64 (metrics_ref.band_yardstick), as the analysis kernel's `ex` for the same 960 samples does; counts match the float64 restatement (tests/metrics_ref.py) exactly, the time-
  domain sums within 1e-12 relative, the log-domain sums (computed from the GPU's own band energies) within 1e-12.
- Split invariance: calls of 1, 7 and 64 frames give byte-identical records; clear on a subset.
- Alignment with the denoiser at atten_lim_db = 0 (noise_gain = 0): near-exact, and far worse when shifted by a frame.
- End to end: evaluate against a hand-written loop, repeated and permuted variants, two geometries, reruns.
- Refusals change nothing."""
import os

import numpy as np
import pytest

import nnnoiseless_b200 as nb
from metrics_ref import MetricsRef, band_excess, band_yardstick, share
from nnnoiseless_b200 import NnnoiselessError
from nnnoiseless_b200 import evaluate as ev
from nnnoiseless_b200 import metrics as mt
from nnnoiseless_b200 import training as tr
from test_training_pool import corpus  # noqa: F401  (the module-scoped WAV fixture)
from test_metrics_cpu import other_geometry
from test_training_waves import new_trainer, run_waves

pytestmark = pytest.mark.gpu
F = 480
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIME = ("ec", "ey", "ed")
LOG = ("seg_snr", "lsd", "speech_dev", "noise_level")


def frames(B, T, seed):
    """clean and out [B][T][480] float32 mixing speech-like noise, all-zero clean, y == c (delayed), scaled copies,
    full-scale int16-range values and tiny values; targets in {0, 0.5, 1} and network vads including 0.5."""
    rng = np.random.default_rng(seed)
    c = rng.normal(0, 2000, (B, T, F)).astype(np.float32)
    y = np.zeros_like(c)
    y[:, 1:] = c[:, :-1]
    kind = rng.integers(0, 6, (B, T))
    noise = rng.normal(0, 300, (B, T, F)).astype(np.float32)
    y = np.where((kind == 1)[..., None], np.float32(0.5) * y, y)
    y = np.where((kind == 2)[..., None], y + noise, y)
    c = np.where((kind == 3)[..., None], np.float32(0.0), c)
    full = np.round(rng.uniform(-32768, 32767, (B, T, F))).astype(np.float32)
    y = np.where((kind == 4)[..., None], full, y)
    tiny = (rng.normal(0, 1, (B, T, F)) * 1e-30).astype(np.float32)
    c = np.where((kind == 5)[..., None], tiny, c)
    y = np.where((kind == 5)[..., None], tiny[:, ::-1], y)
    tgt = rng.choice(np.array([0.0, 0.5, 1.0], np.float32), (B, T))
    vad = rng.choice(np.array([0.0, 0.3, 0.5, 0.7, 1.0], np.float32), (B, T))
    return np.ascontiguousarray(y), np.ascontiguousarray(c), tgt, vad


def run(m, y, c, tgt, vad, calls, torch, after_each=None):
    """Feed [B][T] arrays in calls of the given sizes; after_each(records) after every call."""
    B, T = y.shape[:2]
    dy, dc = torch.from_numpy(y).cuda(), torch.from_numpy(c).cuda()
    dt, dv = torch.from_numpy(tgt).cuda(), torch.from_numpy(vad).cuda()
    f0 = 0
    for n in calls:
        m.accumulate_device(dy[:, f0].data_ptr(), dc[:, f0].data_ptr(), n, T * F, F, dv[:, f0].data_ptr(), dt[:, f0].data_ptr(), T, 1)
        f0 += n
        if after_each is not None:
            after_each(m.records())
    assert f0 == T
    return m.records()


def calls_of(k, T):
    return [k] * (T // k) + ([T % k] if T % k else [])


def rel_close(a, b, scale=None, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.abs(b) if scale is None else scale
    return bool((np.abs(a - b) <= tol * np.maximum(s, 1e-300)).all() or np.array_equal(a, b))


@pytest.mark.parametrize("B", [1, 33, 130])
def test_kernel_against_the_restatement(B):
    import torch
    T = 64
    y, c, tgt, vad = frames(B, T, seed=B)
    per_frame = []
    one = run(nb.Metrics(B), y, c, tgt, vad, [1] * T, torch, after_each=lambda r: per_frame.append(r["last_bands"].copy()))
    for k in (7, 64):
        other = run(nb.Metrics(B), y, c, tgt, vad, calls_of(k, T), torch)
        assert one.tobytes() == other.tobytes(), k  # split invariance, byte for byte
    # the GPU's band energies of frame j are last_bands after call j (frame 0 is not counted)
    bands = [np.zeros((2, B, 22))] + [np.transpose(per_frame[j], (1, 0, 2)) for j in range(1, T)]
    ref = MetricsRef(B).accumulate(y, c, vad=vad, target=tgt, bands=bands)
    for k in ("frames", "vad_counts"):
        assert np.array_equal(one[k], ref[k]), k
    for k in TIME:
        assert rel_close(one[k], ref[k]), k
    absprod = np.zeros((B, 3))
    for s in range(B):
        for q in range(3):
            absprod[s, q] = ref["ec"][s, q] + ref["ey"][s, q]  # bounds sum |c y|
    assert rel_close(one["ecy"], ref["ecy"], scale=absprod)
    for k in LOG:
        scale = np.abs(ref[k]) + (one["frames"][:, 1:2] if k != "noise_level" else one["frames"][:, 2:3])
        assert rel_close(one[k], ref[k], scale=scale.reshape(ref[k].shape[0], -1) if ref[k].ndim > 1 else scale[:, 0]), k
    # the band energies of every counted frame against float64, per band (metrics_ref.band_yardstick)
    cpad = np.concatenate([np.zeros((B, 2, F), np.float32), c], axis=1)  # clean frame j - 1 is cpad[:, j + 1]
    for k, prev, cur in ((0, y[:, :-1], y[:, 1:]), (1, cpad[:, 1:T], cpad[:, 2:T + 1])):
        e64, tol = band_yardstick(prev.reshape(-1, F), cur.reshape(-1, F))
        got = np.stack([per_frame[j][:, k] for j in range(1, T)], axis=1).reshape(-1, 22)
        sh = share(band_excess(got, e64), tol)
        assert (sh <= 1.0).all(), (k, np.argwhere(sh > 1.0)[:5], sh.max())


def test_band_energies_match_the_analysis_kernels_ex():
    """The same 960 samples through the analysis kernel (a DenoiseBatch frame: its window is input_mem[768:1728] of the
    state record after the frame) and through the metrics kernel, on synth_streams and the constructed streams of
    tests/metrics_cases.py: Yb, Cb and ex within the same per-band bound of float64."""
    from conftest import synth_streams
    import metrics_cases
    x = np.concatenate([synth_streams(37, 5, seed=11).reshape(37, 5, F), metrics_cases.cases()["y"][:, 3:8]])
    B = len(x)
    b = nb.DenoiseBatch(B)
    for f in range(5):  # one frame per call: the taps are those of the call's frame
        b.process_host(np.ascontiguousarray(x[:, f][None]))
    ex = b.spectral_taps()["ex"]
    rec = b.get_states().view(nb.state_dtype(b.gru_widths)).reshape(-1)
    w = rec["input_mem"][:, 768:1728].astype(np.float32)
    h0, h1 = w[:, :F], w[:, F:]
    z = np.zeros((B, F), np.float32)
    # frame 2 pairs output [h0 | h1] with clean [h0 | h1]
    out = np.ascontiguousarray(np.stack([z, h0, h1], axis=1))
    clean = np.ascontiguousarray(np.stack([h0, h1, z], axis=1))
    import torch
    m = nb.Metrics(B)
    dout, dclean = torch.from_numpy(out).cuda(), torch.from_numpy(clean).cuda()
    m.accumulate_device(dout.data_ptr(), dclean.data_ptr(), 3, 3 * F, F)
    lb = m.records()["last_bands"]
    # Not bit for bit: the two kernels' FMA contractions of the same FFT and band-sum source differ (first run on an
    # H100: up to 48 ulps in a quiet band, most bands within 4).  Both lie within the same per-band bound of float64.
    ref, tol = band_yardstick(h0, h1)
    ulps = np.abs(lb[:, 0].view(np.int32).astype(np.int64) - ex.view(np.int32).astype(np.int64))
    print("\nmetrics Yb against analysis ex: %d ulps at most, %.1f %% of bands equal" % (ulps.max(), 100.0 * (ulps == 0).mean()))
    worst = {}
    for name, got in (("ex", ex), ("Yb", lb[:, 0]), ("Cb", lb[:, 1])):
        sh = share(band_excess(got, ref), tol)
        worst[name] = sh.max()
        assert (sh <= 1.0).all(), (name, np.argwhere(sh > 1.0)[:5])
    print("largest share of the per-band bound: " + ", ".join("%s %.3f" % kv for kv in worst.items()))


def test_clear_subset_keeps_pairing_and_other_records():
    import torch
    B, T, cut = 33, 40, 17
    y, c, tgt, vad = frames(B, T, seed=5)
    a, b = nb.Metrics(B), nb.Metrics(B)
    sub = [0, 5, 32]
    run_part = lambda m, lo, hi: run(m, np.ascontiguousarray(y[:, lo:hi]), np.ascontiguousarray(c[:, lo:hi]),  # noqa: E731
                                     np.ascontiguousarray(tgt[:, lo:hi]), np.ascontiguousarray(vad[:, lo:hi]), [hi - lo], torch)
    run_part(a, 0, cut)
    run_part(b, 0, cut)
    before = a.records()
    a.clear(sub)
    after = a.records()
    others = np.setdiff1d(np.arange(B), sub)
    assert after[others].tobytes() == before[others].tobytes()
    assert not after[sub].tobytes().strip(b"\0")
    b.clear()  # a handle that starts counting at frame `cut` with the same pairing
    ra, rb = run_part(a, cut, T), run_part(b, cut, T)
    assert ra[sub].tobytes() == rb[sub].tobytes()


def _aligned_windows():
    """The §7k alignment setup: noise_gain = 0, so noisy is the speech and clean its high-passed copy."""
    L, T = 6, 60
    rng = np.random.default_rng(3)
    pool_len = 480 * (T + 1) + 2450 * L
    X = np.fft.rfft(rng.normal(0, 3000, pool_len))
    X[np.fft.rfftfreq(pool_len, 1 / 48000.0) > 15000] = 0
    pool = np.clip(np.round(np.fft.irfft(X, pool_len)), -32768, 32767).astype(np.int16)
    sig_at = (2450 * np.arange(L) + 7 * np.arange(L))[None, :] + 480 * np.arange(T)[:, None]
    prm = tr.randomize(L, rng)
    prm["noise_gain"] = 0.0
    prm["signal_gain"] = np.abs(prm["signal_gain"]) + 0.5
    noisy, clean, _, _ = run_waves(new_trainer(L, pool), sig_at, sig_at[::-1].copy(), [T], {0: prm})
    return noisy, clean


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
    tgt = torch.ones((L, T), device="cuda")
    dc = torch.from_numpy(clean).cuda()
    res = {}
    for name, o in (("aligned", out), ("shifted", torch.cat([out[:, 1:], out[:, -1:]], dim=1).contiguous())):
        m = nb.Metrics(L)
        m.accumulate_device(o.data_ptr(), dc.data_ptr(), 2, T * F, F, 0, tgt.data_ptr(), T, 1)
        m.clear()  # the onset frames
        m.accumulate_device(o[:, 2].data_ptr(), dc[:, 2].data_ptr(), T - 2, T * F, F, 0, tgt[:, 2].data_ptr(), T, 1)
        res[name] = mt.summarize(m.records())
    a, s = res["aligned"], res["shifted"]
    print("\naligned: LSD %s dB, segmental SNR %s dB; shifted: LSD %s, segmental SNR %s"
          % (np.round(a["lsd"], 4), np.round(a["seg_snr"], 2), np.round(s["lsd"], 3), np.round(s["seg_snr"], 2)))
    # first run on an H100: aligned LSD 0.003-0.078 dB and segmental SNR 35.0 (the cap) on every lane; shifted by a frame
    # LSD 2.40-2.61 dB and segmental SNR -2.4 dB
    assert (a["lsd"] < 0.2).all() and (a["seg_snr"] > 34.0).all()
    assert (s["lsd"] > 1.0).all() and (s["seg_snr"] < 5.0).all()


def _hand_loop(sig, noise, L, T, frames_, warmup, seed, models, limits):
    """evaluate's computation written out for one geometry: -> records per variant."""
    import torch
    wc = tr.WaveformCorpus(sig, noise, L)
    wc.start(L * (warmup + frames_), seed)
    specs = [("unprocessed", None, 0.0)] + [(mname, mobj, a) for mname, mobj in models for a in limits]
    V = len(specs)
    b = nb.DenoiseBatch(V * L)
    ids, k = [], {}
    for name, mobj, _ in specs:
        if name in ("unprocessed", "builtin"):
            ids.append(0)
        else:
            if name not in k:
                k[name] = b.add_model(mobj)
            ids.append(k[name])
    b.set_stream_models(np.repeat(ids, L).astype(np.int32))
    b.set_stream_controls(atten_lim_db=np.repeat([a for _, _, a in specs], L).astype(np.float32))
    m = nb.Metrics(V * L)
    noisy, clean = (torch.empty((L, T, F), device="cuda") for _ in range(2))
    vt = torch.empty((L, T), device="cuda")
    rep, out = (torch.empty((V, L, T, F), device="cuda") for _ in range(2))
    vad, tg = torch.empty((T, V * L), device="cuda"), torch.empty((T, V, L), device="cuda")
    done = 0
    for n in [warmup] + calls_of(T, frames_):
        wc.next(n, noisy.data_ptr(), clean.data_ptr(), T * F, F, vad_ptr=vt.data_ptr(), vad_stream_stride=T, vad_frame_stride=1)
        rep.copy_(noisy.unsqueeze(0).expand(V, L, T, F))
        b.process_device(out.data_ptr(), rep.data_ptr(), vad.data_ptr(), n, T * F, F)
        torch.cuda.synchronize()
        rep.copy_(clean.unsqueeze(0).expand(V, L, T, F))
        tg.copy_(vt.t().unsqueeze(1).expand(T, V, L))
        torch.cuda.synchronize()
        m.accumulate_device(out.data_ptr(), rep.data_ptr(), n, T * F, F, vad.data_ptr(), tg.data_ptr(), 1, V * L)
        done += n
        if done == warmup:
            m.clear()
    r = m.records()
    return [r[v * L:(v + 1) * L] for v in range(V)]


@pytest.fixture(scope="module")
def heldout(corpus, tmp_path_factory):  # noqa: F811
    """The pool fixture's corpus plus tests/golden/testing.raw written as a speech WAV."""
    sig, noise = corpus
    d = tmp_path_factory.mktemp("heldout")
    p = str(d / "testing.wav")
    pcm = np.fromfile(os.path.join(ROOT, "tests", "golden", "testing.raw"), dtype="<i2")
    from nnnoiseless_b200.files import write_audio
    write_audio(p, pcm, wav=True)
    return sig + [p], noise


def test_evaluate_end_to_end(heldout, tmp_path):
    sig, noise = heldout
    L, T, frames_, warmup, seed = 8, 50, 150, 40, 3
    sh = os.path.join(ROOT, "tests", "golden", "sh.rnnn")  # the built-in model's geometry: an added model of its batch
    gen = other_geometry(tmp_path / "small.rnn")  # a batch of its own
    rep = ev.evaluate(sig, noise, ["builtin", gen, sh], [np.inf, 12.0], L, frames_, seed=seed, window=T, warmup_frames=warmup)
    names = [v["name"] for v in rep["variants"]]
    assert names == ["unprocessed"] + ["%s@%s" % (m, a) for m in ("builtin", gen, sh) for a in ("inf", "12")]
    assert len(rep["batches"]) == 2 and rep["batches"][1]["variants"] == [gen + "@inf", gen + "@12"]
    # the built-in geometry's variants equal a hand-written loop bit for bit
    hand = _hand_loop(sig, noise, L, T, frames_, warmup, seed, [("builtin", None)], [np.inf, 12.0])
    for v in range(3):
        assert rep["variants"][v]["records"].tobytes() == hand[v].tobytes(), names[v]
    # reruns, a repeated variant and a permutation
    rep2 = ev.evaluate(sig, noise, [sh, gen, "builtin", "builtin"], [12.0, np.inf], L, frames_, seed=seed, window=T,
                       warmup_frames=warmup)
    by = {v["name"]: v["records"].tobytes() for v in rep2["variants"]}
    for v in rep["variants"]:
        assert by[v["name"]] == v["records"].tobytes(), v["name"]
    assert rep2["variants"][5]["records"].tobytes() == rep2["variants"][7]["records"].tobytes()
    print("\n" + ev.format_table(rep))
    # on real speech (testing.raw; the fixture's speech files are tone-and-noise bursts) the built-in model gains
    rep3 = ev.evaluate(sig[-1:], noise, ["builtin"], [np.inf], L, frames_, seed=seed, window=T, warmup_frames=warmup)
    f = rep3["variants"][1]["figures"]
    print("built-in model on testing.raw against the unprocessed mix: delta SI-SDR %.2f +- %.2f dB, noise attenuation "
          "%.2f +- %.2f dB" % (f["delta_si_sdr"]["mean"], f["delta_si_sdr"]["ci95"], f["noise_atten"]["mean"], f["noise_atten"]["ci95"]))
    print(ev.format_table(rep3))
    assert f["delta_si_sdr"]["mean"] > 0 and f["noise_atten"]["mean"] > 0


def test_evaluate_refuses_what_the_device_cannot_hold(heldout):
    sig, noise = heldout
    with pytest.raises(NnnoiselessError, match="MB of device memory"):
        ev.evaluate(sig, noise, ["builtin"], [np.inf], 1 << 16, 100, window=1 << 14)


def test_refusals_change_nothing():
    import torch
    B, T = 5, 6
    y, c, tgt, vad = frames(B, T, seed=9)
    m = nb.Metrics(B)
    dy, dc = torch.from_numpy(y).cuda(), torch.from_numpy(c).cuda()
    with pytest.raises(NnnoiselessError, match="overlap"):
        m.accumulate_device(dy.data_ptr(), dc.data_ptr(), T, F, F)  # stream rows overlap frames
    with pytest.raises(NnnoiselessError, match="overlap"):
        m.accumulate_device(dy.data_ptr(), dc.data_ptr(), T, T * F, F, torch.zeros(B * T, device="cuda").data_ptr(), 0, 1, 1)
    with pytest.raises(NnnoiselessError, match="out of range"):
        m.clear([5])
    with pytest.raises(NnnoiselessError, match="twice"):
        m.records([1, 1])
    with pytest.raises(NnnoiselessError, match="negative"):
        m.accumulate_device(dy.data_ptr(), dc.data_ptr(), -1, T * F, F)
    fresh = nb.Metrics(B)
    for h in (m, fresh):
        h.accumulate_device(dy.data_ptr(), dc.data_ptr(), T, T * F, F)
    assert m.records().tobytes() == fresh.records().tobytes()
