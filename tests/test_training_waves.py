"""Waveform windows from the training simulators (rnnoise_train_waves_device, WaveformCorpus; DESIGN.md §7k).

The kernel against a numpy restatement of train_front_kernel's statements without the combined stream's high-pass, bit for
bit; the corpus path against generate_rows (the features of `noisy` through a DenoiseBatch equal the rows' features);
the alignment of `clean` with the denoiser's output; a GRU trained through synthesis on corpus windows; refusals."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import NnnoiselessError
from nnnoiseless_b200 import training as tr
from train_ref import F32, HP_A, HP_B, biquad, default_params, frame_energy
from test_training_pool import _offsets, _pool, corpus  # noqa: F401  (corpus: the module-scoped WAV fixture)

pytestmark = pytest.mark.gpu
F, NBF, NBB = 480, 42, 22


def bits(x):
    import torch
    if isinstance(x, torch.Tensor):
        x = x.cpu().numpy()
    return np.ascontiguousarray(x).view(np.uint32)


class WaveRef:
    """train_front_kernel's per-sample statements (train_ref.FrontRef's order and precision) minus the combined
    stream's high-pass: -> noisy z, clean hp(s), noise hp(n), vad per frame."""

    def __init__(self, L):
        self.L = L
        self.params = default_params(L)
        self.resp_mem = np.zeros((L, 4), F32)
        self.vad_count = np.zeros(L, np.int32)
        self.hp = np.zeros((2, L, 2), F32)

    def frames(self, pool, sig_at, noise_at):
        """sig_at, noise_at [T][L] -> (noisy, clean, noise) [L][T][480], vad [L][T]."""
        T, L = sig_at.shape
        out = np.zeros((3, L, T, F), F32)
        vad = np.zeros((L, T), F32)
        a = np.broadcast_to(np.array(HP_A, F32), (L, 2))
        b = np.broadcast_to(np.array(HP_B, F32), (L, 2))
        p = self.params
        for t in range(T):
            raw = []
            for at in (sig_at[t], noise_at[t]):
                x = pool[np.maximum(at, 0)[:, None] + np.arange(F)].astype(F32)
                x[at < 0] = 0.0
                raw.append(x)
            with np.errstate(over="ignore", invalid="ignore"):
                energy = frame_energy(raw[0])
                s = biquad(raw[0] * p["signal_gain"][:, None], p["sig_a"], p["sig_b"], self.resp_mem[:, 0:2])
                n = biquad(raw[1] * p["noise_gain"][:, None], p["noise_a"], p["noise_b"], self.resp_mem[:, 2:4])
                out[0, :, t] = s + n
                out[1, :, t] = biquad(s, a, b, self.hp[0])
                out[2, :, t] = biquad(n, a, b, self.hp[1])
            vc = self.vad_count.astype(np.int64)
            vc = np.where(energy > F32(1e9), 0, np.where(energy > F32(1e8), vc - 5, np.where(energy > F32(1e7), vc + 1, vc + 2)))
            self.vad_count = np.clip(vc, 0, 15).astype(np.int32)
            vad[:, t] = np.where(self.vad_count >= 10, F32(0.0), np.where(self.vad_count > 0, F32(0.5), F32(1.0)))
        return out[0], out[1], out[2], vad


def new_trainer(L, pool):
    t = tr.TrainingBatch(L)
    t.pool_reserve(len(pool))
    t.pool_write(0, pool[:len(pool) // 2])  # in two pieces
    t.pool_write(len(pool) // 2, pool[len(pool) // 2:])
    return t


def run_waves(t, sig_at, noise_at, calls, params=None, with_noise=True, with_vad=True, stream_stride=None):
    """calls: frame counts of consecutive calls; params {call index: params set before it} -> numpy outputs
    (noisy, clean, noise, vad) [L][T][..] (noise / vad None when not requested).  stream_stride (elements) defaults to a
    batch-first [L][T][480] layout; another value lays lane l's frames out from l * stream_stride."""
    import torch
    T, L = sig_at.shape
    ss = T * F if stream_stride is None else stream_stride
    bufs = [torch.full((L * ss + 16,), float("nan"), device="cuda") for _ in range(3)]
    vad = torch.full((L, T), float("nan"), device="cuda")
    f0 = 0
    for k, n in enumerate(calls):
        if params and k in params:
            t.set_params(params[k])
        d = 4 * f0 * F
        t.waves_device(sig_at[f0:f0 + n], noise_at[f0:f0 + n], bufs[0].data_ptr() + d, bufs[1].data_ptr() + d, ss, F,
                       bufs[2].data_ptr() + d if with_noise else None, vad[:, f0].data_ptr() if with_vad else None, T, 1)
        f0 += n
    torch.cuda.synchronize()
    got = [x[:L * ss].view(L, ss)[:, :T * F].reshape(L, T, F).cpu().numpy() for x in bufs]
    return got[0], got[1], got[2] if with_noise else None, vad.cpu().numpy() if with_vad else None


# ---- 1. the kernel against the restatement, bit for bit ---------------------------------------------------------------------
@pytest.mark.parametrize("L", [1, 63, 64, 65, 130])
def test_waves_equal_the_restatement(L):
    rng = np.random.default_rng(100 + L)
    T, pool_len = 48, 480 * 41 + 5
    pool = _pool(pool_len, L)
    sig_at, noise_at = _offsets(rng, T, L, pool_len), _offsets(rng, T, L, pool_len)
    p1, p2 = tr.randomize(L, rng), tr.randomize(L, rng)
    p2["noise_gain"][0] = 0.0
    p2["signal_gain"][-1] = 0.0
    calls, params = [1, 7, 40], {1: p1, 2: p2}  # T = 1, 7, 40 per call; the parameters change between calls
    got = run_waves(new_trainer(L, pool), sig_at, noise_at, calls, params)
    ref = WaveRef(L)
    want, f0 = [], 0
    for k, n in enumerate(calls):
        if k in params:
            ref.params[:] = params[k]
        want.append(ref.frames(pool, sig_at[f0:f0 + n], noise_at[f0:f0 + n]))
        f0 += n
    for i, name in enumerate(("noisy", "clean", "noise", "vad")):
        w = np.concatenate([x[i] for x in want], axis=1)
        assert np.array_equal(bits(got[i]), bits(w)), name
    assert set(np.unique(got[3])) <= {0.0, 0.5, 1.0} and len(np.unique(got[3])) > 1


def test_one_call_equals_split_calls():
    L, T = 65, 12
    rng = np.random.default_rng(7)
    pool_len = 480 * 30 + 1
    pool = _pool(pool_len, 7)
    sig_at, noise_at = _offsets(rng, T, L, pool_len), _offsets(rng, T, L, pool_len)
    prm = {0: tr.randomize(L, rng)}
    runs = [run_waves(new_trainer(L, pool), sig_at, noise_at, c, prm) for c in ([T], [1, T - 1], [1] * T)]
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert np.array_equal(bits(a), bits(b))


def test_optional_outputs_and_layouts_leave_noisy_and_clean():
    L, T = 70, 9
    rng = np.random.default_rng(11)
    pool_len = 480 * 25 + 3
    pool = _pool(pool_len, 11)
    sig_at, noise_at = _offsets(rng, T, L, pool_len), _offsets(rng, T, L, pool_len)
    prm = {0: tr.randomize(L, rng)}
    full = run_waves(new_trainer(L, pool), sig_at, noise_at, [T], prm)
    for kw in (dict(with_noise=False), dict(with_vad=False), dict(with_noise=False, with_vad=False),
               dict(stream_stride=T * F + 1)):  # an odd stride: scalar stores
        got = run_waves(new_trainer(L, pool), sig_at, noise_at, [T], prm, **kw)
        for a, b in zip(full, got):
            if b is not None:
                assert np.array_equal(bits(a), bits(b)), kw


# ---- 2. the corpus: reproducible, and tied to the rows ----------------------------------------------------------------------
def corpus_windows(wc, count, T, seed, shuffle=False, noise=False):
    """Every window of a plan, T frames a call -> device tensors noisy, clean [L][F][480] and vad [L][F]."""
    import torch
    p = wc.start(count, seed, shuffle)
    L, Fr = wc.n_lanes, p.n_frames
    noisy, clean, nz = (torch.empty((L, Fr, F), device="cuda") for _ in range(3))
    vad = torch.empty((L, Fr), device="cuda")
    f0 = 0
    while wc.frames_left:
        d = 4 * f0 * F
        n = wc.next(T, noisy.data_ptr() + d, clean.data_ptr() + d, Fr * F, F, nz.data_ptr() + d if noise else None,
                    vad[:, f0].data_ptr(), Fr, 1)
        f0 += n
    assert f0 == Fr and wc.next(T, noisy.data_ptr(), clean.data_ptr(), Fr * F, F) == 0
    torch.cuda.synchronize()
    return noisy, clean, vad


def test_same_seed_same_bytes(corpus):
    sig_paths, noise_paths = corpus
    wc = tr.WaveformCorpus(sig_paths, noise_paths, 5)
    a = corpus_windows(wc, 5 * 300, 37, seed=4, shuffle=True)
    b = corpus_windows(tr.WaveformCorpus(sig_paths, noise_paths, 5), 5 * 300, 64, seed=4, shuffle=True, noise=True)
    for x, y in zip(a, b):
        assert np.array_equal(bits(x), bits(y))


def test_features_equal_the_rows(corpus):
    """Through generate_rows and through WaveformCorpus with the same arguments, over a plan that crosses randomize
    frame 2821 and file changes: the features of `noisy` (a DenoiseBatch of L streams, window after window, never reset)
    are the rows' 42 features bit for bit and `vad` is their last column.  Then, on these noisy lanes, the rows' target
    gains (masked bands at 1) bring the output closer to `clean` than gains of 1 do."""
    import torch
    sig_paths, noise_paths = corpus
    L, count, T, seed = 3, 3 * (tr.RANDOMIZE_PERIOD + 60), 64, 17
    rows = tr.generate_rows(sig_paths, noise_paths, count, lanes=L, seed=seed, shuffle=True)
    wc = tr.WaveformCorpus(sig_paths, noise_paths, L)
    noisy, clean, vad = corpus_windows(wc, count, T, seed, shuffle=True)
    p = wc.plan
    assert len(p.randomize) == 1 and any(len(s) > 1 for s in p.signal) and any(len(s) > 1 for s in p.noise)
    Fr = p.n_frames
    b = nb.DenoiseBatch(L)
    CB = nb.SYNTH_CONTEXT_BYTES
    feats = torch.empty((L, Fr, NBF), device="cuda")
    ones = torch.ones((L, Fr, NBB), device="cuda")
    tgt = torch.from_numpy(np.ascontiguousarray(np.where(rows[..., 42:64] < 0, 1.0, rows[..., 42:64]).transpose(1, 0, 2))).cuda()
    outs = {}
    for name, g in (("ones", ones), ("target", tgt)):
        b.reset()
        out = torch.empty((L, Fr, F), device="cuda")
        ctx = torch.empty((L, T, CB), dtype=torch.uint8, device="cuda")
        for f0 in range(0, Fr, T):
            n = min(T, Fr - f0)
            b.analyze_window_device(noisy[:, f0].data_ptr(), feats[:, f0].data_ptr(), 0, n, Fr * F, F, Fr * NBF, NBF, ctx.data_ptr(), T, 1)
            b.synthesize_window_device(out[:, f0].data_ptr(), g[:, f0].data_ptr(), n, Fr * F, F, Fr * NBB, NBB, ctx.data_ptr(), T, 1)
        torch.cuda.synchronize()
        outs[name] = out.cpu().numpy()
        if name == "ones":
            f = feats.cpu().numpy().transpose(1, 0, 2)
            assert np.array_equal(bits(f), bits(np.ascontiguousarray(rows[..., :42])))
    assert np.array_equal(vad.cpu().numpy().T, rows[..., 86])
    c = clean.cpu().numpy()[:, :-1]

    def snr(y):
        e = y[:, 1:] - c
        return 10 * np.log10((c.astype(np.float64) ** 2).sum() / (e.astype(np.float64) ** 2).sum())
    s1, s2 = snr(outs["ones"]), snr(outs["target"])
    print("\nSNR against clean: gains of 1 %.2f dB, the rows' target gains %.2f dB" % (s1, s2))
    assert s2 > s1


# ---- 3. alignment: clean[t] is output frame t + 1 at gains of 1 -------------------------------------------------------------
def test_clean_is_the_output_one_frame_later():
    """With noise_gain = 0, output frame t + 1 at gains of 1 is clean[t] below 18 kHz, from t = 1 on.
    - Synthesis interpolates the band gains only up to the last band edge (bin 400, 20 kHz), as the reference's
      interp_band_gain does, so bins 400..480 leave at gain 0 whatever the gains: broadband frames (white noise at
      random offsets) missed clean by 28-54 % relative RMS for that alone.  Each lane here reads consecutive frames of
      noise low-passed at 15 kHz, and both sides are compared after one low-pass at 18 kHz, since the pool's int16
      rounding leaves energy above 20 kHz (5e-5 relative RMS in the float64 restatement of tests/spectral_ref.py).
    - Output frame 1 is left out: frame 0's analysis window steps from the zero history into the signal, and that
      onset's energy above 20 kHz is dropped too (0.8 % of the frame in the same restatement, 0 in later frames)."""
    import torch
    L, T = 6, 30
    rng = np.random.default_rng(3)
    pool_len = 480 * (T + 1) + 2450 * L
    X = np.fft.rfft(rng.normal(0, 3000, pool_len))
    X[np.fft.rfftfreq(pool_len, 1 / 48000.0) > 15000] = 0
    pool = np.clip(np.round(np.fft.irfft(X, pool_len)), -32768, 32767).astype(np.int16)
    sig_at = (2450 * np.arange(L) + 7 * np.arange(L))[None, :] + 480 * np.arange(T)[:, None]
    noise_at = sig_at[::-1].copy()
    prm = tr.randomize(L, rng)
    prm["noise_gain"] = 0.0
    prm["signal_gain"] = np.abs(prm["signal_gain"]) + 0.5
    noisy, clean, _, _ = run_waves(new_trainer(L, pool), sig_at, noise_at, [T], {0: prm})
    b = nb.DenoiseBatch(L)
    CB = nb.SYNTH_CONTEXT_BYTES
    xd = torch.from_numpy(noisy).cuda()
    feats = torch.empty((L, T, NBF), device="cuda")
    out = torch.empty((L, T, F), device="cuda")
    ones = torch.ones((L, T, NBB), device="cuda")
    ctx = torch.empty((L, T, CB), dtype=torch.uint8, device="cuda")
    b.analyze_window_device(xd.data_ptr(), feats.data_ptr(), 0, T, T * F, F, T * NBF, NBF, ctx.data_ptr(), T, 1)
    b.synthesize_window_device(out.data_ptr(), ones.data_ptr(), T, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1)
    n = (T - 2) * F
    keep = np.fft.rfftfreq(n, 1 / 48000.0) <= 18000
    low = lambda x: np.fft.irfft(np.fft.rfft(x.reshape(L, n), axis=1) * keep, n, axis=1)  # noqa: E731
    y = low(out.cpu().numpy().astype(np.float64)[:, 2:])
    c = low(clean.astype(np.float64)[:, 1:-1])
    rel = np.sqrt(((y - c) ** 2).sum(axis=1) / (c ** 2).sum(axis=1))
    print("\nrelative RMS of output frame t + 1 against clean[t], per lane:", rel)
    assert (rel < 1e-5).all(), rel


# ---- 4. training through synthesis on corpus windows ------------------------------------------------------------------------
class GruGains:
    def __init__(self, seed):
        import torch
        torch.manual_seed(seed)
        self.gru = torch.nn.GRU(NBF, 32, batch_first=True).cuda()
        self.out = torch.nn.Linear(32, NBB).cuda()

    def parameters(self):
        return list(self.gru.parameters()) + list(self.out.parameters())

    def __call__(self, f):
        import torch
        return torch.sigmoid(self.out(self.gru(f / 10.0)[0]))


def window_loss(b, net, noisy, clean, grad):
    """One whole window [B][T][480]: analyze_window -> net -> synthesize_window -> synthesis_grad, the MSE of output
    frame t + 1 against clean[t]."""
    import torch
    from nnnoiseless_b200.autograd import synthesis_grad
    B, T = noisy.shape[0], noisy.shape[1]
    CB = nb.SYNTH_CONTEXT_BYTES
    b.reset()
    feats = torch.empty((B, T, NBF), device="cuda")
    out = torch.empty((B, T, F), device="cuda")
    ctx = torch.empty((B, T, CB), dtype=torch.uint8, device="cuda")
    b.analyze_window_device(noisy.data_ptr(), feats.data_ptr(), 0, T, T * F, F, T * NBF, NBF, ctx.data_ptr(), T, 1)
    with torch.set_grad_enabled(grad):
        g = net(feats)
        gd = g.detach().contiguous()
        b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1)
        y = synthesis_grad(g, out, ctx) if grad else out
        loss = ((y[:, 1:] - clean[:, :-1]) * (1.0 / 32768.0)).pow(2).mean()
    if grad:
        loss.backward()
    return float(loss.detach())


def test_gru_trained_on_corpus_windows(corpus):
    import torch
    sig_paths, noise_paths = corpus
    B, T, n_win = 16, 32, 6
    wc = tr.WaveformCorpus(sig_paths, noise_paths, B)
    wc.start(B * T * n_win, seed=5)
    wins = []
    for _ in range(n_win):
        noisy, clean = torch.empty((B, T, F), device="cuda"), torch.empty((B, T, F), device="cuda")
        assert wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F) == T
        wins.append((noisy, clean))
    held = wins.pop()
    b = nb.DenoiseBatch(B)
    net = GruGains(1)
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    before = window_loss(b, net, *held, grad=False)
    for k in range(40):
        opt.zero_grad()
        window_loss(b, net, *wins[k % len(wins)], grad=True)
        opt.step()
    after = window_loss(b, net, *held, grad=False)
    print("\nheld-out waveform MSE %.4g -> %.4g (40 Adam steps on corpus windows)" % (before, after))
    assert after < 0.9 * before


# ---- 5. refusals change nothing ---------------------------------------------------------------------------------------------
def test_refusals_change_nothing():
    import torch
    L, T = 5, 6
    rng = np.random.default_rng(9)
    pool_len = 480 * 20 + 1
    pool = _pool(pool_len, 9)
    sig_at, noise_at = _offsets(rng, T, L, pool_len), _offsets(rng, T, L, pool_len)
    out = [torch.empty((L, T, F), device="cuda") for _ in range(3)]
    vad = torch.empty((L, T), device="cuda")
    P = [x.data_ptr() for x in out]

    def call(t, n=T, s=sig_at, z=noise_at, p=P, ss=T * F, fs=F, v=vad.data_ptr()):
        L_ = nb.lib()
        ptr = lambda q: q or None  # noqa: E731
        s, z = np.ascontiguousarray(s[:max(n, 0)], np.int64), np.ascontiguousarray(z[:max(n, 0)], np.int64)
        rc = L_.rnnoise_train_waves_device(t._h, nb._np_ptr(s), nb._np_ptr(z), n, ptr(p[0]), ptr(p[1]), ptr(p[2]), ptr(v), ss, fs, T, 1, None)
        if rc != 0:
            raise NnnoiselessError(nb.last_error())

    t = tr.TrainingBatch(L)
    with pytest.raises(NnnoiselessError, match="no sample pool"):
        call(t)
    t.pool_reserve(pool_len)
    with pytest.raises(NnnoiselessError, match="runs outside the pool"):
        t.pool_write(pool_len - 10, pool[:11])
    with pytest.raises(NnnoiselessError, match="runs outside the pool"):
        t.pool_write(-1, pool[:1])
    t.pool_write(0, pool)
    with pytest.raises(NnnoiselessError, match="does not fit on the device|does not fit on device"):
        t.pool_reserve(1 << 50)
    assert t.pool_samples == pool_len
    bad_s, bad_n = sig_at.copy(), noise_at.copy()
    bad_s[3, 2] = pool_len - 479
    bad_n[4, 1] = -2
    for kw, what in ((dict(s=bad_s), "sig_at = %d at frame 3, lane 2" % (pool_len - 479)), (dict(z=bad_n), "noise_at = -2 at frame 4, lane 1"),
                     (dict(ss=F), "overlap"), (dict(fs=0), "overlap"), (dict(p=[0, P[1], P[2]]), "null"),
                     (dict(p=[P[0], 0, P[2]]), "null"), (dict(n=-1), "negative")):
        with pytest.raises(NnnoiselessError, match=what):
            call(t, **kw)
    call(t, n=0)  # a no-op, and it fixes no mode
    r = tr.TrainingBatch(L)
    r.process_pool_host(pool, sig_at, noise_at)  # a rows trainer refuses waveform frames
    r.pool_reserve(pool_len)
    r.pool_write(0, pool)
    with pytest.raises(NnnoiselessError, match="has made rows"):
        call(r)
    call(t)
    got = [x.cpu().numpy() for x in out + [vad]]
    with pytest.raises(NnnoiselessError, match="has made waveform frames"):
        t.process_pool_host(pool, sig_at, noise_at)
    with pytest.raises(NnnoiselessError, match="has made waveform frames"):
        t.process_host(np.zeros((1, L, F), np.float32), np.zeros((1, L, F), np.float32))
    # a trainer that never saw a refused call
    fresh = new_trainer(L, pool)
    call(fresh)
    want = [x.cpu().numpy() for x in out + [vad]]
    for a, b in zip(got, want):
        assert np.array_equal(bits(a), bits(b))
    # after reset: rows and waveforms again, as from new trainers
    r.reset()
    call(r)
    assert all(np.array_equal(bits(x.cpu().numpy()), bits(w)) for x, w in zip(out + [vad], want))
    t.reset()
    rows = t.process_pool_host(pool, sig_at, noise_at)
    assert np.array_equal(bits(rows), bits(tr.TrainingBatch(L).process_pool_host(pool, sig_at, noise_at)))
