"""The analysis and synthesis kernels (K3 and K5: spectral_warp.cu) one frame at a time against a float64 restatement
of the two stages (tests/spectral_ref.py).

Each frame is checked from the kernel's own inputs as the GPU had them, so that errors do not compound:
- K3 from input_mem (the state record after the frame: the high-pass is exact), the pitch tap, and the cepstral ring
  and mem_id of the record before the frame; checked: X, P, ex, ep, exp, the features, the silence flag, the new
  cepstral row and mem_id.
- K5 from X, P, ex, ep, exp and the silence flag (spectral taps), the raw gains (rnn taps), and lastg and
  synthesis_mem of the record before the frame; checked: the output frame, lastg and synthesis_mem after it.

The yardstick is the oracle's own f32 arithmetic on the same inputs (tests/oracle_state.c), run with both of its f32
FFT orders: d32 is the larger of their two deviations from float64.  Bounds (all per stream, never per batch: the
streams span 1/32768 to 1e4 x int16 full scale):
- X, P: K x max over bins of d32 (FFT rounding is spread over all bins in absolute terms).
- ex, ep, exp: per band, K x max(d32 of the band, the spectrum's d32 propagated through the band weights to first
  order), so that a quiet band cannot hide behind a loud one.
- features and the new cepstral row: K x max(d32 over the array, the band bounds propagated to first order through the
  log energies, the DCTs and the spectral variability).  A stream on a silence tie where neither oracle order took
  the reference's branch has no d32: it is held to the propagated bound alone, with the rounding of the f32
  arithmetic after the FFT added (spectral_ref.analysis_bounds with arith).
- output, synthesis_mem: K x max(d32 over the array).
- The only absolute floor is the smallest normal f32, and only where the float64 value is below it.
- lastg, the cepstral rows not written, mem_id, and everything on silent frames that the kernels leave alone: bit for
  bit.  lastg = max(g, 0.6 lastg) is rounded once in f32, so it must equal the oracle's bit for bit.
The silence test e < 0.04 is the one discontinuity the inputs do not fix: where the float64 margin |e - 0.04| is inside
the propagated bound of e, the reference follows the GPU's branch (the tie rule; counted and printed).  The pitch
filter's `exp > g` compares the GPU's own f32 exp and g on both sides, so its branch is fixed by the inputs.

K = 10: on an H100 (80GB HBM3, 400 W power limit) no quantity of any model used more than 0.46 of its bound
(P; X 0.40, ex 0.34, output and synthesis_mem 0.30), a factor of two of headroom.  The
tie rule fired on 22 of the 5,496 stream-frames.
"""
import hashlib
import os
from contextlib import contextmanager

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle_state as ost
import rnn_ref
import spectral_ref as sr
from conftest import synth_streams

K = 10.0
B, T = 229, 24
EBAND_5MS = sr.EBAND_5MS


# ---- signals ------------------------------------------------------------------------------------------------------
def _tone(k, amp, phase, n):
    """A tone on (fractional) bin k of the 960-point transform: k * 50 Hz."""
    t = np.arange(n, dtype=np.float64)
    if k == 480:
        return amp * np.where(t % 2 == 0, 1.0, -1.0)
    return amp * np.cos(2 * np.pi * k * t / 960.0 + phase)


def _band_noise(k0, k1, rms, n, rng):
    """White noise confined to bins [k0, k1) of the 960-point transform (and their images in the long transform)."""
    spec = np.fft.rfft(rng.standard_normal(n))
    fb = np.arange(len(spec)) * 960.0 / n
    spec[(fb < k0 - 0.5) | (fb >= k1 - 0.5)] = 0.0
    x = np.fft.irfft(spec, n)
    return x * rms / max(np.sqrt(np.mean(x * x)), 1e-30)


def _pulses(period, amp, n):
    x = np.zeros(n)
    x[::period] = amp
    return x


def _hp(x):
    """The input high-pass (src/util.rs:95-107) in float64: only used to place signal levels."""
    a0, a1 = float(np.float32(-1.99599)), float(np.float32(0.99600))
    y = np.empty_like(x)
    m0 = m1 = 0.0
    for i, v in enumerate(x):
        o = v + m0
        m0 = m1 + (-2.0 * v - a0 * o)
        m1 = v - a1 * o
        y[i] = o
    return y


def _band_energy_sum(x):
    """sum_b ex of the last full window of x (float64, after the high-pass)."""
    h = _hp(x)
    X = sr.rfft_windowed(h[None, -960:])
    return float((np.abs(X) ** 2 @ sr.tables()["W"].T).sum())


LADDER = (0.9, 0.95, 0.98, 0.99, 0.995, 1.0, 1.005, 1.01, 1.02, 1.05, 1.1)


def spectral_signals(seed=7):
    """[B][T][480] float32 and the name of each stream: the edges where spectral kernels go wrong, then ordinary
    white + sine streams."""
    rng = np.random.default_rng(seed)
    n = T * 480
    rows, names = [], []

    def add(x, name):
        rows.append(np.asarray(x, np.float64))
        names.append(name)

    # tones exactly on DC, bin 1, every band edge, the middle of the even/odd split, the end of the banded region and
    # Nyquist; tones halfway between bins, which leak across the band edges; a slow chirp over 0 - 24 kHz
    for k in sorted({0, 1, 239, 240, 241, 399, 400, 401, 479, 480} | {4 * e for e in EBAND_5MS}):
        add(_tone(k, 3000.0, rng.uniform(0, 2 * np.pi), n), "tone %d" % k)
    for k in (3.5, 7.5, 39.5, 47.5, 79.5, 135.5, 239.5, 311.5, 399.5, 479.5):
        add(_tone(k, 3000.0, rng.uniform(0, 2 * np.pi), n), "tone %.1f" % k)
    t = np.arange(n, dtype=np.float64)
    add(3000.0 * np.cos(np.pi * 480.0 * t * t / (960.0 * n)), "chirp 0-24 kHz")
    # band-limited noise: band 0 alone, a middle band, band 21 (bins 320-399), and only bins 400-480 (outside every band)
    for k0, k1 in ((0, 4), (48, 56), (320, 400), (400, 481)):
        add(_band_noise(k0, k1, 2000.0, n, rng), "noise bins %d-%d" % (k0, k1 - 1))
    # pulse trains at the smallest, an odd, an even and the largest period the pitch search returns
    for p in (60, 61, 120, 767):
        add(_pulses(p, 8000.0, n), "pulses %d" % p)
    # int16 full scale, float audio left unscaled, 1e4 x full scale
    add(np.where((t // 48) % 2 == 0, 32767.0, -32768.0), "full-scale square")
    add(np.clip(np.rint(rng.uniform(-32768, 32767, n)), -32768, 32767), "full-scale noise")
    base = synth_streams(4, T, seed=seed).astype(np.float64)
    add(base[0] / 32768.0, "float audio")
    add(base[1] / 32768.0, "float audio")
    add(1e4 * rng.uniform(-32768, 32767, n), "1e4 x full-scale noise")
    add(1e4 * _pulses(61, 32767.0, n), "1e4 x full-scale pulses")
    # a ladder of levels around the silence threshold: a tone inside band 8 whose sum of band energies is placed with
    # the float64 reference at 0.9 ... 1.1 x 0.04
    unit = _tone(37, 1.0, 0.3, n)
    e1 = _band_energy_sum(unit[: 12 * 480])
    for q in LADDER:
        add(unit * np.sqrt(sr.C_SIL * q / e1), "level %.3f x threshold" % q)
    # signal -> digital zero (the ill-conditioned frames after a cut) and zero -> signal onsets, where the pitch-lagged
    # window still reaches into silence
    for f0 in (6, 10, 14, 18):
        x = base[2].copy()
        x[f0 * 480:] = 0.0
        add(x, "cut at frame %d" % f0)
    for f0 in (3, 9, 15):
        x = base[3].copy()
        x[: f0 * 480] = 0.0
        add(x, "onset at frame %d" % f0)
    # quiet noise with gaps of digital zero at different offsets: the silent frames stall mem_id at different slots
    for o in range(8):
        x = 2.0 * rng.standard_normal(n)
        for g0 in (2 + o, 13 + o):
            x[g0 * 480:(g0 + 3) * 480] = 0.0
        add(x, "gaps at %d" % o)
    rest = B - len(rows)
    assert rest > 0
    for r in synth_streams(rest, T, seed=seed + 1):
        add(r, "white + sine")
    x = np.stack(rows).astype(np.float32).reshape(B, T, 480)
    return x, names


# ---- running the GPU frame by frame -------------------------------------------------------------------------------
KERNELS = {"warp": {}}


@contextmanager
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


def run_frames(model: bytes, x, kernel, n_frames=T):
    """x [B][T][480] one frame per call on a fresh batch -> per frame dict(before, after (state records), pitch, silence,
    features, gains (raw), vad (raw), vad_out, X, P, ex, ep, exp, out)."""
    with env(**KERNELS[kernel]):
        batch = nb.DenoiseBatch(x.shape[0], nb.RnnModel.from_bytes(model))
    dt = nb.state_dtype(batch.gru_widths)
    prev = batch.get_states()
    frames = []
    for f in range(n_frames):
        out, vad = batch.process_host(np.ascontiguousarray(x[:, f][None]))
        rec = batch.get_states()
        t, r = batch.taps(), batch.rnn_taps()
        frames.append(dict(before=prev, after=rec, rb=prev.view(dt).reshape(-1), ra=rec.view(dt).reshape(-1), pitch=t["pitch"],
                           silence=t["silence"], features=t["features"], gains=r["gains"], vad=r["vad"], vad_out=vad[0],
                           out=out[0], **batch.spectral_taps()))
        prev = rec
    return frames


# ---- checks -------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24


def _share(err, tol):
    """err / tol elementwise, with 0 / 0 = 0 (a zero bound requires a zero error)."""
    err, tol = np.broadcast_arrays(np.asarray(err, np.float64), np.asarray(tol, np.float64))
    out = np.zeros(err.shape)
    nz = tol > 0
    out[nz] = err[nz] / tol[nz]
    out[~nz & (err > 0)] = np.inf
    return out


F32_TINY = float(np.finfo(np.float32).tiny)


def _array_err(got, r64):
    """Per stream, the largest error over the array, less an absolute floor of the smallest normal f32 where the float64
    value is below f32 resolution (an f32 computation may flush it to zero)."""
    e = np.abs(got - r64)
    e = np.where(np.abs(r64) < F32_TINY, np.maximum(e - F32_TINY, 0.0), e)
    return e.reshape(len(e), -1).max(axis=1)


def _array_bound(d32, prop=0.0):
    """Per stream: K x max(d32 over the array, the inputs' bounds propagated to it)."""
    return K * np.maximum(d32.reshape(len(d32), -1).max(axis=1), prop)


class Worst:
    """Largest error and largest share of the bound per quantity, over frames."""

    def __init__(self):
        self.q = {}

    def add(self, name, err, tol):
        sh = _share(err, tol)
        e0, s0 = self.q.get(name, (0.0, 0.0))
        self.q[name] = (max(e0, float(np.max(err, initial=0.0))), max(s0, float(np.max(sh, initial=0.0))))
        return sh

    def line(self):
        return ", ".join("%s %.2e (%.2f)" % (k, e, s) for k, (e, s) in self.q.items())


_K3_YARDSTICK = {}


def oracle_analysis(omodel, frames, x, f):
    """The oracle's analysis of frame f of every stream from the GPU's record before it, under FFT orders 0 and 2.  It
    depends only on the analysis state in the records and the input frame, not on the model: runs of the same kernel
    pair under different models share it (cached by the bytes of those inputs)."""
    fr = frames[f]
    rb = fr["rb"]
    key = hashlib.sha1(b"".join(np.ascontiguousarray(a).tobytes() for a in (
        rb["input_mem"], rb["mem_hp_x"], rb["cepstral_mem"], rb["mem_id"], rb["last_period"], rb["last_gain"], x[:, f]))).digest()
    if key not in _K3_YARDSTICK:
        res = []
        for mode in (0, 2):
            ost.set_fft_mode(mode)
            try:
                res.append([ost.analysis_frame(omodel, fr["before"][s], x[s, f]) for s in range(len(x))])
            finally:
                ost.set_fft_mode(0)
        _K3_YARDSTICK[key] = [{k: np.stack([o[k] for o in r]) for k in r[0]} for r in res]
    return _K3_YARDSTICK[key]


def check_analysis(fr, o32, worst, cov):
    """K3 of one frame against the float64 reference; o32: the oracle's results under the two FFT orders."""
    rb, ra = fr["rb"], fr["ra"]
    # the oracle's high-pass and pitch on the record before: the GPU's input_mem after the frame and its pitch, exactly
    assert np.array_equal(o32[0]["input_mem"].view(np.uint32), ra["input_mem"].view(np.uint32))
    assert np.array_equal(o32[0]["pitch"], fr["pitch"]) and np.array_equal(o32[1]["pitch"], fr["pitch"])
    ref = sr.analysis(ra["input_mem"], fr["pitch"], rb["cepstral_mem"], rb["mem_id"])
    W = sr.tables()["W"]
    d = lambda q, n=None: np.max([np.abs(o[q][:, :n].astype(np.complex128 if o[q].dtype.kind == "c" else np.float64)  # noqa: E731
                                         - ref[q][:, :n]) for o in o32], axis=0)
    # spectra: one bound per stream for every bin
    dX, dP = d("X"), d("P", sr.NB_BINS_BANDED)
    for q, dq, n in (("X", dX, sr.FREQ_SIZE), ("P", dP, sr.NB_BINS_BANDED)):
        err = np.abs(fr[q].astype(np.complex128) - ref[q][:, :n]).max(axis=1)
        assert (worst.add(q, err, K * dq.max(axis=1)) <= 1.0).all(), (q, np.flatnonzero(_share(err, K * dq.max(axis=1)) > 1))
    # band quantities: per band, the band's own d32 or the spectra's propagated through the band weights; then on to the
    # features through the log energies, both DCTs and the spectral variability (spectral_ref.analysis_bounds)
    dx, dp = dX.max(axis=1)[:, None], dP.max(axis=1)[:, None]
    b = sr.analysis_bounds(ref, dx, dp, band={q: d(q) for q in ("ex", "ep", "exp")})
    for q in ("ex", "ep", "exp"):
        tol = K * b[q]
        err = np.abs(fr[q] - ref[q])
        sh = worst.add(q, err, tol)
        assert (sh <= 1.0).all(), (q, np.argwhere(sh > 1.0)[:5], sh.max())
    dex = b["ex"]
    prop_row, prop_feat = b["row"].max(axis=1), b["features"].max(axis=1)
    # the same with the rounding of the f32 arithmetic after the FFT, for streams that have no d32 to carry it
    ba = sr.analysis_bounds(ref, dx, dp, band={q: d(q) for q in ("ex", "ep", "exp")}, arith=True)
    arith_row, arith_feat = ba["row"].max(axis=1), ba["features"].max(axis=1)
    # the silence test: the GPU's branch must be the float64 one unless the margin is inside the bound of e
    tol_e = K * dex.sum(axis=1) + sr.NB_BANDS * U32 * ref["e"]
    tie = np.abs(ref["e"] - sr.C_SIL) <= tol_e
    gsil = fr["silence"] != 0
    sil = np.where(tie, gsil, ref["silence"])
    assert np.array_equal(gsil, sil), np.flatnonzero(gsil != sil)
    for o in o32:
        assert ((o["silence"] != 0) == sil)[~tie].all()
    cov["ties"] += int(tie.sum())
    cov["tie_flips"] += int((tie & (gsil != ref["silence"])).sum())
    near = np.abs(ref["e"] / sr.C_SIL - 1.0) < 0.1
    cov["near_silent"] |= bool((near & sil).any())
    cov["near_live"] |= bool((near & ~sil).any())
    # silent frames: zero features; the cepstral ring and mem_id untouched
    assert not fr["features"][sil].any()
    assert np.array_equal(ra["cepstral_mem"][sil].view(np.uint32), rb["cepstral_mem"][sil].view(np.uint32))
    assert np.array_equal(ra["mem_id"][sil], rb["mem_id"][sil])
    live = np.flatnonzero(~sil)
    if not len(live):
        return sil
    # mem_id advances; the rows other than the one written are unchanged, bit for bit
    mid = rb["mem_id"][live]
    assert np.array_equal(ra["mem_id"][live], (mid + 1) % 8)
    keep = np.ones((len(live), 8), bool)
    keep[np.arange(len(live)), mid] = False
    assert np.array_equal(ra["cepstral_mem"][live][keep].view(np.uint32), rb["cepstral_mem"][live][keep].view(np.uint32))
    # features and the new row, from the oracle's FFT orders whose silence flag is the reference's.  A tie may split them:
    # a stream where neither order took the reference's branch is held to the propagated bound alone (counted)
    match = np.stack([(o["silence"][live] != 0) == sil[live] for o in o32])
    has = match.any(axis=0)
    cov["no_yardstick"] += int((~has).sum())
    rows = np.arange(len(live))
    for q, got, r64, o_of, pq in (("features", fr["features"][live], ref["features"][live], lambda o: o["features"][live],
                                   np.where(has, prop_feat[live], arith_feat[live])),
                                  ("ceps row", ra["cepstral_mem"][live][rows, mid], ref["row"][live],
                                   lambda o: o["ceps"][live][rows, mid], np.where(has, prop_row[live], arith_row[live]))):
        d32 = np.max([np.where(m[:, None], np.abs(o_of(o) - r64), 0.0) for o, m in zip(o32, match)], axis=0)
        err = _array_err(got, r64)
        sh = worst.add(q, err, _array_bound(d32, pq))
        assert (sh <= 1.0).all(), (q, live[sh > 1.0], sh.max())
    p = fr["pitch"][live]
    cov["pitch_odd"] |= bool((p % 2 == 1).any())
    cov["pitch_even"] |= bool((p % 2 == 0).any())
    cov["pitch_min"] = min(cov["pitch_min"], int(p.min()))
    cov["pitch_max"] = max(cov["pitch_max"], int(p.max()))
    cov["mem_ids"] |= set(int(m) for m in mid)
    return sil


def check_synthesis(fr, worst, cov):
    """K5 of one frame against the float64 reference, from the GPU's own spectra, band quantities and raw gains."""
    rb, ra = fr["rb"], fr["ra"]
    sil = fr["silence"] != 0
    nst = len(sil)
    args = (fr["X"], fr["P"], fr["ex"], fr["ep"], fr["exp"], fr["gains"], rb["lastg"], rb["synthesis_mem"], sil)
    ref = sr.synthesis(*args)
    Pf = np.zeros((nst, sr.FREQ_SIZE), np.complex64)
    Pf[:, :sr.NB_BINS_BANDED] = fr["P"]
    o32 = []
    for mode in (0, 2):
        ost.set_fft_mode(mode)
        try:
            o32.append([ost.synthesis_from(fr["X"][s], Pf[s], fr["ex"][s], fr["ep"][s], fr["exp"][s], fr["gains"][s],
                                           rb["lastg"][s], rb["synthesis_mem"][s], sil[s]) for s in range(nst)])
        finally:
            ost.set_fft_mode(0)
    o_out = [np.stack([o[0] for o in r]) for r in o32]
    o_lastg = [np.stack([o[1] for o in r]) for r in o32]
    o_mem = [np.stack([o[2] for o in r]) for r in o32]
    # lastg = max(g, 0.6 lastg) is one f32 rounding: the oracle's bits; silent frames leave it alone and report vad 0
    assert np.array_equal(ra["lastg"].view(np.uint32), o_lastg[0].view(np.uint32)), np.flatnonzero((ra["lastg"] != o_lastg[0]).any(1))
    assert np.array_equal(ra["lastg"][sil].view(np.uint32), rb["lastg"][sil].view(np.uint32))
    assert not fr["vad_out"][sil].any()
    for q, got, r64, o in (("out", fr["out"], ref["out"], o_out), ("synth_mem", ra["synthesis_mem"], ref["synth_mem"], o_mem)):
        d32 = np.maximum(np.abs(o[0] - r64), np.abs(o[1] - r64))
        err = _array_err(got, r64)
        sh = worst.add(q, err, _array_bound(d32))
        assert (sh <= 1.0).all(), (q, np.flatnonzero(sh > 1.0))
    live = ~sil
    cov["branch_r1"] |= bool(ref["branch"][live].any())
    cov["branch_ratio"] |= bool((~ref["branch"][live]).any())
    cov["floor"] |= bool(ref["floor"][live].any())
    g = fr["gains"][live]
    if g.size:
        cov["g_min"] = min(cov["g_min"], float(g.min()))
        cov["g_max"] = max(cov["g_max"], float(g.max()))


def new_coverage():
    return dict(ties=0, tie_flips=0, no_yardstick=0, near_silent=False, near_live=False, pitch_odd=False, pitch_even=False, pitch_min=10 ** 9,
                pitch_max=-1, mem_ids=set(), branch_r1=False, branch_ratio=False, floor=False, g_min=np.inf, g_max=-np.inf,
                silent=False, live=False)


# ---- models -------------------------------------------------------------------------------------------------------
def _ramp_model():
    """A model whose sigmoid output layer spans the raw gains over [0, 1] (synthesis sees the model only through g)."""
    return rnn_ref.make_model(24, 24, 48, 96, seed=11)


MODELS = ["builtin", "sh", "ramp"]


@pytest.fixture(scope="module")
def signals():
    return spectral_signals()


_RUNS = {}


def _model_bytes(name, builtin_bytes, sh_bytes):
    return {"builtin": builtin_bytes, "sh": sh_bytes}.get(name) or _ramp_model()


def _run(name, kernel, model, x):
    if (name, kernel) not in _RUNS:
        _RUNS[(name, kernel)] = run_frames(model, x, kernel)
    return _RUNS[(name, kernel)]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("model_name", MODELS)
def test_spectral_kernels_one_frame_against_float64(model_name, kernel, signals, builtin_bytes, sh_bytes):
    x, names = signals
    model = _model_bytes(model_name, builtin_bytes, sh_bytes)
    frames = _run(model_name, kernel, model, x)
    omodel = ost.Model(model)
    wa, ws, cov = Worst(), Worst(), new_coverage()
    for f, fr in enumerate(frames):
        sil = check_analysis(fr, oracle_analysis(omodel, frames, x, f), wa, cov)
        cov["silent"] |= bool(sil.any())
        cov["live"] |= bool((~sil).any())
        check_synthesis(fr, ws, cov)
    print("\n%-7s %-5s K3: %s" % (model_name, kernel, wa.line()))
    print("%-7s %-5s K5: %s" % (model_name, kernel, ws.line()))
    print("%-7s %-5s silence tie rule: %d stream-frames inside the bound, %d where the GPU left the float64 branch, %d "
          "without an oracle order on the same branch; raw gains %.3f .. %.3f"
          % (model_name, kernel, cov["ties"], cov["tie_flips"], cov["no_yardstick"], cov["g_min"], cov["g_max"]))
    # the signal set reached what it is there for
    assert cov["pitch_odd"] and cov["pitch_even"] and cov["pitch_min"] == 60 and cov["pitch_max"] >= 765, cov
    assert cov["mem_ids"] == set(range(8)), cov
    assert cov["branch_r1"] and cov["branch_ratio"] and cov["floor"], cov
    assert cov["silent"] and cov["live"] and cov["near_silent"] and cov["near_live"], cov
    if model_name == "ramp":
        assert cov["g_min"] < 0.05 and cov["g_max"] > 0.95, cov


@pytest.mark.gpu
def test_spectral_taps_many_rounds_bitwise(signals, builtin_bytes):
    """2 x (SMs x 12 resident warps) + 37 streams, permuted copies of the 229: every warp of the persistent analysis grid
    takes at least two streams and the last round is partial.  The spectral taps and the features at every position
    are the bits of the same stream in the 229-stream batch, frame by frame."""
    import torch

    x, _ = signals
    small = _run("builtin", "warp", builtin_bytes, x)
    n_big = 2 * torch.cuda.get_device_properties(0).multi_processor_count * 12 + 37
    rng = np.random.default_rng(5)
    perm = rng.integers(0, B, n_big)
    perm[:B] = rng.permutation(B)
    big = run_frames(builtin_bytes, np.ascontiguousarray(x[perm]), "warp", n_frames=10)
    for f in range(10):
        for q in ("X", "P", "ex", "ep", "exp", "features"):
            a, b = big[f][q], small[f][q][perm]
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (f, q)
