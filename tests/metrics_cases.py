"""Constructed streams for the metrics kernel's edges (TEST INFRASTRUCTURE; DESIGN.md 7p, "Checks").

cases() -> dict(y, c [B][T][480] float32, tgt, vad [B][T] float32, mode [T] int, names [B]).  Output y and clean c are
chosen per stream: tones on DC, bin 1, every band edge, halfway between bins, bin 400 and Nyquist; noise confined to
one band with the others 60-100 dB below; a 60 dB spectral tilt; cuts and onsets inside a window; amplitudes from 1e-20
to 1e4 x int16 full scale and exact zero; y = delayed c exactly and at half scale; the three segmental-SNR branches.
Targets and vads take the class and VAD edges in a pattern that gives every stream every value.  mode[t] is how call t
of a one-frame run passes its vad and target pointers: 0 both, 1 the vad only, 2 neither.  tgt holds 0.5 on frames
whose call passes no target, which is what the kernel sees then, so runs that pass every target give the same
records."""
import numpy as np

F = 480
T = 24
EBAND_5MS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 34, 40, 48, 60, 78, 100]
TARGETS = np.array([1.0, np.nextafter(np.float32(1), np.float32(0)), 0.0, -0.0, 1e-45, 0.5, np.nan, 2.0], np.float32)
VADS = np.array([0.5, np.nextafter(np.float32(0.5), np.float32(0)), np.nan, -0.0, 1.0], np.float32)
FULL = 32767.0


def _tone(k, amp, phase, n):
    t = np.arange(n, dtype=np.float64)
    if k == 480:
        return amp * np.where(t % 2 == 0, 1.0, -1.0)
    return amp * np.cos(2 * np.pi * k * t / 960.0 + phase)


def _shaped(gain_of_bin, n, rng):
    """White noise with amplitude gain gain_of_bin(bin of the 960-point transform), unit rms before shaping."""
    spec = np.fft.rfft(rng.standard_normal(n))
    spec *= gain_of_bin(np.arange(len(spec)) * 960.0 / n)
    return np.fft.irfft(spec, n)


def _rms(x):
    return max(float(np.sqrt(np.mean(x * x))), 1e-300)


def _band_noise(band, rms, floor_db, n, rng):
    """Noise in band `band`'s bins (4 eband[b] .. 4 eband[b + 1]) at `rms`, everything else floor_db below it."""
    k0, k1 = 4 * EBAND_5MS[band], 4 * EBAND_5MS[band + 1]
    x = _shaped(lambda k: np.where((k >= k0) & (k < k1), 1.0, 0.0), n, rng)
    x *= rms / _rms(x)
    return x + rng.standard_normal(n) * rms * 10.0 ** (-floor_db / 20.0)


def _delayed(c):
    y = np.zeros_like(c)
    y[F:] = c[:-F]
    return y


def cases(seed=3):
    rng = np.random.default_rng(seed)
    n = T * F
    ys, cs, names = [], [], []

    def add(y, c, name):
        ys.append(np.asarray(y, np.float64))
        cs.append(np.asarray(c, np.float64))
        names.append(name)

    noise = lambda s: rng.standard_normal(n) * s  # noqa: E731
    # tones: on DC, bin 1, every band edge, halfway between bins, bin 400 (past the last band) and Nyquist; the clean
    # tone at another amplitude and phase
    for k in sorted({0, 1, 480} | {4 * e for e in EBAND_5MS}) + [1.5, 3.5, 39.5, 79.5, 239.5, 399.5]:
        add(_tone(k, 3000.0, rng.uniform(0, 2 * np.pi), n), _tone(k, 2000.0, rng.uniform(0, 2 * np.pi), n), "tone %s" % k)
    # one loud band, the others 60-100 dB below; output and clean with different floors
    for b in (0, 1, 7, 12, 16, 19, 20):
        add(_band_noise(b, 2000.0, 60.0, n, rng), _band_noise(b, 2000.0, 100.0, n, rng), "band %d alone" % b)
    add(_band_noise(3, 2000.0, 80.0, n, rng), _band_noise(18, 2000.0, 80.0, n, rng), "band 3 against band 18")
    # a 60 dB tilt over 0 - 24 kHz, both ways
    up = _shaped(lambda k: 10.0 ** (-3.0 * (480.0 - k) / 480.0), n, rng)
    down = _shaped(lambda k: 10.0 ** (-3.0 * k / 480.0), n, rng)
    add(up * 3000.0 / _rms(up), down * 3000.0 / _rms(down), "tilt up / down")
    add(down * 3000.0 / _rms(down), _delayed(down * 3000.0 / _rms(down)), "tilt down, clean ahead")
    # cuts and onsets inside a window: every other frame zero (each window has one live and one dead half), and a cut
    # and an onset in mid-stream
    alt = (np.arange(n) // F) % 2 == 0
    add(np.where(alt, noise(2000.0), 0.0), np.where(~alt, noise(2000.0), 0.0), "alternating frames")
    add(np.where(np.arange(n) < 9 * F, noise(2000.0), 0.0), np.where(np.arange(n) >= 13 * F, noise(2000.0), 0.0),
        "cut at 9 / onset at 13")
    # amplitudes
    for name, s in (("1/32768", 1.0 / 32768.0), ("int16 full scale", None), ("1e4 x full scale", 1e4 * FULL),
                    ("1e-20", 1e-20)):
        if s is None:
            y, c = (np.clip(np.rint(rng.uniform(-32768, 32767, n)), -32768, 32767) for _ in range(2))
        else:
            y, c = noise(s), noise(s)
        add(y, c, name)
    add(np.zeros(n), np.zeros(n), "zero")
    add(noise(1e4 * FULL), noise(1e-20), "1e4 x full scale against 1e-20")
    add(noise(1e-20), noise(1.0 / 32768.0), "1e-20 against 1/32768")
    # exact copies and half scale
    for k in range(3):
        c = noise(2000.0)
        add(_delayed(c), c, "delayed clean")
        c = noise(2000.0)
        add(np.float32(0.5) * _delayed(c), c, "half delayed clean")
    # the segmental-SNR branches: Ec = 0 with Ed > 0, Ed = 0 (a copy), both zero (frames alternate with a live one)
    add(noise(2000.0), np.zeros(n), "clean zero")
    c = np.where(alt, 0.0, noise(2000.0))
    add(_delayed(c), c, "copy with zero frames")
    # ordinary noisy outputs
    rest = 200 - len(names)
    for _ in range(rest):
        c = noise(rng.uniform(100.0, 5000.0))
        add(_delayed(c) + noise(rng.uniform(10.0, 3000.0)), c, "noisy")
    B = len(names)
    y = np.stack(ys).astype(np.float32).reshape(B, T, F)
    c = np.stack(cs).astype(np.float32).reshape(B, T, F)
    s, t = np.arange(B)[:, None], np.arange(T)[None, :]
    tgt = TARGETS[(s + 3 * t) % len(TARGETS)]
    vad = VADS[(2 * s + t) % len(VADS)]
    mode = np.zeros(T, np.int64)
    mode[[5, 11]] = 1  # the vad without a target
    mode[[6, 17]] = 2  # neither (a target pointer in one call and none in the next)
    tgt = np.where((mode > 0)[None, :], np.float32(0.5), tgt).astype(np.float32)
    return dict(y=np.ascontiguousarray(y), c=np.ascontiguousarray(c), tgt=np.ascontiguousarray(tgt), vad=np.ascontiguousarray(vad),
                mode=mode, names=names)


def coverage(out, clean, tgt, vad):
    """Stream-frames of a run from a fresh handle (frame 0 uncounted) per class, segmental-SNR branch and VAD cell."""
    out, clean = np.asarray(out, np.float64), np.asarray(clean, np.float64)
    B, Tn = out.shape[:2]
    cprev = np.concatenate([np.zeros((B, 1, F)), clean[:, :-1]], axis=1)
    ec = (cprev ** 2).sum(axis=2)[:, 1:]
    ed = ((out - cprev) ** 2).sum(axis=2)[:, 1:]
    tc = np.asarray(tgt, np.float64)[:, :-1]
    tn = np.asarray(tgt, np.float64)[:, 1:]
    said = np.asarray(vad)[:, 1:] >= 0.5
    with np.errstate(divide="ignore", invalid="ignore"):
        snr = 10.0 * np.log10(ec / ed)
    live = (ed > 0) & (ec > 0)
    voted = (tn == 0.0) | (tn == 1.0)
    is_ = tn == 1.0
    return {
        "speech": int((tc == 1.0).sum()), "noise": int((tc == 0.0).sum()),
        "neither": int(((tc != 1.0) & (tc != 0.0)).sum()),
        "ed=0": int((ed == 0).sum()), "ec=0<ed": int(((ec == 0) & (ed > 0)).sum()), "ec=ed=0": int(((ec == 0) & (ed == 0)).sum()),
        "clamp low": int((live & (snr < -10.0)).sum()), "clamp high": int((live & (snr > 35.0)).sum()),
        "inside": int((live & (snr >= -10.0) & (snr <= 35.0)).sum()),
        "tp": int((voted & said & is_).sum()), "fp": int((voted & said & ~is_).sum()),
        "fn": int((voted & ~said & is_).sum()), "tn": int((voted & ~said & ~is_).sum()),
    }
