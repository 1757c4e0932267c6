"""Float64 restatement of STOI / ESTOI as rnnoise_intelligibility_device defines them (include/rnnoise.h, DESIGN.md 7q).

Each stage is a function of its own inputs, so the GPU tests can feed it the GPU's intermediate results (the workspace
taps) and check one stage at a time.  ``score`` performs the double tail's operations in the kernel's order, unfused
(the unit is built with -fmad=false), so from the same float bands it gives the kernel's scores to rounding of the
final sums."""
import math

import numpy as np
import scipy.signal as ss

EPS = 2.0 ** -52
FRAME, HOP, NFFT, NBANDS, NSEG = 256, 128, 512, 15, 30
EDGES = np.array([7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219])
CLIP = 1.0 + 10.0 ** (15.0 / 20.0)
U32 = 2.0 ** -24


def gamma(k, u=U32):
    return k * u / (1.0 - k * u)


def sizes(n, rate):
    """(up, down, half, n10, F)."""
    g = math.gcd(int(rate), 10000)
    up, down = 10000 // g, int(rate) // g
    half = 0 if up == down == 1 else 10 * max(up, down)
    n10 = -(-int(n) * up // down)
    return up, down, half, n10, ((n10 - FRAME) // HOP + 1 if n10 >= FRAME else 0)


def filter_taps(rate):
    """The float32 taps h of step 1 (None at 10 kHz): firwin(2 half + 1, 1 / max(up, down), kaiser 5) * up."""
    up, down, half, _, _ = sizes(0, rate)
    if half == 0:
        return None
    return (ss.firwin(2 * half + 1, 1.0 / max(up, down), window=("kaiser", 5.0)) * up).astype(np.float32)


def resample(x, rate, h=None, absolute=False):
    """x10[m] = sum_n x[n] h[half + m down - n up] in float64 (with absolute=True: of |x| and |h|, the sum the
    rounding bound scales)."""
    x = np.asarray(x, np.float64)
    up, down, half, n10, _ = sizes(len(x), rate)
    if half == 0:
        return np.abs(x) if absolute else x.copy()
    h = filter_taps(rate) if h is None else h
    h = np.asarray(h, np.float64)
    if absolute:
        x, h = np.abs(x), np.abs(h)
    full = ss.upfirdn(h, x, up, 1)  # full[t] = sum_n x[n] h[t - n up]
    idx = half + np.arange(n10) * down
    out = np.zeros(n10)
    ok = idx < len(full)
    out[ok] = full[idx[ok]]
    return out


def window():
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * (np.arange(FRAME) + 1) / (FRAME + 1))


def frames_of(x10):
    F = (len(x10) - FRAME) // HOP + 1 if len(x10) >= FRAME else 0
    if F == 0:
        return np.zeros((0, FRAME))
    return np.lib.stride_tricks.sliding_window_view(np.asarray(x10, np.float64), FRAME)[::HOP][:F] * window()


def frame_db(x10):
    """E_f = 20 log10(||w x10 frame f|| + EPS)."""
    fr = frames_of(x10)
    return 20.0 * np.log10(np.sqrt((fr * fr).sum(axis=1)) + EPS)


def kept_frames(x10):
    """Indices of the frames kept by the strict 40 dB rule on the clean signal."""
    e = frame_db(x10)
    if len(e) == 0:
        return np.zeros(0, np.int64)
    return np.flatnonzero(e > e.max() - 40.0)


def stft_frames(x10, kept):
    """The M = K - 1 windowed frames of the overlap-add of the kept frames, [M][256]."""
    K = len(kept)
    if K < 2:
        return np.zeros((0, FRAME))
    w = window()
    x10 = np.asarray(x10, np.float64)
    sig = np.zeros((K - 1) * HOP + FRAME)
    for k, f in enumerate(kept):
        sig[k * HOP:k * HOP + FRAME] += w * x10[f * HOP:f * HOP + FRAME]
    return np.lib.stride_tricks.sliding_window_view(sig, FRAME)[::HOP][:K - 1] * w


def bands_of_frames(fr):
    """[M][256] windowed frames -> [15][M] third-octave band magnitudes in float64."""
    p = np.abs(np.fft.rfft(fr, NFFT, axis=1)) ** 2
    return np.sqrt(np.stack([p[:, EDGES[b]:EDGES[b + 1]].sum(axis=1) for b in range(NBANDS)]))


def bands(x10, kept):
    return bands_of_frames(stft_frames(x10, kept))


def band_edges_argmin(fs=10000, nfft=NFFT, num_bands=NBANDS, min_freq=150):
    """The usual third-octave construction: the bins nearest to 150 * 2^((2k - 1) / 6) Hz, k = 0..15."""
    f = np.linspace(0, fs, nfft + 1)[:nfft // 2 + 1]
    k = np.arange(num_bands + 1)
    lo = min_freq * 2.0 ** ((2 * k - 1) / 6.0)
    return np.array([int(np.argmin((f - v) ** 2)) for v in lo])


def _normalise(v, axis):
    """Centre and divide by norm + EPS along `axis`, sums in index order (the kernel's)."""
    v = np.moveaxis(np.array(v, np.float64), axis, -1)
    n = v.shape[-1]
    m = np.zeros(v.shape[:-1])
    for i in range(n):
        m = m + v[..., i]
    m = m / n
    d = v - m[..., None]
    q = np.zeros(v.shape[:-1])
    for i in range(n):
        q = q + d[..., i] * d[..., i]
    return np.moveaxis(d / (np.sqrt(q) + EPS)[..., None], -1, axis)


def score(bx, by):
    """STOI and ESTOI of [15][M] band matrices (any float dtype, taken as float64) -> (stoi, estoi, S)."""
    bx, by = np.asarray(bx, np.float64), np.asarray(by, np.float64)
    M = bx.shape[1]
    S = M - NSEG + 1
    if S < 1:
        return float("nan"), float("nan"), 0
    X = np.lib.stride_tricks.sliding_window_view(bx, NSEG, axis=1)[:, :S].transpose(1, 0, 2)  # [S][15][30]
    Y = np.lib.stride_tricks.sliding_window_view(by, NSEG, axis=1)[:, :S].transpose(1, 0, 2)
    z = np.zeros(X.shape[:2])
    nx, ny = z.copy(), z.copy()
    for i in range(NSEG):
        nx = nx + X[..., i] * X[..., i]
        ny = ny + Y[..., i] * Y[..., i]
    alpha = np.sqrt(nx) / (np.sqrt(ny) + EPS)
    Yc = np.minimum(alpha[..., None] * Y, CLIP * X)
    mx, my = z.copy(), z.copy()
    for i in range(NSEG):
        mx = mx + X[..., i]
        my = my + Yc[..., i]
    mx, my = mx / NSEG, my / NSEG
    sxy, sxx, syy = z.copy(), z.copy(), z.copy()
    for i in range(NSEG):
        dx, dy = X[..., i] - mx, Yc[..., i] - my
        sxy = sxy + dx * dy
        sxx = sxx + dx * dx
        syy = syy + dy * dy
    stoi = sxy / ((np.sqrt(sxx) + EPS) * (np.sqrt(syy) + EPS))
    xh = _normalise(_normalise(X, 2), 1)
    yh = _normalise(_normalise(Y, 2), 1)
    prod = np.zeros((S, NSEG))
    for b in range(NBANDS):
        prod = prod + xh[:, b, :] * yh[:, b, :]
    return float(stoi.sum() / (NBANDS * S)), float(prod.sum() / (NSEG * S)), S


def intelligibility(out, clean, rate):
    """The whole definition in float64 (bands rounded to float32 as specified) -> dict of the record's fields and the
    stages."""
    h = filter_taps(rate)
    x10, y10 = resample(clean, rate, h), resample(out, rate, h)
    kept = kept_frames(x10)
    bx, by = bands(x10, kept), bands(y10, kept)
    s, e, S = score(bx.astype(np.float32), by.astype(np.float32))
    F = sizes(len(clean), rate)[4]
    return dict(stoi=s, estoi=e, frames=F, kept=len(kept), segments=S, x10=x10, y10=y10, kept_list=kept, bx=bx, by=by)
