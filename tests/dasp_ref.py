"""Float64 restatement of the file resampler (dasp_interpolate 0.11.0 `Sinc<[f32; 16]>` driven by Resample::next_sample,
csrc/frontend.cuh), with every tap's f32 rounding certified.

Output k of a source x [n][C] is Sinc::interpolate at (m_k, pos_k), where m_k source frames have been pushed and pos_k
is the fractional position (pos_table).  Each tap is first * second * frame in float64, rounded to f32, and the taps
are summed in f32 in the order left(n), right(n).  The only arithmetic that is not fully specified is `sin` and `cos`:
the oracle calls glibc's, the kernel CUDA's (documented at 2 ulp for double sin and cos), and this restatement
numpy's, which may run SIMD code of a few ulps.  So every tap is widened to an interval that covers a disagreement of
up to 2^-46 in `first` (relative: sin's error is relative to its result) and in `second` (absolute: it goes to 0 at the
window's edge, where a relative bound would say nothing), together with the tap's own two roundings:

    |tap' - tap| <= 2^-46 * (|first * frame| + |tap|)

A tap is *ambiguous* when that interval holds an f32 rounding boundary, i.e. its two ends round to different floats.
A sample without ambiguous taps has exactly one correct f32 value; a sample with some has a candidate set, the f32 sums
over each ambiguous tap's two roundings.
"""
import itertools
import math

import numpy as np

DEPTH, LEN = 8, 16
EPS = 2.0 ** -46
RATIOS = (8000, 11025, 16000, 22050, 44100, 47999, 48001, 96000, 192000)   # over 48000
LONG_N = 2 ** 23 + 12345


_TABLES = {}


def pos_table(ratio, n_in):
    """(m, pos) per output sample of a source of n_in frames: Resample::next_sample's `pos += ratio; while pos >= 1
    { pos -= 1; push }`, until a push would need frame n_in.  The recurrence does not depend on n_in, so the table of
    the longest source asked for so far serves the shorter ones; it is a sequential loop, run once per ratio."""
    ratio = float(ratio)
    if not ratio > 0.0:
        return np.zeros(0, np.int64), np.zeros(0)
    if ratio not in _TABLES or _TABLES[ratio][0] < n_in:
        pos, m, M, P = 0.0, 0, [], []
        while True:
            pos += ratio
            while pos >= 1.0:
                pos -= 1.0
                m += 1
            if m > n_in:
                break
            M.append(m)
            P.append(pos)
        _TABLES[ratio] = (n_in, np.array(M, np.int64), np.array(P, np.float64))
    _, M, P = _TABLES[ratio]
    k = int(np.searchsorted(M, n_in, side="right"))
    return M[:k], P[:k]


def _f32(v):
    with np.errstate(over="ignore"):
        return v.astype(np.float32)


def taps(x, M, P, ks):
    """Taps of output samples ks of source x [n][C] float32, in summation order: (t32, alt, amb), each [len(ks)][16][C].
    t32 is the f32 rounding of this restatement's f64 tap, alt the other candidate where amb (the certified interval
    holds an f32 boundary).  Inactive steps (n >= max_depth) are +0, which leaves an f32 sum unchanged."""
    x = np.asarray(x, np.float32)
    K, C = len(ks), x.shape[1]
    m = M[ks]
    phil = P[ks]
    phir = 1.0 - phil
    idx = np.minimum(m, DEPTH)
    nl, nr = idx, idx + 1
    md = np.where(nl + DEPTH >= LEN, LEN - DEPTH, np.where(nr - DEPTH < 0, DEPTH + nr - DEPTH, DEPTH))
    xz = np.concatenate([np.zeros((1, C)), x.astype(np.float64)])   # row 0: the ring's initial zeros
    t32 = np.zeros((K, 2 * DEPTH, C), np.float32)
    alt = np.zeros_like(t32)
    amb = np.zeros(t32.shape, bool)
    for n in range(DEPTH):
        for side, (ph, j) in enumerate(((phil, nl - n), (phir, nr + n))):
            a = math.pi * (ph + float(n))
            with np.errstate(divide="ignore", invalid="ignore"):
                first = np.where(a == 0.0, 1.0, np.sin(a) / a)
            second = 0.5 + 0.5 * np.cos(a / float(DEPTH))
            si = m - LEN + (j & (LEN - 1))
            fr = xz[np.where((si >= 0) & (n < md), si + 1, 0)]   # an inactive step (n >= max_depth) reads a zero
            tap = (first * second)[:, None] * fr
            err = EPS * (np.abs(first[:, None] * fr) + np.abs(tap))
            lo, hi, mid = _f32(tap - err), _f32(tap + err), _f32(tap)
            s = 2 * n + side
            t32[:, s] = mid
            amb[:, s] = lo != hi
            alt[:, s] = np.where(mid == lo, hi, lo)
    return t32, alt, amb


def _sum(t):
    v = np.zeros((t.shape[0], t.shape[2]), np.float32)
    for s in range(t.shape[1]):
        v = v + t[:, s]
    return v


def interpolate(x, ratio, ks=None, M=None, P=None):
    """The restatement at output samples ks (None: all) of source x [n][C] (or [n]) at `ratio` = input rate / 48000.
    Returns (value [K][C] float32, amb [K][C] bool, cands {(k, c): set of candidate values as float} for amb).

    f32 addition rounds monotonically, so every choice of an ambiguous tap's two roundings gives a sum between the sums
    of all the low and all the high choices.  Where those two are equal the sample has one correct value although some
    of its taps are ambiguous (a tap of 1e-30 next to one of 1e4).  Where they differ the sample is *ambiguous*, and
    its candidate set is the sums over every choice."""
    x = np.asarray(x, np.float32)
    if x.ndim == 1:
        x = x[:, None]
    if M is None:
        M, P = pos_table(ratio, x.shape[0])
    ks = np.arange(len(M)) if ks is None else np.asarray(ks, np.int64)
    vals, ambs, cands = [], [], {}
    for c0 in range(0, len(ks), 1 << 15):
        kc = ks[c0: c0 + (1 << 15)]
        t32, alt, amb = taps(x, M, P, kc)
        v = _sum(t32)
        a = _sum(np.where(amb, np.minimum(t32, alt), t32)) != _sum(np.where(amb, np.maximum(t32, alt), t32))
        for i, c in zip(*np.nonzero(a)):
            steps = np.nonzero(amb[i, :, c])[0]
            picks = np.array(list(itertools.product((0, 1), repeat=len(steps))), bool)   # [2^a][a]
            t = np.repeat(t32[i, :, c][None], len(picks), axis=0)
            t[:, steps] = np.where(picks, alt[i, steps, c], t32[i, steps, c])
            cands[(int(kc[i]), int(c))] = set(_sum(t[:, :, None])[:, 0].tolist())
        vals.append(v)
        ambs.append(a)
    C = x.shape[1]
    return (np.concatenate(vals) if vals else np.zeros((0, C), np.float32),
            np.concatenate(ambs) if ambs else np.zeros((0, C), bool), cands)


def check(got, x, ratio, ks=None):
    """Holds `got` (the outputs at ks, default all) to the restatement: equal bit for bit at every sample that is not
    ambiguous, inside the candidate set at the others.  Returns (ambiguous samples, those where `got` is not the
    restatement's own rounding)."""
    got = np.asarray(got, np.float32)
    if got.ndim == 1:
        got = got[:, None]
    ref, amb, cands = interpolate(x, ratio, ks)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    ks_ = np.arange(len(got)) if ks is None else np.asarray(ks)
    bad = np.nonzero(~amb & (got.view(np.uint32) != ref.view(np.uint32)))
    assert len(bad[0]) == 0, "%d certain samples differ, the first at (k, c) = (%d, %d): %r, restated %r" % (
        len(bad[0]), ks_[bad[0][0]], bad[1][0], got[bad[0][0], bad[1][0]], ref[bad[0][0], bad[1][0]])
    flips = 0
    for i, c in zip(*np.nonzero(amb)):
        cs = cands[(int(ks_[i]), int(c))]
        assert float(got[i, c]) in cs, (int(ks_[i]), int(c), float(got[i, c]), cs)
        flips += int(got[i, c] != ref[i, c])
    return int(amb.sum()), flips


def signal(n, ch, seed, scale=12000.0):
    """n frames of ch channels, each channel a different mix of tones and noise, rounded to int16 values."""
    rng = np.random.default_rng(seed)
    t = np.arange(n)[:, None]
    f = rng.uniform(0.001, 0.45, (1, ch))
    x = np.sin(2 * np.pi * f * t + rng.uniform(0, 6, (1, ch))) * scale * 0.6 + rng.standard_normal((n, ch)) * scale * 0.2
    return np.clip(np.round(x), -32768, 32767).astype(np.float32)


def cases():
    """(name, source [n][C] float32, ratio) of the file resampler's test list, the long source excepted."""
    out = []
    for r in RATIOS:
        out.append(("rate %d" % r, signal(12000, 1, seed=r), r / 48000.0))
    for n in (0, 1, 7, 15, 16, 17):
        for r in (8000, 44100, 96000):
            out.append(("n %d at %d" % (n, r), signal(n, 1, seed=100 + n), r / 48000.0))
    for C in (1, 2, 3, 300):
        out.append(("%d channels" % C, signal(1500 if C == 300 else 6000, C, seed=200 + C), 22050 / 48000.0))
    n = 6000
    full = np.full((n, 1), 32767.0, np.float32)
    full[::3] = -32768.0
    alt = np.where(np.arange(n) % 2 == 0, 32767.0, -32767.0).astype(np.float32)[:, None]
    zeros = signal(n, 1, seed=7)
    zeros[(np.arange(n) // 40) % 3 != 0] = 0.0
    tiny = (np.random.default_rng(8).standard_normal((n, 1)) * 1e-30).astype(np.float32)
    big = (np.random.default_rng(9).standard_normal((n, 1)) * 60000.0).astype(np.float32)
    for name, x in (("full scale", full), ("alternating", alt), ("zeros", zeros), ("1e-30", tiny), ("float beyond 32768", big)):
        for r in (44100, 16000, 96000):
            out.append(("%s at %d" % (name, r), x, r / 48000.0))
    return out
