"""Float64 restatement of the streaming resampler stages (include/rnnoise.h, DESIGN.md 7g), frame by frame with the
input history carried from call to call.

A stage at stream rate R is scipy.signal.upfirdn(h, x, up, down): up (R -> 48 kHz) has up = 48000/g, down = R/g, the
down stage the mirror, g = gcd(48000, R), and h = firwin(20 max + 1, 1 / max, window=('kaiser', 5.0)) * up.  Every
frame of R/100 (or 480) input samples gives 480 (or R/100) output samples, so a frame's output is the upfirdn of the
frame with enough of the previous input in front of it."""
import math

import numpy as np
from scipy.signal import firwin, upfirdn

RATES = (8000, 12000, 16000, 24000, 32000, 44100, 48000)


def factors(rate, direction):
    """(up, down) of the up (direction 0) or down (1) stage."""
    g = math.gcd(48000, int(rate))
    U, D = 48000 // g, int(rate) // g
    return (U, D) if direction == 0 else (D, U)


def filter64(rate, direction):
    """resample_poly's default filter of the stage in float64: (h, up, down).  48 kHz: the identity."""
    up, down = factors(rate, direction)
    if up == down:
        return np.ones(1), 1, 1
    M = max(up, down)
    return firwin(20 * M + 1, 1.0 / M, window=("kaiser", 5.0)) * up, up, down


class Stage:
    """One stream's stage.  process(x) takes any whole number of frames and returns their output, in float64; the
    history is the last `hist` input samples, a multiple of `down` long so that the outputs of the history line up."""

    def __init__(self, rate, direction, h=None):
        h64, self.up, self.down = filter64(rate, direction)
        self.h = np.asarray(h64 if h is None else h, np.float64)
        self.nin, self.nout = (int(rate) // 100, 480) if direction == 0 else (480, int(rate) // 100)
        need = -(-(len(self.h) - 1) // self.up)
        self.hist_len = -(-need // self.down) * self.down
        self.hist = np.zeros(self.hist_len)

    def process(self, x):
        x = np.asarray(x, np.float64).reshape(-1)
        assert len(x) % self.nin == 0
        n_out = len(x) // self.nin * self.nout
        if self.up == self.down:
            return x.copy()
        xx = np.concatenate([self.hist, x])
        skip = self.hist_len * self.up // self.down
        y = upfirdn(self.h, xx, self.up, self.down)[skip: skip + n_out]
        self.hist = xx[len(xx) - self.hist_len:]
        return y


def stream(rate, direction, x, chunks=None, h=None):
    """The stage's output for x fed in calls of `chunks` frames each (None: one call)."""
    st = Stage(rate, direction, h)
    x = np.asarray(x, np.float64).reshape(-1)
    step = (chunks or (len(x) // st.nin)) * st.nin
    return np.concatenate([st.process(x[i: i + step]) for i in range(0, len(x), step)])


# ---- the stages' f32 arithmetic, bit for bit --------------------------------------------------------------------------
def fmaf(a, b, c):
    """fmaf(a, b, c) on float32 arrays, exactly: a * b is exact in float64, TwoSum gives a * b + c = s + e exactly, and
    s rounds to the correctly rounded float32 except where s is an exact float32 midpoint and e != 0, where the sign of
    e decides."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    with np.errstate(over="ignore", invalid="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        r = s.astype(np.float32)
        big = np.float64(2.0 ** 128)   # where float32 rounding overflows, inf stands for 2^128 in the distances
        r64 = np.where(np.isinf(r), np.copysign(big, r), r.astype(np.float64))
        other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        o64 = np.where(np.isinf(other), np.copysign(big, other), other.astype(np.float64))
        tie = np.isfinite(s) & (r64 != s) & (np.abs(s - r64) == np.abs(o64 - s)) & (e != 0)
        toward = (o64 > r64) == (e > 0)
    return np.where(tie & toward, other, r).astype(np.float32)


def fma_chain(H, X, h0, hstep, x0, nt):
    """acc = 0; for m < nt: acc = fmaf(H[h0 + m hstep], X[x0 - m], acc), per element of the index arrays."""
    order = np.argsort(-nt, kind="stable")            # longest chains first: step m works on a prefix
    h0, hstep, x0, nt = h0[order], hstep[order], x0[order], nt[order]
    acc = np.zeros(len(h0), np.float32)
    for m in range(int(nt[0]) if len(nt) else 0):
        k = int(np.count_nonzero(nt > m))
        acc[:k] = fmaf(H[h0[:k] + m * hstep[:k]], X[x0[:k] - m], acc[:k])
    out = np.empty_like(acc)
    out[order] = acc
    return out


def stages_bits(rates, direction, xs, hists=None):
    """The kernels' output of the up (direction 0) or down (1) stage, bit for bit, for streams at `rates` fed xs[s]
    (float32, whole frames: R/100 samples each up, 480 down) after the stage history hists[s] (None: zeros).  Output i
    of a frame is the fmaf chain over ascending m of h[p + m up] * x[j0 - m], i down = j0 up + p, from 0, with h the
    library's own f32 taps (nb.resampler_filter).  48 kHz streams pass through."""
    import nnnoiseless_b200 as nb
    hist_len = 20 if direction == 0 else 120
    Hs, Xs, idx, outs, h_off, x_off = [], [], [], [], 0, 0
    for s, R in enumerate(rates):
        x = np.asarray(xs[s], np.float32)
        h, up, down = nb.resampler_filter(int(R), direction)
        nin, nout = (R // 100, 480) if direction == 0 else (480, R // 100)
        n_out = len(x) // nin * nout
        if up == down:
            outs.append(("copy", x[:n_out].copy()))
            continue
        hist = np.zeros(hist_len, np.float32) if hists is None or hists[s] is None else np.asarray(hists[s], np.float32)
        i = np.arange(n_out, dtype=np.int64)
        j0, p = np.divmod(i * down, up)
        nt = (len(h) - 1 - p) // up + 1
        idx.append((h_off + p, up, x_off + hist_len + j0, nt))
        outs.append(("chain", n_out))
        Hs.append(h)
        Xs.append(np.concatenate([hist, x]))
        h_off += len(h)
        x_off += hist_len + len(x)
    if idx:
        H, X = np.concatenate(Hs), np.concatenate(Xs)
        h0 = np.concatenate([a for a, _, _, _ in idx])
        hs = np.concatenate([np.full(len(a), u, np.int64) for a, u, _, _ in idx])
        x0 = np.concatenate([c for _, _, c, _ in idx])
        nt = np.concatenate([d for _, _, _, d in idx])
        flat = fma_chain(H, X, h0, hs, x0, nt)
    res, k = [], 0
    for kind, v in outs:
        if kind == "copy":
            res.append(v)
        else:
            res.append(flat[k: k + v])
            k += v
    return res


def pcm16(v):
    """The int16 conversion of the Rust front-end, `x.max(-32768.).min(32767.).round() as i16`, in float64: NaN gives
    -32768 (f32::max returns the other operand), ties go away from zero."""
    v = np.asarray(v, np.float32).astype(np.float64)
    v = np.where(np.isnan(v), -32768.0, np.minimum(np.maximum(v, -32768.0), 32767.0))
    return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int16)
