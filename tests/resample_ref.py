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
