"""CPU tests of the streaming stages' bit-exact restatement (resample_ref.fmaf / stages_bits): the fmaf emulation against
exact rational arithmetic on random triples and on constructed midpoint, cancellation and subnormal ones, and the
stage emulation against float64 upfirdn."""
from fractions import Fraction

import numpy as np
import pytest
from scipy.signal import upfirdn

import nnnoiseless_b200 as nb
from resample_ref import fmaf, pcm16, stages_bits


def f32_round(q):
    """The float32 nearest to the rational q, ties to even (q inside the finite range)."""
    f = np.float32(float(q))
    best = None
    for c in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
        d = abs(Fraction(float(c)) - q)
        if best is None or d < best[0] or (d == best[0] and int(np.array(c).view(np.uint32)) & 1 == 0):
            best = (d, c)
    return best[1]


def exact_fma(a, b, c):
    q = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if q == 0:
        neg = (np.signbit(a) != np.signbit(b)) and np.signbit(c) and (a == 0 or b == 0)
        return np.float32(-0.0 if neg else 0.0)
    return f32_round(q)


def check_triples(a, b, c):
    got = fmaf(a, b, c)
    want = np.array([exact_fma(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.nonzero(got.view(np.uint32) != want.view(np.uint32))


def test_fmaf_random_triples():
    rng = np.random.default_rng(1)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(np.float32)
    check_triples(a, b, c)


def test_fmaf_midpoints():
    """a b + c a hair off a float32 midpoint: s rounds to the midpoint in float64 and e's sign decides; a plain
    float64 -> float32 rounding would pick the even neighbour instead in half of these."""
    ks = np.arange(1, 300)
    a, b, c = [], [], []
    rng = np.random.default_rng(2)
    for k in ks:
        e = int(rng.integers(-20, 20))
        cv = np.float32((1 + int(rng.integers(0, 1 << 23)) * 2.0 ** -23) * 2.0 ** e)
        h = 2.0 ** (e - 24)                                   # half an ulp of c
        av = np.float32(1 + k * 2.0 ** -23)
        bv = np.float32(h * (1 - k * 2.0 ** -23))             # a b = h (1 - k^2 2^-46): just under the midpoint
        for sa, sc in ((1, 1), (-1, -1), (1, -1)):
            a.append(np.float32(sa * av)), b.append(bv), c.append(np.float32(sc * cv))
    a, b, c = (np.array(v, np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    s = p + c.astype(np.float64)
    assert np.mean(s.astype(np.float32).view(np.uint32) != fmaf(a, b, c).view(np.uint32)) > 0.2   # the ties matter
    check_triples(a, b, c)


def test_fmaf_cancellation_and_subnormals():
    rng = np.random.default_rng(3)
    n = 1000
    a = (rng.standard_normal(n) * 300).astype(np.float32)
    b = (rng.standard_normal(n) * 300).astype(np.float32)
    c = (-(a.astype(np.float64) * b.astype(np.float64))).astype(np.float32)      # a b + c is the product's rounding error
    check_triples(a, b, c)
    # products and sums below the normal range (2^-126): a build without flush-to-zero keeps them
    a = (rng.standard_normal(n) * 1e-20).astype(np.float32)
    b = (rng.standard_normal(n) * 1e-19).astype(np.float32)
    c = (rng.standard_normal(n) * 1e-39).astype(np.float32)
    assert np.mean(np.abs(fmaf(a, b, c)) < 2.0 ** -126) > 0.5
    check_triples(a, b, c)
    z = np.float32(0.0)
    check_triples(np.array([z, -z, 1e-45, -1e-45], np.float32), np.array([-z, -z, 0.5, 0.5], np.float32),
                  np.array([-z, z, z, -z], np.float32))


@pytest.mark.parametrize("rate", [8000, 8100, 11000, 44100, 47900])
@pytest.mark.parametrize("direction", [0, 1])
def test_stages_bits_are_upfirdn(rate, direction):
    """The emulated stage lies within a few f32 roundings of float64 upfirdn on the library's own taps."""
    nin = rate // 100 if direction == 0 else 480
    x = (np.random.default_rng(rate).standard_normal(4 * nin) * 4000.0).astype(np.float32)
    got = stages_bits([rate], direction, [x])[0].astype(np.float64)
    h, up, down = nb.resampler_filter(rate, direction)
    ref = upfirdn(h.astype(np.float64), x.astype(np.float64), up, down)[: len(got)]
    tol = 32 * 2.0 ** -24 * upfirdn(np.abs(h.astype(np.float64)), np.abs(x.astype(np.float64)), up, down)[: len(got)]
    assert np.all(np.abs(got - ref) <= tol)


def test_pcm16_rule():
    v = np.array([0.0, -0.0, 0.49999997, -0.49999997, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 32766.5, -32766.5, 32767.5, -32767.5,
                  32768.0, -32768.5, -32769.0, 1e30, -1e30, np.inf, -np.inf, np.nan], np.float32)
    assert pcm16(v).tolist() == [0, 0, 0, 0, 1, -1, 2, -2, 3, -3, 32767, -32767, 32767, -32768, 32767, -32768, -32768, 32767, -32768,
                                 32767, -32768, -32768]
