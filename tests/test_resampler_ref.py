"""CPU tests of the per-stream resampler's contract (include/rnnoise.h, DESIGN.md 7g): the library's filters are
resample_poly's, the float64 restatement of the streaming stages is scipy's upfirdn however the frames are split into
calls, the reported delay follows from the filter lengths, and bad rates are refused before any device is needed."""
import numpy as np
import pytest
from scipy.signal import upfirdn

import nnnoiseless_b200 as nb
from resample_ref import RATES, Stage, filter64, stream

ALL_RATES = tuple(range(8000, 48001, 100))   # every valid stream rate: 401


@pytest.mark.parametrize("direction", [0, 1])
@pytest.mark.parametrize("rate", ALL_RATES)
def test_filter_is_resample_poly_default(rate, direction):
    h, up, down = nb.resampler_filter(rate, direction)
    h64, up64, down64 = filter64(rate, direction)
    assert (up, down) == (up64, down64)
    assert h.dtype == np.float32 and h.shape == h64.shape
    if rate == 48000:
        assert h.tolist() == [1.0]
        return
    assert len(h) == 20 * max(up, down) + 1
    # designed in double, stored as float: at most one float ulp from scipy's double taps
    ulp = np.spacing(np.abs(h64).astype(np.float32)).astype(np.float64)
    assert np.all(np.abs(h.astype(np.float64) - h64) <= ulp)
    assert np.mean(h == h64.astype(np.float32)) > 0.99


@pytest.mark.parametrize("chunks", [1, 3, 7])
@pytest.mark.parametrize("direction", [0, 1])
@pytest.mark.parametrize("rate", RATES)
def test_restatement_is_upfirdn_prefix(rate, direction, chunks):
    T = 21
    st = Stage(rate, direction)
    x = np.random.default_rng(rate + direction).standard_normal(T * st.nin) * 1000.0
    y = stream(rate, direction, x, chunks)
    assert len(y) == T * st.nout
    ref = x if rate == 48000 else upfirdn(st.h, x, st.up, st.down)[: len(y)]
    np.testing.assert_allclose(y, ref, rtol=0, atol=1e-9 * np.abs(x).max())


@pytest.mark.parametrize("rate", ALL_RATES)
def test_delay_follows_filter_lengths(rate):
    hu, up_u, down_u = nb.resampler_filter(rate, 0)
    hd, up_d, down_d = nb.resampler_filter(rate, 1)
    # a symmetric filter of L taps delays by (L - 1) / 2 samples of the up-sampled rate, i.e. (L - 1) / (2 * 48000 / ...)
    # 48 kHz samples: the up stage's up-sampled rate is 48 kHz * down_u, the down stage's 48 kHz * up_d
    expect = (len(hu) - 1) / (2.0 * down_u) + (len(hd) - 1) / (2.0 * up_d)
    assert nb.resampler_delay(rate) == pytest.approx(expect, rel=1e-12, abs=0)
    assert nb.resampler_delay(rate) * rate / 48000.0 == pytest.approx(0 if rate == 48000 else 20, rel=1e-14)   # 20 native samples
    assert nb.resampler_delay(16000) == 60.0


@pytest.mark.parametrize("bad", [7900, 8050, 48100, 0])
def test_bad_rates_are_refused(bad):
    with pytest.raises(nb.NnnoiselessError, match="rate %d Hz" % bad):
        nb.resampler_filter(bad, 0)
    with pytest.raises(nb.NnnoiselessError, match="rate %d Hz" % bad):
        nb.resampler_delay(bad)
    # checked before the device is touched: the error names the stream, with or without a GPU
    with pytest.raises(nb.NnnoiselessError, match="stream 2: rate %d Hz" % bad):
        nb.Resampler(4, rates=[16000, 48000, bad, 8000])


def test_bad_arguments_are_refused():
    with pytest.raises(nb.NnnoiselessError, match="direction"):
        nb.resampler_filter(16000, 2)
    with pytest.raises(nb.NnnoiselessError, match="n_streams"):
        nb.Resampler(0)
