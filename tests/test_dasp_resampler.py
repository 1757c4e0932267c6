"""GPU tests of the file resampler (rnnoise_resample_host -> resample_kernel / dasp_sample, csrc/frontend.cuh) sample by
sample: every output equals the oracle bit for bit, except at samples tests/dasp_ref.py certifies ambiguous (CUDA's and
glibc's sin/cos a few ulps apart), where it must be one of the certified candidates.  Cases: nine ratios, sources of 0
to 17 frames, the output cap, 1 to 300 interleaved channels, edge values and a source of 2^23 + 12,345 frames."""
import ctypes as C

import numpy as np
import pytest

import dasp_ref
import nnnoiseless_b200 as nb
import oracle
from nnnoiseless_b200 import files

pytestmark = pytest.mark.gpu

CASES = dasp_ref.cases()


def resample_host(x, ratio, cap):
    """rnnoise_resample_host with an explicit cap; rows past the returned count keep their NaN fill."""
    x = np.ascontiguousarray(x, np.float32)
    out = np.full((max(cap, 1), x.shape[1]), np.nan, np.float32)
    k = nb.lib().rnnoise_resample_host(out.ctypes.data_as(C.c_void_p), cap, x.ctypes.data_as(C.c_void_p), x.shape[0], x.shape[1],
                                       float(ratio), -1)
    assert k >= 0, nb.last_error()
    return k, out


@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_resampler_is_the_oracle(case):
    name, x, ratio = CASES[case]
    got = files.resample(x, ratio)
    want = oracle.resample(x, ratio)
    assert got.shape == want.shape
    n_amb, flips = dasp_ref.check(got, x, ratio)
    differ = int((got.view(np.uint32) != want.view(np.uint32)).sum())
    print("%s: %d outputs, %d ambiguous, %d off the restatement's rounding, %d differ from the oracle" % (
        name, got.size, n_amb, flips, differ))
    assert n_amb == (50 if name == "zeros at 16000" else 0)
    assert differ == flips == 0


@pytest.mark.parametrize("ratio", [8000 / 48000.0, 44100 / 48000.0, 96000 / 48000.0])
def test_startup_and_cap(ratio):
    """The first 17 outputs (the ring partly zeros, then the wrap of nr + n = 16 to the oldest frame), the output cap
    below, at and above the table's length, and the last output before the source runs dry."""
    x = dasp_ref.signal(300, 2, seed=31)
    M, _ = dasp_ref.pos_table(ratio, len(x))
    K = len(M)
    want = oracle.resample(x, ratio)
    for cap in (0, 1, 17, K - 1, K, K + 5):
        k, out = resample_host(x, ratio, cap)
        assert k == min(cap, K), (cap, k, K)
        assert out[:k].tobytes() == want[:k].tobytes(), cap
        assert np.isnan(out[k:]).all(), cap                   # nothing written past the count
    assert dasp_ref.check(want[:17], x, ratio, ks=np.arange(17)) == (0, 0)
    # one frame more lets exactly the outputs of the longer table through, and the shorter call's last output is the
    # longer one's at the same index
    longer = files.resample(np.concatenate([x, x[:1]]), ratio)
    assert len(longer) == len(dasp_ref.pos_table(ratio, len(x) + 1)[0]) and longer[:K].tobytes() == want.tobytes()


def test_channels_are_independent():
    """Channel c of a C-channel call is that channel resampled alone, bit for bit, for 1, 2, 3 and 300 channels."""
    ratio = 22050 / 48000.0
    for C_ in (2, 3, 300):
        x = dasp_ref.signal(900, C_, seed=40 + C_)
        got = files.resample(x, ratio)
        for c in range(C_):
            alone = files.resample(np.ascontiguousarray(x[:, c:c + 1]), ratio)
            assert got[:, c:c + 1].tobytes() == alone.tobytes(), (C_, c)


def test_long_source():
    """2^23 + 12,345 source frames at 44.1 kHz: the host's (int m, double pos) table follows the recurrence over
    9 million steps.  Every output equals the oracle's; any that did not would be checked against the candidates."""
    x = dasp_ref.signal(dasp_ref.LONG_N, 1, seed=5)
    ratio = 44100 / 48000.0
    got = files.resample(x, ratio)
    want = oracle.resample(x, ratio)
    assert got.shape == want.shape
    diff = np.nonzero(got[:, 0].view(np.uint32) != want[:, 0].view(np.uint32))[0]
    rng = np.random.default_rng(1)
    ks = np.unique(np.concatenate([diff, np.arange(20), rng.integers(0, len(got), 4000), np.arange(len(got) - 20, len(got))]))
    n_amb, flips = dasp_ref.check(got[ks], x, ratio, ks=ks)
    print("long source: %d outputs, %d differ from the oracle, %d ambiguous among %d checked" % (len(got), len(diff), n_amb, len(ks)))
    assert len(diff) == 0
