"""CPU tests of the file resampler's restatement (tests/dasp_ref.py) against the oracle's Sinc::interpolate: bit for bit
at every sample that is not certified ambiguous, inside the candidate set at the others.  These hold the restatement
that tests/test_dasp_resampler.py holds the GPU kernel to."""
import numpy as np
import pytest

import dasp_ref
import oracle

CASES = dasp_ref.cases()


@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_restatement_is_the_oracle(case):
    name, x, ratio = CASES[case]
    want = oracle.resample(x, ratio)
    M, _ = dasp_ref.pos_table(ratio, x.shape[0])
    assert want.shape == (len(M), x.shape[1])
    n_amb, flips = dasp_ref.check(want, x, ratio)
    print("%s: %d outputs, %d ambiguous, %d off the restatement's rounding" % (name, want.size, n_amb, flips))
    # only the zero runs at 16 kHz put a window edge's tap (cos near -1) alone in a sum
    assert n_amb == (50 if name == "zeros at 16000" else 0)


def test_restatement_is_the_oracle_on_a_long_source():
    """2^23 + 12,345 source frames at 44.1 kHz: the position table over millions of steps, checked at the first and
    last outputs and at 4,000 sampled ones."""
    x = dasp_ref.signal(dasp_ref.LONG_N, 1, seed=5)
    ratio = 44100 / 48000.0
    want = oracle.resample(x, ratio)
    M, P = dasp_ref.pos_table(ratio, len(x))
    assert len(M) == len(want) and M[-1] <= len(x)
    ks = np.unique(np.concatenate([np.arange(20), np.random.default_rng(0).integers(0, len(M), 4000), np.arange(len(M) - 20, len(M))]))
    assert dasp_ref.check(want[ks], x, ratio, ks=ks) == (0, 0)


def test_candidate_sets_are_honest():
    """One nonzero frame: at exactly one output it is the window edge's tap (`second` near 0) alone in its sum.  The
    certification marks that sample, and only that one, ambiguous and offers both roundings."""
    ratio = 16000 / 48000.0
    x = np.zeros((64, 1), np.float32)
    x[20] = 30000.0
    v, amb, cands = dasp_ref.interpolate(x, ratio)
    assert amb.sum() == 1
    for k in np.nonzero(amb[:, 0])[0]:
        assert len(cands[(int(k), 0)]) >= 2 and float(v[k, 0]) in cands[(int(k), 0)]
    want = oracle.resample(x, ratio)
    assert dasp_ref.check(want, x, ratio)[1] == 0
