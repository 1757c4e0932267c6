"""The persistent analysis kernel (spectral_warp.cu): a warp takes streams w, w + G, w + 2G, ... of the batch and stages
each stream's history window and cepstral ring with bulk copies a round ahead.  Every case is checked two ways:
bit-identical outputs whatever the stream's position and the batch size, and parity with the oracle (pitch exact)."""
import numpy as np
import pytest

import oracle
import nnnoiseless_b200 as nb
from conftest import synth_streams
from test_gpu_parity import check_against_oracle

pytestmark = pytest.mark.gpu

# 12 frames: the history window starts in every one of the 8 ring slots, so it wraps at every place it can.
T = 12


def _pulses(period, amp=8000.0):
    x = np.zeros(T * 480, np.float32)
    x[::period] = amp
    return x


def _unique_streams():
    """37 streams (not a multiple of the warps per block): white + sine, pulse trains whose pitch is the smallest (60),
    odd (61), even (120) and largest (767) period the search returns, digital silence, and silence turning to signal."""
    sig = synth_streams(28, T, seed=31)
    rows = list(sig[:28])
    rows += [_pulses(60), _pulses(61), _pulses(120), _pulses(767), _pulses(767)]
    rows += [np.zeros(T * 480, np.float32)] * 2
    late = sig[0].copy()
    late[: 5 * 480] = 0.0
    rows += [late, np.zeros(T * 480, np.float32)]
    return np.stack(rows).reshape(len(rows), T, 480)


@pytest.fixture(scope="module")
def small(builtin_bytes):
    """The 37 streams as their own batch (far less than one wave of the persistent grid), frame by frame."""
    x = _unique_streams()
    U = x.shape[0]
    b = nb.DenoiseBatch(U)
    outs, vads, pitch, sil = [], [], [], []
    for t in range(T):
        o, v = b.process_host(np.ascontiguousarray(x[:, t][None]))
        outs.append(o[0])
        vads.append(v[0])
        tp = b.taps()
        pitch.append(tp["pitch"].copy())
        sil.append(tp["silence"].copy())
    return dict(x=x, out=np.stack(outs), vad=np.stack(vads), pitch=np.stack(pitch, 1), silence=np.stack(sil, 1),
                ref=oracle.run_batch(oracle.Model(builtin_bytes), x, n_threads=0))


def _positions(B, U, seed):
    """Stream at batch position s = unique stream perm[s]; every unique stream appears."""
    rng = np.random.default_rng(seed)
    perm = rng.integers(0, U, B)
    perm[:U] = np.arange(U)
    return perm


def test_small_batch_vs_oracle(small):
    ref = small["ref"]
    assert np.array_equal(small["pitch"], ref["pitch"])
    check_against_oracle(small["out"], small["vad"], None, ref, small["x"])
    p = small["pitch"][small["silence"] == 0]
    assert (p % 2 == 1).any() and (p % 2 == 0).any()
    assert p.min() == 60 and p.max() >= 765
    assert small["silence"].any() and not small["silence"].all()


def test_many_rounds_bitwise(small):
    """5,003 streams: every warp of the grid takes at least two streams, the last round is partial, and B is not a
    multiple of the warps per block.  Each position gives the bits of its stream in the small batch."""
    U = small["x"].shape[0]
    B = 5003
    perm = _positions(B, U, seed=1)
    x = np.ascontiguousarray(small["x"][perm].transpose(1, 0, 2))
    b = nb.DenoiseBatch(B)
    o, v = b.process_host(x)
    assert np.array_equal(o, small["out"][:, perm])
    assert np.array_equal(v, small["vad"][:, perm])
    assert np.array_equal(b.taps()["pitch"], small["pitch"][perm, -1])


def test_subset_call_bitwise(small):
    """Frames 0..5 for the whole batch, then frames 6.. for a subset through the work state."""
    U = small["x"].shape[0]
    B = 301
    perm = _positions(B, U, seed=2)
    x = np.ascontiguousarray(small["x"][perm].transpose(1, 0, 2))
    b = nb.DenoiseBatch(B)
    o0, _ = b.process_host(x[:6])
    assert np.array_equal(o0, small["out"][:6, perm])
    idx = np.arange(3, B, 7, dtype=np.int32)
    o1, v1 = b.process_streams_host(idx, np.ascontiguousarray(x[6:, idx]))
    assert np.array_equal(o1, small["out"][6:, perm[idx]])
    assert np.array_equal(v1, small["vad"][6:, perm[idx]])


def test_pcm16_output(small):
    """int16 in and out: the float path's output clamped to int16 and rounded half away from zero."""
    x16 = np.ascontiguousarray(small["x"].transpose(1, 0, 2)).astype(np.int16)
    assert np.array_equal(x16.astype(np.float32), small["x"].transpose(1, 0, 2))
    b = nb.DenoiseBatch(x16.shape[1])
    o, v = b.process_pcm16_host(x16)
    f = np.clip(small["out"], -32768.0, 32767.0)
    want = (np.sign(f) * np.floor(np.abs(f) + 0.5)).astype(np.int16)
    assert np.array_equal(o, want)
    assert np.array_equal(v, small["vad"])
