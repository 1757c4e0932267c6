"""The two GRU network kernels (wgmma rnn_tc.cu, mma.sync rnn_mma.cu) against a float64 restatement of
the network (tests/rnn_ref.py), one step at a time, over model geometries that reach every wgmma phase width, the
padding guards of layers that are not multiples of 8, weight-ring sequences that do not start at ring stage 0, models
over the wgmma budget (which run on the mma.sync kernel) and layers of zero neurons.

Each frame, the reference starts from the state the GPU left after the previous frame and takes the GPU's own
features, so errors do not compound and the FFT plays no part; the GPU's new state, raw gains and vad must match.
The yardstick is the reference's own f32 arithmetic (the oracle's rnn_compute) on the same inputs: with d32 its
largest deviation from float64 in a frame, the GPU's must stay within max(K * d32, FLOOR).  On an H100 (80GB HBM3,
400 W power limit) no kernel and geometry used more than 23 % of max(16 d32, 2e-6) (largest errors: state 2.2e-5 at
|state| ~ 10, gains 4.9e-6, vad 3.7e-7), so K = 8 and FLOOR = 1e-6 leave a factor of two.  f16-only activations (no lo half) exceed this
tolerance some 200-fold, a reset gate that reads the update gate's bias more than 2,500-fold.  Streams whose frame is silent
must keep their state bit for bit and report vad 0."""
import ctypes as C
import os
from contextlib import contextmanager

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle
import rnn_ref
from conftest import synth_streams

K, FLOOR = 8.0, 1e-6

# (nd, nv, nn, ndn): the built-in shape; every wgmma phase width 16 ... 192; widths that are not multiples of 8; slab
# counts 17, 25, 26 and 31 (not multiples of the 3 ring stages); models over the wgmma budget; zero-width layers
GEOMETRIES = [(24, 24, 48, 96), (1, 1, 1, 1), (5, 13, 37, 45), (56, 24, 56, 64), (12, 72, 12, 80), (24, 24, 48, 88),
              (24, 24, 40, 96), (80, 5, 80, 8), (24, 24, 48, 97), (43, 42, 43, 127), (7, 78, 7, 127),
              (0, 24, 48, 96), (24, 0, 48, 96), (24, 24, 0, 96), (24, 24, 48, 0)]


def _random_geometries(n, seed=2026):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        nd, nv = rng.integers(0, 86, size=2)
        nn, ndn = rng.integers(1, 86), rng.integers(1, 128)
        if 42 + nd + nv <= 127 and 42 + nv + nn <= 127:
            out.append((int(nd), int(nv), int(nn), int(ndn)))
    return out


GEOMETRIES += _random_geometries(4)
ZERO_WIDTH = [g for g in GEOMETRIES if 0 in g]


def acts_for(i):
    """Activations of the six layers for geometry i: rotating through tanh, sigmoid and ReLU, so that every layer sees
    each of the three in the sweep."""
    return tuple((i + layer) % 3 for layer in range(6))


def model_for(i):
    return rnn_ref.make_model(*GEOMETRIES[i], acts=acts_for(i), seed=100 + i)


def pack_selftest(model: bytes, seed=0) -> float:
    """The wgmma packing replayed on the host: >= 0 the largest deviation (the model runs on the wgmma kernel), -2 the
    model does not fit the wgmma budget (it runs on the mma.sync kernel)."""
    L = nb.lib()
    L.nnb_tc_pack_selftest.restype = C.c_double
    L.nnb_tc_pack_selftest.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    return L.nnb_tc_pack_selftest(model, len(model), seed)


KERNELS = {"default": {}, "mma": {"NNB_RNN_MMA": "1"}}


@contextmanager
def env(**kv):
    """The kernel selection is read from the environment when a batch is created."""
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def run_frames(model: bytes, x, kernel):
    """x [T][B][480] one frame per call on a fresh batch -> per frame dict(prev, gru_state, gains, vad, features,
    silence, vad_out): the GRU state before and after the frame, the raw network outputs, the features the network
    read, the silence flags and the vad the process call returned."""
    with env(**KERNELS[kernel]):
        batch = nb.DenoiseBatch(x.shape[1], nb.RnnModel.from_bytes(model))
    prev = np.zeros((x.shape[1], sum(batch.gru_widths)), np.float32)
    frames = []
    for f in range(len(x)):
        _, vad_out = batch.process_host(x[f:f + 1])
        t, r = batch.taps(), batch.rnn_taps()
        frames.append(dict(prev=prev, features=t["features"], silence=t["silence"], vad_out=vad_out[0], **r))
        prev = r["gru_state"]
    return frames


def one_step_errors(model: bytes, frames, tile=None):
    """Checks every frame against one float64 step from the GPU's previous state.  Returns the largest GPU error and
    the largest K * d32 / FLOOR ratio of each output over all frames, {name: (error, ratio)}; with `tile`, the errors
    of each `tile`-stream block are checked separately too."""
    layers, omodel = rnn_ref.parse(model), oracle.Model(model)
    widths = (layers[1]["nn"], layers[2]["nn"], layers[3]["nn"])
    worst = {q: (0.0, 0.0) for q in ("gru_state", "gains", "vad")}
    for f, fr in enumerate(frames):
        sil = fr["silence"] != 0
        # silent frames: the network leaves the state alone, bit for bit, and the stream reports vad 0
        assert np.array_equal(fr["gru_state"][sil].view(np.uint32), fr["prev"][sil].view(np.uint32)), f
        assert not fr["vad_out"][sil].any(), f
        live = np.flatnonzero(~sil)
        if not len(live):
            continue
        ref = rnn_ref.step(layers, fr["prev"][live], fr["features"][live])
        f32 = rnn_ref.oracle_step(omodel, widths, fr["prev"][live], fr["features"][live])
        for q, r64, r32 in zip(("gru_state", "gains", "vad"), ref, f32):
            if not r64.size:
                continue
            got = fr[q][live].astype(np.float64)
            assert np.isfinite(got).all(), (f, q)
            err = np.abs(got - r64).reshape(len(live), -1).max(axis=1)
            tol = max(K * float(np.abs(r32 - r64).max()), FLOOR)
            e = float(err.max())
            worst[q] = (max(worst[q][0], e), max(worst[q][1], e / tol))
            if tile:
                for t0 in np.unique(live // tile):
                    assert err[live // tile == t0].max() <= tol, (f, q, int(t0), tol)
    return worst


def streams(B, T, seed):
    """[T][B][480]: every 11th stream digitally silent from the start; every 23rd from the 5th a quiet stream that
    goes digitally silent after frame 3 (the high-pass filter's tail makes it silent a few frames later)."""
    x = synth_streams(B, T, seed=seed).reshape(B, T, 480)
    x[::11] = 0.0
    fading = np.arange(5, B, 23)
    x[fading] *= 0.05
    x[fading, 3:] = 0.0
    return np.ascontiguousarray(x.transpose(1, 0, 2)), fading


@pytest.mark.gpu
@pytest.mark.parametrize("gi", range(len(GEOMETRIES)), ids=["-".join(map(str, g)) for g in GEOMETRIES])
def test_gru_kernels_one_step_against_float64(gi):
    """B = 229 streams: a partial last tile for the 64-stream wgmma tiles and the 32-stream mma.sync tiles."""
    model = model_for(gi)
    B, T = 229, 12
    x, fading = streams(B, T, seed=900 + gi)
    fit = pack_selftest(model)
    assert fit >= 0 or fit == -2
    wgmma = fit >= 0  # else the default is the mma.sync kernel: checked below, bit for bit
    results, worst = {}, {}
    for kernel in KERNELS:
        frames = run_frames(model, x, kernel)
        assert frames[0]["silence"][::11].all() and frames[-1]["silence"][fading].all()
        assert not frames[0]["silence"][1::11].any()
        results[kernel] = frames
        worst[kernel] = one_step_errors(model, frames)
        name = kernel if kernel != "default" else ("wgmma" if wgmma else "default=mma")
        print("%-11s %-18s" % (name, GEOMETRIES[gi]),
              ", ".join("%s %.2e (%.2f of tol)" % (q, e, r) for q, (e, r) in worst[kernel].items()))
    for kernel, w in worst.items():
        assert all(r <= 1.0 for _, r in w.values()), (kernel, w)
    if not wgmma:  # a model over the wgmma budget runs on the mma.sync kernel: the same bits
        for a, b in zip(results["default"], results["mma"]):
            for q in ("gru_state", "gains", "vad"):
                assert np.array_equal(a[q], b[q])
