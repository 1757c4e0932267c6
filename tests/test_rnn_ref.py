"""CPU tests of the GRU network's test infrastructure and of the wgmma packing over model geometries: the float64
reference (tests/rnn_ref.py) against the oracle's f32 network step, and the wgmma packing self-test over every
geometry test_rnn_kernels.py runs on the GPU, zero-width layers included."""
import os
import subprocess
import sys

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle
import rnn_ref
from conftest import ROOT
from test_rnn_kernels import GEOMETRIES, ZERO_WIDTH, acts_for, model_for, pack_selftest

# the geometries whose layers fit the wgmma kernel's shared-memory and register budget (the rest, fixed rows and random
# ones alike, must be rejected with -2 and run on the mma.sync kernel)
FITS_WGMMA = {(24, 24, 48, 96), (1, 1, 1, 1), (5, 13, 37, 45), (56, 24, 56, 64), (12, 72, 12, 80), (24, 24, 48, 88),
              (24, 24, 40, 96), (80, 5, 80, 8)}
OVER_BUDGET = {(24, 24, 48, 97), (43, 42, 43, 127), (7, 78, 7, 127)}


def test_activations_match_oracle():
    xs = np.concatenate([np.linspace(-9, 9, 4001), [-8.0, 8.0, -7.98, 7.98, 0.02, -0.02, 0.0, np.nan]]).astype(np.float32)
    t = np.array([oracle.lib().nno_tansig(float(v)) for v in xs])
    s = np.array([oracle.lib().nno_sigmoid(float(v)) for v in xs])
    dt, ds = np.abs(rnn_ref.tansig(xs) - t), np.abs(rnn_ref.sigmoid(xs) - s)
    # the formula jumps by a few 1e-6 where the nearest table entry changes (25 |x| + 0.5 an integer): there f32 and
    # f64 may pick neighbouring entries; everywhere else they agree to f32 rounding
    def inner(u):
        v = 25.0 * np.abs(u.astype(np.float64)) + 0.5
        return np.abs(v - np.round(v)) > 1e-4
    assert dt[inner(xs)].max() < 1e-6 and ds[inner(0.5 * xs)].max() < 1e-6
    assert dt[~np.isnan(xs)].max() < 1e-5 and ds[~np.isnan(xs)].max() < 1e-5
    assert rnn_ref.tansig(np.float32(np.nan)) == 1.0


def test_make_model_is_accepted_and_extreme():
    for i, g in enumerate(GEOMETRIES):
        m = model_for(i)
        assert nb.RnnModel.from_bytes(m) is not None and oracle.model_accepts(m)
        layers = rnn_ref.parse(m)
        assert [L["nn"] for L in layers] == [g[0], g[1], g[2], g[3], 22, 1]
        assert [L["act"] for L in layers] == list(acts_for(i))
        for L in layers:
            for k in ("w", "r", "b"):
                if k in L and L[k].size >= 2:
                    assert L[k].min() == -128 and L[k].max() == 127
    # every layer sees tanh, sigmoid and ReLU somewhere in the sweep
    for layer in range(6):
        assert {acts_for(i)[layer] for i in range(len(GEOMETRIES))} == {0, 1, 2}


@pytest.mark.parametrize("gi", range(len(GEOMETRIES)), ids=["-".join(map(str, g)) for g in GEOMETRIES])
def test_float64_reference_against_oracle_f32_step(gi):
    """rnn_ref.step (float64) and the oracle's f32 rnn_compute agree to f32 rounding on random states and features,
    for every geometry under each of three activation assignments."""
    g = GEOMETRIES[gi]
    rng = np.random.default_rng(gi)
    B = 32
    for rot in range(3):
        m = rnn_ref.make_model(*g, acts=acts_for(gi + rot), seed=gi)
        layers, om = rnn_ref.parse(m), oracle.Model(m)
        state = rng.uniform(-1.0, 1.0, (B, sum(g[1:]))).astype(np.float32)
        feat = (3.0 * rng.standard_normal((B, 42))).astype(np.float32)
        ref = rnn_ref.step(layers, state, feat)
        f32 = rnn_ref.oracle_step(om, g[1:], state, feat)
        for r64, r32 in zip(ref, f32):
            assert r64.shape == r32.shape
            assert np.abs(r64 - r32).max(initial=0.0) <= 2e-5 * max(1.0, np.abs(r64).max(initial=0.0))
        # the network is not trivial: the outputs move with the state
        if sum(g[1:]):
            moved = rnn_ref.step(layers, state + np.float32(0.25), feat)
            assert not np.array_equal(moved[0], ref[0])


@pytest.mark.parametrize("gi", [i for i, g in enumerate(GEOMETRIES) if 0 not in g],
                         ids=["-".join(map(str, g)) for g in GEOMETRIES if 0 not in g])
def test_wgmma_packing_selftest_over_geometries(gi):
    g, m = GEOMETRIES[gi], model_for(gi)
    for seed in range(4):
        r = pack_selftest(m, seed)
        if g in FITS_WGMMA:
            assert 0.0 <= r < 2e-5, (seed, r)
        elif g in OVER_BUDGET:
            assert r == -2.0
        else:
            assert r == -2.0 or 0.0 <= r < 2e-5, (seed, r)


def test_wgmma_packing_of_zero_width_layers(tmp_path):
    """A layer of 0 neurons once made the wgmma packing divide by zero (SIGFPE inside rnnoise_batch_create).  Such a
    model now falls back to the mma.sync kernel (-2).  Each runs in a child process, so that a crash is reported
    instead of ending the test session."""
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "from test_rnn_kernels import pack_selftest\n"
            "print(pack_selftest(open(sys.argv[1], 'rb').read()))\n") % (ROOT, os.path.join(ROOT, "tests"))
    assert len(ZERO_WIDTH) >= 4
    for g in ZERO_WIDTH:
        p = tmp_path / "m.rnn"
        p.write_bytes(model_for(GEOMETRIES.index(g)))
        r = subprocess.run([sys.executable, "-c", code, str(p)], capture_output=True, text=True, cwd=ROOT, timeout=120)
        assert r.returncode == 0, (g, r.returncode, r.stderr[-2000:])
        assert float(r.stdout.split()[-1]) == -2.0, g
