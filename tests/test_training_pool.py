"""Training rows from a WAV corpus on the GPU: rnnoise_train_process_pool_host against the float entry point bit for
bit, generate_rows against the oracle fed the frames the plan names, reproducibility, and the three commands
corpus -> rows -> .rnn -> denoised file."""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle
import nnnoiseless_b200 as nb
from nnnoiseless_b200 import NnnoiselessError
from nnnoiseless_b200 import training as tr
from nnnoiseless_b200.files import CLI_PATH, read_audio, write_audio
from nnnoiseless_b200.synth import synth_streams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _pool(n, seed):
    """int16 samples whose 480-sample stretches sweep the VAD thresholds (frame energies 1e6 .. 1e10)."""
    rng = np.random.default_rng(seed)
    amp = rng.choice([30.0, 300.0, 1000.0, 3000.0, 9000.0], size=n // 480 + 1).repeat(480)[:n]
    return np.clip(np.round(rng.normal(0.0, 1.0, n) * amp), -32768, 32767).astype(np.int16)


def _offsets(rng, T, L, pool_len):
    at = rng.integers(0, pool_len - 480 + 1, (T, L))
    at[rng.random((T, L)) < 0.05] = -1                 # frames of zeros
    at.flat[rng.integers(0, T * L, 3)] = pool_len - 480  # frames ending at the pool's last sample
    return at


def _floats(pool, at):
    x = pool[np.maximum(at, 0)[..., None] + np.arange(480)].astype(np.float32)
    x[at < 0] = 0.0
    return x


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


@pytest.mark.parametrize("L", [1, 63, 64, 65, 130])
def test_pool_rows_are_the_float_rows(L):
    rng = np.random.default_rng(L)
    T, pool_len = 14, 480 * 37 + 7
    pool = _pool(pool_len, L)
    sig_at, noise_at = _offsets(rng, T, L, pool_len), _offsets(rng, T, L, pool_len)
    assert (sig_at % 2 == 1).any()  # odd offsets: 2-byte aligned reads
    sig, noise = _floats(pool, sig_at), _floats(pool, noise_at)
    a, b = tr.TrainingBatch(L), tr.TrainingBatch(L)
    p1, p2 = tr.randomize(L, rng), tr.randomize(L, rng)
    p2["noise_gain"][0] = 0.0
    got, want = [], []
    for (f0, f1), prm in (((0, 5), None), ((5, 9), p1), ((9, T), p2)):  # parameters change between calls
        if prm is not None:
            a.set_params(prm)
            b.set_params(prm)
        got.append(a.process_pool_host(pool, sig_at[f0:f1], noise_at[f0:f1]))
        want.append(b.process_host(sig[f0:f1], noise[f0:f1]))
    assert np.array_equal(_bits(np.concatenate(got)), _bits(np.concatenate(want)))


def test_pool_call_across_the_staging_bound():
    L, T = 8192, 100  # rows staging holds 94 frames of 8192 lanes: one call, two chunks
    rng = np.random.default_rng(5)
    pool_len = 480 * 501 + 3
    pool = _pool(pool_len, 5)
    sig_at, noise_at = _offsets(rng, T, L, pool_len), _offsets(rng, T, L, pool_len)
    got = tr.TrainingBatch(L).process_pool_host(pool, sig_at, noise_at)
    b = tr.TrainingBatch(L)
    for f0 in range(0, T, 20):
        want = b.process_host(_floats(pool, sig_at[f0:f0 + 20]), _floats(pool, noise_at[f0:f0 + 20]))
        assert np.array_equal(_bits(got[f0:f0 + 20]), _bits(want)), f0


def test_pool_offsets_out_of_range_run_nothing():
    L, T = 5, 6
    rng = np.random.default_rng(9)
    pool_len = 480 * 20 + 1
    pool = _pool(pool_len, 9)
    sig_at, noise_at = _offsets(rng, T, L, pool_len), _offsets(rng, T, L, pool_len)
    t = tr.TrainingBatch(L)
    for arr, bad, what in ((sig_at, pool_len - 479, "sig_at"), (noise_at, -2, "noise_at"), (sig_at, pool_len, "sig_at")):
        x = arr.copy()
        x[3, 2] = bad
        args = (x, noise_at) if what == "sig_at" else (sig_at, x)
        with pytest.raises(NnnoiselessError, match="%s = %d at frame 3, lane 2" % (what, bad)):
            t.process_pool_host(pool, *args)
    assert nb.lib().rnnoise_train_process_pool_host(t._h, nb._np_ptr(np.empty(87, np.float32)), nb._np_ptr(pool), 1 << 28,
                                                    nb._np_ptr(sig_at), nb._np_ptr(noise_at), 1) != 0
    assert "pool_len" in nb.last_error()
    got = t.process_pool_host(pool, sig_at, noise_at)
    want = tr.TrainingBatch(L).process_pool_host(pool, sig_at, noise_at)
    assert np.array_equal(_bits(got), _bits(want))


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    """Speech-like (tone + noise with a slow on/off envelope) and noise WAV files; one of each long enough to seek in."""
    d = tmp_path_factory.mktemp("wavs")
    rng = np.random.default_rng(3)
    sig, noise = [], []
    for i, frames in enumerate((1500, 2300, 9000, 700)):
        x = synth_streams(1, frames, seed=40 + i)[0]
        env = np.repeat(rng.choice([0.02, 0.2, 1.0], size=frames // 50 + 1), 50 * 480)[:len(x)]
        p = str(d / ("speech%d.wav" % i))
        write_audio(p, np.clip(np.round(x * env), -32768, 32767).astype(np.int16), wav=True)
        sig.append(p)
    for i, frames in enumerate((2000, 8000, 1200)):
        p = str(d / ("noise%d.wav" % i))
        write_audio(p, np.round(rng.normal(0, rng.uniform(100, 2000), frames * 480)).astype(np.int16), wav=True)
        noise.append(p)
    return sig, noise


def test_corpus_rows_match_oracle(corpus):
    sig_paths, noise_paths = corpus
    L, count = 3, 3 * (2 * tr.RANDOMIZE_PERIOD + 40)  # two randomize frames per lane
    got = tr.generate_rows(sig_paths, noise_paths, count, lanes=L, seed=21)
    p = tr.plan(sig_paths, noise_paths, count, L, seed=21)
    assert got.shape == (p.n_frames, L, 87) and len(p.randomize) == 2
    assert any((s["offset"] > 0).any() for s in p.signal) and any((s["offset"] > 0).any() for s in p.noise)
    audio = {}

    def frames(kind, l):
        files, offs = p.frames_at(kind, l)
        paths = p.signal_paths if kind == "signal" else p.noise_paths
        for i in set(files.tolist()):
            if paths[i] not in audio:
                audio[paths[i]] = read_audio(paths[i])[0][:, 0]
        return np.stack([audio[paths[i]][o:o + 480] for i, o in zip(files, offs)])

    params = dict(p.randomize)
    want = np.empty_like(got)
    for l in range(L):
        t = oracle.Trainer()
        s, n = frames("signal", l), frames("noise", l)
        for f in range(p.n_frames):
            if f in params:
                t.set_params(params[f][l:l + 1])
            want[f, l] = t.frame(s[f], n[f])
    # test_training_rows_match_oracle's tolerances
    assert np.array_equal(got[:, :, 86], want[:, :, 86])
    gm, wm = got[:, :, 42:64] == -1.0, want[:, :, 42:64] == -1.0
    assert (gm != wm).mean() < 1e-3
    ok = ~(gm | wm)
    assert np.max(np.abs(got[:, :, 42:64][ok] - want[:, :, 42:64][ok])) < 1e-4
    assert np.max(np.abs(got[:, :, 64:86] - want[:, :, 64:86])) < 1e-4
    df = np.abs(got[:, :, :42] - want[:, :, :42])
    assert np.sqrt(np.mean(df[:, 2:] ** 2)) < 1e-4
    assert np.array_equal(got[:, :, 40], want[:, :, 40])
    assert set(np.unique(got[:, :, 86])) == {0.0, 0.5, 1.0}


def test_corpus_rows_reproducible(corpus, tmp_path):
    sig_paths, noise_paths = corpus
    kw = dict(count=3 * 3000, lanes=3, seed=8, shuffle=True)
    a, b, c = (str(tmp_path / n) for n in ("a.npy", "b.npy", "c.npy"))
    tr.generate_rows(sig_paths, noise_paths, out=a, **kw)
    tr.generate_rows(sig_paths, noise_paths, out=b, **kw)
    timings = {}
    tr.generate_rows(sig_paths, noise_paths, out=c, pool_bytes=3 * 2 * 480 * 2 * 97, timings=timings, **kw)
    assert timings["calls"] == -(-2821 // 97) + -(-(3000 - 2821) // 97)  # 97 frames a call, and a cut at the randomize frame
    data = [open(x, "rb").read() for x in (a, b, c)]
    assert data[0] == data[1] == data[2]
    assert np.load(a).shape == (3000, 3, 87)


def test_three_commands(corpus, tmp_path):
    sig_paths, noise_paths = corpus
    d = os.path.dirname(sig_paths[0])
    rows, weights = str(tmp_path / "rows.npy"), str(tmp_path / "weights.rnn")
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "nnnoiseless_b200.training", "--signal-glob", os.path.join(d, "speech*.wav"),
                        "--noise-glob", os.path.join(d, "noise*.wav"), "--count", "6000", "--lanes", "3", "--shuffle",
                        "-o", rows], capture_output=True, text=True, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    assert "Found 4 clean files, reading about 1501 frames from each" in r.stderr
    assert "Found 3 noise files, reading about 2001 frames from each" in r.stderr
    assert np.load(rows, mmap_mode="r").shape == (2000, 3, 87)
    r = subprocess.run([sys.executable, "-m", "nnnoiseless_b200.fit", rows, "--epochs", "1", "--window", "200", "-o", weights],
                       capture_output=True, text=True, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    src, out = sig_paths[0], str(tmp_path / "out.wav")
    r = subprocess.run([CLI_PATH, "--model", weights, src, out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    y, rate = read_audio(out)
    assert rate == 48000 and y.shape == ((1500 - 1) * 480, 1) and np.isfinite(y).all()
    with open(weights, "rb") as f:
        model = nb.RnnModel.from_bytes(f.read())
    batch = nb.DenoiseBatch(2, device=0)
    assert batch.add_model(model) == 1
    batch.set_stream_models([1], streams=[1])
    x = synth_streams(2, 10, seed=1).reshape(2, 10, 480).transpose(1, 0, 2)
    o, v = batch.process_host(np.ascontiguousarray(x))
    assert np.isfinite(o).all() and np.isfinite(v).all()
