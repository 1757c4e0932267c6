"""Waveform windows without a GPU: the window offsets WaveformCorpus computes from a plan, the refusal of a corpus
that does not fit on the device, the C++ mirror, and null trainers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import NnnoiselessError
from nnnoiseless_b200 import training as tr
from nnnoiseless_b200.files import write_audio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def wavs(tmp_path_factory):
    d = tmp_path_factory.mktemp("wavs")
    rng = np.random.default_rng(1)
    out = []
    for kind, frames in (("s", (300, 1100, 90, 2600)), ("n", (700, 150, 1900))):
        paths = []
        for i, n in enumerate(frames):
            p = str(d / ("%s%d.wav" % (kind, i)))
            write_audio(p, rng.integers(-3000, 3000, n * 480 + i).astype(np.int16), wav=True)
            paths.append(p)
        out.append(paths)
    return out


@pytest.mark.parametrize("shuffle", [False, True])
def test_window_offsets_follow_the_plan(wavs, shuffle):
    """Offsets of windows that cut segments anywhere (and cross the randomize frame) are Plan.frames_at mapped through
    the pool's file bases."""
    sig_paths, noise_paths = wavs
    L = 4
    p = tr.plan(sig_paths, noise_paths, L * (tr.RANDOMIZE_PERIOD + 300), L, seed=3, shuffle=shuffle)
    assert p.randomize and all(len(s) > 2 for s in p.signal) and all(len(s) > 2 for s in p.noise)
    _, sig_len, _ = tr.probe_corpus(sig_paths)
    _, noise_len, _ = tr.probe_corpus(noise_paths)
    sig_base, noise_base, total = tr.pool_layout(sig_len, noise_len)
    assert total == sig_len.sum() + noise_len.sum() and sig_base[0] == 0 and noise_base[0] == sig_len.sum()
    base = {x: b for x, b in zip(sig_paths, sig_base)}, {x: b for x, b in zip(noise_paths, noise_base)}
    tables = []
    for k, kind in enumerate(("signal", "noise")):
        paths = p.signal_paths if kind == "signal" else p.noise_paths
        b = np.array([base[k][x] for x in paths], np.int64)
        tables.append(tr.segment_table(getattr(p, kind), b, p.n_frames))
        want = np.stack([b[f] + o for f, o in (p.frames_at(kind, l) for l in range(L))], axis=1)  # [F][L]
        assert (want >= 0).all() and (want + 480 <= total).all()
        assert want.max() + 480 <= (sig_len.sum() if kind == "signal" else total)
        got, f0 = [], 0
        rng = np.random.default_rng(k)
        while f0 < p.n_frames:
            n = int(rng.integers(1, 500))
            got.append(tr.window_offsets(tables[-1], f0, min(f0 + n, p.n_frames)))
            f0 += n
        assert np.array_equal(np.concatenate(got), want), kind


def test_corpus_that_does_not_fit_is_refused():
    hour = 3600 * 48000
    assert tr.HOUR_BYTES == 345_600_000
    tr.check_fits(hour, 2 * hour, 80 << 30, 7)  # exactly fits
    with pytest.raises(NnnoiselessError, match=r"7 files, 172800001 samples \(345.6 MB, 1.00 h at 48 kHz\).*345.6 MB free of 85899.3 MB"):
        tr.check_fits(hour + 1, 2 * hour, 80 << 30, 7)


def test_cpp_mirror_wave_methods_compile(tmp_path):
    inc, libdir = os.path.join(ROOT, "include"), os.path.join(ROOT, "nnnoiseless_b200", "lib")
    src = tmp_path / "t.cpp"
    src.write_text('#include "nnnoiseless.hpp"\n'
                   "void epoch(nnnoiseless::TrainingBatch& t, const short* pcm, long long n, const long long* at, float* noisy,\n"
                   "           float* clean, int T, void* stream) {\n"
                   "    t.pool_reserve(n);\n"
                   "    t.pool_write(0, pcm, n);\n"
                   "    t.reset();\n"
                   "    if (t.pool_samples() == n) t.waves(at, at, T, noisy, clean, nullptr, nullptr, T * 480L, 480, T, 1, stream);\n"
                   "}\n"
                   "int main(int argc, char**) {\n"
                   "    if (argc > 1) { nnnoiseless::TrainingBatch t(1); epoch(t, nullptr, 0, nullptr, nullptr, nullptr, 1, nullptr); }\n"
                   "    return 0;\n"
                   "}\n")
    exe = tmp_path / "t"
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-I", inc, str(src), "-o", str(exe), "-L", libdir, "-lnnnoiseless_b200",
                        "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0


def test_null_trainer_refused_without_device():
    L = nb.lib()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    at = (C.c_longlong * 4)()
    for rc in (L.rnnoise_train_reset(None), L.rnnoise_train_pool_reserve(None, 10),
               L.rnnoise_train_waves_device(None, at, at, 1, p, p, None, None, 480, 480, 1, 1, None)):
        assert rc != 0
        assert "null trainer" in nb.last_error()
    assert L.rnnoise_train_pool_write(None, 0, None, 0) != 0 and "null argument" in nb.last_error()
    assert L.rnnoise_train_pool_room(None, p, p) != 0
    assert L.rnnoise_train_pool_samples(None) == 0
