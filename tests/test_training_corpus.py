"""Reading a WAV corpus for the training-row generator (nnnoiseless_b200.training, src/training.rs SignalReader):
the segment plan against a frame-by-frame restatement, the refusals, and rnnoise_audio_probe.  CPU only."""
import os
import struct

import numpy as np
import pytest

import corpus_ref
import oracle
from nnnoiseless_b200 import NnnoiselessError
from nnnoiseless_b200 import training as tr
from nnnoiseless_b200.files import probe_audio, read_audio, write_audio

HERE = os.path.dirname(os.path.abspath(__file__))
LENGTHS = (480, 481, 100 * 480, 100 * 480 + 1, 5000 * 480)  # whole-file and seek branches, at 100 and more frames per file


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("corpus")
    rng = np.random.default_rng(7)
    paths = []
    for i, n in enumerate(LENGTHS):
        p = str(d / ("f%d.wav" % i))
        write_audio(p, rng.integers(-3000, 3000, n).astype(np.int16), wav=True)
        paths.append(p)
    return paths


def _expand(p, kind):
    at = np.stack([np.stack(p.frames_at(kind, l), -1) for l in range(p.n_lanes)], 1)  # [F][L][2]
    assert at.shape == (p.n_frames, p.n_lanes, 2)
    return at


@pytest.mark.parametrize("lanes", [1, 3, 7])
@pytest.mark.parametrize("shuffle", [False, True])
def test_plan_matches_frame_by_frame_restatement(corpus, lanes, shuffle):
    # 90 copies of the list make the signal side take 100 frames per file (seek draws on the 48,001-sample file);
    # the noise side takes thousands (seek draws on the long file only)
    sig_paths, noise_paths = corpus * 90, corpus
    count = lanes * (2 * tr.RANDOMIZE_PERIOD + 57)  # two randomize frames per lane
    p = tr.plan(sig_paths, noise_paths, count, lanes, seed=11 + lanes, shuffle=shuffle)
    lens = np.array(LENGTHS * 90)
    at_s, at_n, params, ps, pn = corpus_ref.run(lens, np.array(LENGTHS), count, lanes, 11 + lanes, shuffle)
    assert p.signal_paths == [sig_paths[i] for i in ps] and p.noise_paths == [noise_paths[i] for i in pn]
    assert p.n_frames == -(-count // lanes) and p.signal_frames_per_file == 100 and p.noise_frames_per_file > 1000
    assert np.array_equal(_expand(p, "signal"), at_s)
    assert np.array_equal(_expand(p, "noise"), at_n)
    assert [f for f, _ in p.randomize] == sorted(params) == [2821, 2821 + 2822]
    for f, prm in p.randomize:
        assert prm.tobytes() == params[f].tobytes()
    # both branches ran: seeks (an offset past 0) and whole files
    offs = np.concatenate([s["offset"] for s in p.signal + p.noise])
    assert (offs > 0).any() and (offs == 0).any()
    # the plan is per segment: no more entries than files opened
    assert sum(len(s) for s in p.signal) < p.n_frames * lanes // 50


def _wav(path, channels=1, rate=48000, bits=16, tag=1, n=960, data_len=None):
    block = channels * bits // 8
    data = bytes(n * block)
    dl = len(data) if data_len is None else data_len
    fmt = struct.pack("<HHIIHH", tag, channels, rate, rate * block, block, bits)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt) + 8 + len(data)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", dl) + data)
    return str(path)


@pytest.fixture
def no_trainer(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("a trainer was created before the error")
    monkeypatch.setattr(tr, "TrainingBatch", fail)


@pytest.mark.parametrize("kw, spec", [
    (dict(channels=2), "WavSpec { channels: 2, sample_rate: 48000, bits_per_sample: 16, sample_format: Int }"),
    (dict(rate=44100), "WavSpec { channels: 1, sample_rate: 44100, bits_per_sample: 16, sample_format: Int }"),
    (dict(bits=24), "WavSpec { channels: 1, sample_rate: 48000, bits_per_sample: 24, sample_format: Int }"),
    (dict(bits=32, tag=3), "WavSpec { channels: 1, sample_rate: 48000, bits_per_sample: 32, sample_format: Float }"),
])
def test_unsupported_format_refused(tmp_path, corpus, no_trainer, kw, spec):
    bad = _wav(tmp_path / "bad.wav", **kw)
    with pytest.raises(NnnoiselessError) as e:
        tr.generate_rows(corpus + [bad], corpus, 1000, lanes=1)
    assert str(e.value) == "unsupported wav format %s in %s" % (spec, bad)
    with pytest.raises(NnnoiselessError, match="unsupported wav format"):
        tr.generate_rows(corpus, [bad], 1000, lanes=1)


def test_short_file_refused(tmp_path, corpus, no_trainer):
    short = str(tmp_path / "short.wav")
    write_audio(short, np.ones(479, np.int16), wav=True)
    with pytest.raises(NnnoiselessError, match="short.wav has 479 samples, fewer than one 480-sample frame"):
        tr.generate_rows(corpus, corpus + [short], 1000, lanes=2)


def test_truncated_data_chunk_refused(tmp_path, corpus, no_trainer):
    cut = _wav(tmp_path / "cut.wav", n=960, data_len=2 * 961)
    with pytest.raises(NnnoiselessError) as e:
        tr.generate_rows([cut] + corpus, corpus, 1000, lanes=1)
    assert str(e.value) == "Failed to read enough bytes. in %s" % cut


def test_empty_glob_refused(tmp_path, corpus, no_trainer):
    paths = tr.glob_paths([str(tmp_path / "nothing*.wav")])
    assert paths == []
    with pytest.raises(NnnoiselessError, match="^cannot read from an empty set of files$"):
        tr.generate_rows(paths, corpus, 1000)
    with pytest.raises(NnnoiselessError, match="^cannot read from an empty set of files$"):
        tr.generate_rows(corpus, paths, 1000)


def test_h5_output_refused(tmp_path, corpus, no_trainer, capsys):
    with pytest.raises(NnnoiselessError, match="HDF5 output is not supported"):
        tr.generate_rows(corpus, corpus, 1000, out=str(tmp_path / "rows.h5"))
    with pytest.raises(SystemExit):
        tr.main(["--signal-glob", corpus[0], "--noise-glob", corpus[0], "--count", "10", "-o", str(tmp_path / "rows.h5")])
    assert "HDF5 output is not supported" in capsys.readouterr().err
    assert not os.path.exists(tmp_path / "rows.h5")


def test_default_lanes_and_warmup_share():
    assert tr.default_lanes(1) == 1 and tr.default_lanes(2_000_000) == 7 and tr.default_lanes(10 ** 10) == 4096
    for count in (282_200, 2_000_000, 50_000_000):
        assert tr.warmup_share(count, tr.default_lanes(count)) <= 0.0101


@pytest.mark.parametrize("name", ["mono.wav", "stereo.wav", "mono-float.wav"])
def test_audio_probe_locates_the_samples(name):
    path = os.path.join(HERE, "golden", "wav", name)
    a = probe_audio(path)
    with open(path, "rb") as f:
        want, rate = oracle.decode_wav(f.read())
    assert (a.channels, a.sample_rate, a.n_frames) == (want.shape[1], rate, want.shape[0])
    dt = "<f4" if a.is_float else "<i%d" % (a.bits_per_sample // 8)
    mm = np.memmap(path, dtype=dt, mode="r", offset=a.data_offset, shape=(a.n_frames * a.channels,))
    got = np.asarray(mm, np.float32).reshape(-1, a.channels)
    if a.is_float:
        got = got * np.float32(32767.0)
    assert np.array_equal(got, want)
    assert np.array_equal(got, read_audio(path)[0])


def test_audio_probe_errors_are_read_audio_errors(tmp_path):
    for p in (_wav(tmp_path / "cut.wav", data_len=10 ** 6), str(tmp_path / "missing.wav")):
        with pytest.raises(NnnoiselessError) as a:
            probe_audio(p)
        with pytest.raises(NnnoiselessError) as b:
            read_audio(p)
        assert str(a.value) == str(b.value)
