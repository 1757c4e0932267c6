"""The metrics accumulator's restatement on hand-worked cases, summarize, the record layout, the C ABI's refusals that
need no device, the C++ mirror and the evaluate CLI's planning (DESIGN.md 7p).  No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nnnoiseless_b200 as nb
from metrics_ref import MetricsRef, band_energies
from nnnoiseless_b200 import evaluate as ev
from nnnoiseless_b200 import metrics as mt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 480


def speech(B, T, seed=0, scale=3000.0):
    rng = np.random.default_rng(seed)
    return (rng.normal(0, scale, (B, T, F))).astype(np.float32)


def delayed(c):
    """The output a perfect denoiser gives: output frame t is clean frame t - 1 (frame 0 is zeros)."""
    y = np.zeros_like(c)
    y[:, 1:] = c[:, :-1]
    return y


def test_delayed_clean_is_exact():
    B, T = 3, 12
    c = speech(B, T)
    ref = MetricsRef(B)
    r = ref.accumulate(delayed(c), c, target=np.ones((B, T), np.float32))
    assert (r["frames"][:, 0] == T - 1).all() and (r["frames"][:, 1] == T - 1).all()
    assert (r["ed"] == 0).all()
    assert np.allclose(r["seg_snr"], 35.0 * (T - 1))
    assert (r["lsd"] == 0).all() and (r["speech_dev"] == 0).all()
    s = mt.summarize(r)
    assert (s["snr"] == np.inf).all() and (s["si_sdr"] == np.inf).all()
    assert np.allclose(s["seg_snr"], 35.0) and (s["lsd"] == 0).all()


def test_half_scale():
    B, T = 2, 9
    c = speech(B, T, 1)
    r = MetricsRef(B).accumulate(0.5 * delayed(c), c, target=np.ones((B, T)))
    s = mt.summarize(r)
    assert np.allclose(s["snr"], 6.020599913279624, rtol=0, atol=1e-12)
    assert (s["si_sdr"] == np.inf).all()
    assert np.allclose(s["speech_level"], -6.020599913279624)
    # every band 6.02 dB down (the 0.01 floor is far below these energies)
    assert np.allclose(s["speech_dev"], -6.0206, atol=1e-3)


def test_white_noise_of_known_power():
    B, T = 4, 200
    c = speech(B, T, 2, scale=1000.0)
    rng = np.random.default_rng(9)
    n = rng.normal(0, 100.0, c.shape).astype(np.float32)
    r = MetricsRef(B).accumulate(delayed(c) + n, c)
    s = mt.summarize(r)
    assert np.allclose(s["snr"], 20.0, atol=0.1), s["snr"]
    assert np.allclose(s["si_sdr"], 20.0, atol=0.1), s["si_sdr"]
    assert np.isnan(s["seg_snr"]).all() and s["nan_counts"]["seg_snr"] == B  # no targets: no speech frames


def test_targets_and_classes():
    """Targets 0, 0.5, 1 and a call without targets; the class of a frame is its paired clean frame's target."""
    B, T = 1, 6
    c = speech(B, 2 * T, 3)
    y = delayed(c)
    tg = np.array([[1, 0, 0.5, 1, 1, 0]], np.float32)
    ref = MetricsRef(B)
    ref.accumulate(y[:, :T], c[:, :T], target=tg)
    r = ref.accumulate(y[:, T:], c[:, T:]).copy()  # no targets: frame T pairs with clean T - 1 (target 0), then 0.5
    # counted frames 1..11; paired targets: 1, 0, 0.5, 1, 1, 0 (from the first call) for frames 1..6, then 0.5
    assert r["frames"][0].tolist() == [11, 3, 2]


def test_vad_counts_half_is_speech():
    B, T = 1, 5
    c = speech(B, T, 4)
    tg = np.array([[1, 1, 0, 0.5, 0]], np.float32)
    vad = np.array([[0.5, 0.49, 0.5, 0.9, 0.1]], np.float32)
    r = MetricsRef(B).accumulate(delayed(c), c, vad=vad, target=tg)
    # counted frames 1..4: (0.49, 1) fn, (0.5, 0) fp, (0.9, 0.5) none, (0.1, 0) tn; frame 0 is not counted
    assert r["vad_counts"][0].tolist() == [0, 1, 1, 1]
    r = MetricsRef(B).accumulate(delayed(c), c, vad=np.full((1, T), 0.5, np.float32), target=np.ones((1, T), np.float32))
    assert r["vad_counts"][0].tolist() == [T - 1, 0, 0, 0]


def test_split_invariance_of_the_restatement():
    B, T = 2, 10
    c = speech(B, T, 5)
    y = speech(B, T, 6)
    tg = np.random.default_rng(1).choice([0.0, 0.5, 1.0], (B, T)).astype(np.float32)
    a = MetricsRef(B).accumulate(y, c, target=tg).copy()
    ref = MetricsRef(B)
    for lo, hi in ((0, 1), (1, 4), (4, 10)):
        ref.accumulate(y[:, lo:hi], c[:, lo:hi], target=tg[:, lo:hi])
    for k in ("frames", "vad_counts"):
        assert np.array_equal(a[k], ref.rec[k])
    for k in ("ec", "ey", "ecy", "ed", "seg_snr", "lsd", "speech_dev", "noise_level"):
        assert np.allclose(a[k], ref.rec[k], rtol=1e-12, atol=0)


def test_band_energies_match_the_analysis_reference():
    import spectral_ref as sr
    x = speech(2, 4, 7)[:, :, :]
    mem = np.zeros((2, 1728))
    mem[:, 768:] = x[:, 2:].reshape(2, 960)
    ref = sr.analysis(mem, np.zeros(2, np.int64), np.zeros((2, 8, 22)), np.zeros(2, np.int64))
    assert np.allclose(band_energies(x[:, 2], x[:, 3]), ref["ex"], rtol=1e-12)


def test_summarize_nans_and_baseline():
    rec = np.zeros(3, nb.METRICS_DTYPE)
    rec["frames"][1] = [10, 4, 6]
    rec["ec"][1] = [100.0, 80.0, 20.0]
    rec["ey"][1] = [50.0, 40.0, 5.0]
    rec["ecy"][1] = [60.0, 50.0, 10.0]
    rec["ed"][1] = [10.0, 8.0, 2.0]
    rec["seg_snr"][1], rec["lsd"][1] = 40.0, 2.0
    rec["noise_level"][1] = 6 * -3.0
    rec["vad_counts"][1] = [3, 1, 1, 5]
    rec["frames"][2] = [5, 0, 0]  # no speech, no noise frames
    rec["ec"][2], rec["ed"][2] = [1.0, 0, 0], [1.0, 0, 0]
    base = rec.copy()
    base["ey"][1, 2] = 50.0
    base["noise_level"][1] = 6 * 7.0
    s = mt.summarize(rec, base)
    assert np.isnan(s["snr"][0]) and np.isclose(s["snr"][1], 10.0) and np.isclose(s["snr"][2], 0.0)
    assert np.isclose(s["si_sdr"][1], 10 * np.log10(3600.0 / (5000.0 - 3600.0)))
    assert np.isclose(s["seg_snr"][1], 10.0) and np.isclose(s["lsd"][1], 0.5)
    assert np.isclose(s["vad_precision"][1], 0.75) and np.isclose(s["vad_recall"][1], 0.75)
    assert np.isclose(s["noise_atten"][1], 10.0) and np.allclose(s["noise_atten_bands"][1], 10.0)
    assert np.isnan(s["noise_atten"][[0, 2]]).all()
    assert s["nan_counts"]["snr"] == 1 and s["nan_counts"]["seg_snr"] == 2 and s["nan_counts"]["noise_atten"] == 2
    assert np.isclose(s["delta_snr"][1], 0.0)


def test_dtype_matches_the_c_struct(tmp_path):
    src = tmp_path / "off.c"
    fields = ["frames", "ec", "ey", "ecy", "ed", "seg_snr", "lsd", "speech_dev", "noise_level", "vad_counts", "last_bands"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rnnoise.h"\nint main(void) {\n'
                   + "".join('printf("%%zu\\n", offsetof(RNNoiseMetricsRecord, %s));\n' % f for f in fields)
                   + 'printf("%zu\\n", sizeof(RNNoiseMetricsRecord));\nreturn 0;\n}\n')
    exe = tmp_path / "off"
    subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    want = [nb.METRICS_DTYPE.fields[f][1] for f in fields] + [nb.METRICS_DTYPE.itemsize]
    assert got == want


def test_cpp_mirror_compiles(tmp_path):
    src = tmp_path / "m.cpp"
    src.write_text('#include "nnnoiseless.hpp"\nint main() {\n  nnnoiseless::Metrics m(4);\n'
                   '  std::vector<RNNoiseMetricsRecord> r = m.records();\n  m.clear();\n'
                   '  m.accumulate_device(nullptr, nullptr, 1, 480, 480);\n  return (int)r.size();\n}\n')
    subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)], check=True)


def test_refusals_without_a_device():
    L = nb.lib()
    before = nb.last_error()
    buf = (C.c_float * 960)()
    assert L.rnnoise_metrics_accumulate_device(None, buf, buf, 960, 480, None, None, 0, 0, 1, None) == -1
    assert "null metrics handle" in nb.last_error()
    assert L.rnnoise_metrics_accumulate_device(None, None, buf, 960, 480, None, None, 0, 0, 1, None) == -1
    assert "null out or clean" in nb.last_error()
    assert L.rnnoise_metrics_accumulate_device(None, buf, buf, 960, 480, None, None, 0, 0, -1, None) == -1
    assert "negative n_frames" in nb.last_error()
    assert L.rnnoise_metrics_clear(None, None, 1) == -1 and "null metrics handle" in nb.last_error()
    assert L.rnnoise_metrics_get(None, None, 1, None) == -1 and "null metrics handle" in nb.last_error()
    assert not L.rnnoise_metrics_create(0, -1) and "n_streams must be positive" in nb.last_error()
    L.rnnoise_metrics_destroy(None)
    del before


def other_geometry(path):
    """A generated model of another geometry than the built-in one, written to `path`."""
    import rnn_ref
    with open(path, "wb") as f:
        f.write(rnn_ref.make_model(16, 16, 32, 64, seed=4))
    return str(path)


def test_variants_and_geometry_groups(tmp_path):
    builtin = ev.load_model("builtin")
    sh = ev.load_model(os.path.join(ROOT, "tests", "golden", "sh.rnnn"))  # the built-in model's geometry
    gen = ev.load_model(other_geometry(tmp_path / "small.rnn"))
    models = [builtin, gen, sh, builtin]
    variants = ev.plan_variants(models, [np.inf, 12.0])
    assert [v["name"] for v in variants] == ["unprocessed"] + ["%s@%s" % (m[0], a) for m in models for a in ("inf", "12")]
    groups = ev.group_batches(variants, models, builtin[2])
    assert len(groups) == 2
    assert groups[0]["variants"] == [0, 1, 2, 5, 6, 7, 8] and groups[0]["models"] == [-1, 2]
    assert groups[1]["variants"] == [3, 4] and groups[1]["models"] == [1]
    assert groups[0]["geometry"] == (24, 24, 48, 96) and groups[1]["geometry"] == (16, 16, 32, 64)
    assert ev.device_bytes(groups, 1024, 100) == 2 * 9 * 1024 * 100 * 1920
    with pytest.raises(ValueError):
        ev.parse_limits("inf,-3")


def test_cli_refuses_bad_arguments(capsys):
    with pytest.raises(SystemExit):
        ev.main(["--signal-glob", "x", "--noise-glob", "y", "--model", "builtin", "--frames", "10", "--atten-lim-db", "nan"])
    with pytest.raises(SystemExit):
        ev.main(["--signal-glob", "x", "--noise-glob", "y", "--model", "builtin", "--frames", "0"])
