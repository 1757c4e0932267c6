"""CPU tests of the STOI / ESTOI definition (tests/stoi_ref.py), the record layout and the argument checks of
rnnoise_intelligibility_device made before any CUDA call (DESIGN.md 7q)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.signal as ss

import nnnoiseless_b200 as nb
import stoi_ref as sr
from nnnoiseless_b200 import evaluate as ev

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def speech_like(n, seed, scale=3000.0, rate=48000):
    """Noise shaped by a slowly varying envelope with pauses: syllable-rate modulation as in speech."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    env = np.maximum(np.sin(2 * np.pi * 3.1 * t + rng.uniform(0, 6)), 0.0) ** 2 * (0.3 + np.abs(np.sin(2 * np.pi * 0.7 * t)))
    b, a = ss.butter(2, [200.0 / (rate / 2), min(3500.0 / (rate / 2), 0.99)], btype="band")
    return (scale * env * ss.lfilter(b, a, rng.normal(0, 1, n))).astype(np.float32)


def golden_speech():
    return np.fromfile(os.path.join(ROOT, "tests", "golden", "testing.raw"), dtype="<i2").astype(np.float32)


@pytest.mark.parametrize("rate", [48000, 44100, 16000, 8000, 10000, 22000])
def test_resample_matches_resample_poly(rate):
    x = np.random.default_rng(rate).normal(0, 1000, 2345).astype(np.float32)
    h = sr.filter_taps(rate)
    up, down, half, n10, _ = sr.sizes(len(x), rate)
    got = sr.resample(x, rate, h)
    assert len(got) == n10
    if h is None:
        assert np.array_equal(got, x.astype(np.float64)) and np.array_equal(ss.resample_poly(x.astype(np.float64), up, down), got)
        return
    assert len(h) == 2 * half + 1
    want = ss.resample_poly(x.astype(np.float64), up, down, window=h.astype(np.float64) / up)
    scale = sr.resample(x, rate, h, absolute=True)
    assert np.all(np.abs(got - want) <= 1e-12 * scale + 1e-300)


def test_band_edges_are_the_argmin_construction():
    assert np.array_equal(sr.band_edges_argmin(), sr.EDGES)


def test_identical_and_negated_pairs_score_one():
    x = speech_like(3 * 48000, 1)
    for y in (x, -x):
        r = sr.intelligibility(y, x, 48000)
        assert r["segments"] > 50
        assert abs(r["stoi"] - 1.0) < 1e-12 and abs(r["estoi"] - 1.0) < 1e-12


def test_independent_noise_scores_near_zero():
    y = np.random.default_rng(5).normal(0, 3000, 3 * 48000).astype(np.float32)
    x = np.random.default_rng(9).normal(0, 3000, len(y)).astype(np.float32)
    r = sr.intelligibility(y, x, 48000)
    assert abs(r["stoi"]) < 0.1 and abs(r["estoi"]) < 0.1, (r["stoi"], r["estoi"])
    # Against a clean signal with deep pauses STOI's clipping y' = min(alpha y, c x) makes y' follow x's envelope
    # wherever x dips 15 dB under its segment's level, so STOI is about 0.3; ESTOI, without clipping, stays near 0.
    r = sr.intelligibility(y, speech_like(len(y), 2), 48000)
    assert 0.2 < r["stoi"] < 0.4 and abs(r["estoi"]) < 0.1, (r["stoi"], r["estoi"])


def test_stoi_falls_with_the_snr_on_golden_speech():
    x = golden_speech()
    noise = np.random.default_rng(11).normal(0, 1, len(x))
    px = float(np.mean(x.astype(np.float64) ** 2))
    got = []
    for snr in (20, 10, 0, -10):
        y = (x + noise * np.sqrt(px / 10 ** (snr / 10))).astype(np.float32)
        got.append(sr.intelligibility(y, x, 48000))
    s = [g["stoi"] for g in got]
    print("\nSTOI at 20, 10, 0, -10 dB SNR: %s; ESTOI %s" % (np.round(s, 4), np.round([g["estoi"] for g in got], 4)))
    assert all(a > b for a, b in zip(s, s[1:]))


def test_segment_count_edges():
    rng = np.random.default_rng(7)
    for M, S in ((30, 1), (29, 0)):
        n10 = 256 + M * 128  # F = M + 1 frames, all kept (white noise): K = M + 1
        x = rng.normal(0, 1000, n10).astype(np.float32)
        r = sr.intelligibility(x * 0.5, x, 10000)
        assert r["frames"] == M + 1 and r["kept"] == M + 1 and r["segments"] == S
        assert (np.isfinite(r["stoi"]) and abs(r["stoi"] - 1) < 1e-12) if S else np.isnan(r["stoi"]) and np.isnan(r["estoi"])


def test_all_zero_clean_keeps_every_frame():
    x = np.zeros(48000, np.float32)
    e = sr.frame_db(sr.resample(x, 48000))
    assert np.all(e == 20 * np.log10(sr.EPS))
    r = sr.intelligibility(np.ones_like(x), x, 48000)
    assert r["kept"] == r["frames"] == 77


def test_dtype_matches_the_c_struct(tmp_path):
    src = tmp_path / "off.c"
    fields = list(nb.INTELLIGIBILITY_DTYPE.names)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rnnoise.h"\nint main(void) {\n'
                   + "".join('printf("%%zu\\n", offsetof(RNNoiseIntelligibility, %s));\n' % f for f in fields)
                   + 'printf("%zu\\n", sizeof(RNNoiseIntelligibility));\nreturn 0;\n}\n')
    exe = tmp_path / "off"
    subprocess.run(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [nb.INTELLIGIBILITY_DTYPE.fields[f][1] for f in fields] + [32]


def test_workspace_layout():
    for B, n, rate in ((1, 0, 48000), (3, 48000, 48000), (5, 12345, 44100), (2, 4096, 10000), (7, 300, 8000)):
        up, down, n10, F = nb.intelligibility_sizes(n, rate)
        assert (up, down, n10, F) == tuple(v for i, v in enumerate(sr.sizes(n, rate)) if i != 2)
        r = lambda v: (v + 255) // 256 * 256  # noqa: E731
        regions = r(2 * B * n10 * 4) + r(B * F * 4) + r(2 * B * 15 * max(F - 1, 0) * 4)
        assert nb.intelligibility_workspace_bytes(B, n, rate) > regions
    assert nb.intelligibility_workspace_bytes(1 << 20, 1 << 40, 48000) == 0  # past SIZE_MAX... or absurd: refused
    for args in ((0, 100, 48000), (1, -1, 48000), (1, 100, 7999), (1, 100, 10050), (1, 100, 48100)):
        assert nb.intelligibility_workspace_bytes(*args) == 0


def test_refusals_without_a_device():
    L = nb.lib()
    fake = 1 << 20  # never dereferenced: every refusal happens before any CUDA call
    need = nb.intelligibility_workspace_bytes(4, 1000, 48000)
    ok = dict(out=fake, clean=fake, B=4, n=1000, stride=1000, rate=48000, res=fake, ws=fake, wsb=need)

    def call(**kw):
        a = {**ok, **kw}
        p = lambda v: C.c_void_p(v) if v else None  # noqa: E731
        return L.rnnoise_intelligibility_device(p(a["out"]), p(a["clean"]), a["B"], a["n"], a["stride"], a["rate"], p(a["res"]), p(a["ws"]),
                                                a["wsb"], -1, None)

    for kw, msg in ((dict(B=0), "n_pairs must be positive"), (dict(B=-3), "n_pairs must be positive"),
                    (dict(n=-1), "negative n_samples"), (dict(rate=7999), "rate 7999"), (dict(rate=10050), "rate 10050"),
                    (dict(rate=48100), "rate 48100"), (dict(stride=999), "rows overlap"), (dict(wsb=need - 1), "needed"),
                    (dict(out=0), "null argument"), (dict(clean=0), "null argument"), (dict(res=0), "null argument"),
                    (dict(ws=0), "null argument"), (dict(ws=fake + 128), "256-byte aligned"), (dict(res=fake + 4), "8-byte"),
                    (dict(out=fake + 2), "float-aligned")):
        assert call(**kw) == -1, kw
        assert msg in nb.last_error(), (kw, nb.last_error())


def test_evaluate_intelligibility_sizes_and_cli(capsys):
    grp = [dict(variants=[0, 1, 2])]
    base = ev.device_bytes(grp, 64, 300)
    assert ev.device_bytes(grp, 64, 300, intelligibility=False) == base
    assert ev.device_bytes(grp, 64, 300, intelligibility=True) == base + nb.intelligibility_workspace_bytes(3 * 64, 299 * 480, 48000)
    with pytest.raises(SystemExit):
        ev.main(["--signal-glob", "x", "--noise-glob", "y", "--model", "builtin", "--frames", "10", "--intelligibility", "--window", "0"])
    with pytest.raises(SystemExit):
        ev.main(["--signal-glob", "x", "--noise-glob", "y", "--model", "builtin", "--frames", "10", "--intelligibility", "--window", "1"])


def test_overlapping_rows_are_refused():
    """Rows that share samples (an unfold with hop < n, an expand) are refused before any device work: passing their
    real stride would read past the tensor, and passing n instead would score other samples."""
    import torch
    sig = torch.arange(10.0)
    for out in (sig.unfold(0, 4, 2), sig[:4].expand(3, 4)):
        with pytest.raises(ValueError, match="rows must not overlap"):
            nb.intelligibility(out, out.clone())  # clean is contiguous, so the row strides differ as well
        with pytest.raises(ValueError, match="rows must not overlap"):
            nb.intelligibility(out, out)
