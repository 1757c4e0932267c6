"""The metrics kernel's yardstick and bounds without a GPU (DESIGN.md 7p, "Checks"): the oracle's f32 band energies lie
inside the per-band bound on the constructed set (tests/metrics_cases.py), the bound is not vacuous, and the float64
restatement (tests/metrics_ref.py) gives hand-worked values on the class, VAD and segmental-SNR edges."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import metrics_cases as mc
import metrics_ref as mr
from metrics_ref import MetricsRef

F = 480
U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def windows():
    """Every counted frame's output and clean windows of the constructed set -> (prev, cur) [n][480] each."""
    d = mc.cases()
    y, c = d["y"], d["c"]
    B, T = y.shape[:2]
    z = np.zeros((B, 1, F), np.float32)
    cpad = np.concatenate([z, z, c], axis=1)  # clean frame j - 1 is cpad[j + 1]
    prev = np.concatenate([y[:, :-1], cpad[:, 1:T]], axis=0).reshape(-1, F)
    cur = np.concatenate([y[:, 1:], cpad[:, 2:T + 1]], axis=0).reshape(-1, F)
    return prev, cur


def test_oracle_bands_inside_the_bound(windows):
    """Both f32 orders the bound is built from, and the f64 DFT rounded once, which it is not built from."""
    prev, cur = windows
    ex, tol = mr.band_yardstick(prev, cur)
    worst = {}
    for mode in (0, 1, 2):
        sh = mr.share(mr.band_excess(mr.oracle_bands(prev, cur, mode), ex), tol)
        worst[mode] = sh.max()
        assert (sh <= 1.0).all(), (mode, np.argwhere(sh > 1.0)[:5])
    print("\noracle band energies, largest share of the bound: order 0 %.3f, f64 DFT %.3f, order 2 %.3f"
          % (worst[0], worst[1], worst[2]))
    assert (tol[(ex == 0).all(axis=1)] == 0).all()  # an all-zero window must give exact zeros


def test_bound_is_not_vacuous(windows):
    prev, cur = windows
    ex, tol = mr.band_yardstick(prev, cur)
    live = ex.max(axis=1) > 1e-10  # not the subnormal or zero streams
    with np.errstate(divide="ignore", invalid="ignore"):
        db = 10.0 * np.log10(ex / ex.max(axis=1, keepdims=True))
    # where the bound is tightest (loud bands) a relative error of 4 K u already fails
    fails = mr.share(mr.band_excess(ex * (1.0 + 4 * mr.K * U32), ex), tol) > 1.0
    assert fails.sum() >= 100, fails.sum()
    # in bands 40 - 80 dB below their frame's loudest one, +1 dB fails everywhere (the earlier tolerance of 1e-4 ex +
    # 1e-5 sum ex let such a band read 10 dB high); the largest bound there is printed
    quiet = live[:, None] & (db < -40.0) & (db > -80.0)
    assert quiet.sum() >= 500, quiet.sum()
    up = mr.share(mr.band_excess(ex * 10.0 ** 0.1, ex), tol)
    assert (up[quiet] > 1.0).all()
    print("\nbands 40-80 dB below the frame's peak: the bound allows at most %.3f dB"
          % (10.0 * np.log10(1.0 + (tol[quiet] / ex[quiet]).max())))


def _float_compares(tmp_path):
    """C's float compares, as the kernel writes them: (t == 1.0f, t == 0.0f) and v >= 0.5f."""
    src = tmp_path / "cmp.c"
    src.write_text("int cls(float t) { return (t == 1.0f) | ((t == 0.0f) << 1); }\n"
                   "int said(float v) { return v >= 0.5f; }\n")
    so = tmp_path / "cmp.so"
    subprocess.run(["gcc", "-O2", "-shared", "-fPIC", str(src), "-o", str(so)], check=True)
    L = C.CDLL(str(so))
    L.cls.argtypes = [C.c_float]
    L.said.argtypes = [C.c_float]
    return L


def test_python_compares_match_c_on_the_edges(tmp_path):
    L = _float_compares(tmp_path)
    for t in mc.TARGETS:
        v = float(np.float64(t))  # what MetricsRef compares
        assert L.cls(t) == ((v == 1.0) | ((v == 0.0) << 1)), t
    for v in mc.VADS:
        assert L.said(v) == (float(v) >= 0.5), v


def _classes(tg, vad=None, **kw):
    B, T = tg.shape
    c = np.random.default_rng(0).normal(0, 1000, (B, T, F)).astype(np.float32)
    y = np.zeros_like(c)
    y[:, 1:] = c[:, :-1]
    return MetricsRef(B).accumulate(y, c, target=tg, vad=vad, **kw)


def test_class_edges_by_hand():
    """Frame t is classed by the target of frame t - 1; only exactly 1 is speech and only +-0 is noise."""
    tg = mc.TARGETS[None, :].copy()  # 1, 1 - ulp, 0, -0, 1e-45, 0.5, nan, 2
    t9 = np.concatenate([tg, np.float32([[0.0]])], axis=1)
    r = _classes(t9)
    # counted frames 1..8 paired with targets 1, 1 - ulp, 0, -0, 1e-45, 0.5, nan, 2
    assert r["frames"][0].tolist() == [8, 1, 2]
    assert r["seg_snr"][0] == 35.0  # one speech frame, an exact copy
    vad = np.tile(mc.VADS, 2)[None, :9].astype(np.float32)  # 0.5, 0.5 - ulp, nan, -0, 1, 0.5, 0.5 - ulp, nan, -0
    r = _classes(t9, vad=vad)
    # the vad is scored against the frame's own target where it is 0 or +-0 or 1: frames 2 (0; vad nan: tn),
    # 3 (-0; vad -0: tn), and frame 8's target 0 (vad -0: tn); frame 1 (1 - ulp) and frames 4..7 are not scored
    assert r["vad_counts"][0].tolist() == [0, 0, 0, 3]
    r = _classes(np.float32([[0.0, 1.0, 1.0, 0.0]]), vad=np.float32([[1.0, np.nextafter(np.float32(0.5), 0), 0.5, 0.5]]))
    # frames 1 (target 1, vad 0.5 - ulp: fn), 2 (1, 0.5: tp), 3 (0, 0.5: fp)
    assert r["vad_counts"][0].tolist() == [1, 1, 1, 0]


def test_target_pointer_in_one_call_and_not_the_next():
    B = 1
    rng = np.random.default_rng(1)
    c = rng.normal(0, 1000, (B, 9, F)).astype(np.float32)
    y = rng.normal(0, 1000, (B, 9, F)).astype(np.float32)
    ref = MetricsRef(B)
    ref.accumulate(y[:, :3], c[:, :3], target=np.float32([[0.5, 0.5, 1.0]]))
    r = ref.accumulate(y[:, 3:6], c[:, 3:6], vad=np.ones((B, 3), np.float32)).copy()
    # frame 3 pairs with clean frame 2 (target 1, from the call before); frames 4, 5 have no target: neither class;
    # the vad without a target pointer counts nothing
    assert r["frames"][0].tolist() == [5, 1, 0] and r["vad_counts"][0].tolist() == [0, 0, 0, 0]
    r = ref.accumulate(y[:, 6:], c[:, 6:], vad=np.ones((B, 3), np.float32), target=np.zeros((B, 3), np.float32))
    # frame 6 pairs with clean 5 (no target: neither), frames 7, 8 with target 0; all three vote fp
    assert r["frames"][0].tolist() == [8, 1, 2] and r["vad_counts"][0].tolist() == [0, 3, 0, 0]


def test_seg_snr_branches_by_hand():
    assert mr.seg_snr(1.0, 0.0) == 35.0 and mr.seg_snr(0.0, 0.0) == 35.0  # Ed = 0, whatever Ec
    assert mr.seg_snr(0.0, 1.0) == -10.0  # Ec = 0 < Ed
    assert mr.seg_snr(1e4, 1.0) == 35.0 and mr.seg_snr(1.0, 1e2) == -10.0  # clamped
    assert mr.seg_snr(1e2, 1.0) == 20.0 and mr.seg_snr(1.0, 1e1) == -10.0


def test_coverage_of_the_constructed_set():
    """Stream-frames of the constructed set in each class, segmental-SNR branch and VAD cell (pinned: a change to
    metrics_cases that drops an edge fails here)."""
    d = mc.cases()
    cov = mc.coverage(d["y"], d["c"], d["tgt"], d["vad"])
    print("\n", cov)
    assert cov == {"speech": 475, "noise": 950, "neither": 3175, "ed=0": 132, "ec=0<ed": 32, "ec=ed=0": 52,
                   "clamp low": 292, "clamp high": 23, "inside": 4121, "tp": 190, "fp": 380, "fn": 285, "tn": 570}


def test_time_bounds_hold_for_exact_sums():
    """The restatement's double sums against exact rational sums (math.fsum) on the constructed set: inside the bound
    the GPU is held to."""
    import math
    d = mc.cases()
    y, c, tg = d["y"][:40], d["c"][:40], d["tgt"][:40]
    ref = MetricsRef(40)
    r = ref.accumulate(y, c, target=tg)
    tb = ref.time_bounds()
    y64, c64 = y.astype(np.float64), c.astype(np.float64)
    cp = np.concatenate([np.zeros((40, 1, F)), c64[:, :-1]], axis=1)
    for s in range(40):
        exact = math.fsum((cp[s, 1:] * y64[s, 1:]).ravel())
        assert abs(r["ecy"][s, 0] - exact) <= tb["ecy"][s, 0] / 2, s
        exact = math.fsum((cp[s, 1:] ** 2).ravel())
        assert abs(r["ec"][s, 0] - exact) <= tb["ec"][s, 0] / 2, s
