"""The metrics kernel (metrics.cu) band by band and frame by frame against float64, on the constructed edges of
tests/metrics_cases.py (DESIGN.md 7p, "Checks").

- Every frame: one-frame calls, last_bands read after each; Yb and Cb of every band of every counted frame within the
  per-band bound of float64 (metrics_ref.band_yardstick); every record field against MetricsRef fed the GPU's own
  bands (counts exact, time sums within 2 gamma_n sum |terms|, log sums within 1e-12 relative) and fed float64 bands
  (log sums within the band bounds carried through the logs).  Calls of 5 and T frames give the same bytes.
- Grid wrap: 2 x SMs x 64 + 37 streams, permuted copies of the constructed set, so that every warp scores at least two
  streams: records after every call equal the small handle's bit for bit, with a clear of a scattered subset.
- Layouts: seq-first, batch-first, a frame stride that is not a multiple of 4 floats, seq-first vad and target strides.
The largest share of each bound is printed."""
import numpy as np
import pytest

import metrics_cases as mc
import metrics_ref as mr
import nnnoiseless_b200 as nb
from metrics_ref import MetricsRef

pytestmark = pytest.mark.gpu
F = 480
T = mc.T
LOG = ("seg_snr", "lsd", "speech_dev", "noise_level")


@pytest.fixture(scope="module")
def data():
    return mc.cases()


def _dev(d, torch):
    return {k: torch.from_numpy(d[k]).cuda() for k in ("y", "c", "tgt", "vad")}


def feed(m, dv, calls, modes=None, after_each=None, clear_after=None):
    """Calls of the given sizes over batch-first device arrays dv (y, c [B][T][480], tgt, vad [B][T]).  modes: per frame
    of one-frame calls, 0 both vad pointers, 1 the vad only, 2 neither.  clear_after: (call index, streams or None)."""
    y, c, tg, vd = dv["y"], dv["c"], dv["tgt"], dv["vad"]
    f0 = 0
    for i, n in enumerate(calls):
        mode = 0 if modes is None else modes[f0]
        assert modes is None or n == 1
        vp = vd[:, f0].data_ptr() if mode < 2 else 0
        tp = tg[:, f0].data_ptr() if mode == 0 else 0
        m.accumulate_device(y[:, f0].data_ptr(), c[:, f0].data_ptr(), n, T * F, F, vp, tp, T, 1)
        f0 += n
        if clear_after is not None and clear_after[0] == i:
            m.clear(clear_after[1])
        if after_each is not None:
            after_each(m.records())
    assert f0 == T
    return m.records()


@pytest.fixture(scope="module")
def small(data):
    """The constructed set in one-frame calls: records after every call, plain and with every stream cleared after
    call CLEAR_AT."""
    import torch
    dv = _dev(data, torch)
    B = len(data["names"])
    out = {}
    for name, clear in (("plain", None), ("cleared", (CLEAR_AT, None))):
        per = []
        feed(nb.Metrics(B), dv, [1] * T, modes=data["mode"], after_each=lambda r: per.append(r.copy()), clear_after=clear)
        out[name] = per
    return out


CLEAR_AT = 9


def _windows(data):
    """Per counted frame j = 1..T-1 the output and clean windows -> (prev, cur) [T-1][2][B][480]."""
    y, c = data["y"], data["c"]
    B = len(y)
    cpad = np.concatenate([np.zeros((B, 2, F), np.float32), c], axis=1)  # clean frame j - 1 is cpad[:, j + 1]
    prev = np.stack([np.stack([y[:, j - 1], cpad[:, j]]) for j in range(1, T)])
    cur = np.stack([np.stack([y[:, j], cpad[:, j + 1]]) for j in range(1, T)])
    return prev, cur


def test_every_frame_against_float64(data, small):
    import torch
    per = small["plain"]
    one = per[-1]
    B = len(one)
    gpu = np.stack([np.transpose(per[j]["last_bands"], (1, 0, 2)) for j in range(1, T)])  # [T-1][2][B][22]
    prev, cur = _windows(data)
    ex, tol = mr.band_yardstick(prev.reshape(-1, F), cur.reshape(-1, F))
    ex, tol = ex.reshape(gpu.shape), tol.reshape(gpu.shape)
    sh = mr.share(mr.band_excess(gpu, ex), tol)
    shares = {"Yb": sh[:, 0].max(), "Cb": sh[:, 1].max()}
    for q, k in (("Yb", 0), ("Cb", 1)):
        bad = np.argwhere(sh[:, k] > 1.0)
        assert not len(bad), (q, [(int(j) + 1, data["names"][s], int(b), float(sh[j, k, s, b])) for j, s, b in bad[:5]])
    # y = delayed c: the output window is the clean window, through the X and P halves of the same FFT
    cp = [s for s, n in enumerate(data["names"]) if n == "delayed clean"]
    same = gpu[1:, 0][:, cp].view(np.uint32) == gpu[1:, 1][:, cp].view(np.uint32)
    # the records from the GPU's own bands (frame 0 is not counted)
    bands = [np.zeros((2, B, 22))] + list(gpu)
    ref = MetricsRef(B)
    rr = ref.accumulate(data["y"], data["c"], vad=data["vad"], target=data["tgt"], bands=bands)
    for k in ("frames", "vad_counts"):
        assert np.array_equal(one[k], rr[k]), k
    assert one["last_bands"].tobytes() == rr["last_bands"].astype(np.float32).tobytes()
    tb = ref.time_bounds()
    for k in ("ec", "ey", "ecy", "ed"):
        s = mr.share(np.abs(one[k] - rr[k]), tb[k])
        shares[k] = s.max()
        assert (s <= 1.0).all(), (k, np.argwhere(s > 1.0)[:5])
    for k in LOG:
        scale = np.abs(rr[k]) + (one["frames"][:, 1] if k != "noise_level" else one["frames"][:, 2]).reshape((B,) + (1,) * (rr[k].ndim - 1))
        assert (np.abs(one[k] - rr[k]) <= 1e-12 * scale).all(), k
    # the same records from float64 bands: the log sums within the band bounds carried through the logs
    r64 = MetricsRef(B)
    band_tol = [np.zeros((2, B, 22))] + list(tol)
    r64.accumulate(data["y"], data["c"], vad=data["vad"], target=data["tgt"], bands=[np.zeros((2, B, 22))] + list(ex),
                   band_tol=band_tol)
    for k in ("lsd", "speech_dev", "noise_level"):
        scale = np.abs(r64.rec[k]) + (one["frames"][:, 1] if k != "noise_level" else one["frames"][:, 2]).reshape((B,) + (1,) * (r64.rec[k].ndim - 1))
        s = mr.share(np.maximum(np.abs(one[k] - r64.rec[k]) - 1e-12 * scale, 0.0), r64.log_tol[k])
        shares[k + " (f64 bands)"] = s.max()
        assert (s <= 1.0).all(), (k, np.argwhere(s > 1.0)[:5])
    # split invariance with every target passed (0.5 where a one-frame call passed none)
    dv = _dev(data, torch)
    for calls in ([5] * (T // 5) + [T % 5], [T]):
        got = feed(nb.Metrics(B), dv, calls)
        assert got.tobytes() == one.tobytes(), calls
    cov = mc.coverage(data["y"], data["c"], data["tgt"], data["vad"])
    print("\nlargest share of the bound: " + ", ".join("%s %.3f" % kv for kv in shares.items()))
    print("y = delayed c: Yb == Cb bit for bit on %d of %d bands" % (same.sum(), same.size))
    print("coverage (stream-frames): %s" % cov)


def test_grid_wrap_bit_for_bit(data, small):
    import torch
    B = len(data["names"])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = 2 * sms * 64 + 37
    rng = np.random.default_rng(17)
    perm = rng.permutation(np.arange(N) % B)
    sub = np.sort(rng.choice(N, N // 7, replace=False))
    dv = _dev(data, torch)
    idx = torch.from_numpy(perm).cuda()
    big = {k: v.index_select(0, idx).contiguous() for k, v in dv.items()}
    m = nb.Metrics(N)
    insub = np.zeros(N, bool)
    insub[sub] = True
    calls = []

    def check(r):
        t = len(calls)
        want = small["plain"][t][perm]
        if t >= CLEAR_AT:
            want[insub] = small["cleared"][t][perm[insub]]
        diff = (r.view(np.uint8).reshape(N, -1) != want.view(np.uint8).reshape(N, -1)).any(axis=1)
        assert not diff.any(), (t, np.flatnonzero(diff)[:5])
        calls.append(t)

    feed(m, big, [1] * T, modes=data["mode"], after_each=check, clear_after=(CLEAR_AT, sub.astype(np.int32)))
    assert len(calls) == T
    print("\n%d streams on %d SMs, %d cleared after call %d" % (N, sms, len(sub), CLEAR_AT))


def test_layouts_give_the_same_bits(data):
    import torch
    B = len(data["names"])
    y, c, tg, vd = data["y"], data["c"], data["tgt"], data["vad"]
    want = feed(nb.Metrics(B), _dev(data, torch), [T])

    def run(dy, dc, ss, fs, dvad, dtg, vss, vfs, calls):
        m = nb.Metrics(B)
        f0 = 0
        for n in calls:
            m.accumulate_device(dy.data_ptr() + 4 * f0 * fs, dc.data_ptr() + 4 * f0 * fs, n, ss, fs,
                                dvad.data_ptr() + 4 * f0 * vfs, dtg.data_ptr() + 4 * f0 * vfs, vss, vfs)
            f0 += n
        return m.records()

    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    # seq-first samples and seq-first vad / target
    sy, sc = cu(np.transpose(y, (1, 0, 2))), cu(np.transpose(c, (1, 0, 2)))
    stg, svd = cu(tg.T), cu(vd.T)
    for calls in ([T], [5] * (T // 5) + [T % 5]):
        assert run(sy, sc, F, B * F, svd, stg, 1, B, calls).tobytes() == want.tobytes(), ("seq-first", calls)
    # batch-first with a frame stride of 483 floats (not a multiple of 4), batch-first vad / target
    P = 483
    py, pc = (np.full((B, T, P), np.nan, np.float32) for _ in range(2))
    py[:, :, :F], pc[:, :, :F] = y, c
    assert run(cu(py), cu(pc), T * P, P, cu(vd), cu(tg), T, 1, [7, 7, 10]).tobytes() == want.tobytes(), "stride 483"
    # seq-first with a padded frame row (stream stride 483) and seq-first vad / target
    qy, qc = (np.full((T, B, P), np.nan, np.float32) for _ in range(2))
    qy[:, :, :F], qc[:, :, :F] = np.transpose(y, (1, 0, 2)), np.transpose(c, (1, 0, 2))
    assert run(cu(qy), cu(qc), P, B * P, svd, stg, 1, B, [T]).tobytes() == want.tobytes(), "seq-first, stream stride 483"
