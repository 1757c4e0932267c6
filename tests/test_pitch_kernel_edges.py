"""pitch_kernel (pitch.cu) on the constructed cases of pitch_cases.py: coin flips of every certified decision, crowded
coarse scans, exact score ties, degenerate histories, both sides of the range guard and the period extremes.

- Bit-exactness: every case is loaded with set_states and runs one frame, then one speech frame more; after each, the
  pitch tap and the record's last_period / last_gain (as bits) equal the oracle's for every stream.  For the default
  kernel and for NNB_PITCH_EXACT = 1, 2 and 3.
- Tile layouts: batches of 16 k + r streams (r = 1, 7, 15); each class sits at every lane of a 16-stream tile; whole
  tiles of crowded streams (every one recomputes all 147 lags), whole tiles of streams with exactly 8 coarse candidates
  (the kernel's candidate recomputation at capacity: 128 single-lag tasks per tile) and a tile of range-guard cases
  mixed with ordinary streams.
- The certificate must fire: over one frame, ladder_exact >= the streams with a ladder coin flip and coarse_exact >=
  the crowded streams plus the nonzero streams outside the range guard.  There the rounding bound exceeds the margin,
  so any sound certificate sends them to the order-exact path.
- Per tile: a batch of only `overflow` streams (which only the range guard routes) must send every one of them to the
  exact coarse path, and a batch of only `cand8` streams must send none of them there (they take the candidate path).
- A subset call over a shuffled list of streams inside a larger batch gives the same bits.
A failure names the class, the case and the stream."""
import os
from contextlib import contextmanager

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle_state as ost
import pitch_cases as pc
import pitch_ref as pr

pytestmark = pytest.mark.gpu


@contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    for k, v in kv.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def setup(builtin_bytes):
    cs = list(pc.cases())
    nat = pc.natural_buffers(64, seed=11)
    st, ref = pc.measure(cs)
    m = ost.Model(builtin_bytes)
    allc = cs + nat
    speech = pc._speech()
    rng = np.random.default_rng(3)
    follow = np.stack([speech[o:o + 480] for o in rng.integers(0, len(speech) - 480, len(allc))]).astype(np.float32)
    fresh = ost.State(m).export()
    dt = nb.state_dtype(nb.gru_widths(builtin_bytes))
    recs, want = [], []
    for i, c in enumerate(allc):
        r = fresh.copy()
        v = r.view(dt)[0]
        v["input_mem"], v["mem_hp_x"], v["last_period"], v["last_gain"] = c.input_mem, c.mem_hp, c.last_period, c.last_gain
        recs.append(r)
        s = ost.State(m)
        assert s.import_(r)
        w = []
        for fr in (c.frame, follow[i]):
            s.process_frame(fr)
            e = s.export().view(dt)[0]
            w.append((s.pitch(), int(e["last_period"]), np.float32(e["last_gain"]).view(np.uint32)))
        want.append(w)
    return dict(cases=allc, recs=np.stack(recs), want=want, follow=follow, st=st, ref=ref, n_cases=len(cs), dt=dt)


def layout(S, r):
    """Stream order for a batch of 16 k + r: every class in aligned blocks of 16 filled cyclically (each class at every
    lane), a tile of range-guard cases interleaved with natural streams, then natural streams up to the size."""
    cs = S["cases"]
    by = {}
    for i, c in enumerate(cs[:S["n_cases"]]):
        by.setdefault(c.cls, []).append(i)
    nat = list(range(S["n_cases"], len(cs)))
    order = []
    for cls, idx in by.items():
        m = 16 * -(-len(idx) // 16)
        order += [idx[(j + len(order)) % len(idx)] for j in range(m)]
    g = by["guard"]
    order += [g[j // 2] if j % 2 == 0 else nat[j // 2] for j in range(16)]
    k = -(-len(order) // 16)
    n = 16 * k + r
    while len(order) < n:
        order.append(nat[len(order) % len(nat)])
    return np.array(order[:n])


def _check(S, order, tp, st_recs, frame, what):
    dt = S["dt"]
    v = st_recs.view(dt).reshape(-1)
    bad = []
    for s, i in enumerate(order):
        wp, wl, wg = S["want"][i][frame]
        got = (int(tp[s]), int(v["last_period"][s]), np.float32(v["last_gain"][s]).view(np.uint32))
        if got != (wp, wl, wg):
            c = S["cases"][i]
            bad.append("stream %d lane %d class %s (%s): pitch/last_period/last_gain bits %s, oracle %s"
                       % (s, s % 16, c.cls, c.note, got, (wp, wl, int(wg))))
    assert not bad, "%s frame %d: %d streams differ:\n%s" % (what, frame, len(bad), "\n".join(bad[:12]))


def _run(S, order, mode):
    with env(NNB_PITCH_EXACT=mode):
        b = nb.DenoiseBatch(len(order))
    b.set_states(S["recs"][order])
    s0 = b.pitch_stats()
    x0 = np.stack([S["cases"][i].frame for i in order])
    b.process_host(x0[None])
    s1 = b.pitch_stats()
    _check(S, order, b.taps()["pitch"], b.get_states(), 0, "NNB_PITCH_EXACT=%s" % mode)
    b.process_host(S["follow"][order][None])
    _check(S, order, b.taps()["pitch"], b.get_states(), 1, "NNB_PITCH_EXACT=%s" % mode)
    return {k: s1[k] - s0[k] for k in s0}


@pytest.mark.parametrize("r", [1, 7, 15])
@pytest.mark.parametrize("mode", [None, "1", "2", "3"])
def test_pitch_cases_bit_exact(setup, mode, r):
    order = layout(setup, r)
    d = _run(setup, order, mode)
    assert d["stream_frames"] == len(order)
    if mode == "1":
        assert d["coarse_exact"] == len(order) and d["ladder_exact"] == len(order)
    if mode is not None:
        return
    # the certificate must fire where the rounding bound exceeds the margin
    ref, nc = setup["ref"], setup["n_cases"]
    cls = np.array([c.cls for c in setup["cases"][:nc]])
    lm = np.where(ref["l_live"], np.abs(ref["l_m"]), np.inf)
    ladder_flip = (lm < 1).any(1) & ref["in_range"]
    outside = ((ref["ex4"] < 0.95e-18) | (ref["y4tot"] < 0.95e-18) | ~(ref["guard_prod"] < 1.05e37)) & \
        (setup["st"]["pitch_buf"] != 0).any(1)
    crowded = (ref["c_n_near"] >= 9) & ~outside
    in_cases = order[order < nc]
    need_l = int(ladder_flip[in_cases].sum())
    need_c = int((crowded | outside)[in_cases].sum())
    print("r %d: %d streams, ladder_exact %d (>= %d), coarse_exact %d (>= %d)"
          % (r, len(order), d["ladder_exact"], need_l, d["coarse_exact"], need_c))
    assert d["ladder_exact"] >= need_l
    assert d["coarse_exact"] >= need_c
    assert (cls[in_cases] == "crowded").sum() >= 32


def test_pitch_cases_subset_call(setup):
    S = setup
    order = layout(S, 7)
    N = len(order) + 37
    rng = np.random.default_rng(9)
    streams = rng.permutation(N)[:len(order)].astype(np.int32)
    b = nb.DenoiseBatch(N)
    b.set_states(S["recs"][order], streams)
    x0 = np.stack([S["cases"][i].frame for i in order])
    for frame, x in enumerate((x0, S["follow"][order])):
        b.process_streams_host(streams, x[None])
        rec = b.get_states(streams)  # taps describe full-batch frames only: the period is the record's last_period
        _check(S, order, rec.view(S["dt"]).reshape(-1)["last_period"], rec, frame, "subset call")


@pytest.mark.parametrize("cls, exact", [("overflow", True), ("cand8", False)])
def test_pitch_tiles_of_one_class(setup, cls, exact):
    """Whole tiles (and a partial one) of one class: the range guard alone sends every overflow stream to the exact coarse
    path; streams with exactly 8 dominant candidates all stay on the candidate path."""
    idx = [i for i, c in enumerate(setup["cases"][:setup["n_cases"]]) if c.cls == cls]
    order = np.array([idx[j % len(idx)] for j in range(37)])
    d = _run(setup, order, None)
    assert d["coarse_exact"] == (len(order) if exact else 0), (cls, d)
