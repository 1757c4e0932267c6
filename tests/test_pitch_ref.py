"""The pitch search's decisions at their rounding edges, without a GPU: the oracle's staged run
(oracle_state.pitch_stages), the float64 reference of every decision (pitch_ref) and the constructed cases
(pitch_cases) are tied to each other and to the oracle's pitch_process, so that the GPU tests in
test_pitch_kernel_edges.py stand on checked ground.

- The staged run reproduces nno_pitch_only's period and last_gain bit for bit on every case and on natural buffers.
- Every decision whose float64 margin is at least one rounding bound has the oracle's f32 outcome: a mistake in the
  reference cannot pass as a coin flip.
- Every class reaches its minimum count, the ladder cases cover k = 2..12, the three cont branches and both thresh
  formulas, and the set really reaches f32 rounding: among the coin flips of each bisected class the oracle's f32
  outcome differs from float64 in at least 10 % and agrees in at least 10 %."""
import collections

import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle_state as ost
import pitch_cases as pc
import pitch_ref as pr

DECISION = {"coarse_bs": "coarse best/second", "coarse_st": "coarse second/third", "fine": "fine best",
            "ps_offset": "pitch_search offset", "ladder": "ladder"}


@pytest.fixture(scope="module")
def measured():
    cs = list(pc.cases()) + pc.natural_buffers()
    st, ref = pc.measure(cs)
    return cs, st, ref


def test_staged_oracle_equals_pitch_only(measured, builtin_bytes):
    cs, st, _ = measured
    buf = np.stack([c.buf for c in cs])
    period, gain = ost.pitch_only(buf, [c.last_period for c in cs], np.array([c.last_gain for c in cs], np.float32))
    bad = np.flatnonzero((period != st["period"]) | (gain.view(np.uint32) != st["gain"].view(np.uint32)))
    assert len(bad) == 0, [(int(i), cs[i].cls, cs[i].note) for i in bad[:8]]
    # and the buffer is what the oracle's own frame step puts in input_mem
    m = ost.Model(builtin_bytes)
    dt = nb.state_dtype(nb.gru_widths(builtin_bytes))
    for c in cs[::37]:
        rec = ost.State(m).export()
        v = rec.view(dt)[0]
        v["mem_hp_x"], v["input_mem"] = c.mem_hp, c.input_mem
        r = ost.analysis_frame(m, rec, c.frame)
        assert np.array_equal(r["input_mem"].view(np.uint32), c.buf.view(np.uint32)), c.cls


def test_reference_agrees_with_oracle_outside_coin_flips(measured):
    cs, st, ref = measured
    bad = {k: [(int(i), cs[i].cls) for i in v[:5]] for k, v in pr.disagreements(st, ref).items() if len(v)}
    assert not bad, bad


def test_case_classes_reach_their_counts_and_f32_rounding(measured):
    cs, st, ref = measured
    n = collections.Counter(c.cls for c in cs)
    short = {k: (n[k], v) for k, v in pc.MIN_COUNT.items() if n[k] < v}
    assert not short, short
    cls = np.array([c.cls for c in cs])
    for i, c in enumerate(cs):
        if c.cls != "natural":
            assert pc.has_property(c, st[i], {k: v[i] for k, v in ref.items()}), (i, c.cls, c.note)
    flips, differ = pr.coin_flips(ref), pr.f32_outcomes_differ(st, ref)
    lines = []
    for k in pc.BISECTED:
        sel = (cls == k) & flips[DECISION[k]]
        d = differ[DECISION[k]][sel]
        lines.append("%s: %d coin flips, f32 != float64 in %d" % (k, sel.sum(), d.sum()))
        assert sel.sum() >= pc.MIN_COUNT[k], lines[-1]
        assert 0.1 <= d.mean() <= 0.9, lines[-1]
    print("; ".join(lines))
    # ladder coverage: every reachable k, the three cont branches, both thresh formulas, among its coin flips
    lad = np.flatnonzero(cls == "ladder")
    seen_k, seen_cont, seen_formula = set(), set(), set()
    for i in lad:
        for s in np.flatnonzero(np.abs(ref["l_m"][i][:st["nk"][i]]) < 1):
            seen_k.add(s + 2)
            lg = np.float32(cs[i].last_gain)
            cv = st["cont"][i][s]
            seen_cont.add("lg" if cv == lg and cv != 0 else "lg/2" if cv == np.float32(lg / np.float32(2)) and cv != 0 else "0")
            seen_formula.add(bool(st["t1"][i][s] < 90))
    assert seen_k == set(range(2, 13)), sorted(seen_k)
    assert seen_cont == {"lg", "lg/2", "0"} and seen_formula == {True, False}, (seen_cont, seen_formula)


def test_range_guard_cases_straddle_the_guard(measured):
    cs, st, ref = measured
    g = np.array([c.cls == "guard" for c in cs])
    for what, unit in (("ex4", 1e-18), ("y4tot", 1e-18), ("guard_prod", 1e37)):
        f = ref[what][g] / unit
        for target in (0.5, 0.9, 1.1, 2.0):
            assert (np.abs(f / target - 1) < 1e-3).sum() >= 4, (what, target)
    pb = st["pitch_buf"][g]
    sub = (pb != 0) & (np.abs(pb) < np.finfo(np.float32).tiny)
    assert sub.any(axis=1).sum() >= 1                                   # subnormal whitened samples
    assert (~np.isfinite(ref["guard_prod"][g])).sum() + (ref["guard_prod"][g] > 1e45).sum() >= 2  # the overflow regime
