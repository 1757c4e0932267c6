"""The training-row restatement (train_ref.py) against the CPU oracle, bit for bit, on the constructed lanes of
train_cases.py, and each case's defining property.

Every case lane runs through its own oracle trainer and, all lanes together, through train_ref.FrontRef.  After every
frame these are equal as bits: the three streams' history windows and mem_hp_x (from the oracle's state records), both
random-filter memories, vad_count and the VAD column.  The oracle's gain columns equal train_ref's float32 row assembly
fed the oracle's own band energies, and that assembly agrees with a float64 evaluation of the same quotient."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle_state as ost
import train_cases as tc
import train_ref as tr


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def run(builtin_bytes):
    cs = tc.cases()
    L = len(cs)
    lane, sig, noi, table = tc.lay_out(cs, L)
    model = ost.Model(builtin_bytes)
    dt = nb.state_dtype(nb.gru_widths(builtin_bytes))
    oracles = [ost.Trainer(model) for _ in range(L)]
    ref = tr.FrontRef(L)
    T = tc.T
    trace = dict(energy=np.empty((T, L), np.float32), vad_count=np.empty((T, L), np.int32), vad=np.empty((T, L), np.float32),
                 cutoff=np.empty((T, L), np.int32), resp_mem=np.empty((T, L, 4), np.float32),
                 hist=np.empty((T, 3, L, tr.HIST), np.float32), ex=np.empty((T, 3, L, 22), np.float32),
                 silence=np.empty((T, 3, L), bool), gains=np.empty((T, L, 22), np.float32),
                 unclamped=np.empty((T, L, 22), np.float64))
    mismatches = []
    for t in range(T):
        if t in table:
            ref.set_params(table[t])
            for l in range(L):
                oracles[l].set_params(table[t][l:l + 1])
        front = ref.frame(sig[t], noi[t])
        rows = np.stack([oracles[l].frame(sig[t, l], noi[t, l]) for l in range(L)])
        probes = [o.probe() for o in oracles]
        ex = np.stack([p["ex"] for p in probes], axis=1)                  # [3][L][22]
        rec = np.stack([p["records"] for p in probes], axis=1).view(dt)[..., 0]   # [3][L]
        sil = tr.silence_from_ex(ex)
        want_gains = tr.gains_f32(ex[0], ex[2], front["cutoff"], sil[2])
        checks = {
            "history": np.array_equal(bits(rec["input_mem"]), bits(ref.hist)),
            "mem_hp_x": np.array_equal(bits(rec["mem_hp_x"]), bits(ref.hp_mem)),
            "resp_mem": np.array_equal(bits(np.stack([p["resp_mem"] for p in probes])), bits(ref.resp_mem)),
            "vad_count": np.array_equal(np.array([p["vad_count"] for p in probes]), front["vad_count"]),
            "vad column": np.array_equal(bits(rows[:, 86]), bits(front["vad"])),
            "gain columns": np.array_equal(bits(rows[:, 42:64]), bits(want_gains)),
            "silent features": np.array_equal(sil[2], ~rows[:, :42].any(axis=1)),
        }
        for what, ok in checks.items():
            if not ok:
                mismatches.append((t, what))
        trace["energy"][t], trace["vad_count"][t], trace["vad"][t] = front["energy"], front["vad_count"], front["vad"]
        trace["cutoff"][t], trace["resp_mem"][t], trace["hist"][t] = front["cutoff"], ref.resp_mem, ref.hist
        trace["ex"][t], trace["silence"][t], trace["gains"][t] = ex, sil, want_gains
        trace["unclamped"][t] = tr.gains_unclamped_f64(ex[0], ex[2])
    return dict(cases=lane, trace=trace, mismatches=mismatches, params=tc.params_by_frame(table, L))


def test_restatement_matches_oracle_bitwise(run):
    assert run["mismatches"] == []


def test_gain_columns_agree_with_float64(run):
    g, u = run["trace"]["gains"], run["trace"]["unclamped"]
    live = g != -1.0
    assert live.sum() > 1000
    want = np.minimum(u[live], 1.0)
    assert np.all(np.abs(g[live] - want) <= 2.0 ** -23 * want)   # one rounding of the quotient and one of the sqrt


def _lane_trace(run, l):
    t = run["trace"]
    out = {k: v[:, l] for k, v in t.items() if k not in ("hist", "ex", "silence")}
    out["hist"], out["ex"], out["silence"] = t["hist"][:, :, l], t["ex"][:, :, l], t["silence"][:, :, l]
    out["params"] = run["params"][:, l]
    return out


@pytest.mark.parametrize("name", [c.name for c in tc.cases()])
def test_case_reaches_its_edge(run, name):
    l = next(i for i, c in enumerate(run["cases"]) if c.name == name)
    run["cases"][l].check(_lane_trace(run, l))
