"""CPU tests of the per-stream state record (include/rnnoise.h): the oracle's export / import continues a stream bit
for bit, and the record's size and field layout agree between the oracle, nb.state_dtype and the size formula."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle_state as ost
import rnn_ref


def _widths(model_bytes):
    return nb.gru_widths(model_bytes)


@pytest.mark.parametrize("k", [0, 1, 7, 8, 57])
def test_oracle_export_import_continues_bitwise(builtin_bytes, testing_raw, k):
    m = ost.Model(builtin_bytes)
    T = min(len(testing_raw), k + 30)
    x = testing_raw[None, :T]
    whole, whole_vad, whole_pitch, ref_states = ost.run(m, x)
    first = ost.State(m)
    for t in range(k):
        first.process_frame(x[0, t])
    rec = first.export()
    resumed = ost.State(m)
    assert resumed.import_(rec)
    assert np.array_equal(resumed.export(), rec)
    out, vad, pitch, states = ost.run(m, x[:, k:], [resumed])
    assert np.array_equal(out.view(np.uint32), whole[:, k:].view(np.uint32))
    assert np.array_equal(vad.view(np.uint32), whole_vad[:, k:].view(np.uint32))
    assert np.array_equal(pitch, whole_pitch[:, k:])
    assert np.array_equal(states[0].export(), ref_states[0].export())
    d = rec.view(nb.state_dtype(_widths(builtin_bytes)))[0]
    assert d["magic"] == nb.STATE_MAGIC and d["version"] == 1 and d["mem_id"] == k % 8
    if k == 0:
        assert not rec[20:].any()  # a fresh state: every field after the widths is zero


def test_state_size_formula(builtin_bytes, sh_bytes):
    geometry = rnn_ref.make_model(5, 13, 37, 45, seed=3)
    for model in (builtin_bytes, sh_bytes, geometry):
        w = _widths(model)
        size = 9664 + 4 * sum(w)
        size += -size % 16
        dt = nb.state_dtype(w)
        assert dt.itemsize == nb.state_bytes(w) == size == ost.Model(model).state_bytes
        assert dt.fields["denoise_gru"][1] + 4 * w[2] == 9664 + 4 * sum(w)
    assert nb.state_bytes(_widths(builtin_bytes)) == 10336


def test_record_fields_decode(builtin_bytes, testing_raw):
    m = ost.Model(builtin_bytes)
    s = ost.State(m)
    for t in range(11):
        s.process_frame(testing_raw[t])
    rec = s.export()
    d = rec.view(nb.state_dtype(_widths(builtin_bytes)))[0]
    assert (d["nv"], d["nn"], d["nd"]) == _widths(builtin_bytes) == (24, 48, 96)
    assert d["mem_id"] == 11 % 8 and 0 <= d["last_period"] <= 768
    assert d["input_mem"][-480:].any() and d["synthesis_mem"].any() and d["denoise_gru"].any()
    assert not rec[9664 + 4 * 168:].any()  # padding


def test_oracle_import_rejects_bad_records(builtin_bytes, testing_raw):
    m = ost.Model(builtin_bytes)
    s = ost.State(m)
    for t in range(3):
        s.process_frame(testing_raw[t])
    good = s.export()
    dt = nb.state_dtype(_widths(builtin_bytes))
    for field, value in [("magic", 0), ("version", 2), ("nv", 23), ("nd", 95), ("mem_id", 8), ("mem_id", -1),
                         ("last_period", 769), ("last_period", -1)]:
        bad = good.copy()
        bad.view(dt)[0][field] = value
        target = ost.State(m)
        before = target.export()
        assert not target.import_(bad), field
        assert np.array_equal(target.export(), before), field
    ok = good.copy()
    ok.view(dt)[0]["last_period"] = 768
    assert ost.State(m).import_(ok)
