"""The wgmma GRU kernel runs a persistent grid: each CTA loops over 64-stream tiles while its producer warp streams the
weights ahead across tile boundaries.  The other GPU tests stay within one tile; this one gives every resident CTA at
least two tiles plus a partial last tile, with silent streams among them.  It compares tile by tile against one
float64 step of the network from the GPU's previous state (tests/test_rnn_kernels.py) and against the mma.sync GRU kernel,
which tiles the streams differently (32 per block, not persistent).  Besides the built-in model, whose 33 weight slabs per tile are a multiple of the 3 ring stages, it runs a model of 17
slabs, so that consecutive tiles start at different ring stages and parities."""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import rnn_ref
from conftest import synth_streams
from test_gpu_parity import OUT_REL_RMS, VAD_ATOL, rel_rms
from test_rnn_kernels import env, one_step_errors, pack_selftest, run_frames

pytestmark = pytest.mark.gpu


def check_many_tiles(model: bytes, name: str):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert pack_selftest(model) >= 0  # runs on the wgmma kernel
    # two resident CTAs per SM: every CTA runs >= 2 tiles, the last tile holds 37 streams
    B, T = 64 * 2 * 2 * sms + 37, 4
    x = synth_streams(B, T, seed=4242).reshape(B, T, 480)
    x[::97] = 0.0  # digital silence: rows of the tiles whose state, VAD and gains the kernel must leave alone
    x = np.ascontiguousarray(x.transpose(1, 0, 2))
    frames = run_frames(model, x, "default")
    sil = frames[-1]["silence"]
    assert sil[::97].all() and not sil[1::97].any()
    worst = one_step_errors(model, frames, tile=64)
    print("wgmma       %-18s" % name, ", ".join("%s %.2e (%.2f of tol)" % (q, e, r) for q, (e, r) in worst.items()))
    with env(NNB_RNN_MMA="1"):
        mma = nb.DenoiseBatch(B, nb.RnnModel.from_bytes(model))
    tc = nb.DenoiseBatch(B, nb.RnnModel.from_bytes(model))
    o_tc, v_tc = tc.process_host(x)
    o_mma, v_mma = mma.process_host(x)
    assert rel_rms(o_tc, o_mma) <= OUT_REL_RMS and np.abs(v_tc - v_mma).max() <= VAD_ATOL
    # tile by tile, so that one tile left out (or written twice) cannot hide in the batch
    for s0 in range(0, B, 64):
        assert rel_rms(o_tc[:, s0:s0 + 64], o_mma[:, s0:s0 + 64]) <= 10 * OUT_REL_RMS, s0
    assert np.array_equal(v_tc[:, ::97], np.zeros_like(v_tc[:, ::97]))


def test_persistent_tensor_core_kernel_over_many_tiles_agrees_with_mma_kernel(builtin_bytes):
    check_many_tiles(builtin_bytes, "builtin")


def test_persistent_tensor_core_kernel_with_ring_wrap_between_tiles():
    """(5, 13, 37, 45): 17 weight slabs per tile, so tile k starts at ring stage 17 k mod 3."""
    check_many_tiles(rnn_ref.make_model(5, 13, 37, 45, seed=7), "5,13,37,45")
