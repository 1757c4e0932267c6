"""The wgmma GRU kernel runs a persistent grid: each CTA loops over 64-stream tiles while its producer warp streams the
weights ahead across tile boundaries.  The other GPU tests stay within one tile; this one gives every resident CTA at
least two tiles plus a partial last tile, with silent streams among them, and compares against the FP32 GRU kernel."""
import os

import numpy as np
import pytest

import nnnoiseless_b200 as nb
from conftest import synth_streams
from test_gpu_parity import OUT_REL_RMS, VAD_ATOL, rel_rms

pytestmark = pytest.mark.gpu


def test_persistent_tensor_core_kernel_over_many_tiles_agrees_with_fp32_kernel():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # two resident CTAs per SM of one tile each (or one CTA of two tiles): every CTA runs >= 2 units, the last tile
    # holds 37 streams
    B, T = 64 * 2 * 2 * sms + 37, 4
    x = synth_streams(B, T, seed=4242).reshape(B, T, 480)
    x[::97] = 0.0  # digital silence: rows of the tiles whose state, VAD and gains the kernel must leave alone
    x = np.ascontiguousarray(x.transpose(1, 0, 2))
    tc = nb.DenoiseBatch(B)
    o_tc, v_tc = tc.process_host(x)
    sil = tc.taps()["silence"]
    assert sil[::97].all() and not sil[1::97].any()
    os.environ["NNB_RNN_FP32"] = "1"
    try:
        f = nb.DenoiseBatch(B)
    finally:
        del os.environ["NNB_RNN_FP32"]
    o_fp, v_fp = f.process_host(x)
    assert rel_rms(o_tc, o_fp) <= OUT_REL_RMS and np.abs(v_tc - v_fp).max() <= VAD_ATOL
    # tile by tile, so that one tile left out (or written twice) cannot hide in the batch
    for s0 in range(0, B, 64):
        assert rel_rms(o_tc[:, s0:s0 + 64], o_fp[:, s0:s0 + 64]) <= 10 * OUT_REL_RMS, s0
    assert np.array_equal(v_tc[:, ::97], np.zeros_like(v_tc[:, ::97]))
