"""GPU tests of the conventions every C-ABI creator and entry point shares (DESIGN.md §1): a creator refuses a device
index past the last device and leaves the caller's current device as it was, and the batch and the resampler check a
list of stream indices with the same texts.  Every case is an argument error, rejected before any kernel runs."""
import numpy as np
import pytest
import torch

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import files, fit, training

pytestmark = pytest.mark.gpu


def _error(call) -> str:
    with pytest.raises(nb.NnnoiselessError) as e:
        call()
    return str(e.value)


def test_creators_refuse_a_device_index_out_of_range(tmp_path):
    bad = torch.cuda.device_count()
    wav = tmp_path / "in.wav"
    files.write_audio(str(wav), np.zeros((4 * 480, 1), np.int16))  # four 48 kHz frames: enough to need the device
    creators = {
        "DenoiseBatch": lambda: nb.DenoiseBatch(4, device=bad),
        "TrainingBatch": lambda: training.TrainingBatch(4, device=bad),
        "Resampler": lambda: nb.Resampler(4, device=bad),
        "Fit": lambda: fit.Fit(max_sequences=1, window=10, device=bad),
        "resample": lambda: files.resample(np.zeros((480, 1), np.float32), 0.5, device=bad),
        "denoise_files": lambda: files.denoise_files([(str(wav), str(tmp_path / "out.wav"))], device=bad),
    }
    current = torch.cuda.current_device()
    for name, create in creators.items():
        assert "device index out of range" in _error(create), name
        assert torch.cuda.current_device() == current, name


def test_batch_and_resampler_check_stream_lists_alike():
    batch, rs = nb.DenoiseBatch(4), nb.Resampler(4)
    for streams, text in [([0, 4], "stream index 4 out of range"), ([-1], "stream index -1 out of range"),
                          ([1, 2, 1], "stream index 1 given twice")]:
        assert _error(lambda: batch.stream_models(streams)) == text
        assert _error(lambda: rs.stream_rates(streams)) == text
    assert _error(lambda: batch.set_stream_models([0] * 5)) == "more streams than the batch holds"
    assert _error(lambda: rs.set_stream_rates([48000] * 5)) == "more streams than the resampler holds"
