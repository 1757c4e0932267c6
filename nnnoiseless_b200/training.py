"""Training-data rows on the GPU: host-side mirror of the reference's ``nnnoiseless-gen-training-data`` loop.

Reference: ``src/training.rs``.  The split is

* host (this module, plain numpy): ``NoiseSimulator::randomize`` (:352-377) -- the random gains, random biquads and
  the low-pass band, drawn every ``GAIN_CHANGE_COUNT`` frames -- and whatever feeds the frames (the reference's
  ``SignalReader`` reads 48 kHz mono 16-bit WAV files, :183-262);
* device (``rnnoise_train_*`` in include/rnnoise.h): everything arithmetic per frame -- gains, filters, mix, the
  VAD counter, three feature extractors, and the 87-float output row.

There is NO CPU fallback: without the CUDA library / a GPU the constructor raises.
"""
import ctypes as C

import numpy as np

from . import FRAME_SIZE, NB_BANDS, NB_FEATURES, DenoiseBatch, NnnoiselessError, RnnModel, _np_ptr, gru_widths, last_error, lib

TRAIN_ROW = NB_FEATURES + 2 * NB_BANDS + 1  # 87, src/training.rs:90
GAIN_CHANGE_COUNT = 2821                    # src/training.rs:17
FREQ_SIZE = 481

SIM_PARAMS_DTYPE = np.dtype([
    ("signal_gain", np.float32), ("noise_gain", np.float32),
    ("sig_a", np.float32, 2), ("sig_b", np.float32, 2),
    ("noise_a", np.float32, 2), ("noise_b", np.float32, 2),
    ("band_lp", np.int32),
])  # == RNNoiseSimParams
assert SIM_PARAMS_DTYPE.itemsize == 44


def default_params(n: int) -> np.ndarray:
    """``NoiseSimulator::new`` (src/training.rs:319-340) for n lanes."""
    p = np.zeros(n, SIM_PARAMS_DTYPE)
    p["signal_gain"] = 1.0
    p["noise_gain"] = 1.0
    p["band_lp"] = NB_BANDS - 1
    return p


def band_lp_for(lowpass: int) -> int:
    return int(lib().rnnoise_train_band_lp(int(lowpass)))


def randomize(n: int, rng: np.random.Generator) -> np.ndarray:
    """``NoiseSimulator::randomize`` (src/training.rs:352-377) for n lanes: same distributions, numpy's generator
    (the reference draws from ``thread_rng``, so its streams are not reproducible either)."""
    p = np.zeros(n, SIM_PARAMS_DTYPE)
    f32 = np.float32
    sg = np.power(f32(10.0), rng.integers(-40, 20, n).astype(f32) / f32(20.0)).astype(f32)
    ng = np.power(f32(10.0), rng.integers(-20, 20, n).astype(f32) / f32(20.0)).astype(f32) * sg
    sg = np.where(rng.random(n) < 0.1, f32(0.0), sg)  # after noise_gain took the un-zeroed signal gain (:357-366)
    p["signal_gain"], p["noise_gain"] = sg, ng
    for k in ("sig_a", "sig_b", "noise_a", "noise_b"):  # random_filter, :311-317
        p[k] = (f32(0.75) * (rng.random((n, 2), dtype=f32) - f32(0.5))).astype(f32)
    lowpass = (f32(FREQ_SIZE) * f32(3000.0) / f32(24000.0) * np.power(f32(50.0), rng.random(n, dtype=f32))).astype(np.int64)
    p["band_lp"] = [band_lp_for(int(v)) for v in lowpass]
    return p


class TrainingBatch:
    """n_lanes independent (NoiseSimulator + 3 x DenoiseFeatures) on one GPU."""

    def __init__(self, n_lanes: int, device: int = -1):
        self.n_lanes = int(n_lanes)
        self._h = lib().rnnoise_train_create(self.n_lanes, int(device))
        if not self._h:
            raise NnnoiselessError("rnnoise_train_create failed: " + last_error())

    def set_params(self, params: np.ndarray, first_lane: int = 0):
        params = np.ascontiguousarray(params, dtype=SIM_PARAMS_DTYPE)
        if lib().rnnoise_train_set_params(self._h, int(first_lane), len(params), _np_ptr(params)) != 0:
            raise NnnoiselessError(last_error())

    def process_host(self, signal: np.ndarray, noise: np.ndarray) -> np.ndarray:
        """signal, noise: [T][L][480] float32 (i16-valued) -> rows [T][L][87]."""
        signal = np.ascontiguousarray(signal, dtype=np.float32)
        noise = np.ascontiguousarray(noise, dtype=np.float32)
        T, L, F = signal.shape
        if noise.shape != signal.shape or L != self.n_lanes or F != FRAME_SIZE:
            raise ValueError("expected two [T][%d][480] arrays" % self.n_lanes)
        rows = np.empty((T, L, TRAIN_ROW), np.float32)
        if lib().rnnoise_train_process_host(self._h, _np_ptr(rows), _np_ptr(signal), _np_ptr(noise), T) != 0:
            raise NnnoiselessError(last_error())
        return rows

    def process_device(self, rows_ptr, signal_ptr, noise_ptr, n_frames, stream_stride, frame_stride, row_lane_stride,
                       row_frame_stride, cuda_stream=0):
        rc = lib().rnnoise_train_process_device(self._h, C.c_void_p(rows_ptr), C.c_void_p(signal_ptr), C.c_void_p(noise_ptr),
                                                int(n_frames), int(stream_stride), int(frame_stride), int(row_lane_stride),
                                                int(row_frame_stride), C.c_void_p(cuda_stream) if cuda_stream else None)
        if rc != 0:
            raise NnnoiselessError(last_error())

    def feature_batch(self) -> "FeatureBatchView":
        """Debug view of the 3 n_lanes feature extractors (stream l: lane l's clean signal, n_lanes + l: its noise,
        2 n_lanes + l: its combined signal) for the DenoiseBatch reads taps(), spectral_taps(), get_states() and
        state_bytes, which describe the most recent frame.  Borrowed: it keeps this trainer alive."""
        h = lib().rnnoise_train_feature_batch(self._h)
        if not h:
            raise NnnoiselessError(last_error())
        return FeatureBatchView(self, h)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib().rnnoise_train_destroy(h)
            self._h = None


class FeatureBatchView(DenoiseBatch):
    """A TrainingBatch's feature batch, borrowed (rnnoise_train_feature_batch): only the reads are allowed on it."""

    def __init__(self, owner: TrainingBatch, handle):
        self._owner = owner
        self._h = handle
        self.n_streams = 3 * owner.n_lanes
        self.gru_widths = gru_widths(RnnModel().to_bytes())  # the trainer's batch runs the built-in model's geometry

    def __del__(self):
        self._h = None  # the trainer owns the batch
