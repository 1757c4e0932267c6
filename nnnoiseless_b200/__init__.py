"""nnnoiseless_b200 -- H100-native (sm_90a CUDA) implementation of nnnoiseless' per-frame denoise path.

This module is a thin ctypes binding over the C ABI in ``include/rnnoise.h`` (the shared library
``nnnoiseless_b200/lib/libnnnoiseless_b200.so`` built by ``nnnoiseless_b200/build.py``).  The names
mirror the reference's Rust API for the path (``src/denoise.rs``, ``src/rnn.rs``):

* :class:`RnnModel` -- ``RnnModel::{default, from_bytes}`` (+ ``from_text`` for RNNoise text models)
* :class:`DenoiseState` -- ``DenoiseState::{new, with_model, process_frame}``, one stream
* :class:`DenoiseBatch` -- N independent ``DenoiseState``s advanced by one call (additive API); single streams are
  saved, restored, moved and reset as state records (``get_states`` / ``set_states`` / ``reset_streams``, decoded by
  :func:`state_dtype`)

There is NO CPU fallback: if the CUDA library is missing or no GPU is visible the constructors raise.
"""
import ctypes as C
import os

import numpy as np

FRAME_SIZE = 480
NB_BANDS = 22
NB_FEATURES = 42

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NNB_LIB") or os.path.join(_HERE, "lib", "libnnnoiseless_b200.so")  # NNB_LIB: a build variant
BUILTIN_WEIGHTS_PATH = os.path.join(_HERE, "data", "weights.rnn")

# every symbol include/rnnoise.h declares (checked by tests/test_capi_symbols.py)
C_ABI_SYMBOLS = [
    "rnnoise_get_frame_size", "rnnoise_get_size", "rnnoise_init", "rnnoise_create", "rnnoise_destroy",
    "rnnoise_process_frame", "rnnoise_model_from_file", "rnnoise_model_free",
    "rnnoise_model_from_bytes", "rnnoise_model_from_text", "rnnoise_model_bytes",
    "rnnoise_batch_create", "rnnoise_batch_destroy", "rnnoise_batch_streams", "rnnoise_batch_reset",
    "rnnoise_batch_process_device", "rnnoise_batch_process_device_pcm16", "rnnoise_batch_process_device_strided",
    "rnnoise_batch_process_host",
    "rnnoise_batch_process_pcm16_host",
    "rnnoise_batch_state_bytes", "rnnoise_batch_get_states", "rnnoise_batch_set_states", "rnnoise_batch_reset_streams",
    "rnnoise_clone", "rnnoise_batch_process_streams_device", "rnnoise_batch_process_streams_host",
    "rnnoise_batch_get_taps", "rnnoise_batch_get_rnn_taps", "rnnoise_batch_get_spectral_taps",
    "rnnoise_batch_profile_step", "rnnoise_kernel_name", "rnnoise_batch_pitch_stats",
    "rnnoise_train_create", "rnnoise_train_destroy", "rnnoise_train_lanes", "rnnoise_train_set_params",
    "rnnoise_train_band_lp", "rnnoise_train_process_host", "rnnoise_train_process_device",
    "rnnoise_denoise_file", "rnnoise_denoise_files", "rnnoise_resample_host",
    "rnnoise_audio_read", "rnnoise_audio_free", "rnnoise_audio_write",
    "rnnoise_kernel_launches", "rnnoise_last_error",
]

_lib = None


class NnnoiselessError(RuntimeError):
    pass


def lib():
    """Load the CUDA shared library (fails loudly if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NnnoiselessError(
            "CUDA library %s is missing: run `python -m nnnoiseless_b200.build` (there is no CPU fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, ci, cf = C.c_void_p, C.c_int, C.c_float
    L.rnnoise_get_frame_size.restype = ci
    L.rnnoise_get_size.restype = ci
    L.rnnoise_init.restype = ci
    L.rnnoise_init.argtypes = [vp, vp]
    L.rnnoise_create.restype = vp
    L.rnnoise_create.argtypes = [vp]
    L.rnnoise_destroy.argtypes = [vp]
    L.rnnoise_process_frame.restype = cf
    L.rnnoise_process_frame.argtypes = [vp, vp, vp]
    L.rnnoise_model_from_file.restype = vp
    L.rnnoise_model_from_file.argtypes = [vp]
    L.rnnoise_model_free.argtypes = [vp]
    L.rnnoise_model_from_bytes.restype = vp
    L.rnnoise_model_from_bytes.argtypes = [C.c_char_p, C.c_size_t]
    L.rnnoise_model_from_text.restype = vp
    L.rnnoise_model_from_text.argtypes = [C.c_char_p, C.c_size_t]
    L.rnnoise_model_bytes.restype = C.c_size_t
    L.rnnoise_model_bytes.argtypes = [vp, vp, C.c_size_t]
    L.rnnoise_batch_create.restype = vp
    L.rnnoise_batch_create.argtypes = [vp, ci, ci]
    L.rnnoise_batch_destroy.argtypes = [vp]
    L.rnnoise_batch_streams.restype = ci
    L.rnnoise_batch_streams.argtypes = [vp]
    L.rnnoise_batch_reset.restype = ci
    L.rnnoise_batch_reset.argtypes = [vp]
    L.rnnoise_batch_process_device.restype = ci
    L.rnnoise_batch_process_device.argtypes = [vp, vp, vp, vp, ci, C.c_long, C.c_long, vp]
    L.rnnoise_batch_process_device_pcm16.restype = ci
    L.rnnoise_batch_process_device_pcm16.argtypes = [vp, vp, vp, vp, ci, C.c_long, C.c_long, vp]
    L.rnnoise_batch_process_device_strided.restype = ci
    L.rnnoise_batch_process_device_strided.argtypes = [vp, vp, vp, ci, vp, ci, C.c_long, C.c_long, C.c_long, vp]
    L.rnnoise_batch_process_host.restype = ci
    L.rnnoise_batch_process_host.argtypes = [vp, vp, vp, vp, ci]
    L.rnnoise_batch_process_pcm16_host.restype = ci
    L.rnnoise_batch_process_pcm16_host.argtypes = [vp, vp, vp, vp, ci]
    L.rnnoise_batch_state_bytes.restype = C.c_size_t
    L.rnnoise_batch_state_bytes.argtypes = [vp]
    L.rnnoise_batch_get_states.restype = ci
    L.rnnoise_batch_get_states.argtypes = [vp, vp, ci, vp, vp]
    L.rnnoise_batch_set_states.restype = ci
    L.rnnoise_batch_set_states.argtypes = [vp, vp, ci, vp, vp]
    L.rnnoise_batch_reset_streams.restype = ci
    L.rnnoise_batch_reset_streams.argtypes = [vp, vp, ci, vp]
    L.rnnoise_clone.restype = vp
    L.rnnoise_clone.argtypes = [vp]
    L.rnnoise_batch_process_streams_device.restype = ci
    L.rnnoise_batch_process_streams_device.argtypes = [vp, vp, ci, vp, vp, ci, vp, ci, C.c_long, C.c_long, C.c_long, vp]
    L.rnnoise_batch_process_streams_host.restype = ci
    L.rnnoise_batch_process_streams_host.argtypes = [vp, vp, ci, vp, vp, vp, ci]
    L.rnnoise_batch_get_taps.restype = ci
    L.rnnoise_batch_get_taps.argtypes = [vp, vp, vp, vp, vp]
    L.rnnoise_batch_get_rnn_taps.restype = ci
    L.rnnoise_batch_get_rnn_taps.argtypes = [vp, vp, vp, vp]
    L.rnnoise_batch_get_spectral_taps.restype = ci
    L.rnnoise_batch_get_spectral_taps.argtypes = [vp, vp, vp, vp, vp, vp]
    L.rnnoise_batch_pitch_stats.restype = ci
    L.rnnoise_batch_pitch_stats.argtypes = [vp, vp]
    L.rnnoise_batch_profile_step.restype = ci
    L.rnnoise_batch_profile_step.argtypes = [vp, vp, vp, vp, C.c_long, vp, vp, ci]
    L.rnnoise_train_create.restype = vp
    L.rnnoise_train_create.argtypes = [ci, ci]
    L.rnnoise_train_destroy.argtypes = [vp]
    L.rnnoise_train_lanes.restype = ci
    L.rnnoise_train_lanes.argtypes = [vp]
    L.rnnoise_train_set_params.restype = ci
    L.rnnoise_train_set_params.argtypes = [vp, ci, ci, vp]
    L.rnnoise_train_band_lp.restype = ci
    L.rnnoise_train_band_lp.argtypes = [ci]
    L.rnnoise_train_process_host.restype = ci
    L.rnnoise_train_process_host.argtypes = [vp, vp, vp, vp, ci]
    L.rnnoise_train_process_device.restype = ci
    L.rnnoise_train_process_device.argtypes = [vp, vp, vp, vp, ci, C.c_long, C.c_long, C.c_long, C.c_long, vp]
    L.rnnoise_denoise_file.restype = ci
    L.rnnoise_denoise_file.argtypes = [C.c_char_p, C.c_char_p, vp]
    L.rnnoise_denoise_files.restype = ci
    L.rnnoise_denoise_files.argtypes = [ci, vp, vp, vp]
    L.rnnoise_resample_host.restype = C.c_long
    L.rnnoise_resample_host.argtypes = [vp, C.c_long, vp, C.c_long, ci, C.c_double, ci]
    L.rnnoise_audio_read.restype = ci
    L.rnnoise_audio_read.argtypes = [C.c_char_p, ci, ci, C.c_double, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_long),
                                     C.POINTER(ci), C.POINTER(C.c_double)]
    L.rnnoise_audio_free.argtypes = [C.POINTER(C.c_float)]
    L.rnnoise_audio_write.restype = ci
    L.rnnoise_audio_write.argtypes = [C.c_char_p, ci, vp, C.c_long, ci]
    L.rnnoise_kernel_name.restype = C.c_char_p
    L.rnnoise_kernel_name.argtypes = [ci]
    L.rnnoise_kernel_launches.restype = C.c_ulonglong
    L.rnnoise_last_error.restype = C.c_char_p
    _lib = L
    return L


def last_error() -> str:
    return lib().rnnoise_last_error().decode("utf-8", "replace")


def kernel_launches() -> int:
    return int(lib().rnnoise_kernel_launches())


def _np_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class RnnModel:
    """``RnnModel`` (src/rnn.rs:55-94).  ``RnnModel()`` is the built-in model (``Default``)."""

    def __init__(self, _handle=None):
        self._h = _handle  # None = built-in (NULL at the C ABI)

    @classmethod
    def from_bytes(cls, data: bytes):
        """``RnnModel::from_bytes``: returns None for malformed bytes, like the reference's Option."""
        h = lib().rnnoise_model_from_bytes(bytes(data), len(data))
        return cls(h) if h else None

    @classmethod
    def from_text(cls, text):
        """RNNoise text format (train/convert_rnnoise.py) -> model; None if malformed."""
        if isinstance(text, str):
            text = text.encode("ascii")
        h = lib().rnnoise_model_from_text(text, len(text))
        return cls(h) if h else None

    def to_bytes(self) -> bytes:
        n = lib().rnnoise_model_bytes(self._h, None, 0)
        buf = (C.c_ubyte * n)()
        lib().rnnoise_model_bytes(self._h, buf, n)
        return bytes(buf)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None:
            _lib.rnnoise_model_free(h)
            self._h = None


class DenoiseState:
    """``DenoiseState`` (src/denoise.rs:37-116) for ONE stream, through the legacy rnnoise_* ABI."""

    FRAME_SIZE = FRAME_SIZE

    def __init__(self, model: RnnModel = None):
        self._model = model  # borrowed by the state: keep it alive (src/capi.rs:53)
        self._h = lib().rnnoise_create(model._h if model is not None else None)
        if not self._h:
            raise NnnoiselessError("rnnoise_create failed: " + last_error())

    @classmethod
    def new(cls):
        return cls()

    @classmethod
    def with_model(cls, model: RnnModel):
        return cls(model)

    from_model = with_model

    def process_frame(self, output: np.ndarray, input: np.ndarray) -> float:
        """``process_frame(&mut self, output, input) -> f32``; panics (raises) unless both are 480 long."""
        if input.shape != (FRAME_SIZE,) or output.shape != (FRAME_SIZE,):
            raise ValueError("process_frame needs 480-sample input and output")  # assert!, src/features.rs:98
        if input.dtype != np.float32 or output.dtype != np.float32:
            raise TypeError("float32 buffers required")
        if not (input.flags.c_contiguous and output.flags.c_contiguous):
            raise ValueError("contiguous buffers required")
        return float(lib().rnnoise_process_frame(self._h, _np_ptr(output), _np_ptr(input)))

    def clone(self):
        """``impl Clone for DenoiseState`` (src/denoise.rs:36): an independent state with the same model whose next
        frames give the same bits as this one's."""
        h = lib().rnnoise_clone(self._h)
        if not h:
            raise NnnoiselessError("rnnoise_clone failed: " + last_error())
        c = DenoiseState.__new__(DenoiseState)
        c._model, c._h = self._model, h
        return c

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None:
            _lib.rnnoise_destroy(h)
            self._h = None


class DenoiseBatch:
    """N independent ``DenoiseState``s on one GPU, advanced together (rnnoise_batch_* in include/rnnoise.h)."""

    def __init__(self, n_streams: int, model: RnnModel = None, device: int = -1):
        self.n_streams = int(n_streams)
        self._h = lib().rnnoise_batch_create(model._h if model is not None else None, self.n_streams, int(device))
        if not self._h:
            raise NnnoiselessError("rnnoise_batch_create failed: " + last_error())
        self.gru_widths = gru_widths((model or RnnModel()).to_bytes())

    def reset(self):
        if lib().rnnoise_batch_reset(self._h) != 0:
            raise NnnoiselessError(last_error())

    def process_host(self, x: np.ndarray, want_vad=True):
        """x: [T][B][480] float32 host array -> (out [T][B][480], vad [T][B])."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        T, B, F = x.shape
        if B != self.n_streams or F != FRAME_SIZE:
            raise ValueError("expected [T][%d][480]" % self.n_streams)
        out = np.empty_like(x)
        vad = np.empty((T, B), np.float32) if want_vad else None
        rc = lib().rnnoise_batch_process_host(self._h, _np_ptr(out), _np_ptr(x), _np_ptr(vad) if want_vad else None, T)
        if rc != 0:
            raise NnnoiselessError(last_error())
        return out, vad

    def process_pcm16_host(self, x: np.ndarray):
        """x: [T][B][480] int16 -> (out int16 [T][B][480], vad [T][B])."""
        x = np.ascontiguousarray(x, dtype=np.int16)
        T, B, F = x.shape
        if B != self.n_streams or F != FRAME_SIZE:
            raise ValueError("expected [T][%d][480]" % self.n_streams)
        out = np.empty_like(x)
        vad = np.empty((T, B), np.float32)
        rc = lib().rnnoise_batch_process_pcm16_host(self._h, _np_ptr(out), _np_ptr(x), _np_ptr(vad), T)
        if rc != 0:
            raise NnnoiselessError(last_error())
        return out, vad

    def process_device(self, out_ptr: int, in_ptr: int, vad_ptr: int, n_frames: int, stream_stride: int,
                       frame_stride: int, cuda_stream: int = 0, pcm16: bool = False):
        """Raw device pointers (e.g. torch tensors' data_ptr()); strides in samples (float32, or int16 if pcm16)."""
        fn = lib().rnnoise_batch_process_device_pcm16 if pcm16 else lib().rnnoise_batch_process_device
        rc = fn(self._h, C.c_void_p(out_ptr), C.c_void_p(in_ptr),
                                                C.c_void_p(vad_ptr) if vad_ptr else None, int(n_frames),
                                                int(stream_stride), int(frame_stride),
                                                C.c_void_p(cuda_stream) if cuda_stream else None)
        if rc != 0:
            raise NnnoiselessError(last_error())

    def profile_step(self, out_ptr: int, in_ptr: int, vad_ptr: int, stream_stride: int, cuda_stream: int = 0):
        """One frame with CUDA events between the kernels: returns {kernel name: milliseconds}."""
        ms = (C.c_float * 16)()
        n = lib().rnnoise_batch_profile_step(self._h, C.c_void_p(out_ptr), C.c_void_p(in_ptr),
                                             C.c_void_p(vad_ptr) if vad_ptr else None, int(stream_stride),
                                             C.c_void_p(cuda_stream) if cuda_stream else None, ms, 16)
        if n < 0:
            raise NnnoiselessError(last_error())
        return {lib().rnnoise_kernel_name(i).decode(): float(ms[i]) for i in range(n)}

    def pitch_stats(self):
        """Cumulative pitch-kernel certification counters: dict(coarse_exact, ladder_exact, stream_frames)."""
        out = (C.c_ulonglong * 3)()
        if lib().rnnoise_batch_pitch_stats(self._h, out) != 0:
            raise NnnoiselessError(last_error())
        return dict(coarse_exact=int(out[0]), ladder_exact=int(out[1]), stream_frames=int(out[2]))

    def taps(self):
        """Intermediates of the most recent frame: dict(pitch, silence, features, gains)."""
        B = self.n_streams
        pitch = np.empty(B, np.int32)
        silence = np.empty(B, np.int32)
        feats = np.empty((B, NB_FEATURES), np.float32)
        gains = np.empty((B, NB_BANDS), np.float32)
        rc = lib().rnnoise_batch_get_taps(self._h, _np_ptr(pitch), _np_ptr(silence), _np_ptr(feats), _np_ptr(gains))
        if rc != 0:
            raise NnnoiselessError(last_error())
        return dict(pitch=pitch, silence=silence, features=feats, gains=gains)

    def rnn_taps(self):
        """The GRU network's raw outputs of the most recent frame and its state after it: dict(gains [B][22] before
        the gain floor, vad [B], gru_state [B][vad + noise + denoise GRU neurons]).  Streams whose frame was silent
        keep their state, and their gains and vad entries are stale."""
        B = self.n_streams
        gains = np.empty((B, NB_BANDS), np.float32)
        vad = np.empty(B, np.float32)
        state = np.empty((B, sum(self.gru_widths)), np.float32)
        rc = lib().rnnoise_batch_get_rnn_taps(self._h, _np_ptr(gains), _np_ptr(vad), _np_ptr(state))
        if rc != 0:
            raise NnnoiselessError(last_error())
        return dict(gains=gains, vad=vad, gru_state=state)

    def spectral_taps(self):
        """The spectra and band quantities analysis hands to synthesis in the most recent frame: dict(X complex64
        [B][481], P complex64 [B][400] (the banded bins only), ex, ep, exp float32 [B][22]), exp = corr / sqrt(0.001 +
        ex * ep).  Written on silent frames too."""
        B = self.n_streams
        X = np.empty((B, 481), np.complex64)
        P = np.empty((B, 400), np.complex64)
        ex, ep, exp = (np.empty((B, NB_BANDS), np.float32) for _ in range(3))
        rc = lib().rnnoise_batch_get_spectral_taps(self._h, _np_ptr(X), _np_ptr(P), _np_ptr(ex), _np_ptr(ep), _np_ptr(exp))
        if rc != 0:
            raise NnnoiselessError(last_error())
        return dict(X=X, P=P, ex=ex, ep=ep, exp=exp)

    # ---- per-stream state records (layout: state_dtype, include/rnnoise.h) ----
    @property
    def state_bytes(self) -> int:
        """Size of one stream's state record."""
        return int(lib().rnnoise_batch_state_bytes(self._h))

    def _streams(self, streams):
        """-> (int32 array or None, n): None stands for every stream of the batch."""
        if streams is None:
            return None, self.n_streams
        idx = np.ascontiguousarray(streams, dtype=np.int32).reshape(-1)
        return idx, len(idx)

    def get_states(self, streams=None) -> np.ndarray:
        """State records of the given streams (default: all) as uint8 [n][state_bytes]; decode with state_dtype."""
        idx, n = self._streams(streams)
        out = np.empty((n, self.state_bytes), np.uint8)
        if lib().rnnoise_batch_get_states(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out), None) != 0:
            raise NnnoiselessError(last_error())
        return out

    def set_states(self, records, streams=None):
        """Import records (uint8 [n][state_bytes] or an array of state_dtype) into the given streams (default: 0..n-1).
        Every record and index is validated first; on an error nothing changes."""
        rec = np.ascontiguousarray(records)
        rec = rec.view(np.uint8).reshape(-1, self.state_bytes) if rec.size else rec.reshape(0, self.state_bytes)
        idx, n = self._streams(streams)
        if streams is None:
            n = rec.shape[0]
        elif n != rec.shape[0]:
            raise ValueError("%d records for %d streams" % (rec.shape[0], n))
        if lib().rnnoise_batch_set_states(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(rec), None) != 0:
            raise NnnoiselessError(last_error())

    def reset_streams(self, streams):
        """Reset the given streams to the freshly created state; the other streams are not touched."""
        idx, n = self._streams(streams)
        if lib().rnnoise_batch_reset_streams(self._h, _np_ptr(idx) if idx is not None else None, n, None) != 0:
            raise NnnoiselessError(last_error())

    def get_states_device(self, dst_ptr: int, streams=None, cuda_stream: int = 0):
        """get_states into device memory at dst_ptr (e.g. a torch tensor's data_ptr()); asynchronous on cuda_stream."""
        idx, n = self._streams(streams)
        rc = lib().rnnoise_batch_get_states(self._h, _np_ptr(idx) if idx is not None else None, n, C.c_void_p(dst_ptr),
                                            C.c_void_p(cuda_stream) if cuda_stream else None)
        if rc != 0:
            raise NnnoiselessError(last_error())

    def set_states_device(self, src_ptr: int, streams=None, cuda_stream: int = 0):
        """set_states from device memory at src_ptr holding one record per stream; ordered on cuda_stream (the records'
        heads are validated on the host, which waits for cuda_stream)."""
        idx, n = self._streams(streams)
        rc = lib().rnnoise_batch_set_states(self._h, _np_ptr(idx) if idx is not None else None, n, C.c_void_p(src_ptr),
                                            C.c_void_p(cuda_stream) if cuda_stream else None)
        if rc != 0:
            raise NnnoiselessError(last_error())

    # ---- subset calls: advance only the listed streams ----
    def process_streams_host(self, streams, x: np.ndarray, want_vad=True):
        """Advance only the given streams (None: 0..n-1) by T frames; the others are not touched.
        x: [T][n][480] float32, row r of every frame belonging to streams[r] -> (out [T][n][480], vad [T][n])."""
        idx, n = self._streams(streams)
        x = np.ascontiguousarray(x, dtype=np.float32)
        if streams is None:
            n = x.shape[1] if x.ndim == 3 else -1
        if x.ndim != 3 or x.shape[1] != n or x.shape[2] != FRAME_SIZE:
            raise ValueError("expected [T][%d][480]" % n)
        T = x.shape[0]
        out = np.empty_like(x)
        vad = np.empty((T, n), np.float32) if want_vad else None
        rc = lib().rnnoise_batch_process_streams_host(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out), _np_ptr(x),
                                                      _np_ptr(vad) if want_vad else None, T)
        if rc != 0:
            raise NnnoiselessError(last_error())
        return out, vad

    def process_streams_device(self, streams, out_ptr: int, in_ptr: int, vad_ptr: int, n_frames: int, stream_stride: int,
                               frame_stride: int, sample_stride: int = 1, pcm16: int = 0, cuda_stream: int = 0, n: int = None):
        """Advance only the given streams by n_frames frames through raw device pointers: sample (r, t, i) of stream
        streams[r] at ptr[r*stream_stride + t*frame_stride + i*sample_stride] (element strides), vad [n_frames][n] or 0.
        pcm16 as rnnoise_batch_process_device_strided.  streams None: streams 0..n-1 (n required)."""
        idx, k = self._streams(streams)
        if streams is None:
            if n is None:
                raise ValueError("streams=None needs n")
            k = int(n)
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_batch_process_streams_device(self._h, _np_ptr(idx) if idx is not None else None, k, ptr(out_ptr), ptr(in_ptr),
                                                        int(pcm16), ptr(vad_ptr), int(n_frames), int(stream_stride), int(sample_stride),
                                                        int(frame_stride), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None:
            _lib.rnnoise_batch_destroy(h)
            self._h = None


def gru_widths(model_bytes: bytes):
    """Neurons of the vad, noise and denoise GRUs of a model image that RnnModel.from_bytes accepts (src/rnn.rs:116-232:
    a [nb_inputs, nb_neurons, activation] header per layer, then the int8 weights)."""
    b = bytes(model_bytes)
    p = 3 + 42 * b[1] + b[1]  # past input_dense: 42 x nd weights, nd biases
    widths = []
    for _ in range(3):
        ni, nn = b[p], b[p + 1]
        widths.append(nn)
        p += 3 + 3 * nn * (ni + nn + 1)
    return tuple(widths)


STATE_MAGIC = 0x54534E52  # "RNST", RNNOISE_STATE_MAGIC
STATE_VERSION = 1


def state_bytes(widths) -> int:
    """Size of a state record for GRU widths (nv, nn, nd): 9664 + 4 (nv + nn + nd), rounded up to a multiple of 16."""
    return (9664 + 4 * sum(int(w) for w in widths) + 15) & ~15


def state_dtype(widths) -> np.dtype:
    """numpy structured dtype of one state record (include/rnnoise.h) for GRU widths (nv, nn, nd): the persistent fields
    of the reference's DenoiseState under their reference names."""
    nv, nn, nd = (int(w) for w in widths)
    f4, i4 = "<f4", "<i4"
    fields = [("magic", "<u4", 0), ("version", i4, 4), ("nv", i4, 8), ("nn", i4, 12), ("nd", i4, 16), ("mem_id", i4, 20),
              ("last_period", i4, 24), ("last_gain", f4, 28), ("mem_hp_x", (f4, (2,)), 32), ("lastg", (f4, (NB_BANDS,)), 40),
              ("input_mem", (f4, (1728,)), 128), ("cepstral_mem", (f4, (8, NB_BANDS)), 7040),
              ("synthesis_mem", (f4, (FRAME_SIZE,)), 7744), ("vad_gru", (f4, (nv,)), 9664),
              ("noise_gru", (f4, (nn,)), 9664 + 4 * nv), ("denoise_gru", (f4, (nd,)), 9664 + 4 * (nv + nn))]
    return np.dtype({"names": [f[0] for f in fields], "formats": [f[1] for f in fields], "offsets": [f[2] for f in fields],
                     "itemsize": state_bytes((nv, nn, nd))})


def shard_streams(n_streams: int, world_size: int, rank: int):
    """Contiguous block sharding of independent streams over ranks (SURVEY 8(e)): returns (start, count)."""
    base, rem = divmod(int(n_streams), int(world_size))
    start = rank * base + min(rank, rem)
    return start, base + (1 if rank < rem else 0)
