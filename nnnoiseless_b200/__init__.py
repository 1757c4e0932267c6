"""nnnoiseless_b200 -- H100-native (sm_90a CUDA) implementation of nnnoiseless' per-frame denoise path.

This module is a thin ctypes binding over the C ABI in ``include/rnnoise.h`` (the shared library
``nnnoiseless_b200/lib/libnnnoiseless_b200.so`` built by ``nnnoiseless_b200/build.py``).  The names
mirror the reference's Rust API for the path (``src/denoise.rs``, ``src/rnn.rs``):

* :class:`RnnModel` -- ``RnnModel::{default, from_bytes}`` (+ ``from_text`` for RNNoise text models)
* :class:`DenoiseState` -- ``DenoiseState::{new, with_model, process_frame}``, one stream
* :class:`DenoiseBatch` -- N independent ``DenoiseState``s advanced by one call (additive API); single streams are
  saved, restored, moved and reset as state records (``get_states`` / ``set_states`` / ``reset_streams``, decoded by
  :func:`state_dtype`)
* :class:`DenoiseBatch` streams each carry a controls record (``set_stream_controls`` / ``get_stream_controls``,
  :data:`STREAM_CONTROLS_DTYPE`): an attenuation limit and a voice-activity gate applied inside synthesis
* :class:`DenoiseBatch` streams can be linked in groups (``link_streams`` / ``unlink_streams`` / ``stream_links``): the
  group's members share one band-gain curve, e.g. the channels of one recording
* :class:`Metrics` -- quality metrics against clean speech accumulated on the GPU (:data:`METRICS_DTYPE` records;
  ``nnnoiseless_b200.metrics.summarize``, ``nnnoiseless_b200.evaluate``)
* :func:`intelligibility` / :func:`intelligibility_device` -- STOI and ESTOI of clips on the GPU
  (:data:`INTELLIGIBILITY_DTYPE` records); :func:`intelligibility_backward_device` their gradient with respect to the
  processed signal (``nnnoiseless_b200.autograd.intelligibility`` as a torch loss)
* :class:`Resampler` -- per-stream sample rates (8 to 48 kHz) for a batch: ``DenoiseBatch.process_native_host`` /
  ``process_native_device`` resample each stream to and from the 48 kHz path on the GPU

There is NO CPU fallback: if the CUDA library is missing or no GPU is visible the constructors raise.
"""
import ctypes as C
import os

import numpy as np

FRAME_SIZE = 480
NB_BANDS = 22
NB_FEATURES = 42
SYNTH_CONTEXT_BYTES = 7552  # RNNOISE_SYNTH_CONTEXT_BYTES: one saved synthesis context (include/rnnoise.h)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NNB_LIB") or os.path.join(_HERE, "lib", "libnnnoiseless_b200.so")  # NNB_LIB: a build variant
BUILTIN_WEIGHTS_PATH = os.path.join(_HERE, "data", "weights.rnn")

# every symbol include/rnnoise.h declares (checked by tests/test_host_cpu.py::test_header_symbols_exported)
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
    "rnnoise_train_create", "rnnoise_train_destroy", "rnnoise_train_lanes", "rnnoise_train_feature_batch",
    "rnnoise_train_set_params",
    "rnnoise_train_band_lp", "rnnoise_train_process_host", "rnnoise_train_process_device", "rnnoise_train_process_pool_host",
    "rnnoise_train_reset", "rnnoise_train_pool_reserve", "rnnoise_train_pool_write", "rnnoise_train_pool_samples",
    "rnnoise_train_pool_room", "rnnoise_train_waves_device",
    "rnnoise_denoise_file", "rnnoise_denoise_files", "rnnoise_resample_host",
    "rnnoise_audio_read", "rnnoise_audio_free", "rnnoise_audio_write", "rnnoise_audio_probe",
    "rnnoise_kernel_launches", "rnnoise_last_error",
    "rnnoise_batch_add_model", "rnnoise_batch_set_stream_models", "rnnoise_batch_get_stream_models",
    "rnnoise_batch_set_stream_controls", "rnnoise_batch_get_stream_controls",
    "rnnoise_batch_link_streams", "rnnoise_batch_unlink_streams", "rnnoise_batch_get_stream_links",
    "rnnoise_denoise_files_linked", "rnnoise_denoise_corpus",
    "rnnoise_batch_pending_frames", "rnnoise_batch_analyze_device", "rnnoise_batch_synthesize_device",
    "rnnoise_batch_synthesize_saving_device", "rnnoise_synthesis_backward_workspace_bytes", "rnnoise_synthesis_backward_device",
    "rnnoise_batch_window_frames", "rnnoise_batch_analyze_window_device", "rnnoise_batch_synthesize_window_device",
    "rnnoise_fit_create", "rnnoise_fit_destroy", "rnnoise_fit_n_params", "rnnoise_fit_get_params", "rnnoise_fit_set_params",
    "rnnoise_fit_set_params_from_model", "rnnoise_fit_step", "rnnoise_fit_evaluate", "rnnoise_fit_get_grads",
    "rnnoise_fit_get_activations", "rnnoise_fit_export", "rnnoise_fit_export_params", "rnnoise_fit_forward_device",
    "rnnoise_fit_backward_device", "rnnoise_fit_set_taps", "rnnoise_fit_get_taps",
    "rnnoise_resampler_filter", "rnnoise_resampler_delay", "rnnoise_resampler_create", "rnnoise_resampler_destroy",
    "rnnoise_resampler_set_stream_rates", "rnnoise_resampler_get_stream_rates", "rnnoise_resampler_up_device",
    "rnnoise_resampler_down_device", "rnnoise_resampler_get_states", "rnnoise_resampler_set_states",
    "rnnoise_batch_process_native_device", "rnnoise_batch_process_native_host",
    "rnnoise_metrics_create", "rnnoise_metrics_destroy", "rnnoise_metrics_accumulate_device", "rnnoise_metrics_clear",
    "rnnoise_metrics_get", "rnnoise_intelligibility_workspace_bytes", "rnnoise_intelligibility_device",
    "rnnoise_intelligibility_backward_workspace_bytes", "rnnoise_intelligibility_backward_device",
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
    L.rnnoise_train_feature_batch.restype = vp
    L.rnnoise_train_feature_batch.argtypes = [vp]
    L.rnnoise_train_set_params.restype = ci
    L.rnnoise_train_set_params.argtypes = [vp, ci, ci, vp]
    L.rnnoise_train_band_lp.restype = ci
    L.rnnoise_train_band_lp.argtypes = [ci]
    L.rnnoise_train_process_host.restype = ci
    L.rnnoise_train_process_host.argtypes = [vp, vp, vp, vp, ci]
    L.rnnoise_train_process_device.restype = ci
    L.rnnoise_train_process_device.argtypes = [vp, vp, vp, vp, ci, C.c_long, C.c_long, C.c_long, C.c_long, vp]
    L.rnnoise_train_process_pool_host.restype = ci
    L.rnnoise_train_process_pool_host.argtypes = [vp, vp, vp, C.c_long, vp, vp, ci]
    L.rnnoise_train_reset.restype = ci
    L.rnnoise_train_reset.argtypes = [vp]
    L.rnnoise_train_pool_reserve.restype = ci
    L.rnnoise_train_pool_reserve.argtypes = [vp, C.c_longlong]
    L.rnnoise_train_pool_write.restype = ci
    L.rnnoise_train_pool_write.argtypes = [vp, C.c_longlong, vp, C.c_longlong]
    L.rnnoise_train_pool_samples.restype = C.c_longlong
    L.rnnoise_train_pool_samples.argtypes = [vp]
    L.rnnoise_train_pool_room.restype = ci
    L.rnnoise_train_pool_room.argtypes = [vp, vp, vp]
    L.rnnoise_train_waves_device.restype = ci
    L.rnnoise_train_waves_device.argtypes = [vp, vp, vp, ci, vp, vp, vp, vp] + [C.c_long] * 4 + [vp]
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
    L.rnnoise_audio_probe.restype = ci
    L.rnnoise_audio_probe.argtypes = [C.c_char_p, vp]
    L.rnnoise_audio_write.restype = ci
    L.rnnoise_audio_write.argtypes = [C.c_char_p, ci, vp, C.c_long, ci]
    L.rnnoise_batch_add_model.restype = ci
    L.rnnoise_batch_add_model.argtypes = [vp, vp]
    L.rnnoise_batch_set_stream_models.restype = ci
    L.rnnoise_batch_set_stream_models.argtypes = [vp, vp, ci, vp]
    L.rnnoise_batch_get_stream_models.restype = ci
    L.rnnoise_batch_get_stream_models.argtypes = [vp, vp, ci, vp]
    L.rnnoise_batch_link_streams.restype = ci
    L.rnnoise_batch_link_streams.argtypes = [vp, vp, ci, ci]
    L.rnnoise_batch_unlink_streams.restype = ci
    L.rnnoise_batch_unlink_streams.argtypes = [vp, vp, ci]
    L.rnnoise_batch_get_stream_links.restype = ci
    L.rnnoise_batch_get_stream_links.argtypes = [vp, vp, ci, vp, vp]
    L.rnnoise_denoise_files_linked.restype = ci
    L.rnnoise_denoise_files_linked.argtypes = [ci, vp, vp, vp, ci]
    L.rnnoise_denoise_corpus.restype = ci
    L.rnnoise_denoise_corpus.argtypes = [ci, vp, vp, vp, ci, vp, vp]
    for name in ("rnnoise_batch_set_stream_controls", "rnnoise_batch_get_stream_controls"):
        getattr(L, name).restype = ci
        getattr(L, name).argtypes = [vp, vp, ci, vp]
    L.rnnoise_batch_pending_frames.restype = ci
    L.rnnoise_batch_pending_frames.argtypes = [vp]
    L.rnnoise_batch_analyze_device.restype = ci
    L.rnnoise_batch_analyze_device.argtypes = [vp, vp, ci, vp, vp, ci] + [C.c_long] * 5 + [vp]
    L.rnnoise_batch_synthesize_device.restype = ci
    L.rnnoise_batch_synthesize_device.argtypes = [vp, vp, ci, vp, ci] + [C.c_long] * 5 + [vp]
    L.rnnoise_batch_synthesize_saving_device.restype = ci
    L.rnnoise_batch_synthesize_saving_device.argtypes = [vp, vp, vp, ci] + [C.c_long] * 5 + [vp, C.c_long, C.c_long, vp]
    L.rnnoise_batch_window_frames.restype = ci
    L.rnnoise_batch_window_frames.argtypes = [vp]
    L.rnnoise_batch_analyze_window_device.restype = ci
    L.rnnoise_batch_analyze_window_device.argtypes = [vp, vp, ci, vp, vp, ci] + [C.c_long] * 5 + [vp, C.c_long, C.c_long, vp]
    L.rnnoise_batch_synthesize_window_device.restype = ci
    L.rnnoise_batch_synthesize_window_device.argtypes = [vp, vp, ci, vp, ci] + [C.c_long] * 5 + [vp, C.c_long, C.c_long, vp]
    L.rnnoise_synthesis_backward_workspace_bytes.restype = C.c_size_t
    L.rnnoise_synthesis_backward_workspace_bytes.argtypes = [ci, ci]
    L.rnnoise_synthesis_backward_device.restype = ci
    L.rnnoise_synthesis_backward_device.argtypes = [vp, C.c_long, C.c_long] * 3 + [ci, ci, vp, C.c_size_t, ci, vp]
    L.rnnoise_fit_create.restype = vp
    L.rnnoise_fit_create.argtypes = [ci, ci, ci, ci, ci, ci, ci]
    L.rnnoise_fit_destroy.argtypes = [vp]
    L.rnnoise_fit_n_params.restype = C.c_long
    L.rnnoise_fit_n_params.argtypes = [vp]
    for name in ("rnnoise_fit_get_params", "rnnoise_fit_set_params", "rnnoise_fit_set_params_from_model", "rnnoise_fit_get_grads"):
        getattr(L, name).restype = ci
        getattr(L, name).argtypes = [vp, vp]
    L.rnnoise_fit_step.restype = ci
    L.rnnoise_fit_step.argtypes = [vp, vp, vp, ci, vp]
    L.rnnoise_fit_evaluate.restype = ci
    L.rnnoise_fit_evaluate.argtypes = [vp, vp, vp, ci, vp]
    L.rnnoise_fit_get_activations.restype = ci
    L.rnnoise_fit_get_activations.argtypes = [vp, vp, vp, vp]
    L.rnnoise_fit_set_taps.restype = ci
    L.rnnoise_fit_set_taps.argtypes = [vp, ci]
    L.rnnoise_fit_get_taps.restype = ci
    L.rnnoise_fit_get_taps.argtypes = [vp, ci] + [vp] * 10
    L.rnnoise_fit_export.restype = C.c_size_t
    L.rnnoise_fit_export.argtypes = [vp, vp, C.c_size_t]
    L.rnnoise_fit_export_params.restype = C.c_size_t
    L.rnnoise_fit_export_params.argtypes = [ci, ci, ci, ci, vp, vp, C.c_size_t]
    L.rnnoise_fit_forward_device.restype = ci
    L.rnnoise_fit_forward_device.argtypes = [vp, vp, ci] + [vp, C.c_long, C.c_long] * 2 + [vp, vp] + [vp, C.c_long, C.c_long] * 2 + [vp]
    L.rnnoise_fit_backward_device.restype = ci
    L.rnnoise_fit_backward_device.argtypes = [vp, vp] + [vp, C.c_long, C.c_long] * 2 + [vp, vp]
    L.rnnoise_resampler_filter.restype = ci
    L.rnnoise_resampler_filter.argtypes = [ci, ci, vp, ci, vp, vp]
    L.rnnoise_resampler_delay.restype = C.c_double
    L.rnnoise_resampler_delay.argtypes = [ci]
    L.rnnoise_resampler_create.restype = vp
    L.rnnoise_resampler_create.argtypes = [ci, vp, ci]
    L.rnnoise_resampler_destroy.argtypes = [vp]
    for name in ("rnnoise_resampler_set_stream_rates", "rnnoise_resampler_get_stream_rates", "rnnoise_resampler_get_states",
                 "rnnoise_resampler_set_states"):
        getattr(L, name).restype = ci
        getattr(L, name).argtypes = [vp, vp, ci, vp]
    for name in ("rnnoise_resampler_up_device", "rnnoise_resampler_down_device"):
        getattr(L, name).restype = ci
        getattr(L, name).argtypes = [vp, vp, ci, vp, vp, ci, ci, C.c_long, C.c_long, vp]
    L.rnnoise_batch_process_native_device.restype = ci
    L.rnnoise_batch_process_native_device.argtypes = [vp, vp, vp, ci, vp, vp, ci, vp, ci, C.c_long, C.c_long, vp]
    L.rnnoise_batch_process_native_host.restype = ci
    L.rnnoise_batch_process_native_host.argtypes = [vp, vp, vp, ci, vp, vp, ci, vp, ci]
    L.rnnoise_metrics_create.restype = vp
    L.rnnoise_metrics_create.argtypes = [ci, ci]
    L.rnnoise_metrics_destroy.argtypes = [vp]
    L.rnnoise_metrics_accumulate_device.restype = ci
    L.rnnoise_metrics_accumulate_device.argtypes = [vp, vp, vp, C.c_long, C.c_long, vp, vp, C.c_long, C.c_long, ci, vp]
    for name in ("rnnoise_metrics_clear", "rnnoise_metrics_get"):
        getattr(L, name).restype = ci
    L.rnnoise_metrics_clear.argtypes = [vp, vp, ci]
    L.rnnoise_metrics_get.argtypes = [vp, vp, ci, vp]
    L.rnnoise_intelligibility_workspace_bytes.restype = C.c_size_t
    L.rnnoise_intelligibility_workspace_bytes.argtypes = [ci, C.c_long, ci]
    L.rnnoise_intelligibility_device.restype = ci
    L.rnnoise_intelligibility_device.argtypes = [vp, vp, ci, C.c_long, C.c_long, ci, vp, vp, C.c_size_t, ci, vp]
    L.rnnoise_intelligibility_backward_workspace_bytes.restype = C.c_size_t
    L.rnnoise_intelligibility_backward_workspace_bytes.argtypes = [ci, C.c_long, ci]
    L.rnnoise_intelligibility_backward_device.restype = ci
    L.rnnoise_intelligibility_backward_device.argtypes = [ci, C.c_long, ci, vp, vp, C.c_size_t, vp, vp, vp, C.c_long, vp, C.c_size_t, ci, vp]
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


# RNNoiseStreamControls (include/rnnoise.h): one stream's attenuation limit and voice-activity gate, 24 bytes
STREAM_CONTROLS_DTYPE = np.dtype([("atten_lim_db", "<f4"), ("gate_threshold", "<f4"), ("gate_closed_gain", "<f4"),
                                  ("gate_hold_frames", "<i4"), ("gate_hold_left", "<i4"), ("gate_closed", "<i4")])
GATE_MAX_HOLD_FRAMES = 6000  # RNNOISE_GATE_MAX_HOLD_FRAMES


# stream links (include/rnnoise.h): RNNOISE_LINK_MAX / RNNOISE_LINK_MEAN, and the largest group
LINK_MODES = {"max": 1, "mean": 2}
LINK_MAX_MEMBERS = 64


def link_mode_of(mode):
    """'max' or 'mean' -> RNNOISE_LINK_MAX / RNNOISE_LINK_MEAN; ValueError otherwise."""
    if not isinstance(mode, str) or mode not in LINK_MODES:
        raise ValueError("link mode must be 'max' or 'mean', not %r" % (mode,))
    return LINK_MODES[mode]


def check_stream_list(streams, n_streams):
    """streams as an int32 array after the checks of the link calls: integers, in 0..n_streams-1, each once.  The range
    is checked on the values as given: the cast to int32 could wrap an out-of-range index into range."""
    a = np.asarray(streams)
    if a.ndim != 1 or not (np.issubdtype(a.dtype, np.integer) or a.size == 0):
        raise ValueError("streams must be a 1-d list of stream indices")
    bad = [int(v) for v in a if not 0 <= int(v) < n_streams]
    if bad:
        raise ValueError("stream index %d out of range 0..%d" % (bad[0], n_streams - 1))
    idx = a.astype(np.int32)
    u, c = np.unique(idx, return_counts=True)
    if np.any(c > 1):
        raise ValueError("stream index %d given twice" % int(u[c > 1][0]))
    return np.ascontiguousarray(idx)


def check_stream_controls(rec):
    """Raise ValueError naming the first record and field of `rec` (STREAM_CONTROLS_DTYPE) that
    rnnoise_batch_set_stream_controls would refuse."""
    def unit(v):
        return 0.0 <= v <= 1.0  # False for NaN
    for r, c in enumerate(rec):
        a, th, cg = float(c["atten_lim_db"]), float(c["gate_threshold"]), float(c["gate_closed_gain"])
        hold, left, closed = int(c["gate_hold_frames"]), int(c["gate_hold_left"]), int(c["gate_closed"])
        bad = None
        if not a >= 0.0:
            bad = "atten_lim_db must be >= 0 (inf: no limit)"
        elif not unit(th):
            bad = "gate_threshold must be in 0..1"
        elif not unit(cg):
            bad = "gate_closed_gain must be in 0..1"
        elif not 0 <= hold <= GATE_MAX_HOLD_FRAMES:
            bad = "gate_hold_frames must be in 0..%d" % GATE_MAX_HOLD_FRAMES
        elif not 0 <= left <= hold:
            bad = "gate_hold_left must be in 0..gate_hold_frames"
        elif closed not in (0, 1):
            bad = "gate_closed must be 0 or 1"
        if bad:
            raise ValueError("stream controls record %d: %s" % (r, bad))


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

    # ---- per-stream models: a table of models of the batch model's geometry ----
    def add_model(self, model: RnnModel) -> int:
        """Add a model of this batch's geometry to its model table; returns its index (the batch's own model is 0).
        The weights are copied: the model may be freed afterwards."""
        k = lib().rnnoise_batch_add_model(self._h, model._h if model is not None else None)
        if k < 0:
            raise NnnoiselessError(last_error())
        return int(k)

    def set_stream_models(self, model_ids, streams=None):
        """Run streams[r] (None: 0..n-1) on model model_ids[r] from the next frame on; the streams keep their state.
        Every index and id is checked first; on an error nothing changes."""
        ids = np.ascontiguousarray(model_ids, dtype=np.int32).reshape(-1)
        idx, n = self._streams(streams)
        if streams is None:
            n = len(ids)
        elif n != len(ids):
            raise ValueError("%d model ids for %d streams" % (len(ids), n))
        if lib().rnnoise_batch_set_stream_models(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(ids)) != 0:
            raise NnnoiselessError(last_error())

    def stream_models(self, streams=None) -> np.ndarray:
        """The model index of each given stream (None: all), int32."""
        idx, n = self._streams(streams)
        out = np.empty(n, np.int32)
        if lib().rnnoise_batch_get_stream_models(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out)) != 0:
            raise NnnoiselessError(last_error())
        return out

    # ---- per-stream controls: attenuation limit and voice-activity gate (DESIGN.md 7m) ----
    def set_stream_controls(self, streams=None, *, atten_lim_db=np.inf, gate_threshold=0.0, gate_closed_gain=0.0,
                            gate_hold_frames=0):
        """Set the controls of the given streams (None: all) from scalars or per-stream arrays, with fresh gate state
        (hold_left 0, open).  atten_lim_db >= 0 (inf: no limit), gate_threshold and gate_closed_gain in 0..1 (threshold
        0: the gate stays open), gate_hold_frames in 0..6000.  Frames issued afterwards use them."""
        idx, n = self._streams(streams)
        rec = np.zeros(n, STREAM_CONTROLS_DTYPE)
        for name, v in (("atten_lim_db", atten_lim_db), ("gate_threshold", gate_threshold),
                        ("gate_closed_gain", gate_closed_gain), ("gate_hold_frames", gate_hold_frames)):
            a = np.asarray(v)
            if a.ndim > 1 or (a.ndim == 1 and len(a) != n):
                raise ValueError("%s: expected a scalar or %d values" % (name, n))
            # the ranges are checked on the values as given: the cast to the record's int32 / float32 could wrap or round
            # an out-of-range value into range
            if name == "gate_hold_frames":
                if not np.issubdtype(a.dtype, np.integer):
                    raise ValueError("gate_hold_frames must be integers")
                if np.any((a < 0) | (a > GATE_MAX_HOLD_FRAMES)):
                    raise ValueError("gate_hold_frames must be in 0..%d" % GATE_MAX_HOLD_FRAMES)
            else:
                if not (np.issubdtype(a.dtype, np.floating) or np.issubdtype(a.dtype, np.integer)):
                    raise ValueError("%s must be real numbers" % name)
                f = a.astype(np.float64)
                ok = f >= 0.0 if name == "atten_lim_db" else (f >= 0.0) & (f <= 1.0)  # False for NaN
                if not np.all(ok):
                    raise ValueError("%s must be %s" % (name, ">= 0 (inf: no limit)" if name == "atten_lim_db" else "in 0..1"))
            rec[name] = a
        self.set_stream_controls_records(rec, streams)

    def set_stream_controls_records(self, records, streams=None):
        """Set whole controls records (an array of STREAM_CONTROLS_DTYPE, state fields included, e.g. from
        get_stream_controls) on the given streams (None: 0..n-1).  Every field is checked first; on an error nothing
        changes."""
        rec = np.ascontiguousarray(records)
        if rec.dtype != STREAM_CONTROLS_DTYPE:
            raise ValueError("records must be an array of STREAM_CONTROLS_DTYPE")
        rec = rec.reshape(-1)
        idx, n = self._streams(streams)
        if streams is None:
            n = len(rec)
            if n > self.n_streams:
                raise ValueError("%d records for a batch of %d streams" % (n, self.n_streams))
        elif n != len(rec):
            raise ValueError("%d records for %d streams" % (len(rec), n))
        check_stream_controls(rec)
        rc = lib().rnnoise_batch_set_stream_controls(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(rec))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def get_stream_controls(self, streams=None) -> np.ndarray:
        """The controls records of the given streams (None: all), after every frame issued so far: an array of
        STREAM_CONTROLS_DTYPE, which set_stream_controls_records restores."""
        idx, n = self._streams(streams)
        out = np.zeros(n, STREAM_CONTROLS_DTYPE)
        if lib().rnnoise_batch_get_stream_controls(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out)) != 0:
            raise NnnoiselessError(last_error())
        return out

    # ---- stream links: one gain curve for a group of streams (DESIGN.md 7n) ----
    def link_streams(self, streams, mode="max"):
        """Link 2..64 distinct streams as one group: from the next fused frame on, each member's band gains are the max
        ('max') or the float32 mean ('mean') of the non-silent members' raw gains, and its gate decides on their largest
        vad.  A stream in another group leaves it first (a group left with one member dissolves)."""
        m = link_mode_of(mode)
        idx = check_stream_list(streams, self.n_streams)
        if not 2 <= len(idx) <= LINK_MAX_MEMBERS:
            raise ValueError("a group links 2..%d streams, not %d" % (LINK_MAX_MEMBERS, len(idx)))
        if lib().rnnoise_batch_link_streams(self._h, _np_ptr(idx), len(idx), m) != 0:
            raise NnnoiselessError(last_error())

    def unlink_streams(self, streams=None):
        """Take the given streams (None: all) out of their groups; groups left with one member dissolve."""
        idx = None if streams is None else check_stream_list(streams, self.n_streams)
        rc = lib().rnnoise_batch_unlink_streams(self._h, _np_ptr(idx) if idx is not None else None,
                                                self.n_streams if idx is None else len(idx))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def stream_links(self, streams=None):
        """-> (group, mode) int32 arrays for the given streams (None: all): group = the lowest stream of the stream's
        group (itself when unlinked), mode = 1 (max), 2 (mean) or 0 (unlinked)."""
        idx = None if streams is None else check_stream_list(streams, self.n_streams)
        n = self.n_streams if idx is None else len(idx)
        group, mode = np.zeros(n, np.int32), np.zeros(n, np.int32)
        if lib().rnnoise_batch_get_stream_links(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(group),
                                                _np_ptr(mode)) != 0:
            raise NnnoiselessError(last_error())
        return group, mode

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

    # ---- split frames: the caller's network between analysis and synthesis ----
    @property
    def pending_frames(self) -> int:
        """Frames analyzed and not yet synthesized (0 .. 4)."""
        return int(lib().rnnoise_batch_pending_frames(self._h))

    def analyze_device(self, in_ptr: int, features_ptr: int, silence_ptr: int, n_frames: int, stream_stride: int, frame_stride: int,
                       feature_stream_stride: int, feature_frame_stride: int, sample_stride: int = 1, pcm16: int = 0,
                       cuda_stream: int = 0):
        """Analyze the next n_frames frames of every stream through raw device pointers: sample (s, t, i) at
        in[s*stream_stride + t*frame_stride + i*sample_stride] (float32, or int16 if pcm16), feature j of (s, t) at
        features[s*feature_stream_stride + t*feature_frame_stride + j] (float32), silence int32 [n_frames][n_streams] or 0.
        The frames stay pending (at most 4) until synthesize_device takes their gains."""
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_batch_analyze_device(self._h, ptr(in_ptr), int(pcm16), ptr(features_ptr), ptr(silence_ptr), int(n_frames),
                                                int(stream_stride), int(sample_stride), int(frame_stride), int(feature_stream_stride),
                                                int(feature_frame_stride), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def synthesize_device(self, out_ptr: int, gains_ptr: int, n_frames: int, stream_stride: int, frame_stride: int,
                          gain_stream_stride: int, gain_frame_stride: int, sample_stride: int = 1, pcm16: int = 0,
                          cuda_stream: int = 0):
        """Synthesize the n_frames oldest pending frames from raw band gains: gain k of (s, t) at
        gains[s*gain_stream_stride + t*gain_frame_stride + k] (float32, used as given); out laid out as analyze_device's
        input."""
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_batch_synthesize_device(self._h, ptr(out_ptr), int(pcm16), ptr(gains_ptr), int(n_frames), int(stream_stride),
                                                   int(sample_stride), int(frame_stride), int(gain_stream_stride),
                                                   int(gain_frame_stride), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def synthesize_saving_device(self, out_ptr: int, gains_ptr: int, n_frames: int, stream_stride: int, frame_stride: int,
                                 gain_stream_stride: int, gain_frame_stride: int, ctx_ptr: int, ctx_stream_stride: int,
                                 ctx_frame_stride: int, sample_stride: int = 1, pcm16: int = 0, cuda_stream: int = 0):
        """synthesize_device with float32 output that also saves each (stream, frame)'s synthesis context at
        ctx + (s*ctx_stream_stride + t*ctx_frame_stride) * SYNTH_CONTEXT_BYTES, for synthesis_backward_device (strides in
        records).  int16 output (pcm16) is refused: the gradient is defined for float samples."""
        if pcm16:
            raise NnnoiselessError("the saving synthesis writes float samples only: pcm16 output is refused")
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_batch_synthesize_saving_device(self._h, ptr(out_ptr), ptr(gains_ptr), int(n_frames), int(stream_stride),
                                                          int(sample_stride), int(frame_stride), int(gain_stream_stride),
                                                          int(gain_frame_stride), ptr(ctx_ptr), int(ctx_stream_stride),
                                                          int(ctx_frame_stride), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    # ---- window frames: split frames of any length, their spectra in the caller's context records ----
    @property
    def window_frames(self) -> int:
        """Frames analyzed by analyze_window_device and not yet synthesized by synthesize_window_device."""
        return int(lib().rnnoise_batch_window_frames(self._h))

    def analyze_window_device(self, in_ptr: int, features_ptr: int, silence_ptr: int, n_frames: int, stream_stride: int,
                              frame_stride: int, feature_stream_stride: int, feature_frame_stride: int, ctx_ptr: int,
                              ctx_stream_stride: int, ctx_frame_stride: int, sample_stride: int = 1, pcm16: int = 0, cuda_stream: int = 0):
        """analyze_device without a bound on the frames owed: X, P, the band energies and the silence flag of (s, t) go to
        the context record at ctx + (s*ctx_stream_stride + t*ctx_frame_stride) * SYNTH_CONTEXT_BYTES (strides in records,
        16-byte aligned) instead of the batch.  The frames are owed until synthesize_window_device is given those records."""
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_batch_analyze_window_device(self._h, ptr(in_ptr), int(pcm16), ptr(features_ptr), ptr(silence_ptr), int(n_frames),
                                                       int(stream_stride), int(sample_stride), int(frame_stride), int(feature_stream_stride),
                                                       int(feature_frame_stride), ptr(ctx_ptr), int(ctx_stream_stride), int(ctx_frame_stride),
                                                       ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def synthesize_window_device(self, out_ptr: int, gains_ptr: int, n_frames: int, stream_stride: int, frame_stride: int,
                                 gain_stream_stride: int, gain_frame_stride: int, ctx_ptr: int, ctx_stream_stride: int,
                                 ctx_frame_stride: int, sample_stride: int = 1, pcm16: int = 0, cuda_stream: int = 0):
        """synthesize_device of the n_frames oldest owed window frames, from the records their analysis wrote; adds lastg
        and the gains to the records, which then equal synthesize_saving_device's for synthesis_backward_device."""
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_batch_synthesize_window_device(self._h, ptr(out_ptr), int(pcm16), ptr(gains_ptr), int(n_frames), int(stream_stride),
                                                          int(sample_stride), int(frame_stride), int(gain_stream_stride),
                                                          int(gain_frame_stride), ptr(ctx_ptr), int(ctx_stream_stride),
                                                          int(ctx_frame_stride), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    # ---- streams at their own sample rate (a Resampler of this batch's size) ----
    def process_native_host(self, resampler, x: np.ndarray, streams=None, want_vad=True):
        """Denoise native-rate frames: x [T][n][480] float32 or int16 host slots, row r of every frame belonging to
        streams[r] (None: 0..n-1, a full-batch call when n == n_streams); the first R/100 samples of a slot are stream
        streams[r]'s 10 ms frame at its resampler rate R, the rest are ignored.  Returns (out like x, the rest of each
        slot 0; vad [T][n]).  Up-sampling, the denoise frames and down-sampling run on the GPU in one call."""
        x = np.ascontiguousarray(x)
        pcm16 = 1 if x.dtype == np.int16 else 0
        x = x if pcm16 else np.ascontiguousarray(x, dtype=np.float32)
        idx, n = self._streams(streams)
        if streams is None:
            n = x.shape[1] if x.ndim == 3 else -1
        if x.ndim != 3 or x.shape[1] != n or x.shape[2] != FRAME_SIZE:
            raise ValueError("expected [T][%d][480]" % n)
        T = x.shape[0]
        out = np.empty_like(x)
        vad = np.empty((T, n), np.float32) if want_vad else None
        rc = lib().rnnoise_batch_process_native_host(self._h, resampler._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out),
                                                     _np_ptr(x), pcm16, _np_ptr(vad) if want_vad else None, T)
        if rc != 0:
            raise NnnoiselessError(last_error())
        return out, vad

    def process_native_device(self, resampler, out_ptr: int, in_ptr: int, vad_ptr: int, n_frames: int, stream_stride: int,
                              frame_stride: int, streams=None, pcm16: int = 0, cuda_stream: int = 0, n: int = None):
        """process_native_host through raw device pointers: native sample (r, t, k), k < R/100, of stream streams[r] at
        ptr[r*stream_stride + t*frame_stride + k] (element strides; float32, or int16 if pcm16), vad [n_frames][n] or 0.
        streams None: streams 0..n-1 (n defaults to every stream)."""
        idx, k = self._streams(streams)
        if streams is None and n is not None:
            k = int(n)
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_batch_process_native_device(self._h, resampler._h, _np_ptr(idx) if idx is not None else None, k, ptr(out_ptr),
                                                       ptr(in_ptr), int(pcm16), ptr(vad_ptr), int(n_frames), int(stream_stride),
                                                       int(frame_stride), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None:
            _lib.rnnoise_batch_destroy(h)
            self._h = None


RESAMPLER_STATE_MAGIC = 0x54535352  # "RSST", RNNOISE_RESAMPLER_STATE_MAGIC
def synthesis_backward_workspace_bytes(n_streams: int, n_frames: int) -> int:
    """Bytes of device workspace synthesis_backward_device needs for a window of n_frames frames of n_streams streams."""
    return int(lib().rnnoise_synthesis_backward_workspace_bytes(int(n_streams), int(n_frames)))


def synthesis_backward_device(ctx_ptr: int, ctx_stream_stride: int, ctx_frame_stride: int, grad_out_ptr: int, go_stream_stride: int,
                              go_frame_stride: int, grad_gains_ptr: int, gg_stream_stride: int, gg_frame_stride: int, n_streams: int,
                              n_frames: int, workspace_ptr: int, workspace_bytes: int, device: int = -1, cuda_stream: int = 0):
    """dL/d(raw gains) [.][.][22] of a window of saved frames from dL/d(output samples) [.][.][480], through raw device
    pointers (rnnoise_synthesis_backward_device; context strides in records, the others in floats).  Stateless; ordered
    on cuda_stream, or synchronous without one."""
    ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
    rc = lib().rnnoise_synthesis_backward_device(ptr(ctx_ptr), int(ctx_stream_stride), int(ctx_frame_stride), ptr(grad_out_ptr),
                                                 int(go_stream_stride), int(go_frame_stride), ptr(grad_gains_ptr), int(gg_stream_stride),
                                                 int(gg_frame_stride), int(n_streams), int(n_frames), ptr(workspace_ptr),
                                                 int(workspace_bytes), int(device), ptr(cuda_stream))
    if rc != 0:
        raise NnnoiselessError(last_error())


RESAMPLER_STATE_VERSION = 1
RESAMPLER_STATE_BYTES = 576


def resampler_filter(rate: int, direction: int):
    """The float32 filter of one resampler stage at stream rate `rate`, direction 0 = up (rate -> 48 kHz), 1 = down:
    returns (taps, up, down), the stage being scipy.signal.upfirdn(taps, x, up, down).  Needs no GPU."""
    up, down = C.c_int(), C.c_int()
    n = lib().rnnoise_resampler_filter(int(rate), int(direction), None, 0, C.byref(up), C.byref(down))
    if n < 0:
        raise NnnoiselessError(last_error())
    h = np.empty(n, np.float32)
    lib().rnnoise_resampler_filter(int(rate), int(direction), _np_ptr(h), n, None, None)
    return h, up.value, down.value


def resampler_delay(rate: int) -> float:
    """Delay of the up and down stages together at stream rate `rate`, in 48 kHz samples (not counting the denoiser's)."""
    d = lib().rnnoise_resampler_delay(int(rate))
    if d < 0:
        raise NnnoiselessError(last_error())
    return float(d)


class Resampler:
    """Per-stream sample rates for a DenoiseBatch of the same size (rnnoise_resampler_* in include/rnnoise.h): stream s
    gives and gets rate/100 samples per 10 ms frame at its own rate (8000..48000 Hz, a multiple of 100), resampled to and
    from the batch's 48 kHz frames on the GPU with its filter history kept across calls."""

    def __init__(self, n_streams: int, rates=None, device: int = -1):
        self.n_streams = int(n_streams)
        r = None if rates is None else np.ascontiguousarray(np.broadcast_to(np.asarray(rates, dtype=np.int32), (self.n_streams,)))
        self._h = lib().rnnoise_resampler_create(self.n_streams, _np_ptr(r) if r is not None else None, int(device))
        if not self._h:
            raise NnnoiselessError("rnnoise_resampler_create failed: " + last_error())

    def _streams(self, streams):
        return DenoiseBatch._streams(self, streams)

    def set_stream_rates(self, rates, streams=None):
        """Stream streams[r] (None: 0..n-1) gets rate rates[r] and zero histories (also when the rate is unchanged)."""
        rates = np.ascontiguousarray(rates, dtype=np.int32).reshape(-1)
        idx, n = self._streams(streams)
        if streams is None:
            n = len(rates)
        elif n != len(rates):
            raise ValueError("%d rates for %d streams" % (len(rates), n))
        if lib().rnnoise_resampler_set_stream_rates(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(rates)) != 0:
            raise NnnoiselessError(last_error())

    def stream_rates(self, streams=None) -> np.ndarray:
        idx, n = self._streams(streams)
        out = np.empty(n, np.int32)
        if lib().rnnoise_resampler_get_stream_rates(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out)) != 0:
            raise NnnoiselessError(last_error())
        return out

    def _stage(self, fn, out_ptr, in_ptr, n_frames, stream_stride, frame_stride, streams, pcm16, cuda_stream, n):
        idx, k = self._streams(streams)
        if streams is None and n is not None:
            k = int(n)
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = fn(self._h, _np_ptr(idx) if idx is not None else None, k, ptr(out_ptr), ptr(in_ptr), int(pcm16), int(n_frames),
                int(stream_stride), int(frame_stride), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def up_device(self, out_ptr: int, in_ptr: int, n_frames: int, stream_stride: int, frame_stride: int, streams=None, pcm16: int = 0,
                  cuda_stream: int = 0, n: int = None):
        """Native frames (sample (r, t, k) at in[r*stream_stride + t*frame_stride + k], float32 or int16) -> compact
        48 kHz float32 out [n_frames][n][480]."""
        self._stage(lib().rnnoise_resampler_up_device, out_ptr, in_ptr, n_frames, stream_stride, frame_stride, streams, pcm16,
                    cuda_stream, n)

    def down_device(self, out_ptr: int, in_ptr: int, n_frames: int, stream_stride: int, frame_stride: int, streams=None, pcm16: int = 0,
                    cuda_stream: int = 0, n: int = None):
        """Compact 48 kHz float32 in [n_frames][n][480] -> native frames out (layout and pcm16 as up_device)."""
        self._stage(lib().rnnoise_resampler_down_device, out_ptr, in_ptr, n_frames, stream_stride, frame_stride, streams, pcm16,
                    cuda_stream, n)

    def get_states(self, streams=None) -> np.ndarray:
        """State records (rate and histories) of the given streams as uint8 [n][RESAMPLER_STATE_BYTES]."""
        idx, n = self._streams(streams)
        out = np.empty((n, RESAMPLER_STATE_BYTES), np.uint8)
        if lib().rnnoise_resampler_get_states(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out)) != 0:
            raise NnnoiselessError(last_error())
        return out

    def set_states(self, records, streams=None):
        """Import records into the given streams (default: 0..n-1); every record is checked first."""
        rec = np.ascontiguousarray(records, dtype=np.uint8).reshape(-1, RESAMPLER_STATE_BYTES)
        idx, n = self._streams(streams)
        if streams is None:
            n = rec.shape[0]
        elif n != rec.shape[0]:
            raise ValueError("%d records for %d streams" % (rec.shape[0], n))
        if lib().rnnoise_resampler_set_states(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(rec)) != 0:
            raise NnnoiselessError(last_error())

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None:
            _lib.rnnoise_resampler_destroy(h)
            self._h = None


# RNNoiseMetricsRecord (include/rnnoise.h): one stream's quality sums, 696 bytes.  Class index 0 = all counted frames,
# 1 = speech (target 1), 2 = noise only (target 0); vad_counts = tp, fp, fn, tn; last_bands = (Yb, Cb) of the last
# counted frame.
METRICS_DTYPE = np.dtype([("frames", "<i8", (3,)), ("ec", "<f8", (3,)), ("ey", "<f8", (3,)), ("ecy", "<f8", (3,)),
                          ("ed", "<f8", (3,)), ("seg_snr", "<f8"), ("lsd", "<f8"), ("speech_dev", "<f8", (NB_BANDS,)),
                          ("noise_level", "<f8", (NB_BANDS,)), ("vad_counts", "<i8", (4,)),
                          ("last_bands", "<f4", (2, NB_BANDS))])
assert METRICS_DTYPE.itemsize == 696


class Metrics:
    """Quality metrics of n_streams denoised streams against clean speech, accumulated on the GPU (rnnoise_metrics_* in
    include/rnnoise.h; DESIGN.md 7p).  Output frame t of a stream is scored against clean frame t - 1, the denoiser's
    one-frame delay; the pairing is kept on the device across calls.  ``records`` returns METRICS_DTYPE records, which
    ``nnnoiseless_b200.metrics.summarize`` turns into SNR, SI-SDR, segmental SNR, LSD and VAD figures."""

    def __init__(self, n_streams: int, device: int = -1):
        self.n_streams = int(n_streams)
        self._h = lib().rnnoise_metrics_create(self.n_streams, int(device))
        if not self._h:
            raise NnnoiselessError("rnnoise_metrics_create failed: " + last_error())

    def _streams(self, streams):
        return DenoiseBatch._streams(self, streams)

    def accumulate_device(self, out_ptr: int, clean_ptr: int, n_frames: int, stream_stride: int, frame_stride: int,
                          vad_ptr: int = 0, vad_target_ptr: int = 0, vad_stream_stride: int = 0, vad_frame_stride: int = 0,
                          cuda_stream: int = 0):
        """Score n_frames frames of every stream through raw device pointers (float32): sample (s, t, i) of out and clean
        at ptr[s*stream_stride + t*frame_stride + i]; the network's vad and the corpus's target vad (each optional) at
        ptr[s*vad_stream_stride + t*vad_frame_stride].  Ordered after cuda_stream; synchronous without one."""
        ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        rc = lib().rnnoise_metrics_accumulate_device(self._h, ptr(out_ptr), ptr(clean_ptr), int(stream_stride), int(frame_stride),
                                                     ptr(vad_ptr), ptr(vad_target_ptr), int(vad_stream_stride), int(vad_frame_stride),
                                                     int(n_frames), ptr(cuda_stream))
        if rc != 0:
            raise NnnoiselessError(last_error())

    def clear(self, streams=None):
        """Zero the records of the given streams (None: all), keeping their pairing: frames so far are dropped."""
        idx, n = self._streams(streams)
        if lib().rnnoise_metrics_clear(self._h, _np_ptr(idx) if idx is not None else None, n) != 0:
            raise NnnoiselessError(last_error())

    def records(self, streams=None) -> np.ndarray:
        """The records of the given streams (None: all) after every call so far, as METRICS_DTYPE."""
        idx, n = self._streams(streams)
        out = np.zeros(n, METRICS_DTYPE)
        if lib().rnnoise_metrics_get(self._h, _np_ptr(idx) if idx is not None else None, n, _np_ptr(out)) != 0:
            raise NnnoiselessError(last_error())
        return out

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None:
            _lib.rnnoise_metrics_destroy(h)
            self._h = None


# RNNoiseIntelligibility (include/rnnoise.h): one pair's STOI and ESTOI (NaN when segments < 1), its 10 kHz frames F,
# the frames K kept by the silence rule and the segments S = max(K - 30, 0); 32 bytes.
INTELLIGIBILITY_DTYPE = np.dtype([("stoi", "<f8"), ("estoi", "<f8"), ("frames", "<i4"), ("kept", "<i4"), ("segments", "<i4"),
                                  ("reserved", "<i4")])
assert INTELLIGIBILITY_DTYPE.itemsize == 32
STOI_BANDS = 15


def intelligibility_workspace_bytes(n_pairs: int, n_samples: int, rate: int = 48000) -> int:
    """Bytes of device workspace intelligibility_device needs (0 for bad arguments).  Needs no GPU."""
    return int(lib().rnnoise_intelligibility_workspace_bytes(int(n_pairs), int(n_samples), int(rate)))


def intelligibility_device(out_ptr: int, clean_ptr: int, n_pairs: int, n_samples: int, stream_stride: int, rate: int, result_ptr: int,
                           workspace_ptr: int, workspace_bytes: int, device: int = -1, cuda_stream: int = 0):
    """STOI and ESTOI of n_pairs pairs through raw device pointers (rnnoise_intelligibility_device): sample i of pair p
    at out[p*stream_stride + i] and clean[p*stream_stride + i] (float32), one INTELLIGIBILITY_DTYPE record per pair at
    result.  Stateless; ordered on cuda_stream, or synchronous without one."""
    ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
    rc = lib().rnnoise_intelligibility_device(ptr(out_ptr), ptr(clean_ptr), int(n_pairs), int(n_samples), int(stream_stride), int(rate),
                                              ptr(result_ptr), ptr(workspace_ptr), int(workspace_bytes), int(device), ptr(cuda_stream))
    if rc != 0:
        raise NnnoiselessError(last_error())


def intelligibility_sizes(n_samples: int, rate: int):
    """(up, down, n10, F) of a call: the 10 kHz resampling factors, the 10 kHz samples and the 256-sample frames."""
    import math
    g = math.gcd(int(rate), 10000)
    up, down = 10000 // g, int(rate) // g
    n10 = -(-int(n_samples) * up // down)
    return up, down, n10, ((n10 - 256) // 128 + 1 if n10 >= 256 else 0)


def intelligibility(out, clean, rate: int = 48000, cuda_stream=None) -> np.ndarray:
    """STOI and ESTOI of each row of float32 CUDA tensors out (processed) and clean, [B][n] -> INTELLIGIBILITY_DTYPE [B].
    Runs on cuda_stream (default: torch's current stream) and returns when the records are on the host."""
    import torch
    if out.shape != clean.shape or out.dim() != 2:
        raise ValueError("out and clean must be [B][n] tensors of one shape")
    B, n = out.shape
    if n > 1 and (out.stride(1) != 1 or clean.stride(1) != 1):
        raise ValueError("out and clean must have unit sample stride")
    if B > 1 and (out.stride(0) != clean.stride(0) or out.stride(0) < n):
        # e.g. unfold(0, n, hop) with hop < n, or expand(B, n): rows that share samples are not separate clips
        raise ValueError("out and clean must have one row stride of at least n = %d (rows must not overlap); strides %d and %d"
                         % (n, out.stride(0), clean.stride(0)))
    if out.dtype != torch.float32 or clean.dtype != torch.float32 or not out.is_cuda or clean.device != out.device:
        raise ValueError("out and clean must be float32 CUDA tensors on one device")
    nbytes = intelligibility_workspace_bytes(B, n, rate)
    if nbytes == 0:
        raise NnnoiselessError("no workspace size for %d pairs of %d samples at %d Hz" % (B, n, rate))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=out.device)
    res = torch.empty(B * INTELLIGIBILITY_DTYPE.itemsize, dtype=torch.uint8, device=out.device)
    cs = torch.cuda.current_stream(out.device).cuda_stream if cuda_stream is None else cuda_stream
    intelligibility_device(out.data_ptr(), clean.data_ptr(), B, n, out.stride(0) if B > 1 else n, rate, res.data_ptr(), ws.data_ptr(), nbytes,
                           out.device.index, cs)
    return res.cpu().numpy().view(INTELLIGIBILITY_DTYPE).copy()


def intelligibility_taps(workspace, B: int, n: int, rate: int = 48000):
    """Torch views of a workspace's documented regions after intelligibility_device(B pairs of n samples at rate):
    x10 float [2][B][n10] (0: clean, 1: out), kept int32 [B][F] (the k-th kept frame's index, then -1) and bands float
    [2][B][15][max(F - 1, 0)]."""
    import torch
    _, _, n10, F = intelligibility_sizes(n, rate)
    maxM = max(F - 1, 0)
    r = lambda v: (v + 255) & ~255  # noqa: E731
    o_kept = r(2 * B * n10 * 4)
    o_bands = o_kept + r(B * F * 4)
    w = workspace.view(torch.uint8)
    x10 = w[:2 * B * n10 * 4].view(torch.float32).view(2, B, n10)
    kept = w[o_kept:o_kept + B * F * 4].view(torch.int32).view(B, F)
    bands = w[o_bands:o_bands + 2 * B * STOI_BANDS * maxM * 4].view(torch.float32).view(2, B, STOI_BANDS, maxM)
    return x10, kept, bands


def intelligibility_backward_workspace_bytes(n_pairs: int, n_samples: int, rate: int = 48000) -> int:
    """Bytes of device workspace intelligibility_backward_device needs (0 for bad arguments).  Needs no GPU."""
    return int(lib().rnnoise_intelligibility_backward_workspace_bytes(int(n_pairs), int(n_samples), int(rate)))


def intelligibility_backward_device(n_pairs: int, n_samples: int, rate: int, result_ptr: int, fwd_workspace_ptr: int,
                                    fwd_workspace_bytes: int, grad_stoi_ptr: int, grad_estoi_ptr: int, grad_out_ptr: int,
                                    grad_stride: int, workspace_ptr: int, workspace_bytes: int, device: int = -1, cuda_stream: int = 0):
    """dL/d out of n_pairs pairs after intelligibility_device left result and fwd_workspace
    (rnnoise_intelligibility_backward_device): L = sum_p grad_stoi[p] stoi_p + grad_estoi[p] estoi_p (float64 device
    arrays; a null pointer is a zero gradient), written to grad_out[p*grad_stride + i] (float32), overwriting it.
    Stateless; ordered on cuda_stream, or synchronous without one."""
    ptr = lambda p: C.c_void_p(p) if p else None  # noqa: E731
    rc = lib().rnnoise_intelligibility_backward_device(int(n_pairs), int(n_samples), int(rate), ptr(result_ptr), ptr(fwd_workspace_ptr),
                                                       int(fwd_workspace_bytes), ptr(grad_stoi_ptr), ptr(grad_estoi_ptr), ptr(grad_out_ptr),
                                                       int(grad_stride), ptr(workspace_ptr), int(workspace_bytes), int(device), ptr(cuda_stream))
    if rc != 0:
        raise NnnoiselessError(last_error())


def intelligibility_backward_taps(workspace, B: int, n: int, rate: int = 48000):
    """Torch views of a backward workspace's documented regions after intelligibility_backward_device(B pairs of n
    samples at rate): dbands float64 [B][15][max(F - 1, 0)] (dL/d out's bands), inverse int32 [B][F] (the kept index of
    each 10 kHz frame, or -1), dframes float [B][max(F - 1, 0)][256] (dL/d each STFT frame's overlap-added samples,
    before its window) and dy10 float [B][n10]."""
    import torch
    _, _, n10, F = intelligibility_sizes(n, rate)
    maxM = max(F - 1, 0)
    r = lambda v: (v + 255) & ~255  # noqa: E731
    o_inv = r(B * STOI_BANDS * maxM * 8)
    o_du = o_inv + r(B * F * 4)
    o_dy = o_du + r(B * maxM * 256 * 4)
    w = workspace.view(torch.uint8)
    dby = w[:B * STOI_BANDS * maxM * 8].view(torch.float64).view(B, STOI_BANDS, maxM)
    inv = w[o_inv:o_inv + B * F * 4].view(torch.int32).view(B, F)
    du = w[o_du:o_du + B * maxM * 256 * 4].view(torch.float32).view(B, maxM, 256)
    dy10 = w[o_dy:o_dy + B * n10 * 4].view(torch.float32).view(B, n10)
    return dby, inv, du, dy10


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
