"""File front-end: host-side mirror of the reference's ``nnnoiseless`` binary (``src/nnnoiseless.rs``).

``denoise_file`` / ``denoise_files`` = ``main`` (:230-334) for one file / a set of files, on a fixed set of recycled GPU
stream slots; ``denoise_corpus`` = the same call with its slot count, chunk length, pool and threads exposed;
``read_audio`` = ``raw_samples`` / ``wav_samples`` (:179-228); ``resample`` = ``Resample`` (:104-131) on the GPU.
The command-line binary itself is ``nnnoiseless_b200/bin/nnnoiseless-b200`` (``cli/nnnoiseless_cli.cpp``).
"""
import ctypes as C
import os

import numpy as np

from . import NnnoiselessError, RnnModel, _np_ptr, last_error, link_mode_of, lib

CLI_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bin", "nnnoiseless-b200")


class FileOptions(C.Structure):
    _fields_ = [("wav_in", C.c_int), ("wav_out", C.c_int), ("sample_rate", C.c_double), ("channels", C.c_int),
                ("model", C.c_void_p), ("device", C.c_int)]


def _options(wav_in, wav_out, sample_rate, channels, model, device):
    return FileOptions(int(bool(wav_in)), int(bool(wav_out)), float(sample_rate or 0.0), int(channels or 0),
                       model._h if model is not None else None, int(device))


def denoise_files(pairs, wav_in=False, wav_out=False, sample_rate=None, channels=None, model: RnnModel = None, device=-1,
                  link_channels=None):
    """pairs: iterable of (input path, output path), denoised as denoise_corpus does with every default.
    link_channels 'max' or 'mean': the channels of each multi-channel file are one linked group (--link-channels)."""
    link = 0 if link_channels is None else link_mode_of(link_channels)
    pairs = [(os.fsencode(a), os.fsencode(b)) for a, b in pairs]
    n = len(pairs)
    ins = (C.c_char_p * n)(*[a for a, _ in pairs])
    outs = (C.c_char_p * n)(*[b for _, b in pairs])
    opt = _options(wav_in, wav_out, sample_rate, channels, model, device)
    if lib().rnnoise_denoise_files_linked(n, ins, outs, C.byref(opt), link) != 0:
        raise NnnoiselessError(last_error())


class CorpusOptions(C.Structure):
    """== RNNoiseCorpusOptions (0: the documented default of each field)."""
    _fields_ = [("slots", C.c_int), ("chunk_frames", C.c_int), ("device_pool_bytes", C.c_longlong), ("decode_threads", C.c_int)]


class CorpusStats(C.Structure):
    """== RNNoiseCorpusStats."""
    _fields_ = [("files", C.c_longlong), ("useful_stream_frames", C.c_longlong), ("issued_slot_frames", C.c_longlong),
                ("chunks", C.c_longlong), ("peak_pool_bytes", C.c_longlong), ("decode_wait_seconds", C.c_double),
                ("device_wait_seconds", C.c_double), ("write_wait_seconds", C.c_double)]


def _count(name, v, lo, hi):
    if v is None:
        return 0
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
        raise ValueError("%s must be an integer in %d..%d, not %r" % (name, lo, hi, v))
    return int(v)


def denoise_corpus(pairs, slots=None, chunk_frames=None, device_pool_bytes=None, decode_threads=None, link_channels=None,
                   wav_in=False, wav_out=False, sample_rate=None, channels=None, model: RnnModel = None, device=-1) -> dict:
    """pairs: iterable of (input path, output path), any number of them, denoised on `slots` recycled streams in chunks
    of `chunk_frames` frames (rnnoise_denoise_corpus).  Each output is byte for byte what denoise_file writes for that
    input alone with the same options, whatever the slots, chunk and order.  None: the library's default (rnnoise.h).
    Returns the call's RNNoiseCorpusStats as a dict."""
    copt = CorpusOptions(_count("slots", slots, 1, 1 << 20), _count("chunk_frames", chunk_frames, 1, 1 << 16),
                         _count("device_pool_bytes", device_pool_bytes, 1, (1 << 63) - 1),
                         _count("decode_threads", decode_threads, 1, 256))
    link = 0 if link_channels is None else link_mode_of(link_channels)
    pairs = [(os.fsencode(a), os.fsencode(b)) for a, b in pairs]
    n = len(pairs)
    ins = (C.c_char_p * n)(*[a for a, _ in pairs])
    outs = (C.c_char_p * n)(*[b for _, b in pairs])
    opt = _options(wav_in, wav_out, sample_rate, channels, model, device)
    st = CorpusStats()
    if lib().rnnoise_denoise_corpus(n, ins, outs, C.byref(opt), link, C.byref(copt), C.byref(st)) != 0:
        raise NnnoiselessError(last_error())
    return {name: getattr(st, name) for name, _ in CorpusStats._fields_}


def denoise_file(input_path, output_path, **kw):
    denoise_files([(input_path, output_path)], **kw)


def read_audio(path, wav=None, channels=1, sample_rate=48000.0):
    """-> (samples [n_frames][channels] float32 in the i16 range, sample_rate).  wav=None: by extension."""
    p = C.POINTER(C.c_float)()
    n, ch, sr = C.c_long(0), C.c_int(0), C.c_double(0.0)
    mode = 0 if wav is None else (1 if wav else -1)
    if lib().rnnoise_audio_read(os.fsencode(path), mode, int(channels), float(sample_rate), C.byref(p), C.byref(n), C.byref(ch),
                                C.byref(sr)) != 0:
        raise NnnoiselessError(last_error())
    try:
        a = np.ctypeslib.as_array(p, shape=(n.value * ch.value,)).copy() if n.value else np.zeros(0, np.float32)
    finally:
        lib().rnnoise_audio_free(p)
    return a.reshape(n.value, ch.value), float(sr.value)


class AudioInfo(C.Structure):
    """== RNNoiseAudioInfo: a WAV file's format and where its samples are (rnnoise_audio_probe)."""
    _fields_ = [("channels", C.c_int), ("sample_rate", C.c_int), ("bits_per_sample", C.c_int), ("is_float", C.c_int),
                ("data_offset", C.c_longlong), ("n_frames", C.c_longlong)]


def probe_audio(path) -> AudioInfo:
    """A RIFF/WAVE file's header alone, with read_audio's checks and error texts."""
    info = AudioInfo()
    if lib().rnnoise_audio_probe(os.fsencode(path), C.byref(info)) != 0:
        raise NnnoiselessError(last_error())
    return info


def write_audio(path, pcm: np.ndarray, wav=None):
    """pcm: [n_frames][channels] int16 -> raw little-endian i16, or a 48 kHz 16-bit WAV."""
    pcm = np.ascontiguousarray(pcm, dtype=np.int16)
    if pcm.ndim == 1:
        pcm = pcm[:, None]
    mode = 0 if wav is None else (1 if wav else -1)
    if lib().rnnoise_audio_write(os.fsencode(path), mode, _np_ptr(pcm), pcm.shape[0], pcm.shape[1]) != 0:
        raise NnnoiselessError(last_error())


def resample(x: np.ndarray, ratio: float, device=-1) -> np.ndarray:
    """x: [n][channels] float32 -> [k][channels] at 1/ratio times the rate (ratio = input rate / 48000)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if x.ndim == 1:
        x = x[:, None]
    n, ch = x.shape
    cap = int(n / ratio) + 16 if ratio > 0 else 0
    out = np.empty((cap, ch), np.float32)
    k = lib().rnnoise_resample_host(_np_ptr(out), cap, _np_ptr(x), n, ch, float(ratio), int(device))
    if k < 0:
        raise NnnoiselessError(last_error())
    return out[:k]
