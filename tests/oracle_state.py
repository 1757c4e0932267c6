"""The CPU oracle with state records (TEST INFRASTRUCTURE): tests/oracle_state.c compiled together with
oracle/nno_oracle.c, with the flags of oracle/Makefile, into a temporary directory once per process.

State(model).export() gives the record rnnoise_batch_get_states gives for the same stream (include/rnnoise.h), and
State.import_() takes one, so records can be built and checked without a GPU.  analysis_frame and synthesis_from run
the two spectral stages of one frame on their own, from a record and from given inputs, under either of the oracle's
f32 FFT orders (set_fft_mode)."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_lib = None
_dir = None


def _cflags():
    mk = open(os.path.join(_ROOT, "oracle", "Makefile")).read()
    return re.search(r"^CFLAGS \?= (.*)$", mk, re.M).group(1).split()


def lib():
    global _lib, _dir
    if _lib is None:
        _dir = tempfile.mkdtemp(prefix="nno_state_")
        so = os.path.join(_dir, "libnno_state.so")
        subprocess.run(["gcc"] + _cflags() + ["-shared", "-o", so, os.path.join(_HERE, "oracle_state.c"), "-lm"],
                       check=True, capture_output=True)
        L = C.CDLL(so)
        vp = C.c_void_p
        L.nno_model_from_bytes.restype = vp
        L.nno_model_from_bytes.argtypes = [C.c_char_p, C.c_size_t]
        L.nno_model_free.argtypes = [vp]
        L.nno_state_new.restype = vp
        L.nno_state_new.argtypes = [vp]
        L.nno_state_free.argtypes = [vp]
        L.nno_process_frame.restype = C.c_float
        L.nno_process_frame.argtypes = [vp, vp, vp]
        L.nno_get_taps.argtypes = [vp, C.POINTER(oracle.Taps)]
        L.nno_state_bytes.restype = C.c_size_t
        L.nno_state_bytes.argtypes = [vp]
        L.nno_state_export.argtypes = [vp, vp]
        L.nno_state_import.restype = C.c_int
        L.nno_state_import.argtypes = [vp, vp]
        L.nno_set_fft_mode.argtypes = [C.c_int]
        L.nno_analysis_frame.restype = C.c_int
        L.nno_analysis_frame.argtypes = [vp] * 12
        L.nno_synthesis_from.argtypes = [vp] * 8 + [C.c_int, vp]
        L.nno_spectral_tables.argtypes = [vp, vp, vp]
        _lib = L
        import atexit
        atexit.register(shutil.rmtree, _dir, True)
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class Model:
    def __init__(self, data: bytes):
        self._h = lib().nno_model_from_bytes(data, len(data))
        if not self._h:
            raise ValueError("oracle: model bytes rejected")

    @property
    def state_bytes(self) -> int:
        return int(lib().nno_state_bytes(self._h))

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.nno_model_free(self._h)
            self._h = None


class State:
    def __init__(self, model: Model):
        self.model = model
        self._h = lib().nno_state_new(model._h)

    def process_frame(self, frame):
        frame = np.ascontiguousarray(frame, dtype=np.float32)
        out = np.empty(480, np.float32)
        vad = lib().nno_process_frame(self._h, _ptr(out), _ptr(frame))
        return out, np.float32(vad)

    def pitch(self) -> int:
        t = oracle.Taps()
        lib().nno_get_taps(self._h, C.byref(t))
        return int(t.pitch)

    def export(self) -> np.ndarray:
        rec = np.zeros(self.model.state_bytes, np.uint8)
        lib().nno_state_export(self._h, _ptr(rec))
        return rec

    def import_(self, rec) -> bool:
        rec = np.ascontiguousarray(rec, dtype=np.uint8).reshape(-1)
        assert rec.size == self.model.state_bytes
        return lib().nno_state_import(self._h, _ptr(rec)) == 0

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.nno_state_free(self._h)
            self._h = None


def run(model: Model, x, states=None):
    """x: [B][T][480] -> (out [B][T][480], vad [B][T], pitch [B][T], states); continues `states` if given."""
    x = np.asarray(x, np.float32)
    B, T, _ = x.shape
    states = states if states is not None else [State(model) for _ in range(B)]
    out = np.empty_like(x)
    vad = np.empty((B, T), np.float32)
    pitch = np.empty((B, T), np.int32)
    for b in range(B):
        for t in range(T):
            out[b, t], vad[b, t] = states[b].process_frame(x[b, t])
            pitch[b, t] = states[b].pitch()
    return out, vad, pitch, states


def set_fft_mode(mode: int):
    """0: the pinned f32 FFT (radices 4,4,5,3,2); 1: f64 DFT sums rounded once; 2: f32 with radices 2,3,5,4,4."""
    lib().nno_set_fft_mode(int(mode))


def spectral_tables():
    """The oracle's f32 tables: (window [960], dct [22][22], wnorm)."""
    window = np.empty(960, np.float32)
    dct = np.empty((22, 22), np.float32)
    wnorm = np.empty(1, np.float32)
    lib().nno_spectral_tables(_ptr(window), _ptr(dct), _ptr(wnorm))
    return window, dct, wnorm[0]


def analysis_frame(model: Model, record, frame):
    """The oracle's shift_and_filter + compute_frame_features on the state of `record` (taken before the frame) ->
    dict(X, P complex [481], ex, ep, exp [22], features [42], ceps [8][22], mem_id, pitch, silence, input_mem [1728])."""
    st = State(model)
    assert st.import_(record)
    frame = np.ascontiguousarray(frame, dtype=np.float32)
    X = np.empty(481, np.complex64)
    P = np.empty(481, np.complex64)
    ex, ep, exp = (np.empty(22, np.float32) for _ in range(3))
    feat = np.empty(42, np.float32)
    ceps = np.empty((8, 22), np.float32)
    mem_id, pitch = np.empty(1, np.int32), np.empty(1, np.int32)
    inp = np.empty(1728, np.float32)
    sil = lib().nno_analysis_frame(st._h, _ptr(frame), _ptr(X), _ptr(P), _ptr(ex), _ptr(ep), _ptr(exp), _ptr(feat), _ptr(ceps),
                                   _ptr(mem_id), _ptr(pitch), _ptr(inp))
    return dict(X=X, P=P, ex=ex, ep=ep, exp=exp, features=feat, ceps=ceps, mem_id=int(mem_id[0]), pitch=int(pitch[0]),
                silence=int(sil), input_mem=inp)


def synthesis_from(X, P, ex, ep, exp, gains, lastg, synth_mem, silence):
    """The oracle's statements after the network (pitch filter, gain floor, gains applied, inverse FFT, overlap-add) on
    the given f32 inputs: X complex [481], P complex [481] -> (out [480], lastg [22], synth_mem [480])."""
    c = lambda a, dt=np.float32: np.ascontiguousarray(a, dtype=dt)  # noqa: E731
    X, P = c(X, np.complex64), c(P, np.complex64)
    ex, ep, exp, gains = c(ex), c(ep), c(exp), c(gains)
    lastg, synth_mem = np.array(lastg, np.float32), np.array(synth_mem, np.float32)
    out = np.empty(480, np.float32)
    lib().nno_synthesis_from(_ptr(X), _ptr(P), _ptr(ex), _ptr(ep), _ptr(exp), _ptr(gains), _ptr(lastg), _ptr(synth_mem),
                             int(silence), _ptr(out))
    return out, lastg, synth_mem
