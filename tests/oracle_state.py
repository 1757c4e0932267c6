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
        L.nno_band_energies.argtypes = [vp, C.c_int, vp, vp]
        L.nno_pitch_stages_bytes.restype = C.c_size_t
        L.nno_pitch_stages.restype = C.c_int32
        L.nno_pitch_stages.argtypes = [vp, C.c_int32, C.c_float, vp]
        L.nno_pitch_only_from.restype = C.c_int32
        L.nno_pitch_only_from.argtypes = [vp, C.c_int32, C.c_float, vp]
        L.nno_highpass.argtypes = [vp, C.c_int, vp, vp]
        L.nno_train_new.restype = vp
        L.nno_train_free.argtypes = [vp]
        L.nno_train_set_params.argtypes = [vp, vp]
        L.nno_train_frame.argtypes = [vp, vp, vp, vp]
        L.nno_train_probe.argtypes = [vp] * 6
        assert L.nno_pitch_stages_bytes() == PITCH_STAGES.itemsize
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


def band_energies(windows):
    """The oracle's transform_input on given windows [n][960] (float32): window, nno_rfft960 under the current FFT
    order, wnorm, compute_band_corr -> (X complex64 [n][481], ex float32 [n][22])."""
    w = np.ascontiguousarray(np.asarray(windows, np.float32).reshape(-1, 960))
    X = np.empty((len(w), 481), np.complex64)
    ex = np.empty((len(w), 22), np.float32)
    lib().nno_band_energies(_ptr(w), len(w), _ptr(X), _ptr(ex))
    return X, ex


_NK = 14  # ladder steps k = 2..15
PITCH_STAGES = np.dtype([
    ("pitch_buf", "<f4", (864,)),
    ("xcorr4", "<f4", (147,)), ("ysq4", "<f4", (147,)), ("best4", "<i4"), ("second4", "<i4"),
    ("xcorr2", "<f4", (294,)), ("ysq2", "<f4", (294,)), ("best2", "<i4"), ("offset2", "<i4"), ("pitch_idx", "<i4"),
    ("t0", "<i4"), ("xx", "<f4"), ("xy0", "<f4"), ("g0", "<f4"),
    ("yy_raw", "<f4", (385,)), ("yy_lookup", "<f4", (385,)),
    ("nk", "<i4"), ("t1", "<i4", (_NK,)), ("t1b", "<i4", (_NK,)), ("taken", "<i4", (_NK,)),
    ("xy", "<f4", (_NK,)), ("yy", "<f4", (_NK,)), ("g1", "<f4", (_NK,)), ("cont", "<f4", (_NK,)), ("thresh", "<f4", (_NK,)),
    ("xc", "<f4", (3,)), ("t", "<i4"), ("offset", "<i4"), ("period", "<i4"), ("gain", "<f4"),
])


def pitch_stages(buf, last_period, last_gain):
    """pitch_process on buffers [n][1728] (the input_mem the pitch search sees) with the carried last_period [n] /
    last_gain [n], run as the oracle's own static functions in pitch_process's order -> PITCH_STAGES [n]: the whitened
    buffer, the coarse and fine xcorr with the running energies seen at each lag, (best, second), the fine best and
    offset, t0, xx, yy_lookup before and after its clamp, every ladder step (t1, t1b, xy, yy, g1, cont, thresh, taken),
    the final xc[3], offset, period and gain."""
    buf = np.ascontiguousarray(np.asarray(buf, np.float32).reshape(-1, 1728))
    n = len(buf)
    lp = np.broadcast_to(np.asarray(last_period, np.int32), (n,))
    lg = np.broadcast_to(np.asarray(last_gain, np.float32), (n,))
    out = np.zeros(n, PITCH_STAGES)
    L = lib()
    for i in range(n):
        L.nno_pitch_stages(_ptr(buf[i]), int(lp[i]), float(lg[i]), C.c_void_p(out.ctypes.data + i * PITCH_STAGES.itemsize))
    return out


def pitch_only(buf, last_period, last_gain):
    """The oracle's pitch_process entry point (nno_pitch_only) on buffers [n][1728] -> (period [n], last_gain [n])."""
    buf = np.ascontiguousarray(np.asarray(buf, np.float32).reshape(-1, 1728))
    n = len(buf)
    lp = np.broadcast_to(np.asarray(last_period, np.int32), (n,))
    lg = np.broadcast_to(np.asarray(last_gain, np.float32), (n,))
    period, gain, g = np.empty(n, np.int32), np.empty(n, np.float32), np.empty(1, np.float32)
    for i in range(n):
        period[i] = lib().nno_pitch_only_from(_ptr(buf[i]), int(lp[i]), float(lg[i]), _ptr(g))
        gain[i] = g[0]
    return period, gain


def highpass(x, mem=(0.0, 0.0)):
    """The input high-pass (src/util.rs:95-107) over x [n] from filter memory mem -> (y [n] float32, mem after)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.empty_like(x)
    m = np.array(mem, np.float32)
    lib().nno_highpass(_ptr(x), len(x), _ptr(y), _ptr(m))
    return y, m


class Trainer:
    """One lane of the oracle's training-data generator (oracle.Trainer) whose state can be read back: probe()."""

    def __init__(self, model: Model):
        self.model = model
        self._h = lib().nno_train_new()

    def set_params(self, params44):
        buf = np.ascontiguousarray(params44)
        assert buf.nbytes == 44
        lib().nno_train_set_params(self._h, _ptr(buf))

    def frame(self, signal, noise) -> np.ndarray:
        signal = np.ascontiguousarray(signal, dtype=np.float32)
        noise = np.ascontiguousarray(noise, dtype=np.float32)
        assert signal.shape == (480,) and noise.shape == (480,)
        row = np.empty(87, np.float32)
        lib().nno_train_frame(self._h, _ptr(signal), _ptr(noise), _ptr(row))
        return row

    def probe(self):
        """-> dict(vad_count, resp_mem [4] (signal m0 m1, noise m0 m1), ex [3][22], records uint8 [3][state_bytes]) of
        the clean, noise and combined extractors after the most recent frame."""
        vc = np.empty(1, np.int32)
        resp = np.empty(4, np.float32)
        ex = np.empty((3, 22), np.float32)
        rec = np.zeros((3, self.model.state_bytes), np.uint8)
        lib().nno_train_probe(self._h, self.model._h, _ptr(vc), _ptr(resp), _ptr(ex), _ptr(rec))
        return dict(vad_count=int(vc[0]), resp_mem=resp, ex=ex, records=rec)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.nno_train_free(self._h)
            self._h = None


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
