"""Training-data rows on the GPU: host-side mirror of the reference's ``nnnoiseless-gen-training-data`` binary.

Reference: ``src/training.rs``.  The split is

* host (this module, plain numpy): the file side of ``SignalReader`` (:183-262) -- which file, which sample offset,
  how many frames -- planned up front as segments, ``NoiseSimulator::randomize`` (:352-377) -- the random gains,
  random biquads and the low-pass band, drawn every ``GAIN_CHANGE_COUNT`` frames -- and the reads of the WAV samples;
* device (``rnnoise_train_*`` in include/rnnoise.h): everything arithmetic per frame -- gains, filters, mix, the
  VAD counter, three feature extractors, and the 87-float output row.

``generate_rows`` / ``python -m nnnoiseless_b200.training`` is the whole binary: speech and noise WAV files in, rows
``[F][L][87]`` out.  A *lane* is one ``NoiseSimulator`` with its own signal reader and noise reader:

* each reader takes ``frames_per_file = max(count // n_paths + 1, 100)`` frames per file (``count`` is the global row
  count); a file longer than ``480 * frames_per_file`` samples is read from a uniform random sample offset in
  ``[0, len - 480 * frames_per_file]``, a shorter one whole from sample 0 (``len // 480`` frames); after its last
  frame the reader opens the next file, wrapping round the list;
* lane ``l``'s readers start at file ``(l * n_paths) // L``; every lane produces ``F = ceil(count / L)`` frames, so
  the output has ``F * L >= count`` rows;
* randomize runs at frames ``2821 + k * 2822`` (``next_frame`` increments ``gain_change_count`` before testing it);
  before that a lane runs with ``NoiseSimulator::new``'s parameters.

Random draws all come from one ``np.random.default_rng(seed)``, in this order: with ``shuffle``, a permutation of the
signal paths, then of the noise paths; then frame by frame, ``randomize(L, rng)`` if the frame is a randomize frame,
then lane by lane the noise reader's seek draw (if it opens a file here) before the signal reader's.  For ``L = 1``
that is the reference's order (``next_frame`` reads the noise before the signal).

Deliberate departures from the reference:

1. Every file is checked up front, from its header alone, before any GPU work; the reference checks a file when it
   opens it.  A data chunk that runs past the end of its file is refused then (hound fails on it mid-read).
2. A file with fewer than 480 samples is an error naming it: the reference's ``next_reader`` leaves ``cur_idx`` where
   it is when ``frames_left == 0`` and reopens that file forever.
3. An empty set of files is the error "cannot read from an empty set of files", not a panic.
4. The output is ``.npy``, not HDF5 (there is no HDF5 library here); an output path ending in ``.h5`` is refused.
5. numpy's generator replaces ``thread_rng``: the reference is not reproducible, this is, for a fixed seed and ``L``.

There is NO CPU fallback: without the CUDA library / a GPU the trainer raises.
"""
import argparse
import ctypes as C
import glob as _glob
import heapq
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import FRAME_SIZE, NB_BANDS, NB_FEATURES, DenoiseBatch, NnnoiselessError, RnnModel, _np_ptr, gru_widths, last_error, lib

TRAIN_ROW = NB_FEATURES + 2 * NB_BANDS + 1  # 87, src/training.rs:90
GAIN_CHANGE_COUNT = 2821                    # src/training.rs:17
RANDOMIZE_PERIOD = GAIN_CHANGE_COUNT + 1    # randomize at frames 2821 + k * 2822 (:389-393)
FREQ_SIZE = 481
POOL_BYTES = 256 << 20                      # rnnoise_train_process_pool_host's bound on one call's sample pool

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

    def process_pool_host(self, pool: np.ndarray, sig_at: np.ndarray, noise_at: np.ndarray, out: np.ndarray = None) -> np.ndarray:
        """pool: int16 samples; sig_at, noise_at: [T][L] int64 offsets into pool (frame at pool[at:at + 480], -1 =
        zeros) -> rows [T][L][87] (written into ``out`` if given: a C-contiguous float32 [T][L][87] array)."""
        pool = np.ascontiguousarray(pool, dtype=np.int16)
        sig_at = np.ascontiguousarray(sig_at, dtype=np.int64)
        noise_at = np.ascontiguousarray(noise_at, dtype=np.int64)
        if pool.ndim != 1 or sig_at.ndim != 2 or noise_at.shape != sig_at.shape or sig_at.shape[1] != self.n_lanes:
            raise ValueError("expected a 1-d pool and two [T][%d] offset arrays" % self.n_lanes)
        T = sig_at.shape[0]
        if out is None:
            out = np.empty((T, self.n_lanes, TRAIN_ROW), np.float32)
        elif out.dtype != np.float32 or out.shape != (T, self.n_lanes, TRAIN_ROW) or not out.flags.c_contiguous:
            raise ValueError("out must be a C-contiguous float32 [%d][%d][87] array" % (T, self.n_lanes))
        if lib().rnnoise_train_process_pool_host(self._h, _np_ptr(out), _np_ptr(pool), len(pool), _np_ptr(sig_at),
                                                 _np_ptr(noise_at), T) != 0:
            raise NnnoiselessError(last_error())
        return out

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


# ---- the corpus: files, the segment plan, the reads ---------------------------------------------------------------

SEGMENT_DTYPE = np.dtype([("first", np.int64), ("file", np.int64), ("offset", np.int64), ("frames", np.int64)])


def glob_paths(globs) -> list:
    """``glob_paths`` (src/training.rs:19-28): each pattern's matches in sorted order, the patterns in turn."""
    out = []
    for g in globs:
        out += sorted(_glob.glob(g))
    return out


def default_lanes(count: int) -> int:
    """``clamp(count // (100 * 2822), 1, 4096)``: each lane's first 2821 frames run un-randomized, so this keeps
    that warm-up at or below about 1 % of the rows."""
    return int(min(max(count // (100 * RANDOMIZE_PERIOD), 1), 4096))


def warmup_share(count: int, lanes: int) -> float:
    """The share of the output rows made with ``NoiseSimulator::new``'s parameters."""
    F = -(-count // lanes)
    return min(F, GAIN_CHANGE_COUNT) / F if F else 0.0


def probe_corpus(paths) -> tuple:
    """Departures 1-3: checks every file's header -> (paths, samples per file [n] int64, data byte offsets [n] int64)."""
    from .files import probe_audio
    paths = list(paths)
    if not paths:
        raise NnnoiselessError("cannot read from an empty set of files")  # SignalReader::new, :186
    n = np.empty(len(paths), np.int64)
    off = np.empty(len(paths), np.int64)
    for i, p in enumerate(paths):
        try:
            a = probe_audio(p)
        except NnnoiselessError as e:
            raise NnnoiselessError("%s in %s" % (e, p)) from None
        if a.channels != 1 or a.sample_rate != 48000 or a.bits_per_sample != 16 or a.is_float:  # next_reader, :202-213
            raise NnnoiselessError("unsupported wav format WavSpec { channels: %d, sample_rate: %d, bits_per_sample: %d, "
                                   "sample_format: %s } in %s"
                                   % (a.channels, a.sample_rate, a.bits_per_sample, "Float" if a.is_float else "Int", p))
        if a.n_frames < FRAME_SIZE:
            raise NnnoiselessError("%s has %d samples, fewer than one %d-sample frame: the reference's reader would reopen it "
                                   "forever" % (p, a.n_frames, FRAME_SIZE))
        n[i], off[i] = a.n_frames, a.data_offset
    return paths, n, off


class Plan:
    """What every lane reads, frame by frame, and when and how it is randomized.

    ``signal[l]`` / ``noise[l]``: lane l's segments, a SEGMENT_DTYPE array in frame order: frames ``first .. first +
    frames`` read file ``file`` (an index into ``signal_paths`` / ``noise_paths``) from sample ``offset`` on, 480
    samples per frame.  ``randomize``: ``[(frame, params [L])]``, the parameters set before that frame."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def frames_at(self, kind: str, lane: int):
        """-> (file [F], sample offset [F]) of every frame of one lane's signal or noise reader."""
        segs = getattr(self, kind)[lane]
        f = np.repeat(segs["file"], segs["frames"])
        o = np.concatenate([s["offset"] + FRAME_SIZE * np.arange(s["frames"]) for s in segs]) if len(segs) else np.zeros(0, np.int64)
        return f, o


def plan(signal_paths, noise_paths, count: int, lanes: int, seed: int = 0, shuffle: bool = False) -> Plan:
    """The segment plan of ``lanes`` lanes making ``count`` rows, drawn from ``np.random.default_rng(seed)`` in the
    module's documented order.  Every file is probed first (departures 1-3).  Costs O(files opened), not O(frames)."""
    count, L = int(count), int(lanes)
    if count <= 0 or L <= 0:
        raise ValueError("count and lanes must be positive")
    sig_paths, sig_len, sig_off = probe_corpus(signal_paths)
    noise_paths, noise_len, noise_off = probe_corpus(noise_paths)
    rng = np.random.default_rng(seed)
    if shuffle:  # main, :83-86: the signal paths, then the noise paths
        ps, pn = rng.permutation(len(sig_paths)), rng.permutation(len(noise_paths))
        sig_paths, sig_len, sig_off = [sig_paths[i] for i in ps], sig_len[ps], sig_off[ps]
        noise_paths, noise_len, noise_off = [noise_paths[i] for i in pn], noise_len[pn], noise_off[pn]
    F = -(-count // L)
    # reader r = 2 l + k: k = 0 lane l's noise reader, k = 1 its signal reader (next_frame reads noise first)
    lens = (noise_len, sig_len)
    fpf = tuple(max(count // len(x) + 1, 100) for x in lens)  # SignalReader::new, :185-194
    idx = [(l * len(lens[k])) // L for l in range(L) for k in (0, 1)]
    segs = [[] for _ in range(2 * L)]
    rand = []
    # events (frame, key): key -1 = randomize, else the reader that opens its next file; a frame's randomize comes
    # before its reads, and lane l's readers before lane l + 1's
    heap = [(0, r) for r in range(2 * L)]
    if GAIN_CHANGE_COUNT < F:
        heap.append((GAIN_CHANGE_COUNT, -1))
    heapq.heapify(heap)
    while heap:
        f, r = heapq.heappop(heap)
        if r < 0:
            rand.append((f, randomize(L, rng)))
            if f + RANDOMIZE_PERIOD < F:
                heapq.heappush(heap, (f + RANDOMIZE_PERIOD, -1))
            continue
        k = r & 1
        i = idx[r] if idx[r] < len(lens[k]) else 0  # next_reader, :196-231
        n, want = int(lens[k][i]), FRAME_SIZE * fpf[k]
        if n > want:
            off, frames = int(rng.integers(0, n - want, endpoint=True)), fpf[k]
        else:
            off, frames = 0, n // FRAME_SIZE
        idx[r] = i + 1
        segs[r].append((f, i, off, min(frames, F - f)))
        if f + frames < F:
            heapq.heappush(heap, (f + frames, r))
    arr = [np.array(x, SEGMENT_DTYPE) for x in segs]
    return Plan(count=count, n_lanes=L, n_frames=F, seed=seed, shuffle=shuffle,
                signal_paths=sig_paths, noise_paths=noise_paths, signal_len=sig_len, noise_len=noise_len,
                signal_data_offset=sig_off, noise_data_offset=noise_off,
                signal_frames_per_file=fpf[1], noise_frames_per_file=fpf[0],
                signal=arr[1::2], noise=arr[0::2], randomize=rand)


def call_bounds(p: Plan, pool_bytes: int = POOL_BYTES) -> list:
    """[(f0, f1)]: the trainer calls.  A call ends at each randomize frame (its parameters are set between calls) and
    after as many frames as keep its pool of 2 x 480 int16 samples per lane-frame within pool_bytes."""
    step = max(1, int(pool_bytes) // (p.n_lanes * 2 * FRAME_SIZE * 2))
    cuts = sorted({0, p.n_frames} | {f for f, _ in p.randomize})
    out = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        out += [(f, min(f + step, b)) for f in range(a, b, step)]
    return out


def build_pool(p: Plan, f0: int, f1: int):
    """The pool and offsets of frames [f0, f1): -> (pool int16, sig_at [n][L], noise_at [n][L]).  The pool is the
    needed slices of the files' data chunks, memory-mapped as ``<i2`` and concatenated in file order."""
    L, n = p.n_lanes, f1 - f0
    pieces = []  # (kind, file, first sample, frames, lane, first frame - f0)
    for k, kind in enumerate(("noise", "signal")):
        for l, segs in enumerate(getattr(p, kind)):
            first = segs["first"]
            j = max(int(np.searchsorted(first, f0, side="right")) - 1, 0)  # the segment that holds frame f0
            while j < len(segs) and first[j] < f1:
                s = segs[j]
                a, b = max(int(s["first"]), f0), min(int(s["first"] + s["frames"]), f1)
                if a < b:
                    pieces.append((k, int(s["file"]), int(s["offset"]) + FRAME_SIZE * (a - int(s["first"])), b - a, l, a - f0))
                j += 1
    pieces.sort()
    pool = np.empty(2 * n * L * FRAME_SIZE, np.int16)
    at = np.empty((2, n, L), np.int64)
    maps, pos, step = {}, 0, FRAME_SIZE * np.arange(n, dtype=np.int64)
    for k, i, s0, nf, l, a in pieces:
        if (k, i) not in maps:
            path, off, ln = ((p.noise_paths, p.noise_data_offset, p.noise_len), (p.signal_paths, p.signal_data_offset, p.signal_len))[k]
            maps[(k, i)] = np.memmap(path[i], dtype="<i2", mode="r", offset=int(off[i]), shape=(int(ln[i]),))
        ns = nf * FRAME_SIZE
        pool[pos:pos + ns] = maps[(k, i)][s0:s0 + ns]
        at[k, a:a + nf, l] = pos + step[:nf]
        pos += ns
    assert pos == len(pool)
    return pool, at[1], at[0]


def generate_rows(signal_paths, noise_paths, count: int, lanes: int = None, seed: int = 0, shuffle: bool = False,
                  out=None, device: int = -1, pool_bytes: int = POOL_BYTES, timings: dict = None) -> np.ndarray:
    """Rows ``[F][L][87]`` float32 from speech and noise WAV files (``F = ceil(count / L)``, ``L`` = ``lanes`` or
    ``default_lanes(count)``).  out: a path: the rows go into that ``.npy`` through ``np.lib.format.open_memmap``,
    call by call, and the memmap is returned.  One prefetch thread builds the next call's pool while the GPU runs the
    current one.  timings (optional dict): gets the seconds spent planning, building pools and waiting for the GPU."""
    if out is not None and str(out).lower().endswith(".h5"):
        raise NnnoiselessError("HDF5 output is not supported (no HDF5 library): write a .npy file instead")
    t0 = time.perf_counter()
    L = default_lanes(count) if lanes is None else int(lanes)
    p = plan(signal_paths, noise_paths, count, L, seed, shuffle)
    t_plan = time.perf_counter() - t0
    tb = TrainingBatch(L, device)
    shape = (p.n_frames, L, TRAIN_ROW)
    rows = np.lib.format.open_memmap(out, mode="w+", dtype=np.float32, shape=shape) if out is not None else np.empty(shape, np.float32)
    params = dict(p.randomize)
    calls = call_bounds(p, pool_bytes)
    t_pool = t_gpu = 0.0

    def build(c):
        t = time.perf_counter()
        r = build_pool(p, *c)
        return r, time.perf_counter() - t

    with ThreadPoolExecutor(1) as ex:
        nxt = ex.submit(build, calls[0])
        for k, (f0, f1) in enumerate(calls):
            (pool, sig_at, noise_at), dt = nxt.result()
            t_pool += dt
            if k + 1 < len(calls):
                nxt = ex.submit(build, calls[k + 1])
            if f0 in params:
                tb.set_params(params[f0])
            t = time.perf_counter()
            tb.process_pool_host(pool, sig_at, noise_at, out=rows[f0:f1])
            t_gpu += time.perf_counter() - t
    if out is not None:
        rows.flush()
    if timings is not None:
        timings.update(plan=t_plan, pool=t_pool, trainer=t_gpu, calls=len(calls), lanes=L, frames=p.n_frames)
    return rows


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m nnnoiseless_b200.training",
                                 description="Generate data for training nnnoiseless models, on the GPU")
    ap.add_argument("--signal-glob", action="append", required=True, help="wildcard for audio signal data")
    ap.add_argument("--noise-glob", action="append", required=True, help="wildcard for audio noise data")
    ap.add_argument("--shuffle", action="store_true", help="if set, shuffle the signal and noise files")
    ap.add_argument("--count", type=int, required=True, help="number of frames to generate")
    ap.add_argument("-o", dest="output", required=True, help="output file (.npy, rows [frames][lanes][87])")
    ap.add_argument("--lanes", type=int, help="simulators run side by side (default: count // 282200, in [1, 4096])")
    ap.add_argument("--seed", type=int, default=0, help="seed of every random draw")
    ap.add_argument("--device", type=int, default=-1, help="CUDA device (-1: current)")
    a = ap.parse_args(argv)
    if a.count <= 0:
        ap.error("count must be a positive integer")
    if a.lanes is not None and a.lanes <= 0:
        ap.error("lanes must be a positive integer")
    if a.output.lower().endswith(".h5"):
        ap.error("HDF5 output is not supported (no HDF5 library): write a .npy file instead")
    sig, noise = glob_paths(a.signal_glob), glob_paths(a.noise_glob)
    L = default_lanes(a.count) if a.lanes is None else a.lanes
    for what, paths in (("clean", sig), ("noise", noise)):
        if paths:
            print("Found %d %s files, reading about %d frames from each" % (len(paths), what, max(a.count // len(paths) + 1, 100)),
                  file=sys.stderr)
    F = -(-a.count // L)
    print("%d lanes x %d frames = %d rows; %.2f %% of them before the first randomize"
          % (L, F, F * L, 100.0 * warmup_share(a.count, L)), file=sys.stderr)
    try:
        generate_rows(sig, noise, a.count, L, a.seed, a.shuffle, out=a.output, device=a.device)
    except NnnoiselessError as e:
        print("error: %s" % e, file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
