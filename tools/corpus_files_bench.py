"""Denoise a generated file corpus with rnnoise_denoise_corpus (recycled stream slots) at several slot counts and chunk
lengths, DESIGN.md 7o.

    python tools/corpus_files_bench.py [--files 2000] [--dir DIR] [--report PATH] [--rounds 3]
                                       [--slots 256,1024] [--chunks 16,64,256]

The corpus is seeded: `--files` 16-bit WAVs (one in eight stereo) at 16, 44.1 and 48 kHz, lengths spread evenly from
1 to 30 s of white noise plus a sine, written under DIR (default: a temporary directory, removed at the end).  Each
round runs denoise_corpus at every slot count and chunk length, alternating, each writing fresh outputs.  Every run
reports wall time, audio seconds denoised per second, occupancy (useful stream-frames over issued slot-frames), the
call's three waits, and the peak of the device's used memory over the run (sampled every 5 ms with cudaMemGetInfo, less
the use before the run: other work on the card would show up in it).  The outputs of every run are hashed and must
equal the first run's.  `--policy` adds the slot-policy probe: the fused call on all S
streams against a subset call on S/2 and S/8 of them, 64 frames each, the host clock over 20 calls ended by a device synchronise.  One JSON
line per run, then a summary with the card's name and power limit."""
import argparse
import ctypes as C
import hashlib
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import nnnoiseless_b200 as nb  # noqa: E402
from nnnoiseless_b200 import files  # noqa: E402


def query(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def wav16(path, x, rate):
    n, ch = x.shape
    payload = x.astype("<i2").tobytes()
    body = struct.pack("<HHIIHH", 1, ch, rate, rate * ch * 2, ch * 2, 16)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(body) + 8 + len(payload)) + b"WAVE" + b"fmt " + struct.pack("<I", len(body)) +
                body + b"data" + struct.pack("<I", len(payload)))
        f.write(payload)


def make_corpus(d, n_files, seed):
    """-> [(path, channels, rate, seconds)], lengths spread evenly from 1 to 30 s in a seeded random order."""
    rng = np.random.default_rng(seed)
    secs = np.linspace(1.0, 30.0, n_files)[rng.permutation(n_files)]
    out = []
    for i, s in enumerate(secs):
        rate = int(rng.choice([16000, 44100, 48000]))
        ch = 2 if rng.random() < 0.125 else 1
        n = int(s * rate)
        t = np.arange(n, dtype=np.float32) / rate
        x = rng.normal(0.0, 1500.0, (n, ch)).astype(np.float32)
        x += (6000.0 * np.sin(2 * np.pi * rng.uniform(100, 3000) * t))[:, None]
        p = os.path.join(d, "in%05d.wav" % i)
        wav16(p, np.clip(np.round(x), -32768, 32767), rate)
        out.append((p, ch, rate, n / rate))
    return out


class MemPeak:
    """Peak of the device's used bytes (cudaMemGetInfo) over a run, less the use at its start."""

    def __init__(self):
        nb.lib()                                           # loads the CUDA runtime the library links
        self.rt = C.CDLL("libcudart.so.12")

    def used(self):
        free, total = C.c_size_t(0), C.c_size_t(0)
        self.rt.cudaMemGetInfo(C.byref(free), C.byref(total))
        return total.value - free.value

    def __enter__(self):
        self.base = self.peak = self.used()
        self.stop = False
        self.t = threading.Thread(target=self.poll)
        self.t.start()
        return self

    def poll(self):
        while not self.stop:
            self.peak = max(self.peak, self.used())
            time.sleep(0.005)

    def __exit__(self, *exc):
        self.stop = True
        self.t.join()
        self.peak = max(self.peak, self.used())


def digest(paths):
    return [hashlib.sha1(open(p, "rb").read()).hexdigest() for p in paths]


def run_once(corpus, outdir, slots, chunk):
    os.makedirs(outdir)
    pairs = [(p, os.path.join(outdir, "o%05d.wav" % i)) for i, (p, _, _, _) in enumerate(corpus)]
    with MemPeak() as mem:
        t0 = time.perf_counter()
        st = files.denoise_corpus(pairs, slots=slots, chunk_frames=chunk)
        wall = time.perf_counter() - t0
    audio = sum(s for _, _, _, s in corpus)
    h = digest([o for _, o in pairs])
    shutil.rmtree(outdir)
    return dict(slots=slots, chunk_frames=chunk, files=len(corpus), wall_s=round(wall, 3), audio_s_per_s=round(audio / wall, 1),
                occupancy=round(st["useful_stream_frames"] / st["issued_slot_frames"], 4),
                decode_wait_s=round(st["decode_wait_seconds"], 3), device_wait_s=round(st["device_wait_seconds"], 3),
                write_wait_s=round(st["write_wait_seconds"], 3), peak_device_mb=round((mem.peak - mem.base) / 2**20, 1),
                chunks=st["chunks"], peak_pool_mb=round(st["peak_pool_bytes"] / 2**20, 1)), h


def policy_probe(S, chunk):
    """Host-timed fused call over all S streams against subset calls on S/2 and S/8 streams (float in, int16 out)."""
    import torch
    L = nb.lib()
    b = nb.DenoiseBatch(S, device=0)
    x = torch.randn(chunk * 480 * S, device="cuda") * 3000
    y = torch.empty(chunk * 480 * S, dtype=torch.int16, device="cuda")
    res = {}
    for n in (S, S // 2, S // 8):
        idx = np.arange(0, S, S // n, dtype=np.int32)[:n]

        def call():
            if n == S:
                rc = L.rnnoise_batch_process_device_strided(b._h, y.data_ptr(), x.data_ptr(), 2, None, chunk, 1, S, 480 * S, None)
            else:
                rc = L.rnnoise_batch_process_streams_device(b._h, idx.ctypes.data, n, y.data_ptr(), x.data_ptr(), 2, None, chunk, 1, n,
                                                             480 * n, None)
            assert rc == 0, nb.last_error()
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(20):
            call()
        torch.cuda.synchronize()
        res["full" if n == S else "subset_%d" % n] = round((time.perf_counter() - t0) / 20 * 1e3, 3)
    return dict(policy=True, slots=S, chunk_frames=chunk, ms_per_call=res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=2000)
    ap.add_argument("--dir", default=None)
    ap.add_argument("--report", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--slots", default="256,1024")
    ap.add_argument("--chunks", default="16,64,256")
    ap.add_argument("--policy", action="store_true")
    ap.add_argument("--seed", type=int, default=11)
    a = ap.parse_args()
    d = a.dir or tempfile.mkdtemp(prefix="corpus_bench_")
    os.makedirs(d, exist_ok=True)
    lines = []

    def emit(r):
        print(json.dumps(r), flush=True)
        lines.append(r)

    try:
        t0 = time.perf_counter()
        corpus = make_corpus(d, a.files, a.seed)
        emit(dict(generated=len(corpus), audio_hours=round(sum(c[3] for c in corpus) / 3600, 2), seconds=round(time.perf_counter() - t0, 1)))
        configs = [(int(s), int(k)) for s in a.slots.split(",") for k in a.chunks.split(",")]
        ref, runs = None, []
        for rnd in range(a.rounds):
            for s, k in configs:
                r, h = run_once(corpus, os.path.join(d, "out"), s, k)
                r["round"] = rnd
                ref = ref or h
                r["equal"] = h == ref
                emit(r)
                runs.append(r)
        if a.policy:
            for s in a.slots.split(","):
                emit(policy_probe(int(s), 64))
        summ = dict(summary=True, device=query("name"), power_limit=query("power.limit"), sm_clock_max=query("clocks.max.sm"),
                    files=len(corpus), all_equal=all(r["equal"] for r in runs))
        for s, k in configs:
            rs = [r for r in runs if (r["slots"], r["chunk_frames"]) == (s, k)]
            if rs:
                summ["corpus_%s_%s" % (s, k)] = dict(wall_s=[r["wall_s"] for r in rs], median_audio_s_per_s=float(np.median([r["audio_s_per_s"] for r in rs])))
        emit(summ)
    finally:
        if a.report:
            os.makedirs(os.path.dirname(os.path.abspath(a.report)), exist_ok=True)
            with open(a.report, "w") as f:
                f.write("".join(json.dumps(r) + "\n" for r in lines))
        if a.dir is None:
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
