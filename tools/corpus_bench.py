"""Training rows from a WAV corpus on one GPU (nnnoiseless_b200.training.generate_rows), end to end.

Writes a seeded corpus to a temporary directory (speech-like: a tone under a slow on/off envelope plus noise; noise:
coloured noise; mono 48 kHz 16-bit, `--seconds` each), then reports, with the card's name and power limit:

* rows/s of generate_rows at the default lane count and at --wide lanes, with the time spent planning, building the
  call pools (in the prefetch thread, overlapped with the GPU) and inside the trainer calls;
* the same plan driven through the float entry point (rnnoise_train_process_host), the host assembling each call's
  [T][L][480] float arrays from the memory-mapped files;
* the oracle's one-thread rows/s on a sample (what the reference binary does, one frame at a time);
* from torch.profiler over a few calls at equal L: the pool and the float front kernel, the trainer's kernels in all,
  and the host<->device copies.

    python tools/corpus_bench.py [--files 200] [--seconds 60] [--count 2000000] [--wide 4096] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nnnoiseless_b200 import training as tr  # noqa: E402
from nnnoiseless_b200.files import write_audio  # noqa: E402


def write_corpus(d, n_files, seconds, seed=0):
    rng = np.random.default_rng(seed)
    n = 48000 * seconds
    base = rng.standard_normal(n + 48000).astype(np.float32)  # shared white noise, a random window per file
    t = np.arange(n, dtype=np.float32) / np.float32(48000.0)
    sig, noise = [], []
    for i in range(n_files):
        o = int(rng.integers(0, 48000))
        env = np.repeat(rng.choice([0.0, 0.05, 0.3, 1.0], size=n // 24000 + 1), 24000)[:n].astype(np.float32)
        x = env * (rng.uniform(1000, 9000) * np.sin(2 * np.pi * rng.uniform(100, 400) * t)) + rng.uniform(30, 300) * base[o:o + n]
        p = os.path.join(d, "speech%03d.wav" % i)
        write_audio(p, np.clip(np.round(x), -32768, 32767).astype(np.int16), wav=True)
        sig.append(p)
        o = int(rng.integers(0, 48000))
        y = np.cumsum(base[o:o + n]) * np.float32(0.02)
        y = (y - np.convolve(y, np.ones(64, np.float32) / 64, "same")) * rng.uniform(50, 800) + rng.uniform(50, 500) * base[o:o + n][::-1]
        p = os.path.join(d, "noise%03d.wav" % i)
        write_audio(p, np.clip(np.round(y), -32768, 32767).astype(np.int16), wav=True)
        noise.append(p)
    return sig, noise


def run_pool(sig, noise, count, lanes):
    timings = {}
    t0 = time.perf_counter()
    tr.generate_rows(sig, noise, count, lanes=lanes, seed=1, timings=timings)
    wall = time.perf_counter() - t0
    L, F = timings["lanes"], timings["frames"]
    return dict(lanes=L, frames=F, rows=F * L, seconds=wall, rows_per_s=F * L / wall, plan_s=timings["plan"],
                pool_build_s=timings["pool"], trainer_calls_s=timings["trainer"], calls=timings["calls"],
                warmup_share=tr.warmup_share(count, L))


def run_float(sig, noise, count, lanes):
    """The same plan through rnnoise_train_process_host: per call, [T][L][480] float32 gathered on the host."""
    t0 = time.perf_counter()
    p = tr.plan(sig, noise, count, lanes, seed=1)
    t_plan = time.perf_counter() - t0
    tb = tr.TrainingBatch(lanes)
    rows = np.empty((p.n_frames, lanes, tr.TRAIN_ROW), np.float32)
    params = dict(p.randomize)
    t_host = t_call = 0.0
    idx = np.arange(480)
    for f0, f1 in tr.call_bounds(p):
        t = time.perf_counter()
        pool, sa, na = tr.build_pool(p, f0, f1)
        s = pool[sa[..., None] + idx].astype(np.float32)
        n = pool[na[..., None] + idx].astype(np.float32)
        t_host += time.perf_counter() - t
        if f0 in params:
            tb.set_params(params[f0])
        t = time.perf_counter()
        rows[f0:f1] = tb.process_host(s, n)
        t_call += time.perf_counter() - t
    wall = time.perf_counter() - t0
    return dict(lanes=lanes, rows=p.n_frames * lanes, seconds=wall, rows_per_s=p.n_frames * lanes / wall, plan_s=t_plan,
                host_assembly_s=t_host, trainer_calls_s=t_call), rows


def oracle_rate(sig, noise, frames=3000):
    import oracle
    from nnnoiseless_b200.files import read_audio
    s = read_audio(sig[0])[0][:frames * 480, 0].reshape(-1, 480)
    n = read_audio(noise[0])[0][:frames * 480, 0].reshape(-1, 480)
    t = oracle.Trainer()
    t0 = time.perf_counter()
    for f in range(len(s)):
        t.frame(s[f], n[f])
    return len(s) / (time.perf_counter() - t0)


def profile(sig, noise, count, lanes, n_calls=4):
    """Kernel and copy times over the first n_calls calls of the pool path and of the float path, same L."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    p = tr.plan(sig, noise, count, lanes, seed=1)
    calls = tr.call_bounds(p)[:n_calls]
    pools = [tr.build_pool(p, *c) for c in calls]
    idx = np.arange(480)
    floats = [(pool[sa[..., None] + idx].astype(np.float32), pool[na[..., None] + idx].astype(np.float32)) for pool, sa, na in pools]
    out = {}
    for name in ("pool", "float"):
        tb = tr.TrainingBatch(lanes)
        for k in range(2):  # warm-up: module load, staging growth
            (tb.process_pool_host(*pools[k]) if name == "pool" else tb.process_host(*floats[k]))
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(len(calls)):
                (tb.process_pool_host(*pools[k]) if name == "pool" else tb.process_host(*floats[k]))
            torch.cuda.synchronize()
        front = kernels = copies = 0.0
        n_front = 0
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = e.device_time if hasattr(e, "device_time") else e.cuda_time
            if "memcpy" in e.name.lower() or "memset" in e.name.lower():
                copies += us
            else:
                kernels += us
                if "train_front_kernel" in e.name:
                    front += us
                    n_front += 1
        frames = sum(c[1] - c[0] for c in calls)
        out[name] = dict(frames=frames, front_kernel_us_per_frame=front / max(n_front, 1), kernels_us_per_frame=kernels / frames,
                         copies_us_per_frame=copies / frames)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=200)
    ap.add_argument("--seconds", type=int, default=60)
    ap.add_argument("--count", type=int, default=2_000_000)
    ap.add_argument("--wide", type=int, default=4096)
    ap.add_argument("--out", help="also write the result to this JSON file")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("corpus_bench: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = dict(gpu=gpu, files=a.files, seconds=a.seconds, count=a.count)
    with tempfile.TemporaryDirectory() as d:
        t = time.perf_counter()
        sig, noise = write_corpus(d, a.files, a.seconds)
        res["corpus_write_s"] = time.perf_counter() - t
        L0 = tr.default_lanes(a.count)
        run_pool(sig, noise, 20 * L0 * 100, L0)  # warm-up: module load, page cache
        for L in (L0, a.wide):
            res["pool_L%d" % L] = run_pool(sig, noise, a.count, L)
            res["float_L%d" % L], _ = run_float(sig, noise, a.count, L)
            print(json.dumps({k: res[k] for k in ("pool_L%d" % L, "float_L%d" % L)}), flush=True)
        res["oracle_rows_per_s"] = oracle_rate(sig, noise)
        res["profile_L%d" % a.wide] = profile(sig, noise, a.count, a.wide)
        res["profile_L%d" % L0] = profile(sig, noise, a.count, L0, n_calls=2)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
