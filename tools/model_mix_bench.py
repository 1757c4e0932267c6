"""Cost of running the streams of one batch on several models (DESIGN.md 7c), at B = 65,536 streams.

    python tools/model_mix_bench.py [--streams 65536] [--models 1,2,4,16] [--subset 8192] [--frames 40] [--warmup 5]

The built-in model plus K - 1 generated models of its geometry; three assignments: contiguous groups, random, and
round-robin (stream % K, the worst case for grouping).  For each K and assignment it reports
  rnn_ms      the GRU kernel alone (rnnoise_batch_profile_step: serialised, CUDA events), median over --frames frames;
  step_ms     a frame-step of pipelined full-batch device calls (CUDA events around calls of 10 frames);
  subset_ms   a one-frame subset call of --subset random streams;
and, as the workaround without a model table, K batches of B / K streams, each given its share of the subset work,
issued back to back from one thread (workaround_subset_ms).  It also times set_stream_models over every stream.
Prints one JSON line per configuration and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import synth_on_device  # noqa: E402


def query(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def assignment(kind, B, K, rng):
    if kind == "contiguous":
        return (np.arange(B) * K // B).astype(np.int32)
    if kind == "random":
        return rng.integers(0, K, B).astype(np.int32)
    return (np.arange(B) % K).astype(np.int32)


def main():
    import torch
    import nnnoiseless_b200 as nb
    import rnn_ref

    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--models", default="1,2,4,16")
    ap.add_argument("--subset", type=int, default=8192)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("model_mix_bench needs a CUDA device")
    B, n_sub = a.streams, a.subset
    dev = torch.device("cuda", 0)
    Tin = 10
    x = synth_on_device(torch, B, Tin, dev, seed=4321)  # [Tin][B][480]
    out = torch.empty_like(x)
    vad = torch.empty(Tin, B, device=dev)
    sp = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(0)
    gen = [nb.RnnModel.from_bytes(rnn_ref.make_model(24, 24, 48, 96, seed=100 + k)) for k in range(15)]
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), power_limit=query("power.limit"), streams=B,
                          lib=os.environ.get("NNB_LIB", "default"))), flush=True)

    def events_ms(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    for K in (int(k) for k in a.models.split(",")):
        batch = nb.DenoiseBatch(B, device=0)
        for k in range(K - 1):
            batch.add_model(gen[k])
        for kind in ("contiguous", "random", "round_robin"):
            if K == 1 and kind != "contiguous":
                continue
            ids = assignment(kind, B, K, rng)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            batch.set_stream_models(ids)
            torch.cuda.synchronize()
            set_ms = (time.perf_counter() - t0) * 1e3
            rnn = []
            for t in range(a.warmup + a.frames):
                d = batch.profile_step(out[t % Tin].data_ptr(), x[t % Tin].data_ptr(), vad[t % Tin].data_ptr(), 480, sp)
                if t >= a.warmup:
                    rnn.append(d["rnn"])

            def call():
                batch.process_device(out.data_ptr(), x.data_ptr(), vad.data_ptr(), Tin, 480, B * 480, cuda_stream=sp)
            call()
            step_ms = events_ms(call, 3) / Tin
            S = np.sort(rng.choice(B, n_sub, replace=False)).astype(np.int32)
            xs = x[0, :n_sub].contiguous()
            os_ = torch.empty_like(xs)

            def sub():
                batch.process_streams_device(S, os_.data_ptr(), xs.data_ptr(), 0, 1, 480, 480, cuda_stream=sp)
            sub()
            subset_ms = events_ms(sub, 10)
            print(json.dumps(dict(K=K, assignment=kind, rnn_ms=round(float(np.median(rnn)), 4),
                                  rnn_ms_min=round(float(np.min(rnn)), 4), rnn_ms_max=round(float(np.max(rnn)), 4),
                                  step_ms=round(step_ms, 4), subset_ms=round(subset_ms, 4),
                                  set_stream_models_ms=round(set_ms, 3))), flush=True)
        del batch
        torch.cuda.synchronize()
        # the workaround: K batches of B / K streams, each with its share of the subset work, issued from one thread
        if K > 1:
            per = B // K
            batches = [nb.DenoiseBatch(per, gen[k - 1] if k else None, device=0) for k in range(K)]
            share = n_sub // K
            Ss = [np.sort(rng.choice(per, share, replace=False)).astype(np.int32) for _ in range(K)]
            xs = x[0, :share].contiguous()
            os_ = torch.empty_like(xs)

            def tick():
                for b, S in zip(batches, Ss):
                    b.process_streams_device(S, os_.data_ptr(), xs.data_ptr(), 0, 1, 480, 480, cuda_stream=sp)
            tick()
            print(json.dumps(dict(K=K, workaround_subset_ms=round(events_ms(tick, 10), 4))), flush=True)
            del batches
            torch.cuda.synchronize()


if __name__ == "__main__":
    main()
