"""Times rnnoise_intelligibility_device (DESIGN.md 7q) on B pairs of T 48 kHz frames, beside the metrics kernel on the
same windows, and evaluate end to end with and without intelligibility:

    call      the whole call (CUDA events, median of --reps), ms and ns per 48 kHz stream-frame
    kernels   each of the four kernels (torch.profiler in a run of its own, median of --reps), ns per stream-frame
    metrics   Metrics.accumulate_device of the same B streams and T frames (CUDA events), ns per stream-frame
    evaluate  nnnoiseless_b200.evaluate at V = 4 variants and L lanes, seconds with and without intelligibility

    python tools/intelligibility_bench.py [--pairs 1024,16384] [--lanes 256,4096] [--window 300] [--reps 5] [--out FILE]

The clean signals are noise under a syllable-rate envelope with pauses, the outputs the same plus noise, so the silence
rule drops frames as it does on speech.  Prints one JSON line per size with the card's name and power limit.  Needs a
GPU; writes its corpus to a temporary directory and nothing else (the JSON also goes to --out if given)."""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nnnoiseless_b200 as nb  # noqa: E402
from metrics_bench import LIMITS, make_corpus, query, timed  # noqa: E402
from nnnoiseless_b200 import evaluate as ev  # noqa: E402

F = 480
KERNELS = ("stoi_resample_kernel", "stoi_mask_kernel", "stoi_bands_kernel", "stoi_score_kernel")


def signals(B, T, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = T * F
    t = torch.arange(n, device="cuda", dtype=torch.float32) / 48000.0
    phase = torch.rand((B, 1), device="cuda", generator=g) * 6.0
    env = torch.clamp(torch.sin(2 * np.pi * 3.1 * t + phase), min=0.0) ** 2 + 0.01
    clean = 3000.0 * env * torch.randn((B, n), device="cuda", generator=g)
    out = clean + 300.0 * torch.randn((B, n), device="cuda", generator=g)
    return out, clean


def kernel_ms(call, reps):
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    times = {k: [] for k in KERNELS}
    for e in prof.events():
        for k in KERNELS:
            if k in e.name:
                times[k].append(e.time_range.elapsed_us() / 1e3)
    return {k: float(np.median(v)) if v else None for k, v in times.items()}


def bench_call(B, T, reps):
    out, clean = signals(B, T)
    n = T * F
    nbytes = nb.intelligibility_workspace_bytes(B, n, 48000)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    res = torch.empty(B * 32, dtype=torch.uint8, device="cuda")
    cs = torch.cuda.current_stream().cuda_stream
    call = lambda: nb.intelligibility_device(out.data_ptr(), clean.data_ptr(), B, n, n, 48000, res.data_ptr(), ws.data_ptr(),  # noqa: E731
                                             nbytes, cuda_stream=cs)
    ms = timed(call, reps)
    rec = res.cpu().numpy().view(nb.INTELLIGIBILITY_DTYPE)
    m = nb.Metrics(B)
    ms_metrics = timed(lambda: m.accumulate_device(out.data_ptr(), clean.data_ptr(), T, n, F, cuda_stream=cs), reps)
    per = kernel_ms(call, reps)
    sf = B * T
    r = dict(pairs=B, window=T, workspace_mb=nbytes / 1e6, call_ms=ms, call_ns_per_stream_frame=1e6 * ms / sf,
             metrics_ms=ms_metrics, metrics_ns_per_stream_frame=1e6 * ms_metrics / sf,
             kernels_ns_per_stream_frame={k: (None if v is None else 1e6 * v / sf) for k, v in per.items()},
             mean_kept_fraction=float((rec["kept"] / np.maximum(rec["frames"], 1)).mean()), mean_stoi=float(np.nanmean(rec["stoi"])))
    del out, clean, ws
    torch.cuda.empty_cache()
    return r


def bench_evaluate(sig, noise, L, T):
    r = dict(lanes=L, variants=1 + len(LIMITS), window=T)
    for flag in (False, True):
        rep = ev.evaluate(sig, noise, ["builtin"], LIMITS, L, 2 * T, seed=2, window=T, warmup_frames=T, intelligibility=flag)
        r["evaluate_seconds" + ("_intelligibility" if flag else "")] = rep["seconds"]
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1024,16384")
    ap.add_argument("--lanes", default="256,4096")
    ap.add_argument("--window", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    head = dict(device=torch.cuda.get_device_name(0), power_limit=query("power.limit"))
    lines = []
    for B in (int(v) for v in a.pairs.split(",") if v):
        lines.append(dict(head, **bench_call(B, a.window, a.reps)))
        print(json.dumps(lines[-1]), flush=True)
    with tempfile.TemporaryDirectory() as d:
        sig, noise = make_corpus(d)
        for L in (int(v) for v in a.lanes.split(",") if v):
            lines.append(dict(head, **bench_evaluate(sig, noise, L, a.window)))
            print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
