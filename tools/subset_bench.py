"""Time subset calls (rnnoise_batch_process_streams_device) at B = 65,536 streams against a full-batch call and against the
records workaround (get_states of the idle streams, a full-batch call, set_states back), with CUDA events.

    python tools/subset_bench.py [--streams 65536] [--iters 10] [--warmup 3]

Prints one JSON line: the card's name and power limit, and for every (n, n_frames) the milliseconds of one subset call,
of one full-batch call and of the workaround.  The gather and scatter kernels are timed alone with torch.profiler; their
rate counts the bytes each copies per stream (gather 8,396, scatter 10,316 for the built-in model) and is set against a
device-to-device copy of the same number of bytes."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from state_bench import power_limit  # noqa: E402

GATHER_BYTES, SCATTER_BYTES = 8396, 10316  # built-in model, per stream


def timed(fn, iters, warmup, s):
    import torch
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(s)
    for _ in range(iters):
        fn()
    e1.record(s)
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_ms(fn, names, iters):
    """Mean device time of the kernels whose names contain each of `names`, over `iters` calls of fn."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for n in names:
        tot, cnt = 0.0, 0
        for e in prof.key_averages():
            if n in e.key:
                tot += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                cnt += e.count
        out[n] = tot / 1000.0 / cnt if cnt else None
    return out


def main():
    import numpy as np
    import torch
    import nnnoiseless_b200 as nb
    from nnnoiseless_b200.synth import synth_streams

    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--subsets", default="1024,8192,32768,65536")
    ap.add_argument("--frames", default="1,10")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("subset_bench needs a CUDA device")
    B = a.streams
    Ts = [int(t) for t in a.frames.split(",")]
    batch = nb.DenoiseBatch(B, device=0)
    s = torch.cuda.current_stream()
    cs = s.cuda_stream
    base = torch.from_numpy(synth_streams(64, max(Ts), seed=9).reshape(64, max(Ts), 480).transpose(1, 0, 2).copy()).cuda()
    x = base.repeat(1, B // 64 + 1, 1)[:, :B].contiguous()  # [T][B][480]
    out = torch.empty_like(x)
    vad = torch.empty(max(Ts), B, device="cuda")
    batch.process_device(out.data_ptr(), x.data_ptr(), vad.data_ptr(), 2, 480, B * 480, cs)
    rec = torch.empty((B, batch.state_bytes), dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(0)
    res = {}
    full_ms = {T: timed(lambda: batch.process_device(out.data_ptr(), x.data_ptr(), vad.data_ptr(), T, 480, B * 480, cs),
                        a.iters, a.warmup, s) for T in Ts}
    for n in [int(v) for v in a.subsets.split(",")]:
        S = np.sort(rng.choice(B, n, replace=False)).astype(np.int32)
        rng.shuffle(S)
        idle = np.setdiff1d(np.arange(B), S).astype(np.int32)
        copy_src = torch.empty(n * SCATTER_BYTES, dtype=torch.uint8, device="cuda")
        copy_dst = torch.empty_like(copy_src)
        for T in Ts:
            def subset():
                batch.process_streams_device(S, out.data_ptr(), x.data_ptr(), vad.data_ptr(), T, 480, n * 480, cuda_stream=cs)

            def workaround():
                if len(idle):
                    batch.get_states_device(rec.data_ptr(), idle, cs)
                batch.process_device(out.data_ptr(), x.data_ptr(), vad.data_ptr(), T, 480, B * 480, cs)
                if len(idle):
                    batch.set_states_device(rec.data_ptr(), idle, cs)

            r = dict(subset_ms=round(timed(subset, a.iters, a.warmup, s), 4), full_ms=round(full_ms[T], 4),
                     workaround_ms=round(timed(workaround, a.iters, a.warmup, s), 4))
            if T == Ts[0]:
                k = kernel_ms(subset, ["subset_gather_kernel", "subset_scatter_kernel"], a.iters)
                g, sc = k["subset_gather_kernel"], k["subset_scatter_kernel"]
                cg = timed(lambda: copy_dst[:n * GATHER_BYTES].copy_(copy_src[:n * GATHER_BYTES]), a.iters, a.warmup, s)
                csc = timed(lambda: copy_dst.copy_(copy_src), a.iters, a.warmup, s)
                r.update(gather_ms=round(g, 4), gather_gb_s=round(n * GATHER_BYTES / g / 1e6, 1),
                         scatter_ms=round(sc, 4), scatter_gb_s=round(n * SCATTER_BYTES / sc / 1e6, 1),
                         d2d_copy_gb_s=round(n * GATHER_BYTES / cg / 1e6, 1), d2d_copy_scatter_bytes_gb_s=round(n * SCATTER_BYTES / csc / 1e6, 1))
            res["n%d_T%d" % (n, T)] = r
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), streams=B, **res)))


if __name__ == "__main__":
    main()
