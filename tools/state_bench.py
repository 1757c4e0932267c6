"""Time per-stream state export and import (rnnoise_batch_get_states / set_states into and out of a device buffer) at
B = 65,536 streams, against a device-to-device copy of the same number of bytes, with CUDA events.

    python tools/state_bench.py [--streams 65536] [--iters 20] [--warmup 3]

Prints one JSON line: the card's name and power limit, and for each operation its time per call, its rate in GB/s of
record bytes (n_streams x state_bytes) and that rate over the copy's.  set_states includes the validation of every
record: a check kernel, then the host waits for the index of the first bad record."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    import torch
    import nnnoiseless_b200 as nb
    from nnnoiseless_b200.synth import synth_streams

    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("state_bench needs a CUDA device")
    B = a.streams
    batch = nb.DenoiseBatch(B, device=0)
    x = torch.from_numpy(synth_streams(64, 2, seed=9).reshape(64, 2, 480).transpose(1, 0, 2).copy()).cuda()
    x = x.repeat(1, B // 64 + 1, 1)[:, :B].contiguous()  # two frames, so that the records hold live state
    out = torch.empty_like(x)
    s = torch.cuda.current_stream()
    batch.process_device(out.data_ptr(), x.data_ptr(), 0, 2, 480, B * 480, s.cuda_stream)
    nbytes = B * batch.state_bytes
    rec = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dup = torch.empty_like(rec)
    ops = {
        "get_states": lambda: batch.get_states_device(rec.data_ptr(), None, s.cuda_stream),
        "set_states": lambda: batch.set_states_device(rec.data_ptr(), None, s.cuda_stream),
        "d2d_copy": lambda: dup.copy_(rec),
    }
    res = {}
    for name, fn in ops.items():
        for _ in range(a.warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(s)
        for _ in range(a.iters):
            fn()
        e1.record(s)
        e1.synchronize()
        ms = e0.elapsed_time(e1) / a.iters
        res[name] = dict(ms=round(ms, 4), gb_s=round(nbytes / ms / 1e6, 1))
    for name in ops:
        res[name]["vs_copy"] = round(res[name]["gb_s"] / res["d2d_copy"]["gb_s"], 3)
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), streams=B,
                          state_bytes=batch.state_bytes, record_bytes_total=nbytes, **res)))


if __name__ == "__main__":
    main()
