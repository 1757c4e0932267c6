"""Cost of streams at their own sample rate (DESIGN.md 7g) at B = 65,536 streams.

    python tools/resample_bench.py [--streams 65536] [--frames 10] [--reps 20] [--launches 200]

Cases: every stream at 16 kHz, at 8 kHz, at 44.1 kHz, and the rates mixed (8, 12, 16, 24, 32, 44.1, 48 kHz).  For each
case it reports
  up_ms, down_ms   one launch of the up / down kernel over one frame of every stream (CUDA events over --launches launches);
  *_gbs, *_hbm     the bytes each kernel must move (samples in and out, the history read and written), per second, and
                   as a share of the 3.35 TB/s HBM3 bound of the H100 SXM data sheet;
  native_step_ms   a frame-step of rnnoise_batch_process_native_device (float, calls of --frames frames);
  step_ms          a frame-step of rnnoise_batch_process_device on the same batch size (48 kHz frames);
the two step times alternated in one run, median over --reps calls each.  Prints one JSON line per case, after one with
the card's name, power limit and clocks."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
MIXED = (8000, 12000, 16000, 24000, 32000, 44100, 48000)


def query(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    import torch
    import nnnoiseless_b200 as nb

    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("resample_bench needs a CUDA device")
    B, T = a.streams, a.frames
    dev = torch.device("cuda", 0)
    sp = torch.cuda.current_stream().cuda_stream
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), power_limit=query("power.limit"),
                          clocks=query("clocks.max.sm,clocks.max.mem"), streams=B, frames_per_call=T)), flush=True)
    g = torch.Generator(device=dev).manual_seed(7)
    x = (torch.randn((B, T, 480), generator=g, device=dev) * 3000.0).contiguous()  # native slots [B][T][480]
    x48 = (torch.randn((T, B, 480), generator=g, device=dev) * 3000.0).contiguous()
    out = torch.empty_like(x)
    out48 = torch.empty_like(x48)
    vad = torch.empty((T, B), device=dev)

    def events_ms(fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    cases = [("16k", np.full(B, 16000)), ("8k", np.full(B, 8000)), ("44.1k", np.full(B, 44100)),
             ("mixed", np.random.default_rng(0).choice(MIXED, B))]
    batch = nb.DenoiseBatch(B, device=0)
    for name, rates in cases:
        rates = rates.astype(np.int32)
        rs = nb.Resampler(B, rates, device=0)
        nin = rates.astype(np.int64) // 100

        def up():
            rs.up_device(out48.data_ptr(), x.data_ptr(), 1, T * 480, 480, cuda_stream=sp)

        def down():
            rs.down_device(out.data_ptr(), x48.data_ptr(), 1, T * 480, 480, cuda_stream=sp)

        up(), down()
        up_ms, down_ms = events_ms(up, a.launches), events_ms(down, a.launches)
        up_bytes = int((4 * nin + 4 * 480 + 2 * 4 * 20).sum())      # native in, 48 kHz out, history read + written
        down_bytes = int((4 * 480 + 4 * nin + 2 * 4 * 120).sum())   # 48 kHz in, native out, history read + written

        def native():
            batch.process_native_device(rs, out.data_ptr(), x.data_ptr(), vad.data_ptr(), T, T * 480, 480, cuda_stream=sp)

        def plain():
            batch.process_device(out48.data_ptr(), x48.data_ptr(), vad.data_ptr(), T, 480, B * 480, cuda_stream=sp)

        native(), plain()
        nat, pla = [], []
        for _ in range(a.reps):
            nat.append(events_ms(native, 1) / T)
            pla.append(events_ms(plain, 1) / T)
        n_ms, p_ms = float(np.median(nat)), float(np.median(pla))
        print(json.dumps(dict(case=name, up_ms=round(up_ms, 4), down_ms=round(down_ms, 4),
                              up_gbs=round(up_bytes / up_ms / 1e6, 1), up_hbm=round(up_bytes / (up_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                              down_gbs=round(down_bytes / down_ms / 1e6, 1),
                              down_hbm=round(down_bytes / (down_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                              native_step_ms=round(n_ms, 4), step_ms=round(p_ms, 4), overhead=round(n_ms / p_ms - 1.0, 4))), flush=True)
        del rs
        torch.cuda.synchronize()


if __name__ == "__main__":
    main()
