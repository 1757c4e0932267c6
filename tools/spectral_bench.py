"""Time the streaming kernels of a frame-step -- analysis, synthesis and the high-pass filter -- each alone, at
B = 65,536 streams, against a device-to-device copy, with CUDA events.

    python tools/spectral_bench.py [--streams 65536] [--frames 100] [--warmup 10]

Every frame runs the five kernels serialised on one stream with an event between each two (rnnoise_batch_profile_step),
so each kernel runs alone on the GPU; a kernel's time is the mean over the timed frames.  Bytes come from shapes: the
synthesis and high-pass kernels' own bytes per stream-frame are bench.py's KERNEL_BYTES; for analysis the two windows are
counted as their union input_mem[768 - pitch, 1728) with each stream's actual pitch of that frame.  The copy moves the
analysis kernel's bytes of one frame; its rate counts bytes read plus bytes written (what the HBM serves), and each
kernel's rate is given as a fraction of it.  Prints one JSON line with the card's name, power limit and SM clock."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import KERNEL_BYTES, ClockSampler, synth_on_device  # noqa: E402

ANALYSIS_FIXED = KERNEL_BYTES["analysis"] - 2 * 960 * 4  # everything but the two history windows


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
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("spectral_bench needs a CUDA device")
    B = a.streams
    dev = torch.device("cuda", 0)
    Tin = 16  # distinct input frames, used cyclically
    x = synth_on_device(torch, B, Tin, dev, seed=1234)
    out = torch.empty_like(x)
    vad = torch.empty(Tin, B, device=dev)
    batch = nb.DenoiseBatch(B, device=0)
    sp = torch.cuda.current_stream().cuda_stream

    def frame(t):
        k = t % Tin
        return batch.profile_step(out[k].data_ptr(), x[k].data_ptr(), vad[k].data_ptr(), 480, sp)

    for t in range(a.warmup):
        frame(t)
    names = ("analysis", "synthesis", "hp_filter")
    ms = {k: [] for k in names}
    abytes = []
    sampler = ClockSampler(0)
    sampler.start()
    for t in range(a.warmup, a.warmup + a.frames):
        d = frame(t)
        for k in names:
            ms[k].append(d[k])
        p = batch.taps()["pitch"].astype(np.int64)
        abytes.append(int(ANALYSIS_FIXED * B + 4 * (960 + p).sum()))
    clocks = sampler.stop()

    # device-to-device copy of the analysis kernel's bytes of one frame
    nbytes = int(np.mean(abytes)) // 16 * 16
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = 20
    e0.record()
    for _ in range(iters):
        dst.copy_(src)
    e1.record()
    e1.synchronize()
    copy_ms = e0.elapsed_time(e1) / iters
    copy_gbs = 2 * nbytes / (copy_ms * 1e-3) / 1e9  # read + written

    res = {}
    for k in names:
        t = float(np.mean(ms[k]))
        by = float(np.mean(abytes)) if k == "analysis" else float(KERNEL_BYTES[k] * B)
        gbs = by / (t * 1e-3) / 1e9
        res[k] = dict(ms=round(t, 4), ms_spread=round(float(np.max(ms[k]) - np.min(ms[k])), 4),
                      bytes_per_stream_frame=round(by / B, 1), gb_s=round(gbs, 1), frac_of_copy=round(gbs / copy_gbs, 3))
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), power_limit=query("power.limit"),
                          sm_clock_mhz_median=clocks.get("sm_mhz"), sm_clock_max_mhz=clocks.get("sm_max_mhz"),
                          clock_reasons=clocks.get("reasons"), streams=B, frames=a.frames,
                          lib=os.environ.get("NNB_LIB", "default"),
                          copy=dict(bytes=nbytes, ms=round(copy_ms, 4), gb_s_read_plus_write=round(copy_gbs, 1)), **res)))


if __name__ == "__main__":
    main()
