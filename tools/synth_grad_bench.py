"""Times training through synthesis (DESIGN.md 7i) with CUDA events: synthesize_device against
synthesize_saving_device per frame, the backward (its three kernels), and the context bytes per second as a share of a
device-to-device copy of the same bytes.

    python tools/synth_grad_bench.py [--sizes 4096x100,65536x4] [--reps 5]

Prints one JSON line per size.  Needs a GPU; writes nothing.
"""
import argparse
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nnnoiseless_b200 as nb  # noqa: E402
from nnnoiseless_b200.synth import synth_streams  # noqa: E402

F, NBF, NBB, CB = 480, 42, 22, nb.SYNTH_CONTEXT_BYTES


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ms))


def run(B, T, reps):
    x = torch.from_numpy(np.ascontiguousarray(synth_streams(B, 4, seed=1).reshape(B, 4, F).transpose(1, 0, 2))).cuda()
    b = nb.DenoiseBatch(B)
    feats = torch.empty((4, B, NBF), device="cuda")
    gains = torch.rand((B, 4, NBB), device="cuda")
    out = torch.empty((B, 4, F), device="cuda")
    ctx4 = torch.empty((B, 4, CB), dtype=torch.uint8, device="cuda")
    cs = torch.cuda.current_stream().cuda_stream

    def synth(saving):
        b.analyze_device(x.data_ptr(), feats.data_ptr(), 0, 4, F, B * F, NBF, B * NBF, cuda_stream=cs)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        if saving:
            b.synthesize_saving_device(out.data_ptr(), gains.data_ptr(), 4, 4 * F, F, 4 * NBB, NBB, ctx4.data_ptr(), 4, 1, cuda_stream=cs)
        else:
            b.synthesize_device(out.data_ptr(), gains.data_ptr(), 4, 4 * F, F, 4 * NBB, NBB, cuda_stream=cs)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / 4

    for s in (False, True):
        synth(s)
    plain, saving = [], []
    for _ in range(reps):  # alternated
        plain.append(synth(False))
        saving.append(synth(True))
    # the backward over a T-frame window of records (the 4 saved frames repeated: the work does not depend on the values)
    ctx = ctx4.repeat(1, (T + 3) // 4, 1)[:, :T].contiguous()
    go = torch.randn((B, T, F), device="cuda")
    grad = torch.empty((B, T, NBB), device="cuda")
    nbytes = nb.synthesis_backward_workspace_bytes(B, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")

    def bwd():
        nb.synthesis_backward_device(ctx.data_ptr(), T, 1, go.data_ptr(), T * F, F, grad.data_ptr(), T * NBB, NBB, B, T, ws.data_ptr(),
                                     nbytes, cuda_stream=cs)

    bwd()
    bwd_ms = timed(bwd, reps)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        bwd()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        m = re.search(r"(grad_tables_kernel|synthesis_grad_warp_kernel|synthesis_grad_scan_kernel)", e.key)
        if m:
            kern[m.group(1)] = round(e.device_time_total / 1000.0 / e.count, 4)
    # bytes stored per second: the records a saving frame adds, against a device-to-device copy of the same bytes
    dst = torch.empty_like(ctx4)
    copy_ms = timed(lambda: dst.copy_(ctx4), reps)
    extra = float(np.median(saving) - np.median(plain))
    ctx_bytes = B * CB  # per frame
    return dict(B=B, T=T, synth_ms_per_frame=round(float(np.median(plain)), 4), saving_ms_per_frame=round(float(np.median(saving)), 4),
                backward_ms=round(bwd_ms, 3), backward_ms_per_frame=round(bwd_ms / T, 4), backward_kernels_ms=kern,
                ctx_GBps=round(ctx_bytes / max(extra, 1e-6) / 1e6, 1), d2d_copy_GBps=round(4 * ctx_bytes / copy_ms / 1e6, 1),
                ctx_share_of_copy=round((ctx_bytes / max(extra, 1e-6)) / (4 * ctx_bytes / copy_ms), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096x100,65536x4")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    dev = torch.cuda.get_device_properties(0).name
    for sz in a.sizes.split(","):
        B, T = (int(v) for v in sz.split("x"))
        r = run(B, T, a.reps)
        r["device"] = dev
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
