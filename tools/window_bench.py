"""Times window frames (DESIGN.md 7j) against split frames with CUDA events, in ms per frame of analysis + synthesis:

    split    analyze_device + synthesize_device in chunks of 4
    saving   analyze_device + synthesize_saving_device in chunks of 4 (the records of training through synthesis)
    window   analyze_window_device of the whole window, then synthesize_window_device of it (the same records)

The three cases alternate within every repetition; each prints its median and its spread (min, max).  Then one
training step (forward, synthesis_grad, backward, Adam) of a GRU network over whole windows against the same network
stepped in chunks of 4 with its state carried across chunks by hand.

    python tools/window_bench.py [--sizes 65536x4,4096x100] [--reps 7] [--train 256x64]

Prints one JSON line per size, with the card's name and power limit.  Needs a GPU; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nnnoiseless_b200 as nb  # noqa: E402
from nnnoiseless_b200.synth import synth_streams  # noqa: E402

F, NBF, NBB, CB = 480, 42, 22, nb.SYNTH_CONTEXT_BYTES


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_properties(0).name


def stats(ms):
    return dict(median=round(float(np.median(ms)), 4), min=round(float(np.min(ms)), 4), max=round(float(np.max(ms)), 4))


def signal(B, T):
    x = synth_streams(min(B, 256), T, seed=1).reshape(-1, T, F)
    x = np.tile(x, ((B + x.shape[0] - 1) // x.shape[0], 1, 1))[:B]
    return torch.from_numpy(np.ascontiguousarray(x.transpose(1, 0, 2))).cuda()  # [T][B][480]


def frames(B, T, reps):
    x = signal(B, T)
    b = nb.DenoiseBatch(B)
    feats = torch.empty((T, B, NBF), device="cuda")
    gains = torch.rand((T, B, NBB), device="cuda")
    out = torch.empty_like(x)
    ctx = torch.empty((B, T, CB), dtype=torch.uint8, device="cuda")
    cs = torch.cuda.current_stream().cuda_stream

    def case(name):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        if name == "window":
            b.analyze_window_device(x.data_ptr(), feats.data_ptr(), 0, T, F, B * F, NBF, B * NBF, ctx.data_ptr(), T, 1, cuda_stream=cs)
            b.synthesize_window_device(out.data_ptr(), gains.data_ptr(), T, F, B * F, NBB, B * NBB, ctx.data_ptr(), T, 1, cuda_stream=cs)
        else:
            for t0 in range(0, T, 4):
                k = min(4, T - t0)
                b.analyze_device(x[t0].data_ptr(), feats[t0].data_ptr(), 0, k, F, B * F, NBF, B * NBF, cuda_stream=cs)
                if name == "saving":
                    b.synthesize_saving_device(out[t0].data_ptr(), gains[t0].data_ptr(), k, F, B * F, NBB, B * NBB, ctx[:, t0].data_ptr(), T,
                                               1, cuda_stream=cs)
                else:
                    b.synthesize_device(out[t0].data_ptr(), gains[t0].data_ptr(), k, F, B * F, NBB, B * NBB, cuda_stream=cs)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / T

    names = ("split", "saving", "window")
    for n in names:  # warm-up
        case(n)
    ms = {n: [] for n in names}
    for _ in range(reps):
        for n in names:
            ms[n].append(case(n))
    r = {n + "_ms_per_frame": stats(v) for n, v in ms.items()}
    sp, sa, wi = (float(np.median(ms[n])) for n in names)
    r.update(window_over_split=round(wi / sp, 4), saving_minus_window_ms_per_frame=round(sa - wi, 4))
    return r


def training(B, T, reps):
    """ms per training step: a 1-layer GRU (42 -> 64) and a linear layer to the gains, over whole windows or in chunks of 4."""
    from nnnoiseless_b200.autograd import synthesis_grad
    torch.manual_seed(0)
    gru, lin = torch.nn.GRU(NBF, 64, batch_first=True).cuda(), torch.nn.Linear(64, NBB).cuda()
    opt = torch.optim.Adam(list(gru.parameters()) + list(lin.parameters()), lr=1e-3)
    x = signal(B, T)
    clean = x.transpose(0, 1).contiguous() * 0.5
    b = nb.DenoiseBatch(B)
    feats = torch.empty((T, B, NBF), device="cuda")
    out = torch.empty((B, T, F), device="cuda")
    ctx = torch.empty((B, T, CB), dtype=torch.uint8, device="cuda")

    def step(whole):
        b.reset()
        opt.zero_grad()
        if whole:
            b.analyze_window_device(x.data_ptr(), feats.data_ptr(), 0, T, F, B * F, NBF, B * NBF, ctx.data_ptr(), T, 1)
            h, _ = gru(feats.transpose(0, 1) / 10.0)
            g = torch.sigmoid(lin(h))
            gd = g.detach().contiguous()
            b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1)
        else:
            chunks, hn = [], None
            for t0 in range(0, T, 4):
                k = min(4, T - t0)
                b.analyze_device(x[t0].data_ptr(), feats[t0].data_ptr(), 0, k, F, B * F, NBF, B * NBF)
                h, hn = gru(feats[t0:t0 + k].transpose(0, 1) / 10.0, hn)
                gk = torch.sigmoid(lin(h))
                gd = gk.detach().contiguous()
                b.synthesize_saving_device(out[:, t0].data_ptr(), gd.data_ptr(), k, T * F, F, k * NBB, NBB, ctx[:, t0].data_ptr(), T, 1)
                chunks.append(gk)
            g = torch.cat(chunks, 1)
        y = synthesis_grad(g, out, ctx)
        ((y[:, 1:] - clean[:, :-1]) / 32768.0).pow(2).mean().backward()
        opt.step()

    def timed(whole):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        step(whole)
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1])

    for w in (False, True):
        timed(w)
    ms = {"chunked": [], "whole": []}
    for _ in range(reps):
        ms["chunked"].append(timed(False))
        ms["whole"].append(timed(True))
    return dict(train_B=B, train_T=T, chunked_step_ms=stats(ms["chunked"]), whole_window_step_ms=stats(ms["whole"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="65536x4,4096x100")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--train", default="256x64")
    a = ap.parse_args()
    dev = card()
    for sz in a.sizes.split(","):
        B, T = (int(v) for v in sz.split("x"))
        r = dict(B=B, T=T, **frames(B, T, a.reps), device=dev)
        print(json.dumps(r), flush=True)
    if a.train:
        B, T = (int(v) for v in a.train.split("x"))
        print(json.dumps(dict(**training(B, T, a.reps), device=dev)), flush=True)


if __name__ == "__main__":
    main()
