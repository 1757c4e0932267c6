"""Times the STOI / ESTOI backward, rnnoise_intelligibility_backward_device (DESIGN.md 7r), beside the forward on the
same pairs, and a training step through synthesis with and without an ESTOI term:

    forward   rnnoise_intelligibility_device (CUDA events, median of --reps), ns per 48 kHz stream-frame
    backward  rnnoise_intelligibility_backward_device after it (CUDA events), ns per stream-frame
    kernels   each of the four backward kernels (torch.profiler in a run of its own, median of --reps)
    train     one step of DenoiseNetwork -> synthesize_window -> synthesis_grad -> loss -> backward -> Adam at L lanes
              and T frames (CUDA events), with loss = waveform MSE and with loss = MSE + lam (1 - ESTOI)

    python tools/intelligibility_grad_bench.py [--pairs 1024,16384] [--window 300] [--lanes 256] [--train-window 64]
                                               [--reps 5] [--out FILE]

The signals are tools/intelligibility_bench.py's.  Prints one JSON line per size with the card's name and power limit.
Needs a GPU; writes its corpus to a temporary directory and nothing else (the JSON also goes to --out if given)."""
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
from intelligibility_bench import signals  # noqa: E402
from metrics_bench import make_corpus, query, timed  # noqa: E402

F = 480
KERNELS = ("stoi_score_bwd_kernel", "stoi_bands_bwd_kernel", "stoi_ola_bwd_kernel", "stoi_resample_bwd_kernel")


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
    fb = nb.intelligibility_workspace_bytes(B, n, 48000)
    bb = nb.intelligibility_backward_workspace_bytes(B, n, 48000)
    fws = torch.empty(fb, dtype=torch.uint8, device="cuda")
    bws = torch.empty(bb, dtype=torch.uint8, device="cuda")
    res = torch.empty(B * 32, dtype=torch.uint8, device="cuda")
    gs, ge = torch.full((B,), 1.0 / B, dtype=torch.float64, device="cuda"), torch.full((B,), 1.0 / B, dtype=torch.float64, device="cuda")
    g = torch.empty((B, n), device="cuda")
    cs = torch.cuda.current_stream().cuda_stream
    fwd = lambda: nb.intelligibility_device(out.data_ptr(), clean.data_ptr(), B, n, n, 48000, res.data_ptr(), fws.data_ptr(), fb,  # noqa: E731
                                            cuda_stream=cs)
    bwd = lambda: nb.intelligibility_backward_device(B, n, 48000, res.data_ptr(), fws.data_ptr(), fb, gs.data_ptr(), ge.data_ptr(),  # noqa: E731
                                                     g.data_ptr(), n, bws.data_ptr(), bb, cuda_stream=cs)
    ms_f = timed(fwd, reps)
    ms_b = timed(bwd, reps)
    per = kernel_ms(bwd, reps)
    sf = B * T
    r = dict(pairs=B, window=T, backward_workspace_mb=bb / 1e6, forward_ms=ms_f, backward_ms=ms_b,
             forward_ns_per_stream_frame=1e6 * ms_f / sf, backward_ns_per_stream_frame=1e6 * ms_b / sf, backward_over_forward=ms_b / ms_f,
             kernels_ns_per_stream_frame={k: (None if v is None else 1e6 * v / sf) for k, v in per.items()},
             finite_gradient=bool(torch.isfinite(g).all()))
    del out, clean, fws, bws, g
    torch.cuda.empty_cache()
    return r


def bench_train(sig, noise, L, T, reps, lam=0.1):
    from nnnoiseless_b200 import training as tr
    from nnnoiseless_b200.autograd import DenoiseNetwork, intelligibility, synthesis_grad
    wc = tr.WaveformCorpus(sig, noise, L)
    wc.start(L * T, seed=3)
    noisy, clean = torch.empty((L, T, F), device="cuda"), torch.empty((L, T, F), device="cuda")
    wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F)
    net = DenoiseNetwork.from_model(None, L, T)
    opt = torch.optim.Adam([net.params], lr=1e-4)
    b = nb.DenoiseBatch(L, device=0)
    feats = torch.empty((L, T, 42), device="cuda")
    sil = torch.empty((T, L), dtype=torch.int32, device="cuda")
    out = torch.empty((L, T, F), device="cuda")
    ctx = torch.empty((L, T, nb.SYNTH_CONTEXT_BYTES), dtype=torch.uint8, device="cuda")
    r = dict(lanes=L, train_window=T, lam=lam)
    for with_estoi in (False, True):
        def step():
            opt.zero_grad()
            b.analyze_window_device(noisy.data_ptr(), feats.data_ptr(), sil.data_ptr(), T, T * F, F, T * 42, 42, ctx.data_ptr(), T, 1)
            gains, _, _ = net(feats, sil)
            b.synthesize_window_device(out.data_ptr(), gains.detach().contiguous().data_ptr(), T, T * F, F, T * 22, 22, ctx.data_ptr(), T, 1)
            y = synthesis_grad(gains, out, ctx)
            loss = ((y[:, 1:] - clean[:, :-1]) * (1.0 / 32768.0)).pow(2).mean()
            if with_estoi:
                _, e = intelligibility(y[:, 1:].reshape(L, -1), clean[:, :-1].reshape(L, -1))
                loss = loss + lam * (1 - e.nanmean())
            loss.backward()
            opt.step()
            net.clip_()
        r["step_ms_estoi" if with_estoi else "step_ms"] = timed(step, reps)
    r["estoi_share_of_step"] = 1.0 - r["step_ms"] / r["step_ms_estoi"]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1024,16384")
    ap.add_argument("--window", type=int, default=300)
    ap.add_argument("--lanes", type=int, default=256)
    ap.add_argument("--train-window", type=int, default=64)
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
        lines.append(dict(head, **bench_train(sig, noise, a.lanes, a.train_window, a.reps)))
        print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
