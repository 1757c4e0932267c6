"""Times waveform windows from the training simulators (DESIGN.md 7k) at sizes (L lanes, T frames per window):

    kernel    train_wave_kernel alone (torch.profiler, one window per launch)
    call      the device time of WaveformCorpus.next (CUDA events: the offsets' upload and the kernel)
    host      the host time of WaveformCorpus.next with a stream given (it returns without waiting)
    upload    WaveformCorpus's upload rate of a synthetic corpus (memory-mapped WAV files -> the device pool)

Then one training step of the 7j network (42 -> 64 nn.GRU + linear: analyze_window -> net -> synthesize_window ->
synthesis_grad -> Adam) three ways, alternated within each repetition:

    pre       on windows generated beforehand
    same      WaveformCorpus.next on the step's stream, then the step
    side      next for window k + 1 on a side stream while step k runs

    python tools/waveform_bench.py [--sizes 256x64,4096x100] [--reps 7] [--out FILE]

Prints one JSON line per size with the card's name and power limit.  Needs a GPU; writes its corpus to a temporary
directory and nothing else (the JSON also goes to --out if given).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nnnoiseless_b200 as nb  # noqa: E402
from nnnoiseless_b200 import training as tr  # noqa: E402
from nnnoiseless_b200.autograd import synthesis_grad  # noqa: E402
from nnnoiseless_b200.files import write_audio  # noqa: E402

F, NBF, NBB, CB = 480, 42, 22, nb.SYNTH_CONTEXT_BYTES


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_properties(0).name


def stats(ms):
    return dict(median=round(float(np.median(ms)), 4), min=round(float(np.min(ms)), 4), max=round(float(np.max(ms)), 4))


def make_corpus(d, minutes):
    """Speech-like (tones under an on/off envelope) and noise WAV files: `minutes` of each, in 1-minute files."""
    rng = np.random.default_rng(0)
    sig, noise = [], []
    n = 60 * 48000
    t = np.arange(n) / 48000.0
    for i in range(minutes):
        env = np.repeat(rng.choice([0.02, 0.3, 1.0], size=n // 24000 + 1), 24000)[:n]
        x = 3000 * np.sin(2 * np.pi * (150 + 40 * i) * t) * env + rng.normal(0, 200, n)
        p = os.path.join(d, "speech%d.wav" % i)
        write_audio(p, np.clip(np.round(x), -32768, 32767).astype(np.int16), wav=True)
        sig.append(p)
        p = os.path.join(d, "noise%d.wav" % i)
        write_audio(p, np.round(rng.normal(0, 1000, n)).astype(np.int16), wav=True)
        noise.append(p)
    return sig, noise


class Net:
    def __init__(self):
        torch.manual_seed(0)
        self.gru = torch.nn.GRU(NBF, 64, batch_first=True).cuda()
        self.head = torch.nn.Linear(64, NBB).cuda()
        self.opt = torch.optim.Adam(list(self.gru.parameters()) + list(self.head.parameters()), lr=1e-3)


def train_step(b, net, noisy, clean, feats, out, ctx):
    B, T = noisy.shape[0], noisy.shape[1]
    cs = torch.cuda.current_stream().cuda_stream
    b.reset()
    net.opt.zero_grad()
    b.analyze_window_device(noisy.data_ptr(), feats.data_ptr(), 0, T, T * F, F, T * NBF, NBF, ctx.data_ptr(), T, 1, cuda_stream=cs)
    g = torch.sigmoid(net.head(net.gru(feats / 10)[0]))
    gd = g.detach().contiguous()
    b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1, cuda_stream=cs)
    y = synthesis_grad(g, out, ctx)
    loss = ((y[:, 1:] - clean[:, :-1]) / 32768).pow(2).mean()
    loss.backward()
    net.opt.step()


def bench(wc, L, T, reps):
    res = dict(L=L, T=T)
    n_win = 4 * reps + 8
    wc.start(L * T * n_win)
    bufs = [(torch.empty((L, T, F), device="cuda"), torch.empty((L, T, F), device="cuda")) for _ in range(2)]
    cs = torch.cuda.current_stream()

    def nxt(k, stream):
        noisy, clean = bufs[k % 2]
        if wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F, cuda_stream=stream.cuda_stream) != T:
            wc.start(L * T * n_win)
            wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F, cuda_stream=stream.cuda_stream)
        return noisy, clean

    # the call: device time (events) and host time
    for k in range(3):
        nxt(k, cs)
    dev, host = [], []
    for k in range(reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        torch.cuda.synchronize()
        ev[0].record()
        t0 = time.perf_counter()
        nxt(k, cs)
        host.append(1e3 * (time.perf_counter() - t0))
        ev[1].record()
        torch.cuda.synchronize()
        dev.append(ev[0].elapsed_time(ev[1]))
    res["call_ms"], res["host_ms"] = stats(dev), stats(host)
    # the kernel alone
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for k in range(reps):
            nxt(k, cs)
        torch.cuda.synchronize()
    ks = [e.device_time_total / 1e3 for e in prof.events() if "train_wave_kernel" in e.name]
    res["kernel_ms"] = stats(ks) if ks else None
    res["kernel_launches"] = len(ks)
    # the training step three ways
    b = nb.DenoiseBatch(L)
    net = Net()
    feats, out = torch.empty((L, T, NBF), device="cuda"), torch.empty((L, T, F), device="cuda")
    ctx = torch.empty((L, T, CB), dtype=torch.uint8, device="cuda")
    pre = [tuple(x.clone() for x in nxt(k, cs)) for k in range(2)]
    side = torch.cuda.Stream()
    times = {"pre": [], "same": [], "side": []}
    for rep in range(reps + 1):
        for way in times:
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            if way == "pre":
                train_step(b, net, *pre[rep % 2], feats, out, ctx)
            elif way == "same":
                train_step(b, net, *nxt(rep, cs), feats, out, ctx)
            else:
                with torch.cuda.stream(side):
                    side.wait_stream(cs)
                    nxt(rep + 1, side)  # window k + 1 while step k runs on window k
                train_step(b, net, *bufs[rep % 2], feats, out, ctx)
                cs.wait_stream(side)
            ev[1].record()
            torch.cuda.synchronize()
            if rep > 0:
                times[way].append(ev[0].elapsed_time(ev[1]))
    res["step_ms"] = {k: stats(v) for k, v in times.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256x64,4096x100")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--minutes", type=int, default=10, help="minutes of speech and of noise in the synthetic corpus")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    lines = []
    with tempfile.TemporaryDirectory() as d:
        sig, noise = make_corpus(d, a.minutes)
        for size in a.sizes.split(","):
            L, T = (int(v) for v in size.split("x"))
            wc = tr.WaveformCorpus(sig, noise, L)
            r = dict(card=card(), upload_MB_per_s=round(2 * wc.pool_samples / wc.upload_seconds / 1e6, 1),
                     pool_MB=round(2 * wc.pool_samples / 1e6, 1))
            with torch.cuda.stream(torch.cuda.Stream()):  # the default stream's handle is NULL, which makes next() wait
                r.update(bench(wc, L, T, a.reps))
            print(json.dumps(r), flush=True)
            lines.append(r)
            del wc
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
