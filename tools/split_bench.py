"""Cost of split frames (DESIGN.md 7h) at B = 65,536 streams.

    python tools/split_bench.py [--streams 65536] [--chunk 4] [--reps 10] [--frames 40]

Three times per frame, each the median over --reps calls of --frames frames (CUDA events on one torch stream), the three
cases alternated in one run:
  fused_ms    rnnoise_batch_process_device, calls of --chunk frames;
  split_ms    analyze --chunk frames, synthesize them with constant gains: the cost of the split itself;
  network_ms  the same with a float32 torch network of the built-in model's geometry (dense 42->24, GRUs 24, 48, 96,
              dense 96->22) between the calls.
Prints one JSON line, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    from nnnoiseless_b200.synth import synth_streams

    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--chunk", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=40)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("split_bench: no CUDA device")
    B, T, K = a.streams, a.frames, a.chunk
    x = torch.from_numpy(synth_streams(256, T, seed=3).reshape(256, T, 480).transpose(1, 0, 2).copy()).cuda()
    x = x.repeat(1, (B + 255) // 256, 1)[:, :B].contiguous()  # [T][B][480]
    out = torch.empty_like(x)
    feats = torch.empty((T, B, 42), device="cuda")
    sil = torch.empty((T, B), dtype=torch.int32, device="cuda")
    gains = torch.full((T, B, 22), 0.5, device="cuda")

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.dense = torch.nn.Linear(42, 24)
            self.vad = torch.nn.GRUCell(24, 24)
            self.noise = torch.nn.GRUCell(24 + 24 + 42, 48)
            self.den = torch.nn.GRUCell(24 + 48 + 42, 96)
            self.out = torch.nn.Linear(96, 22)

        def forward(self, f, h):
            hv, hn, hd = h
            d = torch.tanh(self.dense(f))
            hv = self.vad(d, hv)
            hn = self.noise(torch.cat([d, hv, f], 1), hn)
            hd = self.den(torch.cat([hv, hn, f], 1), hd)
            return torch.sigmoid(self.out(hd)), (hv, hn, hd)

    net = Net().cuda().eval()
    st = torch.cuda.Stream()
    cs = st.cuda_stream
    batches = {k: nb.DenoiseBatch(B, device=0) for k in ("fused", "split", "network")}

    def fused(b):
        for t0 in range(0, T, K):
            b.process_device(out[t0].data_ptr(), x[t0].data_ptr(), 0, min(K, T - t0), 480, B * 480, cs)

    def split(b, with_net):
        h = tuple(torch.zeros((B, n), device="cuda") for n in (24, 48, 96))
        for t0 in range(0, T, K):
            k = min(K, T - t0)
            b.analyze_device(x[t0].data_ptr(), feats[t0].data_ptr(), sil[t0].data_ptr(), k, 480, B * 480, 42, B * 42, cuda_stream=cs)
            if with_net:
                for t in range(t0, t0 + k):
                    g, h = net(feats[t], h)
                    gains[t] = g
            b.synthesize_device(out[t0].data_ptr(), gains[t0].data_ptr(), k, 480, B * 480, 22, B * 22, cuda_stream=cs)

    cases = {"fused": lambda: fused(batches["fused"]), "split": lambda: split(batches["split"], False),
             "network": lambda: split(batches["network"], True)}
    times = {k: [] for k in cases}
    with torch.no_grad(), torch.cuda.stream(st):
        for fn in cases.values():  # warm-up: module loads, cuBLAS algorithm choice
            fn()
        st.synchronize()
        for _ in range(a.reps):
            for name, fn in cases.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                fn()
                e1.record(st)
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) / T)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    print(json.dumps(dict(gpu=query("name"), power_limit=query("power.limit"), streams=B, chunk=K, frames=T, reps=a.reps,
                          fused_ms=round(med["fused"], 4), split_ms=round(med["split"], 4), network_ms=round(med["network"], 4),
                          spread={k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()})))


if __name__ == "__main__":
    main()
