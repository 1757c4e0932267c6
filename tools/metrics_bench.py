"""Times the held-out evaluation (DESIGN.md 7p) at L lanes, V variants (the baseline + the built-in model at three
attenuation limits), T frames per window:

    metrics   Metrics.accumulate_device of V L streams, T frames (CUDA events), and per stream-frame
    analysis  the analysis kernel of one fused frame of V L streams (DenoiseBatch.profile_step), per stream-frame
    steps     the fused process_device of V L streams, T frames (CUDA events)
    next      WaveformCorpus.next of L lanes, T frames (CUDA events)
    evaluate  nnnoiseless_b200.evaluate end to end: lane-frames (per variant) per second

    python tools/metrics_bench.py [--lanes 256,4096] [--window 100] [--reps 5] [--out FILE]

Prints one JSON line per size with the card's name and power limit.  Needs a GPU; writes its corpus to a temporary
directory and nothing else (the JSON also goes to --out if given)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nnnoiseless_b200 as nb  # noqa: E402
from nnnoiseless_b200 import evaluate as ev  # noqa: E402
from nnnoiseless_b200 import training as tr  # noqa: E402
from nnnoiseless_b200.files import write_audio  # noqa: E402
from nnnoiseless_b200.synth import synth_streams  # noqa: E402

F = 480
LIMITS = [np.inf, 12.0, 6.0]


def query(field):
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + field, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def make_corpus(d, seconds=60):
    rng = np.random.default_rng(5)
    sig, noise = [], []
    for i in range(4):
        n = seconds * 100
        x = synth_streams(1, n, seed=10 + i)[0]
        env = np.repeat(rng.choice([0.02, 0.2, 1.0], size=n // 50 + 1), 50 * F)[:len(x)]
        p = os.path.join(d, "speech%d.wav" % i)
        write_audio(p, np.clip(np.round(x * env), -32768, 32767).astype(np.int16), wav=True)
        sig.append(p)
        p = os.path.join(d, "noise%d.wav" % i)
        write_audio(p, np.round(rng.normal(0, rng.uniform(100, 2000), n * F)).astype(np.int16), wav=True)
        noise.append(p)
    return sig, noise


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def bench(sig, noise, L, T, reps):
    V = 1 + len(LIMITS)
    S = V * L
    cs = torch.cuda.current_stream().cuda_stream
    wc = tr.WaveformCorpus(sig, noise, L)
    wc.start(L * (reps + 2) * T, seed=1)
    noisy, clean = (torch.empty((L, T, F), device="cuda") for _ in range(2))
    vt = torch.empty((L, T), device="cuda")
    nxt = lambda: wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F, vad_ptr=vt.data_ptr(), vad_stream_stride=T,  # noqa: E731
                          vad_frame_stride=1, cuda_stream=cs)
    ms_next = timed(nxt, reps)
    b = nb.DenoiseBatch(S)
    b.set_stream_controls(atten_lim_db=np.repeat([0.0] + LIMITS, L).astype(np.float32))
    rep, out = (torch.empty((V, L, T, F), device="cuda") for _ in range(2))
    rep.copy_(noisy.unsqueeze(0).expand(V, L, T, F))
    vad = torch.empty((T, S), device="cuda")
    ms_steps = timed(lambda: b.process_device(out.data_ptr(), rep.data_ptr(), vad.data_ptr(), T, T * F, F, cuda_stream=cs), reps)
    prof = [b.profile_step(out.data_ptr(), rep.data_ptr(), 0, T * F) for _ in range(reps)]
    ms_analysis = float(np.median([p["analysis"] for p in prof]))
    m = nb.Metrics(S)
    tg = torch.ones((T, S), device="cuda")
    ms_metrics = timed(lambda: m.accumulate_device(out.data_ptr(), rep.data_ptr(), T, T * F, F, vad.data_ptr(), tg.data_ptr(), 1, S,
                                                   cuda_stream=cs), reps)
    rep_e = ev.evaluate(sig, noise, ["builtin"], LIMITS, L, 10 * T, seed=2, window=T, warmup_frames=T)
    return dict(lanes=L, variants=V, window=T, streams=S,
                metrics_ms_per_window=ms_metrics, metrics_ns_per_stream_frame=1e6 * ms_metrics / (S * T),
                analysis_ms_per_frame=ms_analysis, analysis_ns_per_stream_frame=1e6 * ms_analysis / S,
                steps_ms_per_window=ms_steps, next_ms_per_window=ms_next,
                evaluate_seconds=rep_e["seconds"], evaluate_lane_frames_per_second=rep_e["lane_frames_per_second"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", default="256,4096")
    ap.add_argument("--window", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    head = dict(device=torch.cuda.get_device_name(0), power_limit=query("power.limit"))
    lines = []
    with tempfile.TemporaryDirectory() as d:
        sig, noise = make_corpus(d)
        for L in (int(v) for v in a.lanes.split(",")):
            r = dict(head, **bench(sig, noise, L, a.window, a.reps))
            print(json.dumps(r), flush=True)
            lines.append(r)
    if a.out:
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
