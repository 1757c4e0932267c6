"""Time the synthesis kernel alone at B = 65,536 streams with and without per-stream controls (DESIGN.md 7m), with CUDA
events over serialised frame-steps as tools/spectral_bench.py does.

    python tools/controls_bench.py [--controls off|one|on] [--streams 65536] [--frames 100] [--warmup 10]
    python tools/controls_bench.py --alternate PARENT_TREE [--rounds 3]

Every frame runs the five kernels serialised on one stream with an event between each two (rnnoise_batch_profile_step),
so the synthesis kernel runs alone on the GPU; its time is the mean over the timed frames.  --controls on gives every
stream a 12 dB attenuation limit and a gate (threshold 0.9, hold 3 frames, closed gain 0.1): on bench.py's synthetic
signals the vad stays below 0.9 on most frames, so most stream-frames take the gated store path.  --controls one gives
stream 0 alone those controls: the frames take the kernel with controls compiled in, and every other stream runs it on
the defaults (what a single fused kernel would cost a batch without controls).  --alternate runs, in `rounds` rounds, the
package and library of another tree (a built checkout of the commit before the controls), then this tree's with controls
off, one and on, each in its own process, and prints one JSON line per run and a summary line of medians with
the card's name, power limit and SM clock."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def query(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run_one(a):
    sys.path.insert(0, os.path.abspath(a.root))  # the tree whose package, library and bench helpers are measured
    import torch
    import nnnoiseless_b200 as nb
    from bench import ClockSampler, synth_on_device

    if not torch.cuda.is_available():
        sys.exit("controls_bench needs a CUDA device")
    B = a.streams
    dev = torch.device("cuda", 0)
    Tin = 16  # distinct input frames, used cyclically
    x = synth_on_device(torch, B, Tin, dev, seed=1234)
    out = torch.empty_like(x)
    vad = torch.empty(Tin, B, device=dev)
    batch = nb.DenoiseBatch(B, device=0)
    if a.controls != "off":
        batch.set_stream_controls(None if a.controls == "on" else [0], atten_lim_db=12.0, gate_threshold=0.9, gate_closed_gain=0.1,
                                  gate_hold_frames=3)
    sp = torch.cuda.current_stream().cuda_stream

    def frame(t):
        k = t % Tin
        return batch.profile_step(out[k].data_ptr(), x[k].data_ptr(), vad[k].data_ptr(), 480, sp)

    for t in range(a.warmup):
        frame(t)
    ms, closed = [], []
    sampler = ClockSampler(0)
    sampler.start()
    for t in range(a.warmup, a.warmup + a.frames):
        ms.append(frame(t)["synthesis"])
        if a.controls == "on" and t % 10 == 0:
            closed.append(float(np.mean(batch.get_stream_controls()["gate_closed"])))
    clocks = sampler.stop()
    res = dict(device=torch.cuda.get_device_name(0), power_limit=query("power.limit"), sm_clock_median_mhz=clocks.get("sm_mhz"),
               streams=B, frames=a.frames, lib=nb.LIB_PATH, controls=a.controls,
               synthesis_ms=round(float(np.mean(ms)), 4), synthesis_ms_spread=round(float(np.max(ms) - np.min(ms)), 4))
    if closed:
        res["gate_closed_fraction"] = round(float(np.mean(closed)), 3)
    print(json.dumps(res), flush=True)
    return res


def alternate(a):
    runs = {"parent": [], "off": [], "one": [], "on": []}
    last = None
    for _ in range(a.rounds):
        for name, root, controls in (("parent", a.alternate, "off"), ("off", ROOT, "off"), ("one", ROOT, "one"), ("on", ROOT, "on")):
            env = dict(os.environ)
            env.pop("NNB_LIB", None)
            cmd = [sys.executable, os.path.abspath(__file__), "--controls", controls, "--streams", str(a.streams), "--frames",
                   str(a.frames), "--warmup", str(a.warmup), "--root", root]
            r = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True)
            last = json.loads(r.stdout.strip().splitlines()[-1])
            print(json.dumps(dict(run=name, **last)), flush=True)
            runs[name].append(last["synthesis_ms"])
    med = {k: float(np.median(v)) for k, v in runs.items()}
    print(json.dumps(dict(summary=True, device=last["device"], power_limit=last["power_limit"], streams=a.streams, rounds=a.rounds,
                          synthesis_ms_median=med, synthesis_ms_all=runs,
                          off_vs_parent=round(med["off"] / med["parent"] - 1.0, 4),
                          one_vs_parent=round(med["one"] / med["parent"] - 1.0, 4),
                          on_vs_parent=round(med["on"] / med["parent"] - 1.0, 4))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--controls", choices=["off", "one", "on"], default="off")
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--root", default=ROOT, help="tree to measure (default: this one)")
    ap.add_argument("--alternate", default="", metavar="TREE", help="built tree to alternate with this one (e.g. the parent commit)")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if a.alternate:
        alternate(a)
    else:
        run_one(a)


if __name__ == "__main__":
    main()
