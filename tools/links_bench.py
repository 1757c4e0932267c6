"""Time the synthesis kernel alone at B = 65,536 streams with and without stream links (DESIGN.md 7n), with CUDA events
over serialised frame-steps as tools/controls_bench.py does.

    python tools/links_bench.py [--links off|pairs|g8max|g8mean] [--streams 65536] [--frames 100] [--warmup 10]
    python tools/links_bench.py --alternate PARENT_TREE [--rounds 3]

Every frame runs the five kernels serialised on one stream with an event between each two (rnnoise_batch_profile_step),
so the synthesis kernel runs alone on the GPU; its time is the mean over the timed frames.  --links off runs this tree
without groups (the kernel from before the links), pairs links streams 2k and 2k + 1 under MAX, g8max / g8mean link
groups of 8 consecutive streams.  A linked stream-frame reads count x 22 x 4 bytes of its members' raw gains on top of
the kernel's own traffic.  --alternate runs, in `rounds` rounds, the package and library of another tree (a built
checkout of the commit before the links), then this tree's off, pairs, g8max and g8mean, each in its own process, and
prints one JSON line per run and a summary line of medians and round-to-round spreads with the card's name, power limit
and SM clock."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNS = ("off", "pairs", "g8max", "g8mean")


def query(fields):
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def link(batch, B, how):
    """Link the batch's streams as `how` says; returns the member count of a group (1: no groups)."""
    if how == "off":
        return 1
    size, mode = (2, "max") if how == "pairs" else (8, how[2:])
    for s in range(0, B - B % size, size):
        batch.link_streams(np.arange(s, s + size, dtype=np.int32), mode)
    return size


def run_one(a):
    sys.path.insert(0, os.path.abspath(a.root))  # the tree whose package, library and bench helpers are measured
    import torch
    import nnnoiseless_b200 as nb
    from bench import ClockSampler, synth_on_device

    if not torch.cuda.is_available():
        sys.exit("links_bench needs a CUDA device")
    B = a.streams
    dev = torch.device("cuda", 0)
    Tin = 16  # distinct input frames, used cyclically
    x = synth_on_device(torch, B, Tin, dev, seed=1234)
    out = torch.empty_like(x)
    vad = torch.empty(Tin, B, device=dev)
    batch = nb.DenoiseBatch(B, device=0)
    count = link(batch, B, a.links)
    sp = torch.cuda.current_stream().cuda_stream

    def frame(t):
        k = t % Tin
        return batch.profile_step(out[k].data_ptr(), x[k].data_ptr(), vad[k].data_ptr(), 480, sp)

    for t in range(a.warmup):
        frame(t)
    ms = []
    sampler = ClockSampler(0)
    sampler.start()
    for t in range(a.warmup, a.warmup + a.frames):
        ms.append(frame(t)["synthesis"])
    clocks = sampler.stop()
    res = dict(device=torch.cuda.get_device_name(0), power_limit=query("power.limit"), sm_clock_median_mhz=clocks.get("sm_mhz"),
               streams=B, frames=a.frames, lib=nb.LIB_PATH, links=a.links, group_size=count,
               extra_gain_bytes_per_stream_frame=0 if count == 1 else count * 22 * 4,
               synthesis_ms=round(float(np.mean(ms)), 4), synthesis_ms_spread=round(float(np.max(ms) - np.min(ms)), 4))
    print(json.dumps(res), flush=True)
    return res


def alternate(a):
    runs = {k: [] for k in ("parent",) + RUNS}
    last = None
    for _ in range(a.rounds):
        for name, root, links in (("parent", a.alternate, "off"),) + tuple((k, ROOT, k) for k in RUNS):
            env = dict(os.environ)
            env.pop("NNB_LIB", None)
            cmd = [sys.executable, os.path.abspath(__file__), "--links", links, "--streams", str(a.streams), "--frames",
                   str(a.frames), "--warmup", str(a.warmup), "--root", root]
            r = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True)
            last = json.loads(r.stdout.strip().splitlines()[-1])
            print(json.dumps(dict(run=name, **last)), flush=True)
            runs[name].append(last["synthesis_ms"])
    med = {k: float(np.median(v)) for k, v in runs.items()}
    print(json.dumps(dict(summary=True, device=last["device"], power_limit=last["power_limit"],
                          sm_clock_median_mhz=last["sm_clock_median_mhz"], streams=a.streams, frames=a.frames, rounds=a.rounds,
                          synthesis_ms_median=med, synthesis_ms_all=runs,
                          round_spread_ms={k: round(float(np.max(v) - np.min(v)), 4) for k, v in runs.items()},
                          vs_parent={k: round(med[k] / med["parent"] - 1.0, 4) for k in RUNS})))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--links", choices=RUNS, default="off")
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
