"""Per-phase, per-warp cycle account of pitch_kernel at the benchmark's batch size.

Build the profiling variant (NNB_VARIANT=prof python -m nnnoiseless_b200.build), then on a GPU:

    NNB_LIB=nnnoiseless_b200/lib/libnnnoiseless_b200_prof.so python tools/pitch_phase_profile.py [--streams 65536]

The streams are bench.py's signals (synth_on_device).  After `--warm` frames fill the history, one frame is run with the
kernel's clock trace armed: lane 0 of every warp stamps clock64() when it arrives at each barrier.  Per phase and warp
role: busy cycles (previous barrier's release -> arriving at this one) and cycles waiting at the barrier, summed over the
role's warps and averaged over the blocks; the phase's wall time in a tile (release of the
previous barrier -> release of this one) and which role arrived last (the critical path); and the tile's lifetime.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NW, PT_N = 8, 32
# (name, trace point at the warps' arrival at the phase's closing barrier, warps taking part in that barrier)
# A warp's stamp right after a barrier is taken before the warp really blocks (BAR.SYNC.DEFER_BLOCKING), so only the
# arrival stamps are used: a barrier's release is its last arrival.  Ph6x and Ph10x hold barriers of their own (they
# rarely have work); their points are the first stamp after them.
ALL = list(range(NW))
PHASES = [
    ("Ph1 downsample (HBM loads)", 1, ALL),
    ("Ph2 autocorr", 3, ALL),
    ("Ph3 LPC", 5, ALL),
    ("Ph4 FIR", 7, ALL),
    ("Ph5 coarse FMA | chains", 9, ALL),
    ("Ph6a certified select", 11, ALL),
    ("Ph6x exact coarse", 13, ALL),
    ("Ph6b fine windows | yy_lookup", 15, ALL[:-1]),
    ("Ph8 fine select + lags", 17, ALL),
    ("Ph9 rd FMA", 19, ALL),
    ("Ph10g ladder gains (lane-tasks)", 20, ALL),
    ("Ph10a ladder", 21, ALL),
    ("Ph10x exact ladder", 23, ALL),
    ("Ph11 final lane-tasks", 24, ALL),
    ("Ph11 final lane-per-stream", 26, ALL),
]
ROLES = [("w0", [0]), ("w1-4", [1, 2, 3, 4]), ("w5", [5]), ("w6", [6]), ("w7", [7])]


def account(tr):
    """tr: [blocks][NW][PT_N] int64 clock64 stamps -> per-phase averages over blocks.  Per warp and phase: busy =
    arrival - (the later of the previous release and the warp's own previous arrival), wait = release - arrival (0 for a
    warp outside the barrier); wall = release - previous release."""
    t = tr[:, :, :PT_N - 1].astype(np.float64)
    start = t[:, :, 0].min(axis=1)
    life = t[:, :, 26].max(axis=1) - start
    rows = []
    prev_arr = t[:, :, 0]
    prev_rel = start
    for name, a, ws in PHASES:
        arr = t[:, :, a]
        rel = arr[:, ws].max(axis=1)
        busy = np.maximum(arr - np.maximum(prev_rel[:, None], prev_arr), 0.0)
        wait = np.zeros_like(busy)
        wait[:, ws] = rel[:, None] - arr[:, ws]
        last = np.argmax(arr[:, ws], axis=1)
        row = {"phase": name, "wall": float((rel - prev_rel).mean()),
               "last_warp": np.bincount(np.array(ws)[last], minlength=NW).tolist()}
        for rn, wr in ROLES:
            row["busy_" + rn] = float(busy[:, wr].sum(axis=1).mean())
            row["wait_" + rn] = float(wait[:, wr].sum(axis=1).mean())
        rows.append(row)
        prev_arr, prev_rel = arr, rel
    return {"tile_cycles": float(life.mean()), "phases": rows}


def residency(tr):
    """Mean number of tiles resident on an SM while it works (tile lifetimes summed / span of the SM's busy time)."""
    sm = tr[:, 0, PT_N - 1]
    t0 = tr[:, :, 0].min(axis=1)
    t1 = tr[:, :, 26].max(axis=1)
    occ = []
    for s in np.unique(sm):
        m = sm == s
        occ.append((t1[m] - t0[m]).sum() / (t1[m].max() - t0[m].min()))
    return float(np.mean(occ)), int(np.bincount(sm.astype(np.int64)).max())


def nvsmi(fields):
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=" + ",".join(fields), "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return [v.strip() for v in q.split(",")] if q else ["?"] * len(fields)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--warm", type=int, default=4, help="frames run before the traced one")
    ap.add_argument("--json", default="", help="also write the account here")
    ap.add_argument("--trace", default="", help="also write the raw trace here (.npy)")
    args = ap.parse_args()
    import torch
    import nnnoiseless_b200 as nb
    from bench import synth_on_device
    B, T = args.streams, args.warm + 1
    dev = torch.device("cuda", 0)
    x = synth_on_device(torch, B, T, dev, seed=1234)
    out = torch.empty_like(x)
    vad = torch.empty(T, B, device=dev)
    batch = nb.DenoiseBatch(B, device=0)
    L = nb.lib()
    L.nnb_pitch_trace_arm.argtypes = [C.c_void_p]
    for t in range(args.warm):
        batch.process_device(out[t].data_ptr(), x[t].data_ptr(), vad[t].data_ptr(), 1, stream_stride=480, frame_stride=B * 480)
    torch.cuda.synchronize()
    nblk = (B + 15) // 16
    tr = torch.zeros(nblk, NW, PT_N, dtype=torch.int64, device=dev)
    assert L.nnb_pitch_trace_arm(tr.data_ptr()) == 0
    t = args.warm
    batch.process_device(out[t].data_ptr(), x[t].data_ptr(), vad[t].data_ptr(), 1, stream_stride=480, frame_stride=B * 480)
    torch.cuda.synchronize()
    assert L.nnb_pitch_trace_arm(None) == 0
    tr = tr.cpu().numpy()
    if args.trace:
        np.save(args.trace, tr)
    acc = account(tr)
    acc["tiles_per_sm_resident"], acc["tiles_on_busiest_sm"] = residency(tr)
    acc["streams"] = B
    print("%s, power limit %s W, SM clock %s MHz" % (torch.cuda.get_device_name(0), *nvsmi(["power.limit", "clocks.sm"])))
    print("tile lifetime %.0f cycles (mean over %d tiles), %.2f tiles resident per SM, %d tiles on the busiest SM"
          % (acc["tile_cycles"], nblk, acc["tiles_per_sm_resident"], acc["tiles_on_busiest_sm"]))
    hdr = "%-31s %7s %5s" % ("phase", "wall", "%") + "".join(" %13s" % ("busy|wait " + rn) for rn, _ in ROLES) + "  last to arrive (warp: tiles)"
    print(hdr)
    for r in acc["phases"]:
        lw = sorted(((n, w) for w, n in enumerate(r["last_warp"]) if n), reverse=True)[:2]
        print("%-31s %7.0f %5.1f" % (r["phase"], r["wall"], 100.0 * r["wall"] / acc["tile_cycles"])
              + "".join(" %6.0f|%6.0f" % (r["busy_" + rn], r["wait_" + rn]) for rn, _ in ROLES)
              + "  " + ", ".join("w%d: %d" % (w, n) for n, w in lw))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(acc, f, indent=1)


if __name__ == "__main__":
    main()
