"""Time the fitting kernels (csrc/fit.cu) on one GPU: ms per Adam step at S = 32 windows of T = 2,000 frames with the
reference geometry (24, 24, 48, 96), split by kernel family with torch.profiler (forward recurrences, backward
recurrences, GEMMs with their split-K reductions, the rest), training frames/s at S = 32 and S = 1,024, and the float32
torch restatement of the same step (tests/fit_ref.py, autograd) on this machine's CPU cores.  Prints one JSON line.

    python tools/fit_bench.py [--steps 10] [--cpu-steps 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from nnnoiseless_b200 import fit  # noqa: E402

FAMILIES = (("fwd_recurrence", "fit_gru_fwd"), ("bwd_recurrence", "fit_gru_bwd"), ("gemm", "fit_gemm"), ("gemm", "fit_reduce"))


def rows_for(S, T, seed=0):
    rng = np.random.default_rng(seed)
    rows = np.zeros((S, T, 87), np.float32)
    rows[..., :42] = rng.standard_normal((S, T, 42))
    rows[..., 42:64] = rng.random((S, T, 22))
    rows[..., 86] = rng.choice([0.0, 0.5, 1.0], size=(S, T))
    return rows, np.ones((S, T), np.float32)


def time_steps(S, T, steps):
    f = fit.Fit(fit.WIDTHS, S, T, device=0)
    f.set_params(fit.init_params(fit.WIDTHS, 0))
    rows, w = rows_for(S, T)
    f.step(rows, w)  # warm-up: module load, first launches
    t0 = time.perf_counter()
    for _ in range(steps):
        f.step(rows, w)  # each step ends in a device synchronise (the loss is read back)
    ms = (time.perf_counter() - t0) * 1e3 / steps
    return f, rows, w, ms


def split(f, rows, w, steps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            f.step(rows, w)
    out = {"fwd_recurrence": 0.0, "bwd_recurrence": 0.0, "gemm": 0.0, "rest": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        fam = next((k for k, pat in FAMILIES if pat in e.key), "rest")
        out[fam] += t / 1e3 / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--cpu-steps", type=int, default=1)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    T = 2000
    f, rows, w, ms32 = time_steps(32, T, a.steps)
    parts = split(f, rows, w, a.steps)
    del f
    _, _, _, ms1024 = time_steps(1024, T, max(2, a.steps // 4))
    params = fit.init_params(fit.WIDTHS, 0)
    from fit_ref import loss_and_grad
    t0 = time.perf_counter()
    for _ in range(a.cpu_steps):
        loss_and_grad(params, fit.WIDTHS, rows, w, torch.float32)
    cpu_ms = (time.perf_counter() - t0) * 1e3 / a.cpu_steps
    print(json.dumps(dict(
        gpu=gpu, geometry=list(fit.WIDTHS), T=T,
        ms_per_step_S32=round(ms32, 3), split_ms_S32={k: round(v, 3) for k, v in parts.items()},
        frames_per_s_S32=round(32 * T / (ms32 / 1e3)), ms_per_step_S1024=round(ms1024, 3),
        frames_per_s_S1024=round(1024 * T / (ms1024 / 1e3)),
        cpu_torch_f32_ms_per_step_S32=round(cpu_ms, 1), cpu_threads=torch.get_num_threads(),
        cpu_frames_per_s_S32=round(32 * T / (cpu_ms / 1e3)))))


if __name__ == "__main__":
    main()
