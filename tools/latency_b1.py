"""Per-kernel latency of one frame at small batch sizes (the legacy one-stream ABI's regime), per kernel variant.

Run on the GPU box:  python tools/latency_b1.py            (spawns one subprocess per variant: the switches are read at create)
"""
import json
import os
import subprocess
import sys
import time

VARIANTS = {
    "default": {},
    "rnn_mma": {"NNB_RNN_MMA": "1"},
}


def child(B):
    import numpy as np
    import torch
    import nnnoiseless_b200 as nb
    from nnnoiseless_b200 import synth
    dev = torch.device("cuda:0")
    batch = nb.DenoiseBatch(B, device=0)
    T = 60
    x = torch.from_numpy(synth.synth_mixed(B, T, seed=5).reshape(B, T, 480).transpose(1, 0, 2).copy()).to(dev)
    out = torch.empty_like(x)
    vad = torch.empty(T, B, device=dev)
    acc = {}
    for t in range(T):
        d = batch.profile_step(out[t].data_ptr(), x[t].data_ptr(), vad[t].data_ptr(), 480)
        if t >= 20:
            for k, v in d.items():
                acc.setdefault(k, []).append(v * 1e3)
    res = {k: float(np.median(v)) for k, v in acc.items()}
    res["sum_us"] = sum(res.values())
    if B == 1:
        st = nb.DenoiseState()
        xin = np.ascontiguousarray(x[:, 0, :].cpu().numpy())
        o = np.empty(480, np.float32)
        for i in range(20):
            st.process_frame(o, xin[i % T])
        t0 = time.perf_counter()
        n = 400
        for i in range(n):
            st.process_frame(o, xin[i % T])
        res["legacy_us_per_frame"] = 1e6 * (time.perf_counter() - t0) / n
    print(json.dumps(res))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        child(int(sys.argv[2]))
        sys.exit(0)
    for B in (1, 16, 256):
        for name, env in VARIANTS.items():
            e = dict(os.environ)
            e.update(env)
            r = subprocess.run([sys.executable, __file__, "--child", str(B)], env=e, capture_output=True, text=True)
            line = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else r.stderr[-300:]
            print("B=%d %-12s %s" % (B, name, line), flush=True)
