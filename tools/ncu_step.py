"""One frame-step of B streams for ncu: warm-up frames first, then the five kernels of one more frame.
    ncu --set full --import-source on --clock-control none --launch-skip $((5*WARM)) -c 5 -o ncu_step python tools/ncu_step.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nnnoiseless_b200 as nb  # noqa: E402
from nnnoiseless_b200.synth import synth_streams  # noqa: E402

B = int(os.environ.get("NCU_STREAMS", "65536"))
WARM = int(os.environ.get("NCU_WARM", "6"))
T = WARM + 1
base = synth_streams(256, T, seed=1).reshape(256, T, 480)
idx = np.random.default_rng(0).integers(0, 256, B)
x = torch.from_numpy(np.ascontiguousarray(base[idx].transpose(1, 0, 2))).cuda()   # [T][B][480]
out = torch.empty_like(x)
vad = torch.empty((T, B), device="cuda")
b = nb.DenoiseBatch(B)
b.process_device(out.data_ptr(), x.data_ptr(), vad.data_ptr(), T, 480, B * 480)
torch.cuda.synchronize()
print("done", float(out.abs().mean()))
