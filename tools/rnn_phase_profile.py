"""Per-tile clock split of rnn_tc_kernel (the wgmma GRU).  Build the profiling variant here (NNB_VARIANT=prof python -m
nnnoiseless_b200.build), run on a GPU box with NNB_LIB=nnnoiseless_b200/lib/libnnnoiseless_b200_prof.so
python tools/rnn_phase_profile.py [B].  Cycles are per 64-stream tile, summed over the tile's consumer warpgroup
(thread 0's clock); tiles of co-resident CTAs overlap, so the sum over tiles exceeds the kernel's wall time."""
import ctypes as C, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nnnoiseless_b200 as nb
from nnnoiseless_b200.synth import synth_streams
B = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
x = synth_streams(64, 6, seed=3).reshape(64, 6, 480)
xt = np.ascontiguousarray(np.tile(x.transpose(1, 0, 2), (1, B // 64, 1)))
b = nb.DenoiseBatch(B)
b.process_host(xt[:2])
L = nb.lib()
buf = (C.c_ulonglong * 8)()
L.nnb_rnn_prof_read(buf, 1)
b.process_host(xt[2:])
L.nnb_rnn_prof_read(buf, 0)
tiles = max(1, buf[4])
names = ["HBM loads -> operand", "wait for weights", "MMA issue + wait", "epilogue + stores"]
tot = sum(buf[:4])
for i in range(4):
    print("%-22s %9.0f cycles/tile  %5.1f%%" % (names[i], buf[i] / tiles, 100.0 * buf[i] / max(tot, 1)))
print("total %.0f cycles/tile over %d tiles" % (tot / tiles, tiles))
