"""Small end-to-end run used under compute-sanitizer (memcheck / racecheck / initcheck)."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nnnoiseless_b200 as nb
from nnnoiseless_b200.synth import synth_streams
B, T = 37, 6
x = np.ascontiguousarray(synth_streams(B, T, seed=5).reshape(B, T, 480).transpose(1, 0, 2))
b = nb.DenoiseBatch(B)
o, v = b.process_host(x)
o16, _ = nb.DenoiseBatch(B).process_pcm16_host(x.astype(np.int16))
z, _ = nb.DenoiseBatch(3).process_host(np.zeros((3, 3, 480), np.float32))
print("ok", float(np.abs(o).mean()), int(np.abs(o16).max()), float(np.abs(z).max()))
# subset calls: the work state grows (5 -> 20 rows), and a 10-frame call rotates the ring by more than its 8 slots
s1, _ = b.process_streams_host([4, 30, 1, 17, 8], x[:3, :5])
s2, _ = b.process_streams_host(np.arange(36, 16, -1), np.ascontiguousarray(np.concatenate([x, x[:4]])[:, :20]))
o2, _ = b.process_host(x[:2])
print("ok subset", float(np.abs(s1).mean()), float(np.abs(s2).mean()), float(np.abs(o2).mean()))
# a single-stream state and its clone
s = nb.DenoiseState()
f = np.ascontiguousarray(x[0, 0])
s.process_frame(np.empty_like(f), f)
c = s.clone()
c.process_frame(np.empty_like(f), f)
# N4 training rows and N2 resampler / file driver
from nnnoiseless_b200 import training as tr, files
L = 70
sig = np.ascontiguousarray(synth_streams(L, 4, seed=6).reshape(L, 4, 480).transpose(1, 0, 2))
noi = np.ascontiguousarray(synth_streams(L, 4, seed=7).reshape(L, 4, 480).transpose(1, 0, 2)) * np.float32(0.1)
tb = tr.TrainingBatch(L)
tb.set_params(tr.randomize(L, np.random.default_rng(0)))
rows = tb.process_host(sig, noi)
y = files.resample(synth_streams(2, 5, seed=8).T.copy(), 44100 / 48000)
import tempfile
d = tempfile.mkdtemp()
files.write_audio(os.path.join(d, "a.raw"), synth_streams(1, 4, seed=9).T.astype(np.int16))
files.denoise_file(os.path.join(d, "a.raw"), os.path.join(d, "a.wav"), sample_rate=32000)
print("ok2", float(np.abs(rows).mean()), y.shape, os.path.getsize(os.path.join(d, "a.wav")))
# every handle is destroyed here, while the library is loaded (the file driver releases its own buffers in its call)
del b, c, s, tb
print("ok destroyed")
