"""Times training the denoiser's own network through synthesis (DESIGN.md 7l) at sizes (L lanes, T frames per window),
on windows of a synthetic corpus generated beforehand, on a non-default torch stream:

    step      one training step of DenoiseNetwork (the built-in model's network), phase by phase (CUDA events):
              analyze_window, net forward, synthesize_window, synthesis backward (synthesis_grad and the waveform loss),
              net backward, Adam + clip_
    kernels   the net's forward and backward kernels alone (torch.profiler, a run of its own), per call

and, alternated with the step inside each repetition, the same step with two other networks:

    gru7j     the 7j network (42 -> 64 nn.GRU + linear) as tools/waveform_bench.py times it
    torch     the same RNNoise network restated in plain torch (a Python time loop of Keras reset_after=False cells with
              relu / tanh activations, silent frames carried with torch.where, autograd backward): what a user would
              otherwise write to train it

    python tools/fit_synthesis_bench.py [--sizes 256x64,4096x100] [--reps 7] [--out FILE]

Prints one JSON line per size with the card's name, power limit and maximum SM clock.  Needs a GPU; writes its corpus to a
temporary directory and nothing else (the JSON also goes to --out if given).
"""
import argparse
import json
import os
import re
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import nnnoiseless_b200 as nb  # noqa: E402
from nnnoiseless_b200 import fit, training as tr  # noqa: E402
from nnnoiseless_b200.autograd import DenoiseNetwork, synthesis_grad  # noqa: E402
from waveform_bench import Net as Gru7j, card, make_corpus, stats, train_step as gru7j_step  # noqa: E402

F, NBF, NBB, CB = 480, 42, 22, nb.SYNTH_CONTEXT_BYTES
PHASES = ("analyze", "net_forward", "synthesize", "synthesis_backward", "net_backward", "optimiser")


class TorchRNNoise(torch.nn.Module):
    """The RNNoise network in plain torch, with the parameters and activations of a DenoiseNetwork."""

    def __init__(self, net):
        super().__init__()
        data = nb.RnnModel().to_bytes()
        self.widths, self.acts = net.widths, tuple(data[p + 2] for p in layer_offsets(data))
        self.params = torch.nn.Parameter(net.params.detach().clone())

    def _gru(self, x, i, silent, h):
        name, n = ("vad_gru", "noise_gru", "denoise_gru")[i], self.widths[1 + i]
        P = self._P
        U, xw = P[(name, "recurrent_kernel")], x @ P[(name, "kernel")] + P[(name, "bias")]
        out = []
        for t in range(x.shape[1]):
            a, hu = xw[:, t], h @ U[:, :2 * n]
            z = torch.sigmoid(a[:, :n] + hu[:, :n])
            r = torch.sigmoid(a[:, n:2 * n] + hu[:, n:])
            hc = _act(self.acts[1 + i], a[:, 2 * n:] + (r * h) @ U[:, 2 * n:])
            h = torch.where(silent[:, t], h, z * h + (1 - z) * hc)
            out.append(h)
        return torch.stack(out, 1), h

    def forward(self, x, sil, state=None):
        self._P = P = fit.unflatten(self.params, self.widths)
        silent = sil.t().bool()[..., None]
        nw = list(self.widths[1:])
        h0 = torch.split(torch.zeros(x.shape[0], sum(nw), device=x.device) if state is None else state, nw, 1)
        d = _act(self.acts[0], x @ P[("input_dense", "kernel")] + P[("input_dense", "bias")])
        hv, v_last = self._gru(d, 0, silent, h0[0])
        hn, n_last = self._gru(torch.cat([d, hv, x], -1), 1, silent, h0[1])
        hd, d_last = self._gru(torch.cat([hv, hn, x], -1), 2, silent, h0[2])
        gains = _act(self.acts[4], hd @ P[("denoise_output", "kernel")] + P[("denoise_output", "bias")])
        return torch.where(silent, 0.0, gains), torch.cat([v_last, n_last, d_last], 1).detach()


def _act(code, v):
    return torch.tanh(v) if code == 0 else (torch.sigmoid(v) if code == 1 else torch.relu(v))


def layer_offsets(data):
    """Byte offset of each of the six layer headers of a .rnn image."""
    offs, p = [], 0
    for gates in (1, 3, 3, 3, 1, 1):
        offs.append(p)
        ni, n = data[p], data[p + 1]
        p += 3 + gates * n * ni + (3 * n * n if gates == 3 else 0) + gates * n
    return offs


def rnnoise_step(b, net, opt, noisy, clean, feats, sil, out, ctx, ev=None):
    """One training step through synthesis; ev: 7 CUDA events recorded at the phase boundaries (or None)."""
    B, T = noisy.shape[0], noisy.shape[1]
    cs = torch.cuda.current_stream().cuda_stream
    mark = (lambda k: ev[k].record()) if ev else (lambda k: None)  # noqa: E731
    b.reset()
    opt.zero_grad()
    mark(0)
    b.analyze_window_device(noisy.data_ptr(), feats.data_ptr(), sil.data_ptr(), T, T * F, F, T * NBF, NBF, ctx.data_ptr(), T, 1, cuda_stream=cs)
    mark(1)
    g = net(feats, sil)[0]
    mark(2)
    gd = g.detach().contiguous()
    b.synthesize_window_device(out.data_ptr(), gd.data_ptr(), T, T * F, F, T * NBB, NBB, ctx.data_ptr(), T, 1, cuda_stream=cs)
    mark(3)
    gl = gd.requires_grad_()
    y = synthesis_grad(gl, out, ctx)
    ((y[:, 1:] - clean[:, :-1]) / 32768).pow(2).mean().backward()
    mark(4)
    g.backward(gl.grad)
    mark(5)
    opt.step()
    with torch.no_grad():
        for p in net.parameters():
            p.clamp_(-0.499, 0.499)
    mark(6)


def bench(wc, L, T, reps):
    res = dict(L=L, T=T)
    wc.start(L * T * 4)
    wins = []
    for _ in range(2):
        noisy, clean = torch.empty((L, T, F), device="cuda"), torch.empty((L, T, F), device="cuda")
        wc.next(T, noisy.data_ptr(), clean.data_ptr(), T * F, F, cuda_stream=torch.cuda.current_stream().cuda_stream)
        wins.append((noisy, clean))
    b = nb.DenoiseBatch(L)
    feats, out = torch.empty((L, T, NBF), device="cuda"), torch.empty((L, T, F), device="cuda")
    sil = torch.empty((T, L), dtype=torch.int32, device="cuda")
    ctx = torch.empty((L, T, CB), dtype=torch.uint8, device="cuda")
    ours = DenoiseNetwork.from_model(None, L, T)
    ours_opt = torch.optim.Adam([ours.params], lr=1e-3)
    plain = TorchRNNoise(ours)
    plain_opt = torch.optim.Adam([plain.params], lr=1e-3)
    g7 = Gru7j()
    times = {"step": [], "gru7j": [], "torch": []}
    phases = {k: [] for k in PHASES}
    cs = torch.cuda.current_stream()
    for rep in range(reps + 1):
        for way in times:
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            noisy, clean = wins[rep % 2]
            e0.record(cs)
            if way == "step":
                rnnoise_step(b, ours, ours_opt, noisy, clean, feats, sil, out, ctx, ev)
            elif way == "torch":
                rnnoise_step(b, plain, plain_opt, noisy, clean, feats, sil, out, ctx)
            else:
                gru7j_step(b, g7, noisy, clean, feats, out, ctx)
            e1.record(cs)
            torch.cuda.synchronize()
            if rep > 0:
                times[way].append(e0.elapsed_time(e1))
                if way == "step":
                    for k, name in enumerate(PHASES):
                        phases[name].append(ev[k].elapsed_time(ev[k + 1]))
    res["step_ms"] = {k: stats(v) for k, v in times.items()}
    res["phase_ms"] = {k: stats(v) for k, v in phases.items()}
    # the net's kernels alone
    gg = torch.randn(L, T, NBB, device="cuda")
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ours.params.grad = None
            g, v, _ = ours(feats, sil)
            (g * gg).sum().backward()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        m = re.search(r"fit_\w+(<\w+>)?", e.name)
        if m:
            per.setdefault(m.group(0), []).append(e.device_time_total / 1e3)
    res["kernel_ms_per_call"] = {k: round(sum(v) / reps, 4) for k, v in sorted(per.items())}
    fwd = sum(sum(v) for k, v in per.items() if "gru_fwd" in k) / reps
    bwd = sum(sum(v) for k, v in per.items() if "gru_bwd" in k) / reps
    res["recurrences_ms_per_call"] = dict(forward=round(fwd, 4), backward=round(bwd, 4))
    res["net_kernels_ms_per_call"] = round(sum(sum(v) for v in per.values()) / reps, 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256x64,4096x100")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--minutes", type=int, default=4, help="minutes of speech and of noise in the synthetic corpus")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    lines = []
    with tempfile.TemporaryDirectory() as d:
        sig, noise = make_corpus(d, a.minutes)
        for size in a.sizes.split(","):
            L, T = (int(v) for v in size.split("x"))
            wc = tr.WaveformCorpus(sig, noise, L)
            r = dict(card=card())
            with torch.cuda.stream(torch.cuda.Stream()):
                r.update(bench(wc, L, T, a.reps))
            print(json.dumps(r), flush=True)
            lines.append(r)
            del wc
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
