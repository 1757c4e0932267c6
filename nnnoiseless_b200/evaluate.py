"""Score denoise models on held-out corpus windows, on the GPU (DESIGN.md 7p).

    python -m nnnoiseless_b200.evaluate --signal-glob 'heldout/speech/*.wav' --noise-glob 'heldout/noise/*.wav' \\
        --model builtin --model a.rnn --atten-lim-db inf,12 --lanes 1024 --frames 6000 --seed 1 --json out.json

The variants are every model at every attenuation limit, plus the baseline "unprocessed": the built-in model at
atten_lim_db = 0, whose gains are exactly 1.  Variants whose models share a geometry run as one DenoiseBatch of V * L
streams (stream v * L + l = variant v on lane l, through per-stream models and controls); a model of another geometry
gets a batch of its own.  Each window of T frames is one WaveformCorpus.next, then per batch one device copy of `noisy`
into the replicated input, one fused process_device call with vad, one copy of `clean` into the same buffer and one
Metrics.accumulate_device call.  The first --warmup-frames frames are run and then cleared.  The report gives, per
variant, the lane means and 95 % intervals (1.96 sd / sqrt(L)) of every figure of metrics.summarize, the paired ones
against the baseline, the per-band arrays and the raw records.

With --intelligibility (DESIGN.md 7q) every scored window is also scored with STOI and ESTOI, per stream of each batch:
output frames 1..n-1 against clean frames 0..n-2 (the denoiser's one-frame delay, as Metrics pairs them), through one
nb.intelligibility_device call per batch and window.  Each variant then gains stoi and estoi (per lane, the mean over
the windows with finite scores) and delta_stoi and delta_estoi (paired per lane against the baseline), each with its
95 % interval and the counts of windows scored and NaN.  A score needs 30 STFT frames after silence removal, so use
--window 300: a 1 s window leaves about 76 10 kHz frames before it."""
import argparse
import json
import sys
import time

import numpy as np

import nnnoiseless_b200 as nb
from nnnoiseless_b200 import NnnoiselessError
from nnnoiseless_b200 import metrics as mt
from nnnoiseless_b200 import training as tr

BASELINE = "unprocessed"
BAND_FIGURES = ("speech_dev", "noise_atten_bands")


def load_model(spec):
    """'builtin', a binary .rnn model or an RNNoise text model (.rnnn) -> (name, RnnModel or None for the built-in,
    model bytes)."""
    if spec == "builtin":
        with open(nb.BUILTIN_WEIGHTS_PATH, "rb") as f:
            return spec, None, f.read()
    with open(spec, "rb") as f:
        data = f.read()
    m = nb.RnnModel.from_text(data) if spec.endswith(".rnnn") else nb.RnnModel.from_bytes(data)
    if m is None:
        raise NnnoiselessError("%s is not a model nnnoiseless can read" % spec)
    return spec, m, m.to_bytes()


def geometry(model_bytes):
    """The layer widths that decide whether two models can share a batch: dense, vad, noise and denoise neurons."""
    return (int(model_bytes[1]),) + tuple(nb.gru_widths(model_bytes))


def parse_limits(text):
    out = []
    for t in str(text).split(","):
        v = float(t)
        if not v >= 0.0:
            raise ValueError("attenuation limits must be >= 0 (inf: no limit), not %r" % t)
        out.append(v)
    return out


def plan_variants(models, limits):
    """models: [(name, RnnModel or None, bytes)] -> variants [dict(name, model, atten_lim_db, key)]: the baseline first,
    then every model at every limit in the order given.  key indexes the model list (-1: the built-in baseline)."""
    variants = [dict(name=BASELINE, model="builtin", atten_lim_db=0.0, key=-1)]
    for k, (name, _, _) in enumerate(models):
        for a in limits:
            variants.append(dict(name="%s@%s" % (name, "inf" if a == np.inf else "%g" % a), model=name, atten_lim_db=a, key=k))
    return variants


def group_batches(variants, models, builtin_bytes):
    """-> [dict(geometry, variants [indices into variants], models [key per batch model id, first = the batch's own])]
    in order of first appearance; the built-in model counts as key -1."""
    def bytes_of(k):
        return builtin_bytes if k == -1 else models[k][2]
    groups = []
    for v, var in enumerate(variants):
        g = geometry(bytes_of(var["key"]))
        grp = next((x for x in groups if x["geometry"] == g), None)
        if grp is None:
            grp = dict(geometry=g, variants=[], models=[])
            groups.append(grp)
        grp["variants"].append(v)
        # a model listed twice (or the built-in as a model and as the baseline) is one entry of the table
        if not any(bytes_of(k) == bytes_of(var["key"]) for k in grp["models"]):
            grp["models"].append(var["key"])
    return groups


def device_bytes(groups, lanes, window, intelligibility=False):
    """Device memory of the replicated windows: input/clean and output, V L T 480 float32 each, per batch; with
    intelligibility also the largest batch's STOI workspace (V L pairs of (T - 1) 480 samples), which they share."""
    total = sum(2 * len(g["variants"]) * lanes * window * 1920 for g in groups)
    if intelligibility:
        total += max(nb.intelligibility_workspace_bytes(len(g["variants"]) * lanes, (window - 1) * nb.FRAME_SIZE, 48000) for g in groups)
    return total


def _model_id(grp, models, builtin_bytes, key):
    b = builtin_bytes if key == -1 else models[key][2]
    return next(i for i, k in enumerate(grp["models"]) if (builtin_bytes if k == -1 else models[k][2]) == b)


def evaluate(signal_paths, noise_paths, model_specs, limits, lanes, frames, seed=0, window=100, warmup_frames=200, device=-1,
             shuffle=False, intelligibility=False):
    """Runs the evaluation and returns the report (see the module's documentation)."""
    import torch
    models = [load_model(s) for s in model_specs]
    with open(nb.BUILTIN_WEIGHTS_PATH, "rb") as f:
        builtin_bytes = f.read()
    variants = plan_variants(models, limits)
    groups = group_batches(variants, models, builtin_bytes)
    L, T = int(lanes), int(window)
    if L <= 0 or T <= 0 or frames <= 0 or warmup_frames < 0:
        raise ValueError("lanes, frames and window must be positive, warmup_frames >= 0")
    if intelligibility and T < 2:
        raise ValueError("intelligibility needs a window of at least 2 frames")
    dev = torch.device("cuda", device if device >= 0 else torch.cuda.current_device())
    free, total = torch.cuda.mem_get_info(dev)
    need = device_bytes(groups, L, T, intelligibility)
    if need > free:
        raise NnnoiselessError("%d variants x %d lanes x %d frames per window need %.1f MB of device memory for the replicated "
                               "windows (2 V L T 1920 bytes per batch); %.1f MB of %.1f MB are free: use fewer lanes or a "
                               "shorter --window" % (len(variants), L, T, need / 1e6, free / 1e6, total / 1e6))
    with torch.cuda.device(dev):
        return _run(torch, signal_paths, noise_paths, models, builtin_bytes, variants, groups, L, T, int(frames), int(seed),
                    int(warmup_frames), dev.index, shuffle, intelligibility)


def _run(torch, signal_paths, noise_paths, models, builtin_bytes, variants, groups, L, T, frames, seed, warmup, device, shuffle,
         intelligibility=False):
    t_start = time.perf_counter()
    wc = tr.WaveformCorpus(signal_paths, noise_paths, L, device)
    plan = wc.start(L * (warmup + frames), seed, shuffle)
    total = min(plan.n_frames, warmup + frames)
    F = nb.FRAME_SIZE
    noisy = torch.empty((L, T, F), device="cuda")
    clean = torch.empty((L, T, F), device="cuda")
    vad_t = torch.empty((L, T), device="cuda")
    runs = []
    for grp in groups:
        V = len(grp["variants"])
        own = grp["models"][0]
        b = nb.DenoiseBatch(V * L, model=None if own == -1 else models[own][1], device=device)
        for k in grp["models"][1:]:
            b.add_model(nb.RnnModel() if k == -1 else models[k][1])
        ids = np.repeat([_model_id(grp, models, builtin_bytes, variants[v]["key"]) for v in grp["variants"]], L).astype(np.int32)
        b.set_stream_models(ids)
        b.set_stream_controls(atten_lim_db=np.repeat([variants[v]["atten_lim_db"] for v in grp["variants"]], L).astype(np.float32))
        runs.append(dict(batch=b, metrics=nb.Metrics(V * L, device), V=V,
                         rep=torch.empty((V, L, T, F), device="cuda"), out=torch.empty((V, L, T, F), device="cuda"),
                         vad=torch.empty((T, V * L), device="cuda"), tgt=torch.empty((T, V, L), device="cuda"), stoi=[]))
    ws_bytes = device_bytes(groups, L, T, True) - device_bytes(groups, L, T) if intelligibility else 0
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda") if intelligibility else None
    cs = torch.cuda.current_stream().cuda_stream
    done, cleared = 0, warmup == 0
    while done < total:
        n = min(T, (warmup if not cleared else total) - done)
        got = wc.next(n, noisy.data_ptr(), clean.data_ptr(), T * F, F, vad_ptr=vad_t.data_ptr(), vad_stream_stride=T,
                      vad_frame_stride=1, cuda_stream=cs)
        if got != n:
            raise NnnoiselessError("the corpus plan ended after %d frames" % (done + got))
        for r in runs:
            V = r["V"]
            r["rep"].copy_(noisy.unsqueeze(0).expand(V, L, T, F))
            r["batch"].process_device(r["out"].data_ptr(), r["rep"].data_ptr(), r["vad"].data_ptr(), n, T * F, F, cuda_stream=cs)
            r["rep"].copy_(clean.unsqueeze(0).expand(V, L, T, F))
            r["tgt"].copy_(vad_t.t().unsqueeze(1).expand(T, V, L))  # the network's vad layout, [frame][stream]
            r["metrics"].accumulate_device(r["out"].data_ptr(), r["rep"].data_ptr(), n, T * F, F, r["vad"].data_ptr(),
                                           r["tgt"].data_ptr(), 1, V * L, cuda_stream=cs)
            if intelligibility and cleared and n > 1:
                res = torch.empty(V * L * nb.INTELLIGIBILITY_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
                nb.intelligibility_device(r["out"].data_ptr() + F * 4, r["rep"].data_ptr(), V * L, (n - 1) * F, T * F, 48000, res.data_ptr(),
                                          ws.data_ptr(), ws_bytes, device, cs)
                r["stoi"].append(res)
        done += n
        if not cleared and done == warmup:
            torch.cuda.synchronize()
            for r in runs:
                r["metrics"].clear()
            cleared = True
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t_start
    records = [None] * len(variants)
    stoi = [None] * len(variants) if intelligibility else None
    for grp, r in zip(groups, runs):
        rec = r["metrics"].records()
        si = (np.stack([x.cpu().numpy().view(nb.INTELLIGIBILITY_DTYPE) for x in r["stoi"]]) if r["stoi"]
              else np.zeros((0, r["V"] * L), nb.INTELLIGIBILITY_DTYPE))
        for j, v in enumerate(grp["variants"]):
            records[v] = rec[j * L:(j + 1) * L]
            if intelligibility:
                stoi[v] = si[:, j * L:(j + 1) * L]
    return report(variants, records, groups, L, total - warmup, seconds, stoi)


def _stats(x):
    """Lane mean and 95 % half-interval of a figure, over the lanes where it is defined."""
    x = np.asarray(x, np.float64)
    ok = np.isfinite(x)
    n = int(ok.sum())
    if n == 0:
        return dict(mean=float("nan"), ci95=float("nan"), lanes=0)
    m = float(x[ok].mean())
    sd = float(x[ok].std(ddof=1)) if n > 1 else float("nan")
    return dict(mean=m, ci95=1.96 * sd / np.sqrt(n), lanes=n)


def lane_scores(rec, field):
    """[windows][lanes] intelligibility records -> per lane, the mean of `field` over its windows with a finite score
    (NaN where none is), and the counts of windows scored and NaN."""
    x = np.asarray(rec[field], np.float64)
    ok = np.isfinite(x)
    n = ok.sum(axis=0)
    mean = np.where(n > 0, np.where(ok, x, 0.0).sum(axis=0) / np.maximum(n, 1), np.nan)
    return mean, int(ok.sum()), int((~ok).sum())


def intelligibility_figures(rec, base):
    """stoi, estoi, delta_stoi, delta_estoi of one variant's [windows][lanes] records, paired per lane with the
    baseline's."""
    out = {}
    for k in ("stoi", "estoi"):
        m, scored, nan = lane_scores(rec, k)
        out[k] = dict(_stats(m), windows=scored, nan_windows=nan)
        out["delta_" + k] = dict(_stats(m - lane_scores(base, k)[0]), windows=scored, nan_windows=nan)
    return out


def report(variants, records, groups, lanes, frames, seconds, stoi=None):
    base = records[0]
    out = dict(lanes=lanes, frames=frames, seconds=seconds, lane_frames_per_second=lanes * frames * len(variants) / seconds if seconds else None,
               batches=[dict(geometry=list(g["geometry"]), variants=[variants[v]["name"] for v in g["variants"]]) for g in groups],
               variants=[])
    for v, var in enumerate(variants):
        s = mt.summarize(records[v], None if v == 0 else base)
        figures = {k: _stats(x) for k, x in s.items() if k not in BAND_FIGURES and k != "nan_counts"}
        bands = {k: np.nanmean(s[k], axis=0) if np.isfinite(s[k]).any() else np.full(nb.NB_BANDS, np.nan) for k in BAND_FIGURES if k in s}
        if stoi is not None:
            figures.update(intelligibility_figures(stoi[v], stoi[0]))
        out["variants"].append(dict(name=var["name"], model=var["model"], atten_lim_db=var["atten_lim_db"], figures=figures, bands=bands,
                                    nan_counts=s["nan_counts"], records=records[v]))
        if stoi is not None:
            out["variants"][-1]["intelligibility"] = stoi[v]
    return out


def _jsonable(x):
    if isinstance(x, dict):
        return {k: _jsonable(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_jsonable(v) for v in x]
    if isinstance(x, np.ndarray) and x.dtype.names:
        return [{k: _jsonable(r[k]) for k in x.dtype.names} for r in x]
    if isinstance(x, np.ndarray):
        return _jsonable(x.tolist())
    if isinstance(x, (float, np.floating)):
        f = float(x)
        return f if np.isfinite(f) else str(f)
    if isinstance(x, np.integer):
        return int(x)
    return x


TABLE = ("snr", "delta_snr", "si_sdr", "delta_si_sdr", "seg_snr", "lsd", "noise_atten", "speech_level", "vad_precision", "vad_recall")


STOI_TABLE = ("stoi", "delta_stoi", "estoi", "delta_estoi")


def format_table(rep):
    cols = TABLE + (STOI_TABLE if any("stoi" in v["figures"] for v in rep["variants"]) else ())
    head = "%-28s" % "variant" + "".join("%16s" % k for k in cols)
    lines = [head]
    for v in rep["variants"]:
        cells = []
        for k in cols:
            f = v["figures"].get(k)
            d = 3 if k in STOI_TABLE else 2
            cells.append("%16s" % ("-" if f is None or f["lanes"] == 0 else "%.*f+-%.*f" % (d, f["mean"], d, f["ci95"])))
        lines.append("%-28s" % v["name"] + "".join(cells))
    return "\n".join(lines)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m nnnoiseless_b200.evaluate", description="Score denoise models on held-out corpus windows, on the GPU")
    ap.add_argument("--signal-glob", action="append", required=True, help="wildcard for speech WAV files")
    ap.add_argument("--noise-glob", action="append", required=True, help="wildcard for noise WAV files")
    ap.add_argument("--model", action="append", required=True, help="'builtin', a .rnn model or an RNNoise text model (.rnnn); repeatable")
    ap.add_argument("--atten-lim-db", default="inf", help="comma-separated attenuation limits in dB (inf: none)")
    ap.add_argument("--lanes", type=int, default=256, help="corpus lanes scored side by side")
    ap.add_argument("--frames", type=int, required=True, help="frames scored per lane, after the warm-up")
    ap.add_argument("--window", type=int, default=100, help="frames per window")
    ap.add_argument("--warmup-frames", type=int, default=200, help="frames run and then cleared before scoring")
    ap.add_argument("--seed", type=int, default=0, help="seed of the corpus plan")
    ap.add_argument("--shuffle", action="store_true", help="shuffle the speech and noise files")
    ap.add_argument("--device", type=int, default=-1, help="CUDA device (-1: current)")
    ap.add_argument("--json", help="write the whole report here")
    ap.add_argument("--intelligibility", action="store_true",
                    help="also score every window with STOI and ESTOI on the GPU (use --window 300: a score needs 30 STFT frames)")
    a = ap.parse_args(argv)
    try:
        limits = parse_limits(a.atten_lim_db)
    except ValueError as e:
        ap.error(str(e))
    if a.lanes <= 0 or a.frames <= 0 or a.window <= 0 or a.warmup_frames < 0:
        ap.error("lanes, frames and window must be positive, warmup-frames >= 0")
    if a.intelligibility and a.window < 2:
        ap.error("--intelligibility needs a window of at least 2 frames")
    try:
        rep = evaluate(tr.glob_paths(a.signal_glob), tr.glob_paths(a.noise_glob), a.model, limits, a.lanes, a.frames, a.seed, a.window,
                       a.warmup_frames, a.device, a.shuffle, a.intelligibility)
    except (NnnoiselessError, OSError) as e:
        print("error: %s" % e, file=sys.stderr)
        return 1
    print(format_table(rep))
    print("%d lanes x %d frames x %d variants in %.2f s" % (rep["lanes"], rep["frames"], len(rep["variants"]), rep["seconds"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(_jsonable(rep), f)
    return 0


if __name__ == "__main__":
    sys.exit(main())
