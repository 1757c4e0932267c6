"""Float64 restatement of the metrics accumulator (rnnoise_metrics_accumulate_device, DESIGN.md 7p).

TEST INFRASTRUCTURE.  Frame by frame, with the one-frame lag, the classes and the half-window pairing state of the
kernel.  Band energies come from spectral_ref (rfft_windowed and the band weights W), or from the caller: the GPU's own
per-frame last_bands, so that the log-domain sums can be checked from the kernel's own inputs.

Bounds (DESIGN.md 7p, "Checks"):
- band energies (band_yardstick): per band, K x max(d32 of the band, the spectrum's d32 propagated to first order
  through the band weights: spectral_ref.analysis_bounds), where d32 is the larger deviation from float64 of the
  oracle's transform_input under its two f32 FFT orders (0 and 2).  The only absolute floor is the smallest normal
  f32, taken off the error where the float64 value is below it (band_excess).
- time-domain sums (MetricsRef.time_bounds): 2 gamma_n sum |terms| in double, n = 480 per frame + the frame count + 2 (the
  difference y - c and its square are rounded): the kernel's sum and the reference's each lie within gamma_n sum |terms|
  of the exact one."""
import numpy as np

import oracle_state as ost
import spectral_ref as sr

F = 480
NB = 22
K = 10.0
U64 = 2.0 ** -53
F32_TINY = float(np.finfo(np.float32).tiny)


def record_dtype():
    import nnnoiseless_b200 as nb
    return nb.METRICS_DTYPE


def band_energies(prev, cur):
    """The analysis kernel's ex of the windows [prev | cur], [B][480] each -> [B][22] float64."""
    X = sr.rfft_windowed(np.concatenate([prev, cur], axis=1))
    return np.abs(X) ** 2 @ sr.tables()["W"].T


def band_yardstick(prev, cur):
    """The windows [prev | cur] ([n][480] float32 values each) -> (ex [n][22] float64, tol [n][22]): the float64 band
    energies and K x their per-band bound (the module docstring), with the oracle's f32 transform_input as yardstick."""
    w = np.concatenate([np.asarray(prev, np.float32), np.asarray(cur, np.float32)], axis=1)
    n = len(w)
    mem = np.zeros((n, 1728))
    mem[:, 768:] = w
    ref = sr.analysis(mem, np.zeros(n, np.int64), np.zeros((n, 8, NB)), np.zeros(n, np.int64))
    o32 = []
    for mode in (0, 2):
        ost.set_fft_mode(mode)
        try:
            o32.append(ost.band_energies(w))
        finally:
            ost.set_fft_mode(0)
    dX = np.max([np.abs(X.astype(np.complex128) - ref["X"]).max(axis=1) for X, _ in o32], axis=0)[:, None]
    dex = np.max([np.abs(ex.astype(np.float64) - ref["ex"]) for _, ex in o32], axis=0)
    return ref["ex"], K * sr.analysis_bounds(ref, dX, dX, band={"ex": dex})["ex"]


def oracle_bands(prev, cur, mode):
    """The oracle's f32 band energies of the windows [prev | cur] under FFT order `mode` -> [n][22] float32."""
    ost.set_fft_mode(mode)
    try:
        return ost.band_energies(np.concatenate([np.asarray(prev, np.float32), np.asarray(cur, np.float32)], axis=1))[1]
    finally:
        ost.set_fft_mode(0)


def band_excess(got, ref):
    """|got - ref|, less the smallest normal f32 where the float64 value is below it (f32 may flush it to zero)."""
    e = np.abs(np.asarray(got, np.float64) - ref)
    return np.where(np.abs(ref) < F32_TINY, np.maximum(e - F32_TINY, 0.0), e)


def share(err, tol):
    """err / tol elementwise, with 0 / 0 = 0 (a zero bound requires a zero error)."""
    err, tol = np.broadcast_arrays(np.asarray(err, np.float64), np.asarray(tol, np.float64))
    out = np.zeros(err.shape)
    nz = tol > 0
    out[nz] = err[nz] / tol[nz]
    out[~nz & (err > 0)] = np.inf
    return out


def gamma(n):
    """gamma_n = n u / (1 - n u) in double."""
    n = np.asarray(n, np.float64)
    return n * U64 / (1.0 - n * U64)


def log_excess_bound(e, tol):
    """Largest change of 10 log10(E + 0.01) when E >= 0 moves by at most tol from e."""
    down = np.log10((e + 0.01) / (np.maximum(e - tol, 0.0) + 0.01))
    return 10.0 * np.maximum(down, np.log10((e + tol + 0.01) / (e + 0.01)))


def seg_snr(ec, ed):
    if ed == 0.0:
        return 35.0
    if ec == 0.0:
        return -10.0
    return min(max(10.0 * np.log10(ec / ed), -10.0), 35.0)


class MetricsRef:
    def __init__(self, B):
        self.B = B
        self.yh = np.zeros((B, F))
        self.ch = np.zeros((B, F))
        self.cl = np.zeros((B, F))
        self.tl = np.zeros(B)
        self.started = np.zeros(B, bool)
        self.rec = np.zeros(B, record_dtype())
        self.abs_ecy = np.zeros((B, 3))  # sum |c y| per class: the terms of ecy
        self.log_tol = {k: np.zeros(self.rec[k].shape) for k in ("lsd", "speech_dev", "noise_level")}

    def clear(self, streams=None):
        s = np.arange(self.B) if streams is None else np.asarray(streams)
        self.rec[s] = np.zeros(1, record_dtype())
        self.abs_ecy[s] = 0.0
        for v in self.log_tol.values():
            v[s] = 0.0

    def time_bounds(self):
        """Bounds on |GPU - reference| of ec, ey, ecy, ed [B][3] (the module docstring)."""
        r = self.rec
        g = 2.0 * gamma(F + r["frames"] + 2)
        return dict(ec=g * r["ec"], ey=g * r["ey"], ecy=g * self.abs_ecy, ed=g * r["ed"])

    def accumulate(self, out, clean, vad=None, target=None, bands=None, band_tol=None):
        """out, clean [B][T][480] (float32 values); vad, target [B][T] or None; bands: [T][2][B][22] band energies to use
        instead of float64 ones (the GPU's per-frame last_bands), or None.  band_tol [T][2][B][22]: bounds on how far
        band energies computed elsewhere may lie from the ones used here; log_tol then bounds how far the log-domain
        sums computed from those may lie from these (lsd, speech_dev, noise_level)."""
        out = np.asarray(out, np.float64)
        clean = np.asarray(clean, np.float64)
        B, T = out.shape[:2]
        r = self.rec
        for j in range(T):
            y = out[:, j]
            c = self.cl if j == 0 else clean[:, j - 1]
            yh = self.yh if j == 0 else out[:, j - 1]
            ch = self.ch if j == 0 else (self.cl if j == 1 else clean[:, j - 2])
            tgt_c = self.tl if j == 0 else (np.asarray(target, np.float64)[:, j - 1] if target is not None else np.full(B, 0.5))
            tgt_now = np.asarray(target, np.float64)[:, j] if target is not None else np.full(B, 0.5)
            if bands is not None:
                Yb, Cb = np.asarray(bands[j][0], np.float64), np.asarray(bands[j][1], np.float64)
            else:
                Yb, Cb = band_energies(yh, y), band_energies(ch, c)
            Ly, Lc = 10.0 * np.log10(Yb + 0.01), 10.0 * np.log10(Cb + 0.01)
            if band_tol is not None:
                dLy, dLc = log_excess_bound(Yb, band_tol[j][0]), log_excess_bound(Cb, band_tol[j][1])
            for s in range(B):
                if not (self.started[s] or j > 0):
                    continue
                ec, ey, ecy, ed = (c[s] ** 2).sum(), (y[s] ** 2).sum(), (c[s] * y[s]).sum(), ((y[s] - c[s]) ** 2).sum()
                classes = [0] + ([1] if tgt_c[s] == 1.0 else []) + ([2] if tgt_c[s] == 0.0 else [])
                for q in classes:
                    r["frames"][s, q] += 1
                    r["ec"][s, q] += ec
                    r["ey"][s, q] += ey
                    r["ecy"][s, q] += ecy
                    r["ed"][s, q] += ed
                    self.abs_ecy[s, q] += np.abs(c[s] * y[s]).sum()
                d = Ly[s] - Lc[s]
                if tgt_c[s] == 1.0:
                    r["seg_snr"][s] += seg_snr(ec, ed)
                    r["lsd"][s] += np.sqrt((d * d).mean())
                    r["speech_dev"][s] += d
                    if band_tol is not None:  # |rms(d) - rms(d')| <= rms(d - d') <= max |d - d'|
                        self.log_tol["lsd"][s] += (dLy[s] + dLc[s]).max()
                        self.log_tol["speech_dev"][s] += dLy[s] + dLc[s]
                if tgt_c[s] == 0.0:
                    r["noise_level"][s] += Ly[s]
                    if band_tol is not None:
                        self.log_tol["noise_level"][s] += dLy[s]
                if vad is not None and target is not None and tgt_now[s] in (0.0, 1.0):
                    said, is_ = vad[s][j] >= 0.5, tgt_now[s] == 1.0
                    r["vad_counts"][s, 0 if said and is_ else (1 if said else (2 if is_ else 3))] += 1
                r["last_bands"][s, 0] = Yb[s]
                r["last_bands"][s, 1] = Cb[s]
        # the pairing state
        T1 = T - 1
        self.ch = (self.cl if T == 1 else clean[:, T - 2]).copy()
        self.yh = out[:, T1].copy()
        self.cl = clean[:, T1].copy()
        self.tl = np.asarray(target, np.float64)[:, T1].copy() if target is not None else np.full(B, 0.5)
        self.started[:] = True
        return r
