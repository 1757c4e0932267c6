"""Float64 restatement of the metrics accumulator (rnnoise_metrics_accumulate_device, DESIGN.md 7p).

TEST INFRASTRUCTURE.  Frame by frame, with the one-frame lag, the classes and the half-window pairing state of the
kernel.  Band energies come from spectral_ref (rfft_windowed and the band weights W), or from the caller: the GPU's own
per-frame last_bands, so that the log-domain sums can be checked from the kernel's own inputs."""
import numpy as np

import spectral_ref as sr

F = 480
NB = 22


def record_dtype():
    import nnnoiseless_b200 as nb
    return nb.METRICS_DTYPE


def band_energies(prev, cur):
    """The analysis kernel's ex of the windows [prev | cur], [B][480] each -> [B][22] float64."""
    X = sr.rfft_windowed(np.concatenate([prev, cur], axis=1))
    return np.abs(X) ** 2 @ sr.tables()["W"].T


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

    def clear(self, streams=None):
        self.rec[np.arange(self.B) if streams is None else np.asarray(streams)] = np.zeros(1, record_dtype())

    def accumulate(self, out, clean, vad=None, target=None, bands=None):
        """out, clean [B][T][480] (float32 values); vad, target [B][T] or None; bands: [T][2][B][22] band energies to use
        instead of float64 ones (the GPU's per-frame last_bands), or None."""
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
                d = Ly[s] - Lc[s]
                if tgt_c[s] == 1.0:
                    r["seg_snr"][s] += seg_snr(ec, ed)
                    r["lsd"][s] += np.sqrt((d * d).mean())
                    r["speech_dev"][s] += d
                if tgt_c[s] == 0.0:
                    r["noise_level"][s] += Ly[s]
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
