"""Per-stream quality figures from Metrics records (METRICS_DTYPE, DESIGN.md 7p).  Host code; needs no GPU.

``summarize(records, baseline=None)`` -> dict of float64 arrays, one value per record:
- snr: 10 log10(Ec / Ed) over all counted frames;
- si_sdr: 10 log10(Ecy^2 / (Ec Ey - Ecy^2)) over all counted frames (+inf when the denominator is <= 0);
- seg_snr, lsd: means over speech frames;
- speech_level: 10 log10(Ey / Ec) over speech frames;  speech_dev [n][22]: mean Ly_b - Lc_b over speech frames;
- vad_precision, vad_recall: from the tp / fp / fn counts.
With ``baseline`` (the records of the unprocessed stream of the same lanes) also:
- noise_atten: 10 log10(Ey_noise(baseline) / Ey_noise);  noise_atten_bands [n][22]: the per-band noise level's drop;
- delta_snr, delta_si_sdr: the paired differences against the baseline.
A figure with no frames to define it is NaN; ``nan_counts`` counts them per figure."""
import numpy as np

ALL, SPEECH, NOISE = 0, 1, 2


def _db(num, den):
    """10 log10(num / den) in float64: +inf for x / 0, -inf for 0 / x, NaN for 0 / 0."""
    num, den = np.asarray(num, np.float64), np.asarray(den, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where((num == 0) & (den == 0), np.nan, 10.0 * np.log10(num / den))


def _mean(total, n):
    with np.errstate(divide="ignore", invalid="ignore"):
        n = np.asarray(n, np.float64)
        total = np.asarray(total, np.float64)
        nn = n.reshape(n.shape + (1,) * (total.ndim - n.ndim))
        return np.where(nn > 0, total / np.where(nn > 0, nn, 1.0), np.nan)


def si_sdr(ec, ey, ecy):
    """10 log10(Ecy^2 / (Ec Ey - Ecy^2)); +inf when the denominator is <= 0, NaN when Ec or Ecy is 0."""
    ec, ey, ecy = (np.asarray(v, np.float64) for v in (ec, ey, ecy))
    num = ecy * ecy
    den = ec * ey - num
    with np.errstate(divide="ignore", invalid="ignore"):
        v = 10.0 * np.log10(num / np.where(den > 0, den, 1.0))
    return np.where((ec <= 0) | (num <= 0), np.nan, np.where(den <= 0, np.inf, v))


def summarize(records, baseline=None):
    r = np.asarray(records)
    fr = r["frames"]
    out = {
        "snr": np.where(fr[:, ALL] > 0, _db(r["ec"][:, ALL], r["ed"][:, ALL]), np.nan),
        "si_sdr": np.where(fr[:, ALL] > 0, si_sdr(r["ec"][:, ALL], r["ey"][:, ALL], r["ecy"][:, ALL]), np.nan),
        "seg_snr": _mean(r["seg_snr"], fr[:, SPEECH]),
        "lsd": _mean(r["lsd"], fr[:, SPEECH]),
        "speech_level": np.where(fr[:, SPEECH] > 0, _db(r["ey"][:, SPEECH], r["ec"][:, SPEECH]), np.nan),
        "speech_dev": _mean(r["speech_dev"], fr[:, SPEECH]),
    }
    tp, fp, fn = (r["vad_counts"][:, k].astype(np.float64) for k in range(3))
    with np.errstate(divide="ignore", invalid="ignore"):
        out["vad_precision"] = np.where(tp + fp > 0, tp / (tp + fp), np.nan)
        out["vad_recall"] = np.where(tp + fn > 0, tp / (tp + fn), np.nan)
    if baseline is not None:
        b = np.asarray(baseline)
        if b.shape != r.shape:
            raise ValueError("baseline has %d records for %d" % (b.size, r.size))
        fn_v, fn_b = fr[:, NOISE], b["frames"][:, NOISE]
        ok = (fn_v > 0) & (fn_b > 0)
        out["noise_atten"] = np.where(ok, _db(b["ey"][:, NOISE], r["ey"][:, NOISE]), np.nan)
        with np.errstate(invalid="ignore"):
            out["noise_atten_bands"] = np.where(ok[:, None], _mean(b["noise_level"], fn_b) - _mean(r["noise_level"], fn_v), np.nan)
        base = summarize(b)
        with np.errstate(invalid="ignore"):
            out["delta_snr"] = out["snr"] - base["snr"]
            out["delta_si_sdr"] = out["si_sdr"] - base["si_sdr"]
    out["nan_counts"] = {k: int(np.isnan(v).any(axis=tuple(range(1, v.ndim))).sum()) for k, v in out.items()}
    return out
