"""Float64 reference of the two spectral stages of a frame, vectorised over streams.

TEST INFRASTRUCTURE.  `analysis` restates src/features.rs:115-219 and 281-298 with src/lib.rs:65-82 and 139-148 (the
windowed forward FFTs of the current and pitch-lagged windows, band energies and correlation, the 42 features, the
cepstral ring); `synthesis` restates src/features.rs:223-275 with src/lib.rs:84-97 and src/denoise.rs:102-115 (pitch
filter, gain floor, band-gain interpolation, inverse FFT, window, overlap-add).

Constants the kernels receive as f32 enter as those f32 values widened to float64: the window, wnorm and DCT tables (the
oracle's own, which the GPU's tables equal) and the literals 0.001, 1e-8, 0.6, 1e-2, 0.04, 2.1, 12, 4, 1.3 and 0.9.
Everything else is evaluated in float64, so that a comparison measures a kernel's arithmetic and not table rounding.
"""
import numpy as np

import oracle_state as ost

NB_BANDS = 22
NB_FEATURES = 42
NB_DELTA_CEPS = 6
CEPS_MEM = 8
FREQ_SIZE = 481
NB_BINS_BANDED = 400
EBAND_5MS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 34, 40, 48, 60, 78, 100]

f = lambda v: float(np.float32(v))  # noqa: E731  an f32 literal, widened
C_CORR, C_EPS, C_FLOOR, C_LOG, C_SIL, C_SV = f(0.001), f(1e-8), f(0.6), f(1e-2), f(0.04), f(2.1)
C_C0, C_C1, C_P0, C_P1 = f(12.0), f(4.0), f(1.3), f(0.9)

_T = None


def tables():
    """dict(window [960], dct [22][22], wnorm, W [22][481], M [481][22]) in float64.  W: the band-sum weights (exact
    fractions j / size, first and last band doubled); M: the band-gain interpolation (rows >= 400 zero)."""
    global _T
    if _T is None:
        window, dct, wnorm = ost.spectral_tables()
        W = np.zeros((NB_BANDS, FREQ_SIZE))
        M = np.zeros((FREQ_SIZE, NB_BANDS))
        for i in range(NB_BANDS - 1):
            size = (EBAND_5MS[i + 1] - EBAND_5MS[i]) * 4
            for j in range(size):
                k, fr = EBAND_5MS[i] * 4 + j, j / size
                W[i, k] += 1.0 - fr
                W[i + 1, k] += fr
                M[k, i], M[k, i + 1] = 1.0 - fr, fr
        W[0] *= 2.0
        W[-1] *= 2.0
        _T = dict(window=window.astype(np.float64), dct=dct.astype(np.float64), wnorm=float(wnorm), W=W, M=M)
    return _T


def rfft_windowed(frames):
    """frames [B][960] -> rfft(window * frames) * wnorm, [B][481] complex128."""
    t = tables()
    return np.fft.rfft(np.asarray(frames, np.float64) * t["window"], axis=-1) * t["wnorm"]


def _dct(x):
    """src/lib.rs:139-148: out[i] = sqrt(2/22) sum_j x[j] dct[j][i]."""
    return (np.asarray(x, np.float64) @ tables()["dct"]) * np.sqrt(2.0 / NB_BANDS)


def log_energies(ex):
    """src/features.rs:147-158: log10(1e-2 + ex) with the sequential follower -> ly [B][22]."""
    lg = np.log10(C_LOG + np.asarray(ex, np.float64))
    ly = np.empty_like(lg)
    log_max = np.full(lg.shape[0], -2.0)
    follow = np.full(lg.shape[0], -2.0)
    for i in range(NB_BANDS):
        ly[:, i] = np.maximum(np.maximum(lg[:, i], log_max - 7.0), follow - 1.5)
        log_max = np.maximum(log_max, ly[:, i])
        follow = np.maximum(follow - 1.5, ly[:, i])
    return ly


def analysis(input_mem, pitch, ceps_ring, mem_id):
    """K3 for B streams: input_mem [B][1728] (after the frame's high-pass), pitch [B], ceps_ring [B][8][22] and mem_id [B]
    (before the frame) -> dict(X [B][481], P [B][481], ex, ep, corr, exp [B][22], e [B] (sum of ex), ly [B][22],
    features [B][42] (as if the frame were not silent), silence [B] bool, row [B][22] (the new cepstral row), ring [B][8][22]
    and mem_id [B] after a non-silent frame)."""
    x = np.asarray(input_mem, np.float64)
    pitch = np.asarray(pitch, np.int64)
    mem_id = np.asarray(mem_id, np.int64)
    B = len(x)
    W = tables()["W"]
    X = rfft_windowed(x[:, 768:1728])
    lag = 768 - pitch[:, None] + np.arange(960)[None, :]
    P = rfft_windowed(np.take_along_axis(x, lag, axis=1))
    ex = np.abs(X) ** 2 @ W.T
    ep = np.abs(P) ** 2 @ W.T
    corr = (X.real * P.real + X.imag * P.imag) @ W.T
    exp = corr / np.sqrt(C_CORR + ex * ep)
    e = ex.sum(axis=1)
    ly = log_energies(ex)
    feat = np.zeros((B, NB_FEATURES))
    ceps = _dct(ly)
    ceps[:, 0] -= C_C0
    ceps[:, 1] -= C_C1
    pcor = _dct(exp)[:, :NB_DELTA_CEPS]
    pcor[:, 0] -= C_P0
    pcor[:, 1] -= C_P1
    ring = np.array(ceps_ring, np.float64)
    rows = np.arange(B)
    ring[rows, mem_id] = ceps
    c1 = (mem_id - 1) % CEPS_MEM
    c2 = (mem_id - 2) % CEPS_MEM
    a, b, c = ring[rows, mem_id, :NB_DELTA_CEPS], ring[rows, c1, :NB_DELTA_CEPS], ring[rows, c2, :NB_DELTA_CEPS]
    feat[:, :NB_BANDS] = ceps
    feat[:, :NB_DELTA_CEPS] = a + b + c
    feat[:, NB_BANDS:NB_BANDS + NB_DELTA_CEPS] = a - c
    feat[:, NB_BANDS + NB_DELTA_CEPS:NB_BANDS + 2 * NB_DELTA_CEPS] = a - 2.0 * b + c
    feat[:, NB_BANDS + 2 * NB_DELTA_CEPS:NB_BANDS + 3 * NB_DELTA_CEPS] = pcor
    feat[:, NB_BANDS + 3 * NB_DELTA_CEPS] = f(0.01) * (pitch - 300.0)
    d = ((ring[:, :, None, :] - ring[:, None, :, :]) ** 2).sum(axis=3)
    d[:, np.arange(CEPS_MEM), np.arange(CEPS_MEM)] = np.inf
    feat[:, NB_BANDS + 3 * NB_DELTA_CEPS + 1] = d.min(axis=2).sum(axis=1) / CEPS_MEM - C_SV
    return dict(X=X, P=P, ex=ex, ep=ep, corr=corr, exp=exp, e=e, ly=ly, features=feat, silence=e < C_SIL, row=ceps,
                ring=ring, mem_id=(mem_id + 1) % CEPS_MEM)


def synthesis(X, P, ex, ep, exp, raw_gains, lastg, synth_mem, silence):
    """K5 for B streams: X [B][481] and P [B][>= 400] complex, ex, ep, exp, raw_gains, lastg [B][22], synth_mem [B][480],
    silence [B] -> dict(out [B][480], lastg [B][22], synth_mem [B][480], branch [B][22] bool (exp > g: the pitch filter's
    r = 1 branch), floor [B][22] bool (0.6 lastg > g: the gain floor is taken))."""
    t = tables()
    W, M = t["W"], t["M"]
    X = np.asarray(X, np.complex128)
    Pb = np.zeros_like(X)
    Pb[:, :NB_BINS_BANDED] = np.asarray(P, np.complex128)[:, :NB_BINS_BANDED]
    ex, ep, exp = (np.asarray(a, np.float64) for a in (ex, ep, exp))
    g, lg = np.asarray(raw_gains, np.float64), np.asarray(lastg, np.float64)
    sil = np.asarray(silence, bool)
    # pitch filter (src/features.rs:223-257)
    e2, g2 = exp * exp, g * g
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(exp > g, 1.0, e2 * (1.0 - g2) / (C_CORR + g2 * (1.0 - e2)))
    r = np.sqrt(np.clip(r, 0.0, 1.0)) * np.sqrt(ex / (C_EPS + ep))
    rf = r @ M.T
    x = X + Pb * rf
    x = x.real + 1j * np.where(np.arange(FREQ_SIZE) == 0, X.imag, x.imag)  # DC is a real offset: its imaginary part stays
    new_e = np.abs(x) ** 2 @ W.T
    s2 = np.sqrt(ex / (C_EPS + new_e))
    rf2 = s2 @ M.T
    gg = np.maximum(g, C_FLOOR * lg)
    gf = gg @ M.T
    y = np.where(sil[:, None], X, x * rf2 * gf)
    new_lastg = np.where(sil[:, None], lg, gg)
    # frame synthesis (src/features.rs:263-275): the unnormalised inverse FFT, halved and windowed, overlap-added
    w = 960.0 * np.fft.irfft(y, n=960, axis=-1) / 2.0 * t["window"]
    out = w[:, :480] + np.asarray(synth_mem, np.float64)
    return dict(out=out, lastg=new_lastg, synth_mem=w[:, 480:], branch=exp > g, floor=C_FLOOR * lg > g, X=X, Pb=Pb, x=x,
                y=y, w=w, r=r, rf=rf, new_e=new_e, s2=s2, rf2=rf2, gg=gg, gf=gf, e2=e2, g2=g2, silence=sil)


# ---- first-order error bounds -------------------------------------------------------------------------------------
U = 2.0 ** -24  # f32 unit roundoff
MAX_BAND_TERMS = 160  # a band sum takes the frac part of one segment and the (1 - frac) part of the next: <= 72 + 88 bins


def analysis_bounds(ref, dX, dP, band=None, arith=False):
    """Absolute error bounds of the analysis outputs, to first order, from bounds on the spectra: dX [B][481] and dP
    [B][481] per bin (or [B][1] for every bin).  band: dict of per-band bounds [B][22] on ex, ep and exp known
    otherwise (each band takes the larger).  arith: add the rounding of the f32 arithmetic after the FFT (band sums of
    up to 160 terms, the table fractions j / size rounded to f32, the normalisation, log10, both DCTs of 22 terms, the
    delta features, the spectral variability).  -> dict(ex, ep, corr, exp, e [B], row [B][22], features [B][42])."""
    t = tables()
    W, D = t["W"], np.abs(t["dct"]) * np.sqrt(2.0 / NB_BANDS)
    band = band or {}
    aX, aP = np.abs(ref["X"]), np.abs(ref["P"]).copy()
    aP[:, NB_BINS_BANDED:] = 0.0
    dP = np.where(np.arange(FREQ_SIZE) < NB_BINS_BANDED, dP, 0.0)
    ex = (2 * aX * dX + dX * dX) @ W.T
    ep = (2 * aP * dP + dP * dP) @ W.T
    corr = (aX * dP + aP * dX + dX * dP) @ W.T
    if arith:
        ex = ex + (MAX_BAND_TERMS + 5) * U * ref["ex"]
        ep = ep + (MAX_BAND_TERMS + 5) * U * ref["ep"]
        corr = corr + (MAX_BAND_TERMS + 5) * U * ((aX * aP) @ W.T)
    ex = np.maximum(ex, band.get("ex", 0.0))
    ep = np.maximum(ep, band.get("ep", 0.0))
    den = np.sqrt(C_CORR + ref["ex"] * ref["ep"])
    dden = (ref["ex"] * ep + ref["ep"] * ex) / (2 * den)
    exp = corr / den + np.abs(ref["corr"]) * dden / den ** 2 + (4 * U * np.abs(ref["exp"]) if arith else 0.0)
    exp = np.maximum(exp, band.get("exp", 0.0))
    # log energies: the follower (running maxima) moves no output by more than the largest input change so far
    lg = np.abs(np.log10(C_LOG + ref["ex"]))
    dlg = ex / ((C_LOG + ref["ex"]) * np.log(10.0)) + ((2 * lg + 1.0 / np.log(10.0)) * U if arith else 0.0)
    dly = np.maximum.accumulate(dlg, axis=1)
    row = dly @ D
    pcor = exp @ D[:, :NB_DELTA_CEPS]
    if arith:
        row = row + (NB_BANDS + 1) * U * (np.abs(ref["ly"]) @ D) + 3 * U * np.abs(ref["row"])
        pcor = pcor + (NB_BANDS + 1) * U * (np.abs(ref["exp"]) @ D[:, :NB_DELTA_CEPS]) + 3 * U * np.abs(ref["features"][:, 34:40])
    # spectral variability: only the distances to the new row move, each by at most 2 |row - ring_j| |d row| + |d row|^2
    rr = np.sqrt((row ** 2).sum(axis=1))
    dist2 = ((ref["ring"] - ref["row"][:, None, :]) ** 2).sum(axis=2)
    sv = 2 * np.sqrt(dist2.max(axis=1)) * rr + rr * rr
    feat = np.zeros_like(ref["features"])
    n6, nb = NB_DELTA_CEPS, NB_BANDS
    feat[:, :nb] = row
    feat[:, nb:nb + n6] = row[:, :n6]
    feat[:, nb + n6:nb + 2 * n6] = row[:, :n6]
    feat[:, nb + 2 * n6:nb + 3 * n6] = pcor
    feat[:, nb + 3 * n6 + 1] = sv
    if arith:
        rows = np.arange(len(feat))
        mid = (ref["mem_id"] - 1) % CEPS_MEM
        a = np.abs(ref["ring"][rows, mid, :n6])
        b = np.abs(ref["ring"][rows, (mid - 1) % CEPS_MEM, :n6])
        c = np.abs(ref["ring"][rows, (mid - 2) % CEPS_MEM, :n6])
        feat[:, :n6] += 2 * U * (a + b + c)
        feat[:, nb:nb + n6] += U * (a + c)
        feat[:, nb + n6:nb + 2 * n6] += 2 * U * (a + 2 * b + c)
        feat[:, nb + 3 * n6] = U * np.abs(ref["features"][:, nb + 3 * n6])
        mins = ref["features"][:, nb + 3 * n6 + 1] + C_SV
        feat[:, nb + 3 * n6 + 1] += (NB_BANDS + 2 + CEPS_MEM) * U * np.abs(mins) + U * np.abs(ref["features"][:, nb + 3 * n6 + 1])
    return dict(ex=ex, ep=ep, corr=corr, exp=exp, e=ex.sum(axis=1), row=row, features=feat)


def windowing_bounds(input_mem, pitch):
    """Per stream, the error every f32 analysis makes in each bin before its FFT: the products window x input are rounded
    (u |x w| per sample, summed into a bin with weight wnorm) -> (dX [B][1], dP [B][1])."""
    t = tables()
    x = np.abs(np.asarray(input_mem, np.float64))
    lag = 768 - np.asarray(pitch, np.int64)[:, None] + np.arange(960)[None, :]
    dX = U * t["wnorm"] * (x[:, 768:1728] * t["window"]).sum(axis=1)
    dP = U * t["wnorm"] * (np.take_along_axis(x, lag, axis=1) * t["window"]).sum(axis=1)
    return dX[:, None], dP[:, None]


def spectrum_bounds(ref, eps_ratio, dgg=None):
    """First-order absolute bounds of the f32 values every f32 synthesis forms on its way to y, on the inputs of `ref`
    (a `synthesis` result): eps_ratio [B][22] bounds the relative error of the pitch filter's sqrt(ratio) before its own
    rounding; dgg [B][22] bounds gg (default: one rounding of 0.6 lastg).  -> dict(drf, dx, dne, ds2, drf2, dgf): r's
    interpolation with the f32 fractions j / size, x = X + P rf [B][481], the band sums of the new energies (up to
    MAX_BAND_TERMS terms in any order), s2 = sqrt(ex / (1e-8 + new_e)) [B][22] and the interpolated rf2 and gf."""
    M, W = tables()["M"], tables()["W"]
    r = ref["r"]
    eps_r = eps_ratio + 4 * U  # sqrt of the ratio, sqrt(ex / (1e-8 + ep)), the product
    drf = (r * eps_r) @ M.T + 4 * U * (r @ M.T)  # the fractions j / size are rounded to f32
    ax1 = np.abs(ref["x"])
    dx1 = np.abs(ref["Pb"]) * drf + 2 * U * (np.abs(ref["X"]) + np.abs(ref["Pb"]) * ref["rf"])
    dne = (2 * ax1 * dx1 + dx1 * dx1) @ W.T + (MAX_BAND_TERMS + 5) * U * ref["new_e"]
    ds2 = ref["s2"] * (dne / (2 * (C_EPS + ref["new_e"])) + 3 * U)
    drf2 = ds2 @ M.T + 4 * U * ref["rf2"]
    dgg = U * ref["gg"] if dgg is None else dgg  # 0.6 lastg is rounded once
    dgf = dgg @ M.T + 4 * U * ref["gf"]
    return dict(drf=drf, dx=dx1, dne=dne, ds2=ds2, drf2=drf2, dgf=dgf)


def synthesis_bounds(ref):
    """Absolute bounds [B][480] on out and synth_mem for the rounding of the f32 arithmetic every f32 synthesis does
    around its inverse FFT on the same inputs (the FFT itself excluded), to first order: the pitch-filter ratio r (with
    the cancellation in 1 - g^2 and 1 - exp^2), the interpolations with their f32 fractions, x + p rf, the band sums
    of the new energies, the renormalisation and gains (spectrum_bounds), then per time sample the spectrum's error
    through the unnormalised inverse FFT (|y_n| <= |x_0| / 2 + |x_480| / 2 + sum |x_k| after halving) and the window,
    halving and overlap-add.  -> (d_out, d_synth_mem)."""
    t = tables()
    live = ~ref["silence"][:, None]
    e2, g2 = ref["e2"], ref["g2"]
    with np.errstate(divide="ignore", invalid="ignore"):
        cancel = np.nan_to_num(g2 / np.abs(1.0 - g2) + e2 / np.abs(1.0 - e2), posinf=1e30)
    eps_ratio = np.where(ref["branch"], 0.0, 0.5 * (8 * U + U * cancel))
    b = spectrum_bounds(ref, eps_ratio)
    ax1, dx1, drf2, dgf = np.abs(ref["x"]), b["dx"], b["drf2"], b["dgf"]
    dx = dx1 * ref["rf2"] * ref["gf"] + ax1 * (drf2 * ref["gf"] + ref["rf2"] * dgf) + 2 * U * np.abs(ref["y"])
    dx = np.where(live, dx, 0.0)
    c = np.ones(FREQ_SIZE)
    c[0] = c[-1] = 0.5
    dy = (dx * c).sum(axis=1)[:, None] * t["window"] + U * np.abs(ref["w"])
    return dy[:, :480] + U * np.abs(ref["out"]), dy[:, 480:]
