"""Float64 restatement of the STOI / ESTOI backward, rnnoise_intelligibility_backward_device (include/rnnoise.h,
DESIGN.md 7r).

Each stage is a function of its own inputs, so the GPU tests can feed it the GPU's intermediate results (the forward
and backward workspace taps) and check one stage at a time:
- ``score_bwd``: d bands of out from the float bands, the kernel's operations in the kernel's order (unfused, as the
  unit is built), so from the same bands it gives the kernel's d bands to the rounding of a few sums;
- ``bands_bwd``, ``ola_bwd``, ``resample_bwd``: the exact adjoints of the linear stages (and of the band magnitudes at
  given bands), each with the sums of absolute values its rounding bound scales.
``torch_intelligibility`` transcribes stoi_ref's definition into torch, for float64 autograd as an independent check."""
import numpy as np

import stoi_ref as sr

EPS, NSEG, NBANDS, HOP, FRAME = sr.EPS, sr.NSEG, sr.NBANDS, sr.HOP, sr.FRAME
LO, HI = int(sr.EDGES[0]), int(sr.EDGES[-1])
BAND_OF_BIN = np.concatenate([np.full(sr.EDGES[b + 1] - sr.EDGES[b], b) for b in range(NBANDS)])  # bins LO..HI-1


def _sum(v, axis):
    """Sum along axis in index order (the kernel's)."""
    v = np.moveaxis(v, axis, -1)
    s = np.zeros(v.shape[:-1])
    for i in range(v.shape[-1]):
        s = s + v[..., i]
    return s


def _normalise_bwd(d, g, r, axis):
    """dL/dv from g = dL/d(d / (r + EPS)), d = v - mean v centred along axis, r = ||d||: normalise_bwd's operations."""
    d, g = np.moveaxis(d, axis, -1), np.moveaxis(g, axis, -1)
    D = r + EPS
    s = _sum(g * d, -1)
    with np.errstate(divide="ignore", invalid="ignore"):
        coef = np.where(r > 0.0, -(s / (D * D)) / np.where(r > 0, r, 1.0), 0.0)
    g = g / D[..., None] + coef[..., None] * d
    m = _sum(g, -1) / g.shape[-1]
    return np.moveaxis(g - m[..., None], -1, axis)


def _centre(v, axis):
    """(v - mean v, ||v - mean v||) along axis, sums in order."""
    v = np.moveaxis(v, axis, -1)
    m = _sum(v, -1) / v.shape[-1]
    d = v - m[..., None]
    return np.moveaxis(d, -1, axis), np.sqrt(_sum(d * d, -1))


def score_bwd(bx, by, grad_stoi, grad_estoi):
    """dL/d by [15][M] of L = grad_stoi stoi + grad_estoi estoi at float band matrices bx, by [15][M] (taken as
    float64); a None gradient skips its term.  Zeros for S < 1."""
    bx, by = np.asarray(bx, np.float64), np.asarray(by, np.float64)
    M = bx.shape[1]
    S = M - NSEG + 1
    acc = np.zeros((NBANDS, M))
    if S < 1:
        return acc
    X = np.lib.stride_tricks.sliding_window_view(bx, NSEG, axis=1)[:, :S].transpose(1, 0, 2)  # [S][15][30]
    Y = np.lib.stride_tricks.sliding_window_view(by, NSEG, axis=1)[:, :S].transpose(1, 0, 2)
    parts = []
    if grad_stoi is not None:
        gst = grad_stoi / float(NBANDS * S)
        nx, ny = _sum(X * X, 2), _sum(Y * Y, 2)
        sy = np.sqrt(ny)
        alpha = (np.sqrt(nx) / (sy + EPS))[..., None]
        Yc = np.minimum(alpha * Y, sr.CLIP * X)
        mx, my = _sum(X, 2) / NSEG, _sum(Yc, 2) / NSEG
        dx, dy = X - mx[..., None], Yc - my[..., None]
        sxy, sxx, syy = _sum(dx * dy, 2), _sum(dx * dx, 2), _sum(dy * dy, 2)
        ry = np.sqrt(syy)
        Dy = ry + EPS
        den = (np.sqrt(sxx) + EPS) * Dy
        term = sxy / den
        dsxy = gst / den
        with np.errstate(divide="ignore", invalid="ignore"):
            coef = np.where(ry > 0.0, -(gst * term) / (Dy * np.where(ry > 0, ry, 1.0)), 0.0)
        h = dsxy[..., None] * dx + coef[..., None] * dy
        h = h - (_sum(h, 2) / NSEG)[..., None]
        branch = alpha * Y <= sr.CLIP * X  # y' = alpha y on the tie
        dalpha = _sum(np.where(branch, h * Y, 0.0), 2)
        h = np.where(branch, h * alpha, 0.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            cny = np.where(sy > 0.0, -(dalpha * alpha[..., 0]) / ((sy + EPS) * np.where(sy > 0, sy, 1.0)), 0.0)
        parts.append(h + cny[..., None] * Y)
    if grad_estoi is not None:
        gse = grad_estoi / float(NSEG * S)
        xh = sr._normalise(sr._normalise(X, 2), 1)
        A, rc = _centre(sr._normalise(Y, 2), 1)
        G = _normalise_bwd(A, gse * xh, rc, 1)
        d, rr = _centre(Y, 2)
        parts.append(_normalise_bwd(d, G, rr, 2))
    for sg in range(S):
        for part in parts:
            acc[:, sg:sg + NSEG] = acc[:, sg:sg + NSEG] + part[sg]
    return acc


def ola_frames(y10, kept):
    """The linear stage the backward transposes second: u_j[i] [M][256], the overlap-added kept frames that STFT frame
    j windows (v_j = w u_j)."""
    K = len(kept)
    if K < 2:
        return np.zeros((0, FRAME))
    w = sr.window()
    y10 = np.asarray(y10, np.float64)
    sig = np.zeros((K - 1) * HOP + FRAME)
    for k, f in enumerate(kept):
        sig[k * HOP:k * HOP + FRAME] += w * y10[f * HOP:f * HOP + FRAME]
    return np.lib.stride_tricks.sliding_window_view(sig, FRAME)[::HOP][:K - 1].copy()


def band_spectrum(u):
    """The DFT stage: u [M][256] -> V [M][212] complex, bins LO..HI-1 of the 512-point DFT of w u."""
    return np.fft.rfft(np.asarray(u, np.float64) * sr.window(), sr.NFFT, axis=1)[:, LO:HI]


def band_spectrum_adjoint(G):
    """The adjoint of band_spectrum under the real inner product Re <V, G>: [M][212] complex -> [M][256]."""
    full = np.zeros((G.shape[0], sr.NFFT), complex)
    full[:, LO:HI] = G
    return sr.window() * np.real(np.fft.ifft(full, axis=1) * sr.NFFT)[:, :FRAME]


def bands_bwd(y10, kept, by, dby):
    """d u [M][256] from out's 10 kHz signal, the kept list, its float bands by [15][M] and dby [15][M]:
    G(k) = dby[b] V(k) / by[b] (0 where by = 0), then the adjoint.  -> (du, norms of w u_j [M], sum_k |dby / by| [M],
    sum_k |G(k)| [M])."""
    u = ola_frames(y10, kept)
    M = u.shape[0]
    by = np.asarray(by, np.float64)[:, :M]
    sc = np.where(by > 0, np.asarray(dby, np.float64)[:, :M] / np.where(by > 0, by, 1.0), 0.0)[BAND_OF_BIN].T  # [M][212]
    V = band_spectrum(u)
    G = sc * V
    fr = u * sr.window()
    return band_spectrum_adjoint(G), np.sqrt((fr * fr).sum(axis=1)), np.abs(sc).sum(axis=1), np.abs(G).sum(axis=1)


def ola_bwd(du, kept, n10, absolute=False):
    """The adjoint of ola_frames: dy10 [n10] from du [M][256] (with absolute=True: of |du|, the sum the bound
    scales)."""
    du = np.abs(du) if absolute else np.asarray(du, np.float64)
    M = du.shape[0]
    w = sr.window()
    out = np.zeros(n10)
    for j in range(M):
        for k in (j - 1, j, j + 1):
            if k < 0 or k >= len(kept):
                continue
            # sample i of STFT frame j holds kept frame k at offset o = i - 128 (k - j), 0 <= o < 256
            i = np.arange(FRAME)
            o = i - HOP * (k - j)
            ok = (o >= 0) & (o < FRAME)
            np.add.at(out, kept[k] * HOP + o[ok], w[o[ok]] * du[j, i[ok]])
    return out


def read_samples(kept, n10):
    """Mask of the 10 kHz samples some STFT frame reads."""
    r = np.zeros(n10, bool)
    K = len(kept)
    for k, f in enumerate(kept):
        if K < 2:
            break
        lo = 0
        hi = HOP if k == K - 1 else FRAME  # the last kept frame's second half lies past STFT frame K - 2
        r[f * HOP + lo:f * HOP + hi] = True
    return r


def _resample_index(n, rate):
    """(idx [N][P], taps [N][P]) with out[n] = sum_t dy10[idx[n, t]] taps[n, t] (idx -1: no term): the transposed filter
    as a gather over m ascending."""
    up, down, half, n10, _ = sr.sizes(n, rate)
    h = sr.filter_taps(rate).astype(np.float64)
    ntaps = len(h)
    P = ntaps // down + 2
    nn = np.arange(n)
    m0 = -((half - nn * up) // down)  # ceil((n up - half) / down)
    m = m0[:, None] + np.arange(P)[None, :]
    k = half + m * down - nn[:, None] * up
    ok = (m >= 0) & (m < n10) & (k >= 0) & (k < ntaps)
    return np.where(ok, m, -1), np.where(ok, h[np.clip(k, 0, ntaps - 1)], 0.0)


def resample_bwd(dy10, n, rate, absolute=False):
    """d out[n] = sum_m dy10[m] h[half + m down - n up] (with absolute=True: of |dy10| and |h|) -> [n]."""
    dy10 = np.asarray(dy10, np.float64)
    if sr.filter_taps(rate) is None:
        return np.abs(dy10[:n]) if absolute else dy10[:n].copy()
    idx, taps = _resample_index(n, rate)
    v = np.where(idx >= 0, dy10[np.clip(idx, 0, max(len(dy10) - 1, 0))] if len(dy10) else 0.0, 0.0)
    if absolute:
        v, taps = np.abs(v), np.abs(taps)
    return (v * taps).sum(axis=1)


def intelligibility_grad(out, clean, rate, grad_stoi=1.0, grad_estoi=1.0):
    """The whole backward in float64 from the float64 forward stages -> dL/d out [n].  The score's derivative is taken
    at the bands rounded to float, as the forward stores them, and the band magnitudes' at the float64 bands: the
    rounding is the identity.  (The kernels use their float bands for both, a relative difference of u32.)"""
    f = sr.intelligibility(out, clean, rate)
    M = f["bx"].shape[1]
    n = len(out)
    if f["segments"] < 1:
        return np.zeros(n)
    bx, by = f["bx"].astype(np.float32), f["by"].astype(np.float32)
    dby = score_bwd(bx, by, grad_stoi, grad_estoi)
    du = bands_bwd(f["y10"], f["kept_list"], f["by"], dby)[0]
    dy10 = ola_bwd(du, f["kept_list"], len(f["y10"]))
    return resample_bwd(dy10, n, rate) if M else np.zeros(n)


def value64(out, clean, rate, kept=None):
    """(stoi, estoi) of the definition in float64 with no float rounding of the bands, at a given kept list (None: the
    clean signal's): the function whose finite differences the gradient is checked against."""
    h = sr.filter_taps(rate)
    x10, y10 = sr.resample(clean, rate, h), sr.resample(np.asarray(out, np.float64), rate, h)
    kept = sr.kept_frames(x10) if kept is None else kept
    s, e, _ = sr.score(sr.bands(x10, kept), sr.bands(y10, kept))
    return s, e


def torch_intelligibility(out, clean, rate):
    """stoi_ref's definition transcribed into torch, float64, differentiable in out (a float64 tensor [n]); the bands'
    float rounding passes the gradient through unchanged.  -> (stoi, estoi) tensors."""
    import torch
    n = out.shape[0]
    up, down, half, n10, _ = sr.sizes(n, rate)
    h = sr.filter_taps(rate)
    if h is None:
        y10 = out
    else:
        # y10[m] = sum_j h[ph + j up] x[n0 - j], q = half + m down = n0 up + ph
        h = h.astype(np.float64)
        P = -(-len(h) // up)
        q = half + np.arange(n10) * down
        n0, ph = q // up, q % up
        k = ph[:, None] + up * np.arange(P)[None, :]
        src = n0[:, None] - np.arange(P)[None, :]
        ok = (k < len(h)) & (src >= 0) & (src < n)
        taps = torch.from_numpy(np.where(ok, h[np.clip(k, 0, len(h) - 1)], 0.0))
        y10 = (out[torch.from_numpy(np.clip(src, 0, n - 1))] * taps).sum(dim=1)
    x10 = sr.resample(clean, rate)
    kept = sr.kept_frames(x10)
    K = len(kept)
    w = torch.from_numpy(sr.window())

    def bands(sig10):
        fr = sig10.unfold(0, FRAME, HOP)[torch.from_numpy(kept)] * w  # [K][256]
        idx = (torch.arange(K)[:, None] * HOP + torch.arange(FRAME)[None, :]).reshape(-1)
        ola = torch.zeros((K - 1) * HOP + FRAME, dtype=torch.float64).index_add(0, idx, fr.reshape(-1))
        st = ola.unfold(0, FRAME, HOP)[:K - 1] * w
        p = torch.fft.rfft(st, sr.NFFT, dim=1).abs() ** 2
        b = torch.stack([p[:, sr.EDGES[i]:sr.EDGES[i + 1]].sum(dim=1) for i in range(NBANDS)]).sqrt()
        return b + (b.float().double() - b).detach()

    bx, by = bands(torch.from_numpy(x10)), bands(y10)
    M = bx.shape[1]
    S = M - NSEG + 1
    X = bx.unfold(1, NSEG, 1)[:, :S].permute(1, 0, 2)
    Y = by.unfold(1, NSEG, 1)[:, :S].permute(1, 0, 2)
    alpha = X.norm(dim=2, keepdim=True) / (Y.norm(dim=2, keepdim=True) + EPS)
    Yc = torch.minimum(alpha * Y, sr.CLIP * X)
    dx, dy = X - X.mean(dim=2, keepdim=True), Yc - Yc.mean(dim=2, keepdim=True)
    stoi = (dx * dy).sum(dim=2) / ((dx.norm(dim=2) + EPS) * (dy.norm(dim=2) + EPS))

    def nrm(v, d):
        c = v - v.mean(dim=d, keepdim=True)
        return c / (c.norm(dim=d, keepdim=True) + EPS)

    estoi = (nrm(nrm(X, 2), 1) * nrm(nrm(Y, 2), 1)).sum()
    return stoi.sum() / (NBANDS * S), estoi / (NSEG * S)
