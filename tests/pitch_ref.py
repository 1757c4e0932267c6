"""A float64 reference of every decision pitch_process takes (src/pitch.rs:63-221), vectorised over streams (TEST
INFRASTRUCTURE).

It starts from the oracle's f32 operands (oracle_state.pitch_stages): the whitened buffer, the f32 running energies
(find_best_pitch's y_sq_norm at each lag, remove_doubling's yy_lookup, xx) that the pitch kernel also computes in the
reference's order, and the carried last_period / last_gain.  Every dot product the reference rounds -- the 147 coarse
correlations (240 terms), the fine correlations and all inner products of remove_doubling (480 terms) -- is evaluated
in float64, together with the rounding bound gamma_n sum |x_j y_j| of the reference's f32 result (any order, any mix of
fused and unfused roundings).  It follows the oracle's path (the lags it looked at) and gives, for each decision, the
float64 outcome and its margin in units of the bound on that decision:

- coarse scan: best / second and second / third, the number of lags within the bound of the best;
- fine scan: the best;
- the +-1 offset rules of pitch_search and of the end of remove_doubling (two comparisons each);
- every ladder step g1 > thresh.
The clamps of the running energies (y_sq_norm >= 1, yy_lookup >= 0) are not among them: they are sequential f32
recurrences that the kernel repeats in the reference's order, not decisions taken from reordered sums.

A decision with |margin| < 1 is a coin flip: the reference's own f32 rounding decides it, and only arithmetic that
repeats the reference's operations in order is sure to decide it the same way.  Margins also carry the f32 roundings of
the comparison itself (a few units of 2^-24 of the operands)."""
import numpy as np

U = 2.0 ** -24
F7 = float(np.float32(0.7))
F85 = float(np.float32(0.85))
F_FLOOR_LO, F_FLOOR_HI = float(np.float32(0.4)), float(np.float32(0.3))
NL4, NL2, N4, N2, HALF_MAX = 147, 294, 240, 480, 384
CHUNK = 128


def gamma(n):
    return n * U / (1.0 - n * U)


def _ratio(num, den):
    """num / den with 0 / 0 = 0 and x / 0 = +-inf (an exact decision has no bound)."""
    num, den = np.broadcast_arrays(np.asarray(num, np.float64), np.asarray(den, np.float64))
    out = np.where(num == 0, 0.0, np.copysign(np.inf, num))
    nz = den > 0
    out[nz] = num[nz] / den[nz]
    return out


def _dots(p, shifts, n):
    """For each stream b and each k: sum_j p[b, 384 + j] p[b, 384 - shifts[b, k] + j], j < n (stride 1 if n == 480, the
    even samples if n == 240) in float64, and sum |.| -> (value, abs) [B][K]."""
    B, K = shifts.shape
    step = 2 if n == N4 else 1
    j = np.arange(n) * step
    x = p[:, HALF_MAX + j]                                                  # [B][n]
    idx = HALF_MAX - shifts[:, :, None] + j[None, None, :]                  # [B][K][n]
    y = p[np.arange(B)[:, None, None], idx]
    prod = x[:, None, :] * y
    return prod.sum(2), np.abs(prod).sum(2)


def _top3(r, pos):
    """The reference's scan ends with the two largest scores among positive correlations, the earliest lag winning an
    exact tie (strict >).  -> (best, second, third) [B], -1 where there are not that many positive lags."""
    key = np.where(pos, r, -np.inf)
    order = np.argsort(-key, axis=1, kind="stable")
    top = order[:, :3].copy()
    npos = pos.sum(1)
    for k in range(3):
        top[npos <= k, k] = -1
    return top[:, 0], top[:, 1], top[:, 2]


def _at(a, i):
    return np.take_along_axis(a, np.maximum(i, 0)[:, None], 1)[:, 0]


def _scan_margins(c, d, ysq):
    """Scores r = c^2 / y (c > 0) with bounds; top three; margins best/second and second/third; lags near the best."""
    pos = c > 0
    r = np.where(pos, c * c / ysq, 0.0)
    dr = np.where(pos, (2 * np.abs(c) * d + d * d) / ysq + 3 * U * r, 0.0)
    b, s, t = _top3(r, pos)
    rb, rs, rt = _at(r, b), _at(r, s), _at(r, t)
    db, ds, dt = _at(dr, b), _at(dr, s), _at(dr, t)
    m_bs = np.where(s >= 0, _ratio(rb - rs, db + ds), np.inf)
    m_st = np.where(t >= 0, _ratio(rs - rt, ds + dt), np.inf)
    near = (pos & (r + dr >= (rb - db)[:, None])).sum(1)
    return dict(best=b, second=s, third=t, m_bs=m_bs, m_st=m_st, n_near=np.where(b >= 0, near, 0), npos=pos.sum(1))


def _offset_rule(a, b, c, da, db, dc):
    """The +-1 rule of src/pitch.rs:107-113 and :205-218 in float64: (offset, margin of rule 1, margin of rule 2)."""
    v1 = (c - a) - F7 * (b - a)
    e1 = dc + 0.3 * da + F7 * db + 4 * U * (np.abs(a) + np.abs(b) + np.abs(c))
    v2 = (a - c) - F7 * (b - c)
    e2 = da + 0.3 * dc + F7 * db + 4 * U * (np.abs(a) + np.abs(b) + np.abs(c))
    off = np.where(v1 > 0, 1, np.where(v2 > 0, -1, 0))
    return off, _ratio(v1, e1), _ratio(v2, e2)


def reference(st, last_period, last_gain):
    """st: oracle_state.PITCH_STAGES [B] -> dict of float64 outcomes and margins per stream (see the module doc)."""
    out = [_reference(st[i:i + CHUNK], np.asarray(last_period)[i:i + CHUNK] if np.ndim(last_period) else last_period,
                      np.asarray(last_gain)[i:i + CHUNK] if np.ndim(last_gain) else last_gain)
           for i in range(0, len(st), CHUNK)]
    return {k: np.concatenate([o[k] for o in out]) for k in out[0]}


def _reference(st, last_period, last_gain):
    B = len(st)
    p = st["pitch_buf"].astype(np.float64)
    lp = np.broadcast_to(np.asarray(last_period, np.int64), (B,))
    lg = np.broadcast_to(np.asarray(last_gain, np.float32), (B,)).astype(np.float64)
    res = {}

    # ---- range of the coarse search (the kernel's guard: ex4, y4tot, ex4 y4tot (y4tot + 1)) ----
    ex4 = (p[:, HALF_MAX::2] ** 2).sum(1)
    y4tot = (p[:, 0::2] ** 2).sum(1)
    res.update(ex4=ex4, y4tot=y4tot, guard_prod=ex4 * y4tot * (y4tot + 1.0))
    # where the reference's f32 products stay finite and normal in both scans and in remove_doubling; outside it
    # selects on underflowed or infinite values and float64 does not describe it
    ex2, y2 = (p[:, HALF_MAX:] ** 2).sum(1), (p ** 2).sum(1)
    with np.errstate(over="ignore", invalid="ignore"):
        res["in_range"] = ((ex4 > 1e-18) & (y4tot > 1e-18) & (res["guard_prod"] < 1e37) &
                           (ex2 > 1e-18) & (y2 > 1e-18) & (ex2 * y2 * (y2 + 1.0) < 1e37))

    # ---- coarse scan: xcorr4[i] = sum_j x_lp4[j] y_lp4[i + j], x_lp4[j] = p[384 + 2j], y_lp4[j] = p[2j] ----
    lag4 = np.broadcast_to(HALF_MAX - 2 * np.arange(NL4), (B, NL4))
    c4, a4 = _dots(p, lag4, N4)
    d4 = gamma(N4) * a4
    sc = _scan_margins(c4, d4, st["ysq4"].astype(np.float64))
    res.update({"c_" + k: v for k, v in sc.items()})
    res["c4"], res["d4"] = c4, d4

    # ---- fine scan on the oracle's windows (around 2 best4 and 2 second4), xcorr = max(inner_prod, -1) ----
    i2 = np.arange(NL2)[None, :]
    win = (np.abs(i2 - 2 * st["best4"][:, None]) <= 2) | (np.abs(i2 - 2 * st["second4"][:, None]) <= 2)
    c2 = np.zeros((B, NL2))
    d2 = np.zeros((B, NL2))
    cols = np.argsort(~win, axis=1, kind="stable")[:, :10]                 # the (at most 10) window lags
    v, a = _dots(p, HALF_MAX - cols, N2)
    inw = np.take_along_axis(win, cols, 1)
    np.put_along_axis(c2, cols, np.where(inw, np.maximum(v, -1.0), 0.0), 1)
    np.put_along_axis(d2, cols, np.where(inw & (v > -1.0), gamma(N2) * a, 0.0), 1)
    fs = _scan_margins(c2, d2, st["ysq2"].astype(np.float64))
    res.update(f_best=np.maximum(fs["best"], 0), f_m=fs["m_bs"], f_npos=fs["npos"])
    # pitch_search's +-1 rule at the oracle's fine best
    bst = st["best2"].astype(np.int64)
    inner = (bst > 0) & (bst < NL2 - 1)
    g = lambda arr, k: np.take_along_axis(arr, np.clip(bst + k, 0, NL2 - 1)[:, None], 1)[:, 0]  # noqa: E731
    off, m1, m2 = _offset_rule(g(c2, -1), g(c2, 0), g(c2, 1), g(d2, -1), g(d2, 0), g(d2, 1))
    res.update(ps_offset=np.where(inner, off, 0), ps_m1=np.where(inner, m1, np.nan), ps_m2=np.where(inner, m2, np.nan),
               ps_inner=inner)

    # ---- remove_doubling on the oracle's t0: g0, every ladder step, the final +-1 rule ----
    t0 = st["t0"].astype(np.int64)
    nk = st["nk"].astype(np.int64)
    K = st["t1"].shape[1]
    xx = st["xx"].astype(np.float64)
    yyl = st["yy_lookup"].astype(np.float64)
    xy0, axy0 = _dots(p, t0[:, None], N2)
    xy0, dxy0 = xy0[:, 0], gamma(N2) * axy0[:, 0]
    den0 = np.sqrt(1.0 + xx * _at(yyl, t0))
    g0, dg0 = xy0 / den0, dxy0 / den0
    res.update(g0=g0)
    t1, t1b = st["t1"].astype(np.int64), st["t1b"].astype(np.int64)
    live = np.arange(K)[None, :] < nk[:, None]
    va, aa = _dots(p, np.where(live, t1, 1), N2)
    vb, ab = _dots(p, np.where(live, t1b, 1), N2)
    xy = (va + vb) / 2
    dxy = gamma(N2) * (aa + ab) / 2
    yy = st["yy"].astype(np.float64)
    den = np.sqrt(1.0 + xx[:, None] * yy)
    g1, dg1 = xy / den, dxy / den
    cont = st["cont"].astype(np.float64)
    lo = t1 < 90
    coef = np.where(lo, F85, F7)
    floor = np.where(lo, F_FLOOR_LO, F_FLOOR_HI)
    raw = coef * g0[:, None] - cont
    thresh = np.maximum(raw, floor)
    free = raw > floor - coef * dg0[:, None]                                # the floor does not pin thresh
    err = dg1 + np.where(free, coef * dg0[:, None], 0.0) + 4 * U * np.abs(g1) + 2 * U * (coef * np.abs(g0[:, None]) + cont)
    res.update(l_g1=np.where(live, g1, np.nan), l_thresh=np.where(live, thresh, np.nan), l_taken=live & (g1 > thresh),
               l_m=np.where(live, _ratio(g1 - thresh, err), np.nan), l_live=live,
               l_d=np.abs(t1 - (lp // 2)[:, None]), l_floored=~free)
    t = st["t"].astype(np.int64)
    v3, a3 = _dots(p, t[:, None] + np.array([[-1, 0, 1]]), N2)
    d3 = gamma(N2) * a3
    off, m1, m2 = _offset_rule(v3[:, 0], v3[:, 1], v3[:, 2], d3[:, 0], d3[:, 1], d3[:, 2])
    res.update(rd_offset=off, rd_m1=m1, rd_m2=m2)

    return res


KAPPA4, ETA1 = 3.1e-5, 1.00001  # pitch.cu: the coarse certificate's bound factor and slack
CMAX = 8                         # pitch.cu: candidates a stream may recompute in the reference's order


def kernel_candidates(st, ref, band=1e-4):
    """The coarse candidate set of pitch.cu's certificate, emulated on the float64 correlations: delta = KAPPA4
    sqrt(ex4 y4tot) 1.001, intervals [lo, hi] of c^2 / y from c -+ delta, F1, F2 the top two scores, candidates
    {j : hi_j ETA1 >= min(lo_F1, lo_F2)}.  -> (nc [B], robust [B]: the count is the same with the threshold moved by
    +-band (far more than the FMA values' distance from float64), dominant [B]: every candidate's score beats
    ETA1^2 (1 + band) x the largest non-candidate upper bound, so a stream with 3..CMAX candidates stays on the
    candidate path)."""
    c, y = ref["c4"], st["ysq4"].astype(np.float64)
    B = len(c)
    delta = (KAPPA4 * np.sqrt(ref["ex4"] * ref["y4tot"]) * 1.001)[:, None]
    r = np.where(c > 0, c * c / y, 0.0)
    top = np.argsort(-r, axis=1, kind="stable")[:, :2]
    lo = np.where(c - delta > 0, (c - delta) ** 2 / y, 0.0)
    hi = np.maximum(c + delta, 0.0) ** 2 / y
    t0 = np.minimum(_at(lo, top[:, 0]), _at(lo, top[:, 1]))[:, None]
    forced = np.zeros_like(c, bool)
    forced[np.arange(B), top[:, 0]] = forced[np.arange(B), top[:, 1]] = True
    mem = forced | (hi * ETA1 >= t0)
    nc = mem.sum(1)
    robust = ((forced | (hi * ETA1 >= t0 * (1 + band))).sum(1) == nc) & ((forced | (hi * ETA1 >= t0 * (1 - band))).sum(1) == nc)
    mb = np.where(mem, 0.0, hi).max(1)
    dominant = np.where(mem, r, np.inf).min(1) > mb * ETA1 * ETA1 * (1 + band)
    return nc, robust, dominant


def disagreements(st, ref):
    """Decisions with |margin| >= 1 whose float64 outcome differs from the oracle's f32 outcome -> dict name -> stream
    indices.  Such a decision is not a coin flip: the oracle and the reference must agree on it (inside the range where
    the reference's f32 values are finite and normal)."""
    bad = {}
    out = ~ref["in_range"]
    ref = {k: np.where(out.reshape((-1,) + (1,) * (np.ndim(v) - 1)), np.nan, v) if k.endswith(("_m", "_m1", "_m2", "_bs", "_st"))
           else v for k, v in ref.items()}
    robust_bs = np.abs(ref["c_m_bs"]) >= 1
    robust_st = np.abs(ref["c_m_st"]) >= 1
    bad["coarse best"] = np.flatnonzero(robust_bs & robust_st & (ref["c_best"] >= 0) & (ref["c_best"] != st["best4"]))
    two = ref["c_second"] >= 0
    same_set = (np.minimum(ref["c_best"], ref["c_second"]) == np.minimum(st["best4"], st["second4"])) & \
               (np.maximum(ref["c_best"], ref["c_second"]) == np.maximum(st["best4"], st["second4"]))
    bad["coarse second"] = np.flatnonzero(robust_st & two & ~same_set)
    fine_ok = (np.abs(ref["f_m"]) >= 1) & (ref["f_npos"] >= 1)
    bad["fine best"] = np.flatnonzero(fine_ok & (ref["f_best"] != st["best2"]))
    for name, off, m1, m2 in (("pitch_search offset", st["offset2"], ref["ps_m1"], ref["ps_m2"]),
                              ("remove_doubling offset", st["offset"], ref["rd_m1"], ref["rd_m2"])):
        r1 = np.abs(m1) >= 1
        bad[name + " rule 1"] = np.flatnonzero(r1 & ((m1 > 0) != (off == 1)))
        r2 = r1 & (m1 < 0) & (np.abs(m2) >= 1)
        bad[name + " rule 2"] = np.flatnonzero(r2 & ((m2 > 0) != (off == -1)))
    lad = ref["l_live"] & (np.abs(ref["l_m"]) >= 1) & (ref["l_taken"] != (st["taken"] != 0))
    bad["ladder"] = np.flatnonzero(lad.any(1))
    return bad


def coin_flips(ref):
    """Per decision, which streams hold a coin flip (|margin| < 1) -> dict name -> bool [B]."""
    lm = np.where(ref["l_live"], np.abs(ref["l_m"]), np.inf)
    return {
        "coarse best/second": np.abs(ref["c_m_bs"]) < 1,
        "coarse second/third": np.abs(ref["c_m_st"]) < 1,
        "fine best": np.abs(ref["f_m"]) < 1,
        "pitch_search offset": (np.abs(ref["ps_m1"]) < 1) | ((ref["ps_m1"] < 0) & (np.abs(ref["ps_m2"]) < 1)),
        "remove_doubling offset": (np.abs(ref["rd_m1"]) < 1) | ((ref["rd_m1"] < 0) & (np.abs(ref["rd_m2"]) < 1)),
        "ladder": (lm < 1).any(1),
    }


def f32_outcomes_differ(st, ref):
    """Per decision, whether the oracle's f32 outcome differs from the float64 one -> dict name -> bool [B]."""
    lad = ref["l_live"] & (np.abs(ref["l_m"]) < 1) & (ref["l_taken"] != (st["taken"] != 0))
    return {
        "coarse best/second": ref["c_best"] != st["best4"],
        "coarse second/third": (np.minimum(ref["c_best"], ref["c_second"]) != np.minimum(st["best4"], st["second4"])) |
                               (np.maximum(ref["c_best"], ref["c_second"]) != np.maximum(st["best4"], st["second4"])),
        "fine best": ref["f_best"] != st["best2"],
        "pitch_search offset": ref["ps_offset"] != st["offset2"],
        "remove_doubling offset": ref["rd_offset"] != st["offset"],
        "ladder": lad.any(1),
    }
