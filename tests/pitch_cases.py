"""Constructed inputs for the pitch kernel's decisions at their rounding edges (TEST INFRASTRUCTURE).

Each case is a deterministic (state record, next frame) pair: the record's input_mem and mem_hp_x come from the input
high-pass run over the first 1728 samples of a raw signal, the frame is the signal's next 480 samples, and last_period /
last_gain are set per case.  The buffer the pitch search sees is input_mem after that frame.  Every property below is
measured on that buffer with the oracle's staged run (oracle_state.pitch_stages) and the float64 reference
(pitch_ref), and a case is kept only if it has the property of its class:

  coarse_bs     coarse best / second coin flip (two periodic components, amplitude ratio bisected)
  coarse_st     coarse second / third coin flip (three components)
  crowded       >= 9 coarse lags within the bound of the best (a period of 4p samples, p <= 16, plus a little noise)
  ties          exact f32 score ties: strictly periodic at levels where y_sq_norm rounds to 1.0f
  few_pos       fewer than two positive coarse correlations (two short bursts)
  zero          an all-zero history
  one_sample    a history with one nonzero sample
  fine          fine-scan best coin flip (a fractional period bisected across the half-sample point)
  ps_offset     coin flip of pitch_search's +-1 rule (the same, bisected on that rule)
  ladder        coin flips of g1 > thresh: k = 2..12, the three cont branches, both thresh formulas (last_gain set so
                that thresh sits within +-2 ulp of the oracle's g1, or the amplitude of a sub-period bisected)
  guard         ex4, y4tot at 1/2, 0.9, 1.1, 2 x 1e-18 and ex4 y4tot (y4tot + 1) at the same multiples of 1e37;
                subnormal whitened samples; the reference's own overflow regime
  overflow      the reference's own overflow regime where only the range guard sends a stream to the exact path: every
                c^2 (and the kernel's whole certificate) is finite, but the reference's products c^2 y overflow
  cand8         exactly CMAX = 8 coarse candidates, each beating every other lag: the kernel's candidate recomputation
                at its capacity (periods of 72 and 76 samples put 8 equal peaks in the 147 lags)
  t0_clip       t0 clipped at 383 (the fine best at lag 0)
  fine_end      the fine best at lag 293, where the reference skips the offset
  floor60       2 t + offset < 60: the period clipped to the 60 floor

cases() builds them all (about a minute on one CPU core) and caches them per process."""
import functools

import numpy as np

import oracle_state as ost
import pitch_ref as pr

N_RAW = 1728 + 480
MIN_COUNT = dict(coarse_bs=64, coarse_st=32, crowded=32, ties=16, few_pos=8, zero=8, one_sample=8, fine=32, ps_offset=32,
                 ladder=96, guard=48, overflow=16, cand8=16, t0_clip=8, fine_end=8, floor60=8)
BISECTED = ("coarse_bs", "coarse_st", "fine", "ps_offset", "ladder")


class Case:
    __slots__ = ("cls", "input_mem", "mem_hp", "frame", "last_period", "last_gain", "buf", "note")

    def __init__(self, cls, raw=None, last_period=0, last_gain=0.0, input_mem=None, note=""):
        self.cls, self.note = cls, note
        self.last_period, self.last_gain = int(last_period), np.float32(last_gain)
        if raw is not None:
            raw = np.asarray(raw, np.float32)
            self.input_mem, self.mem_hp = ost.highpass(raw[:1728])
            self.frame = raw[1728:].copy()
            tail, _ = ost.highpass(self.frame, self.mem_hp)
        else:
            self.input_mem, self.mem_hp = np.asarray(input_mem, np.float32), np.zeros(2, np.float32)
            self.frame = np.zeros(480, np.float32)
            tail = np.zeros(480, np.float32)
        self.buf = np.concatenate([self.input_mem[480:], tail])


def measure(case_list):
    """-> (oracle stages [n], float64 reference dict) on the buffers the pitch search sees."""
    buf = np.stack([c.buf for c in case_list])
    lp = np.array([c.last_period for c in case_list])
    lg = np.array([c.last_gain for c in case_list], np.float32)
    st = ost.pitch_stages(buf, lp, lg)
    return st, pr.reference(st, lp, lg)


def _one(case):
    st, ref = measure([case])
    return st[0], {k: v[0] for k, v in ref.items()}


# ---- signals ------------------------------------------------------------------------------------------------------
def periodic_noise(period, rng, n=N_RAW, smooth=True):
    """White noise repeated with a (possibly fractional) period, band-limited to a quarter of the band so that the
    pitch search's decimation keeps it: sum of harmonics of 48000 / period Hz with random phases."""
    t = np.arange(n, dtype=np.float64)
    H = max(1, int(period / 4.0)) if smooth else max(1, int(period / 2.0) - 1)
    h = np.arange(1, H + 1)[:, None]
    amp = rng.standard_normal(H)[:, None]
    ph = rng.uniform(0, 2 * np.pi, H)[:, None]
    x = (amp * np.cos(2 * np.pi * h * t[None, :] / period + ph)).sum(0)
    return x / np.sqrt(np.mean(x * x))


def _bisect(make, signed, lo, hi, keep, iters=48):
    """Bisect a parameter on a signed float64 margin: make(param) -> case, signed(st, ref) -> margin or None (path
    changed).  Every evaluated case with |margin| < 1 is kept (at most `keep`, the last ones)."""
    flo = signed(*_one(make(lo)))
    fhi = signed(*_one(make(hi)))
    if flo is None or fhi is None or np.sign(flo) == np.sign(fhi):
        return []
    out = []
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        c = make(mid)
        m = signed(*_one(c))
        if m is None:
            return out[-keep:]
        if abs(m) < 1:
            out.append(c)
        if np.sign(m) == np.sign(flo):
            lo = mid
        else:
            hi = mid
        if hi - lo <= abs(mid) * 1e-15:
            break
    return out[-keep:]


# ---- classes ------------------------------------------------------------------------------------------------------
def _coarse_flip(rng, three):
    cls = "coarse_st" if three else "coarse_bs"
    P = sorted(rng.choice(np.arange(400, 760, 4), 3 if three else 2, replace=False))
    comps = [periodic_noise(p, rng) for p in P]
    noise = 300.0 * rng.standard_normal(N_RAW)

    def make(r):
        if three:  # a dominant best, then second and third traded by the ratio (over a little noise)
            x = 4500.0 * comps[0] + 3000.0 * comps[1] + 3000.0 * r * comps[2] + noise
        else:
            x = 3000.0 * comps[0] + 3000.0 * r * comps[1]
        return Case(cls, x, note="periods %s ratio %.17g" % (P, r))

    key, mk = ("c_second", "c_m_st") if three else ("c_best", "c_m_bs")
    st0, r0 = _one(make(0.5 if not three else 0.7))
    ref_lag = r0[key]

    def signed(st, ref):
        if three and ref["c_best"] != r0["c_best"]:
            return None
        return ref[mk] if ref[key] == ref_lag else -ref[mk]
    return _bisect(make, signed, 0.5 if not three else 0.7, 2.0 if not three else 1.4, keep=4)


def _crowded(rng):
    p = int(rng.integers(4, 17))
    x = 3000.0 * periodic_noise(4 * p, rng, smooth=False) + rng.uniform(0, 1e-3) * rng.standard_normal(N_RAW)
    return Case("crowded", x, note="period %d + noise" % (4 * p))


def _tie(rng):
    P = 4 * int(rng.integers(17, 48))
    x = rng.uniform(2e-6, 1e-5) * periodic_noise(P, rng)
    return Case("ties", x, note="period %d, tiny" % P)


def _few_pos(rng):
    x = np.zeros(N_RAW)
    a, d = int(rng.integers(600, N_RAW - 700)), int(rng.integers(60, 700))
    x[a] = rng.choice([-1, 1]) * rng.uniform(100, 3e4)
    x[a + d] = rng.choice([-1, 1]) * rng.uniform(100, 3e4)
    return Case("few_pos", x, last_period=int(rng.integers(0, 769)), last_gain=rng.uniform(0, 1), note="bursts %d, %d" % (a, a + d))


def _fractional(rng, cls):
    P0 = float(rng.uniform(190, 700))
    comp_seed = int(rng.integers(1 << 30))

    def make(P):
        x = 3000.0 * periodic_noise(P, np.random.default_rng(comp_seed))
        return Case(cls, x, note="period %.17g" % P)
    st0, r0 = _one(make(P0))
    if cls == "fine":
        def signed(st, ref):
            if st["best4"] != st0["best4"] or st["second4"] != st0["second4"]:
                return None
            return ref["f_m"] if ref["f_best"] == r0["f_best"] else -ref["f_m"]
        return _bisect(make, signed, P0, P0 + 2.0, keep=4)

    def signed(st, ref):
        if st["best2"] != st0["best2"] or not ref["ps_inner"]:
            return None
        return ref["ps_m1"] if ref["ps_m1"] > -1 or ref["ps_m2"] < -1 else ref["ps_m2"]
    return _bisect(make, signed, P0, P0 + 1.0, keep=4)


def _ladder(rng, k):
    """Coin flips of ladder step k for one t0 and a random cont branch (the thresh formula follows from t1)."""
    out = []
    t0 = int(rng.integers(max(193, 30 * k - k // 2), 384))  # step k is reached: (2 t0 + k) / 2k >= 30
    t1 = (2 * t0 + k) // (2 * k)
    seed = int(rng.integers(1 << 30))
    branch = rng.choice(["d<=1", "d<=2", "none"])

    def make(b, lp=0, lg=0.0):
        g = np.random.default_rng(seed)
        x = 3000.0 * periodic_noise(2 * t0, g) + 3000.0 * b * periodic_noise(2 * t1, g)
        return Case("ladder", x, last_period=lp, last_gain=lg, note="k %d t0 %d %s b %.17g" % (k, t0, branch, b))

    st, ref = _one(make(0.8))
    if st["t0"] != t0 or st["nk"] < k - 1 or st["t1"][k - 2] != t1:
        return []
    s = k - 2
    coef = np.float32(0.85) if t1 < 90 else np.float32(0.7)
    if branch == "none":
        def signed(st_, ref_):
            if st_["t0"] != t0:
                return None
            return ref_["l_m"][s]
        return _bisect(lambda b: make(b, 0, 0.0), signed, 0.05, 4.0, keep=3)
    if branch == "d<=2" and not 5 * k * k < t0:
        return []
    g1, A = st["g1"][s], np.float32(coef * st["g0"])
    floor = np.float32(0.4) if t1 < 90 else np.float32(0.3)
    if not (floor < g1 < A):
        return []
    lp = 2 * t1 if branch == "d<=1" else 2 * (t1 + 2)
    for j in (-2, -1, 0, 1, 2):
        target = np.float32(g1 + j * np.spacing(g1))
        c = float(A) - float(target)
        for lg in (np.float32(c) if branch == "d<=1" else np.float32(2 * c)) + np.arange(-6, 7) * np.spacing(np.float32(c)):
            lg = np.float32(lg)
            cont = lg if branch == "d<=1" else np.float32(lg / np.float32(2))
            if lg >= 0 and np.float32(A - cont) == target:
                out.append(make(0.8, lp, lg))
                break
    return out


def _guard_cases(rng):
    out = []
    for bi in range(4):
        base = 3000.0 * periodic_noise(float(rng.uniform(200, 700)), rng) + 300.0 * rng.standard_normal(N_RAW)
        for what, deg, unit in (("ex4", 2, 1e-18), ("y4tot", 2, 1e-18), ("guard_prod", 6, 1e37)):
            for f in (0.5, 0.9, 1.1, 2.0):
                s = 1.0
                for _ in range(4):
                    st, ref = _one(Case("guard", s * base))
                    s *= (f * unit / ref[what]) ** (1.0 / deg)
                out.append(Case("guard", s * base, last_period=int(rng.integers(0, 769)), last_gain=rng.uniform(0, 1),
                                note="%s at %.1f x %.0e" % (what, f, unit)))
    # deep in the underflow regime (the reference's products c^2 y turn subnormal or zero), subnormal whitened
    # samples, and the overflow regime
    for s in (3e-9, 1e-10, 3e-12, 1e-13, 3e-15, 1e-16, 1e-36, 1e-40, 1e-43, 1e12, 1e15, 1e18):
        out.append(Case("guard", s * (3000.0 * periodic_noise(float(rng.uniform(200, 700)), rng)), note="scale %.0e" % s))
    return out


def _overflow(rng):
    """Speech or a periodic signal scaled so that sum x_lp4^2 ~ 1e17 .. 3e19 (int16 audio x 1e3 .. 1e4)."""
    if rng.uniform() < 0.5:
        o = int(rng.integers(0, len(_speech()) - N_RAW))
        base, what = _speech()[o:o + N_RAW], "speech at %d" % o
    else:
        P = float(rng.uniform(190, 760))
        base, what = 3000.0 * periodic_noise(P, rng) + 300.0 * rng.standard_normal(N_RAW), "period %.1f" % P
    target = 10.0 ** rng.uniform(17, 19.5)
    s = 1.0
    for _ in range(3):
        st, ref = _one(Case("overflow", s * base))
        if not ref["ex4"] > 0:
            return []
        s *= np.sqrt(target / ref["ex4"])
    return Case("overflow", s * base, last_period=int(rng.integers(0, 769)), last_gain=rng.uniform(0, 1),
                note="%s, ex4 %.1e" % (what, target))


def _cand8(rng):
    P = int(rng.choice([72, 76]))
    x = 3000.0 * periodic_noise(P, rng, smooth=False) + rng.uniform(0, 30) * rng.standard_normal(N_RAW)
    return Case("cand8", x, last_period=int(rng.integers(0, 769)), last_gain=rng.uniform(0, 1), note="period %d" % P)


def _extreme(rng, cls):
    if cls == "t0_clip":
        P = float(rng.uniform(766, 772))
    elif cls == "fine_end":  # speech whose period is shorter than the shortest lag: the scan peaks at its end
        o = int(rng.integers(0, len(_speech()) - N_RAW))
        return Case(cls, rng.uniform(0.1, 2.0) * _speech()[o:o + N_RAW], last_period=int(rng.integers(0, 769)),
                    last_gain=rng.uniform(0, 1), note="speech at %d" % o)
    else:
        P = float(rng.uniform(57.5, 61))
    x = 3000.0 * periodic_noise(P, rng, smooth=cls != "floor60") + rng.uniform(0, 100) * rng.standard_normal(N_RAW)
    return Case(cls, x, last_period=int(rng.integers(0, 769)), last_gain=rng.uniform(0, 1), note="period %.3f" % P)


def has_property(c, st, ref):
    """The measured property that puts a case in its class."""
    cls = c.cls
    if cls == "coarse_bs":
        return abs(ref["c_m_bs"]) < 1
    if cls == "coarse_st":
        return abs(ref["c_m_st"]) < 1
    if cls == "crowded":
        return ref["c_n_near"] >= 9
    if cls == "ties":
        b, s = st["best4"], st["second4"]
        return bool((st["ysq4"] == 1.0).all()) and ref["ex4"] > 1e-18 and \
            int((st["xcorr4"] == st["xcorr4"][b]).sum()) >= 2 and st["xcorr4"][s] == st["xcorr4"][b]
    if cls == "few_pos":
        return ref["c_npos"] < 2 and np.count_nonzero(c.buf) >= 2
    if cls == "zero":
        return not c.buf.any()
    if cls == "one_sample":
        return np.count_nonzero(c.buf) == 1
    if cls == "fine":
        return abs(ref["f_m"]) < 1
    if cls == "ps_offset":
        return abs(ref["ps_m1"]) < 1 or (ref["ps_m1"] < 0 and abs(ref["ps_m2"]) < 1)
    if cls == "ladder":
        return bool((np.abs(ref["l_m"][:st["nk"]]) < 1).any())
    if cls == "guard":
        return True
    if cls == "overflow":
        return overflow_only(st, ref)
    if cls == "cand8":
        nc, robust, dominant = pr.kernel_candidates(st[None], {k: np.asarray(v)[None] for k, v in ref.items()})
        return nc[0] == pr.CMAX and robust[0] and dominant[0]
    if cls == "t0_clip":
        return st["pitch_idx"] // 2 > 383 and st["best2"] == 0
    if cls == "fine_end":
        return st["best2"] == 293
    if cls == "floor60":
        return 2 * st["t"] + st["offset"] < 60
    raise KeyError(cls)


def overflow_only(st, ref):
    """Inside the guard's lower limits, a finite certificate bound and finite kernel scores (|c| + delta)^2 for every
    lag, but ex4 y4tot (y4tot + 1) far above 1e37 and the reference's products c_best^2 y beyond the f32 range: only the
    range guard itself routes the stream to the exact path."""
    delta = pr.KAPPA4 * np.sqrt(ref["ex4"] * ref["y4tot"]) * 1.001
    cmax = np.max(np.abs(ref["c4"]))
    return bool(ref["ex4"] > 1e-18 and ref["y4tot"] > 1e-18 and delta < 1e29 and (cmax + delta) ** 2 < 1e38 and
                ref["guard_prod"] > 1e39 and cmax ** 2 * ref["y4tot"] > 1e39)


def _fill(cls, gen, rng, n_min, max_tries=4000):
    out = []
    for _ in range(max_tries):
        if len(out) >= n_min:
            break
        got = gen(rng)
        got = got if isinstance(got, list) else [got]
        for c in got:
            st, ref = _one(c)
            if has_property(c, st, ref):
                out.append(c)
    return out


@functools.lru_cache(maxsize=None)
def cases(seed=20261016):
    """-> list of Case, every class at least MIN_COUNT of its kind."""
    rng = np.random.default_rng(seed)
    out = []
    out += _fill("coarse_bs", lambda r: _coarse_flip(r, False), rng, MIN_COUNT["coarse_bs"])
    out += _fill("coarse_st", lambda r: _coarse_flip(r, True), rng, MIN_COUNT["coarse_st"] + 16)
    out += _fill("crowded", _crowded, rng, MIN_COUNT["crowded"])
    out += _fill("ties", _tie, rng, MIN_COUNT["ties"])
    out += _fill("few_pos", _few_pos, rng, MIN_COUNT["few_pos"])
    for i in range(MIN_COUNT["zero"]):
        out.append(Case("zero", None, last_period=[0, 60, 61, 100, 383, 384, 767, 768][i], last_gain=i / 7.0, input_mem=np.zeros(1728)))
    for v in (1e-30, 1.0, 32767.0, 1e20, -5.0, -1e4, 3e-3, 7.0):
        h = np.zeros(1728, np.float32)
        h[int(rng.integers(480, 1728))] = v
        out.append(Case("one_sample", None, last_period=int(rng.integers(0, 769)), last_gain=rng.uniform(0, 1), input_mem=h))
    out += _fill("fine", lambda r: _fractional(r, "fine"), rng, MIN_COUNT["fine"])
    out += _fill("ps_offset", lambda r: _fractional(r, "ps_offset"), rng, MIN_COUNT["ps_offset"])
    for k in range(2, 13):  # every reachable step
        out += _fill("ladder", lambda r, k=k: _ladder(r, k), rng, 11)
    out += _guard_cases(rng)
    for cls in ("t0_clip", "fine_end", "floor60"):
        out += _fill(cls, lambda r, c=cls: _extreme(r, c), rng, MIN_COUNT[cls])
    rng = np.random.default_rng(seed + 1)
    out += _fill("overflow", _overflow, rng, MIN_COUNT["overflow"])
    out += _fill("cand8", _cand8, rng, MIN_COUNT["cand8"])
    return tuple(out)


@functools.lru_cache(maxsize=None)
def _speech():
    import os
    return np.fromfile(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "testing.raw"), "<i2").astype(np.float64)


def natural_buffers(n=256, seed=5):
    """Buffers of natural signals (speech at random offsets and gains, white + sine) with random carried
    last_period / last_gain -> list of Case."""
    rng = np.random.default_rng(seed)
    speech = _speech()
    out = []
    for i in range(n):
        if i % 2 == 0:
            o = int(rng.integers(0, len(speech) - N_RAW))
            x = rng.uniform(0.05, 2.0) * speech[o:o + N_RAW]
        else:
            t = np.arange(N_RAW)
            x = rng.uniform(100, 1e4) * np.sin(2 * np.pi * rng.uniform(60, 1000) * t / 48000.0) + rng.uniform(10, 3000) * rng.standard_normal(N_RAW)
        out.append(Case("natural", x, last_period=int(rng.integers(0, 769)), last_gain=rng.uniform(0, 1)))
    return out
