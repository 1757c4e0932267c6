"""Constructed lanes for the training-row path (TEST INFRASTRUCTURE): each case is a lane of T frames -- raw signal and
noise (i16-valued unless said otherwise) and the parameters set before given frames -- built so that one decision of
src/training.rs is taken at its edge.  Every case class states its defining property in check(trace), which the CPU
test asserts on the restatement and the oracle, so a case that stops reaching its edge fails loudly.

trace (one lane, every array over the T frames): energy [T] (float32, before the gain), vad_count [T], vad [T],
cutoff [T], resp_mem [T][4] after the frame, params [T] (in force during the frame), hist [T][3][1728] (clean, noise,
combined after the frame), ex [T][3][22], silence [T][3], gains [T][22] (float32 row columns), unclamped [T][22]
(float64, no clamp)."""
import numpy as np

import train_ref as tr

T = 24
F32 = np.float32
_n = np.arange(tr.FRAME)


def tone(freq, amp, t):
    """An i16-valued sine of frame t (continuous across frames)."""
    return np.round(amp * np.sin(2 * np.pi * freq * (_n + tr.FRAME * t) / 48000.0)).astype(F32)


def spikes(samples, at=100):
    """A frame of zeros with `samples` at positions at, at + 1, ... (their energy is summed in this order)."""
    x = np.zeros(tr.FRAME, F32)
    x[at:at + len(samples)] = samples
    return x


def params(signal_gain=1.0, noise_gain=1.0, sig=((0, 0), (0, 0)), noi=((0, 0), (0, 0)), band_lp=21):
    p = tr.default_params(1)[0]
    p["signal_gain"], p["noise_gain"], p["band_lp"] = signal_gain, noise_gain, band_lp
    p["sig_a"], p["sig_b"] = sig
    p["noise_a"], p["noise_b"] = noi
    return p


def random_filter(rng):
    """random_filter (src/training.rs:291-297): a and b uniform in [-0.375, 0.375)."""
    return tuple(tuple((F32(0.75) * (rng.random(2, dtype=F32) - F32(0.5))).astype(F32)) for _ in range(2))


# energy classes of NoiseSimulator::vad (src/training.rs:368-386), as the counter step they cause
QUIET, MID, LOUD, LOUDER = 2, 1, -5, None
_AMP = {QUIET: 100, MID: 400, LOUD: 1500, LOUDER: 5000}  # 480 a^2 / 2: 2.4e6, 3.8e7, 5.4e8, 6e9


def level_frames(seq, freq=440.0):
    return np.stack([tone(freq, _AMP[c], t) for t, c in enumerate(seq)])


def vad_class(e):
    """The counter step an f32 frame energy causes (None: reset to 0)."""
    return LOUDER if e > F32(1e9) else LOUD if e > F32(1e8) else MID if e > F32(1e7) else QUIET


class Case:
    name = "?"

    def __init__(self, signal, noise, schedule=None):
        self.signal = np.asarray(signal, F32).reshape(T, tr.FRAME)
        self.noise = np.asarray(noise, F32).reshape(T, tr.FRAME)
        self.schedule = schedule or {}   # frame -> parameters set before it

    def check(self, trace):
        raise NotImplementedError


class VadThreshold(Case):
    """Frame 3 has an f32 energy of exactly 1e7, 1e8 or 1e9, or exactly the next float above: the samples are
    i16-valued and every partial sum is exact, or a +1 is absorbed by the sum.  Frames 0-2 take the counter to 6."""
    F = 3

    def __init__(self, label, samples, want_energy, want_step):
        self.name = "vad_threshold_" + label
        self.want_energy, self.want_step = F32(want_energy), want_step
        sig = level_frames([QUIET] * T)
        sig[self.F] = spikes(samples)
        super().__init__(sig, np.stack([tone(1000, 300, t) for t in range(T)]))

    def check(self, tr_):
        e = tr_["energy"][self.F]
        assert e.view(np.uint32) == self.want_energy.view(np.uint32), (self.name, float(e))
        assert tr_["vad_count"][self.F - 1] == 6
        want = 0 if self.want_step is None else 6 + self.want_step
        assert tr_["vad_count"][self.F] == want


def _up(x):
    return np.nextafter(F32(x), F32(np.inf))


def vad_threshold_cases():
    big9 = [20000, 20000, 10000, 10000]  # 1e9 = 4e8 + 4e8 + 1e8 + 1e8, every partial sum exact
    return [
        VadThreshold("1e7", [3000, 1000], 1e7, QUIET),
        VadThreshold("1e7_ulp", [3000, 1000, 1], _up(1e7), MID),                     # ulp 1
        VadThreshold("1e7_ulp_one_first", [1, 3000, 1000], _up(1e7), MID),
        VadThreshold("1e8", [10000], 1e8, MID),
        VadThreshold("1e8_ulp", [2, 2, 10000], _up(1e8), LOUD),                       # ulp 8 = 2^2 + 2^2, summed first
        VadThreshold("1e8_one_first", [1, 10000], 1e8, MID),                          # 1 + 1e8 rounds to 1e8
        VadThreshold("1e8_one_last", [10000, 1], 1e8, MID),
        VadThreshold("1e8_eight_ones_first", [1] * 8 + [10000], _up(1e8), LOUD),      # 8 + 1e8 is exact ...
        VadThreshold("1e8_eight_ones_last", [10000] + [1] * 8, 1e8, MID),             # ... each +1 after 1e8 is lost
        VadThreshold("1e9", big9, 1e9, LOUD),
        VadThreshold("1e9_ulp", [8] + big9, _up(1e9), LOUDER),                        # ulp 64 = 8^2
        VadThreshold("1e9_one_first", [1] + big9, 1e9, LOUD),
        VadThreshold("1e9_one_last", big9 + [1], 1e9, LOUD),
    ]


class VadCounter(Case):
    """A sequence of energy classes that drives vad_count onto a given edge: `event` names it and check finds it."""

    def __init__(self, label, seq, event):
        self.name = "vad_counter_" + label
        self.seq, self.event = list(seq) + [QUIET] * (T - len(seq)), event
        super().__init__(level_frames(self.seq), np.stack([tone(2500, 200, t) for t in range(T)]))

    def check(self, tr_):
        vc = np.concatenate([[0], tr_["vad_count"]])
        raw = [0 if c is None else vc[t] + c for t, c in enumerate(self.seq)]  # the counter before the clamp
        assert [vad_class(e) for e in tr_["energy"]] == self.seq, self.name
        assert np.array_equal(vc[1:], np.clip(raw, 0, 15))
        hit = {"clamp15": any(r > 15 for r in raw), "clamp0_from3": any(vc[t] == 3 and r < 0 for t, r in enumerate(raw)),
               "onto10": any(vc[t + 1] == 10 and vc[t] < 10 for t in range(T)),
               "off10_to9": any(vc[t] >= 10 and vc[t + 1] == 9 for t in range(T))}
        assert hit[self.event], (self.name, vc)
        v = tr_["vad"]
        assert np.array_equal(v, np.where(vc[1:] >= 10, 0.0, np.where(vc[1:] > 0, 0.5, 1.0)).astype(F32))


def vad_counter_cases():
    Q, M, Lo, X = QUIET, MID, LOUD, LOUDER
    return [
        VadCounter("clamp15", [Q] * 9 + [M, Lo, Lo, M], "clamp15"),       # 16 -> 15, 15 + 1 -> 15, then 10, 5, 6
        VadCounter("onto10", [Q] * 5 + [M, Lo, Q, Q, M], "onto10"),       # exactly 10: vad 0
        VadCounter("clamp0_from3", [M] * 3 + [Lo, Q, X, M], "clamp0_from3"),  # 3 - 5 -> 0
        VadCounter("nine_ten_eleven", [Q] * 4 + [M, M, M, Lo, Q], "onto10"),  # 9 (vad 0.5) -> 10 -> 11 -> 6 -> 8
        VadCounter("fourteen_to_nine", [Q] * 7 + [Lo, M, Lo, Q, Q, Q, Q], "off10_to9"),  # 14, 9, 10, 5, ...
    ]


class GainBeforeEnergy(Case):
    """signal_gain = 0 with a loud raw signal: the energy is taken before the gain, so vad_count is 0 every frame, while
    the clean and combined streams are digital silence."""
    name = "energy_before_gain_zero_signal_gain"

    def __init__(self):
        super().__init__(level_frames([LOUDER] * T), np.stack([tone(700, 3000, t) for t in range(T)]),
                         {0: params(signal_gain=0.0, noise_gain=0.0)})

    def check(self, tr_):
        assert np.all(tr_["energy"] > F32(1e9)) and np.all(tr_["vad_count"] == 0) and np.all(tr_["vad"] == 1.0)
        assert not tr_["hist"][:, 0].any() and not tr_["hist"][:, 2].any()
        assert tr_["silence"][:, 0].all() and tr_["silence"][:, 2].all()
        assert np.all(tr_["gains"] == -1.0)


class EnergyOverflow(Case):
    """A raw signal around 1e19 with signal_gain 1e-15: x^2 ~ 1e38 stays finite but the f32 sum overflows to inf,
    which counts as loud; every stream stays finite."""
    name = "energy_overflow"

    def __init__(self):
        sig = np.stack([tone(440, 30000, t) for t in range(T)]) * F32(3.4e14)
        super().__init__(sig.astype(F32), np.stack([tone(3000, 500, t) for t in range(T)]),
                         {0: params(signal_gain=1e-15, noise_gain=1.0)})

    def check(self, tr_):
        assert np.all(np.isinf(tr_["energy"])) and np.all(tr_["vad_count"] == 0)
        assert np.all(np.isfinite(tr_["hist"])) and np.abs(tr_["hist"][:, 0]).max() > 1.0
        assert not tr_["silence"][4:, 0].any()


class GainMask(Case):
    """Band energies either side of 5e-2.  noise_band: the signal is a 300 Hz tone, the noise a 9 kHz tone, so the noise
    bands have ce < 5e-2 <= me, the empty ones both below and the tone bands neither.  cancel: the signal is both tones,
    the noise exactly minus the 300 Hz one (identity filters), so the 300 Hz bands have me < 5e-2 <= ce."""

    def __init__(self, label):
        self.name = "gain_mask_" + label
        a = np.stack([tone(300, 3000, t) for t in range(T)])
        b = np.stack([tone(9000, 3000, t) for t in range(T)])
        self.label = label
        if label == "noise_band":
            super().__init__(a, b)
        else:
            super().__init__(a + b, -a)

    def check(self, tr_):
        ce, me = tr_["ex"][4:, 0], tr_["ex"][4:, 2]
        lo_c, lo_m = ce < F32(5e-2), me < F32(5e-2)
        assert not tr_["silence"][4:, 2].any() and np.all(tr_["cutoff"] == 22)
        assert (lo_c & lo_m).any() and (~lo_c & ~lo_m).any()
        one = (lo_c & ~lo_m) if self.label == "noise_band" else (~lo_c & lo_m)
        assert one.any(), self.name
        g = tr_["gains"][4:]
        assert np.all(g[lo_c & lo_m] == -1.0) and np.all(g[one] >= 0.0)


class ClampAtOne(Case):
    """noise = -signal through the same random filter with noise_gain = signal_gain / 2: the combined stream is exactly
    half the clean one (the scaling by 2^-1 commutes with every rounding), so me = ce / 4 exactly and every unmasked
    gain is sqrt((ce + 1e-3) / (ce / 4 + 1e-3)) > 1, clamped to exactly 1."""
    name = "clamp_at_one"

    def __init__(self, rng):
        sig = np.stack([tone(440, 2000, t) + tone(3100, 800, t) for t in range(T)])
        f = random_filter(rng)
        super().__init__(sig, -sig, {0: params(signal_gain=0.5, noise_gain=0.25, sig=f, noi=f)})

    def check(self, tr_):
        h = tr_["hist"]
        assert np.array_equal(h[:, 2], h[:, 0] * F32(0.5))
        assert np.array_equal(tr_["ex"][:, 2], tr_["ex"][:, 0] * F32(0.25))
        g, u = tr_["gains"], tr_["unclamped"]
        live = g != -1.0
        assert live[4:].sum() > 20 and np.all(g[live] == 1.0) and np.all(u[live] > 1.5)


class ExactCancel(Case):
    """noise = -signal through the same random filter with equal gains: the combined stream is exactly 0 (round to nearest
    is odd-symmetric), so it is silent and every gain is -1 although the clean stream is loud."""
    name = "exact_cancel"

    def __init__(self, rng):
        sig = np.stack([tone(440, 2000, t) + tone(3100, 800, t) for t in range(T)])
        f = random_filter(rng)
        super().__init__(sig, -sig, {0: params(signal_gain=0.7, noise_gain=0.7, sig=f, noi=f)})

    def check(self, tr_):
        assert not tr_["hist"][:, 2].any() and tr_["silence"][:, 2].all()
        assert not tr_["silence"][2:, 0].any() and np.all(tr_["cutoff"] == 22)
        assert np.all(tr_["gains"] == -1.0)


class Cutoff(Case):
    """The gain cutoff: noise_gain = 0 gives 0 while vad == 0 and band_lp + 1 while vad > 0; band_lp = 0 and 21."""

    def __init__(self, label):
        self.name = "cutoff_" + label
        self.label = label
        if label.startswith("noise_gain0"):
            seq = [QUIET] * 6 + [LOUD, LOUD, QUIET, QUIET, QUIET, LOUD, LOUD]  # counter 12 (vad 0) ... 7, 2 (vad 0.5)
            bl = 21 if label == "noise_gain0" else 9
            super().__init__(level_frames(seq + [QUIET] * (T - len(seq))), np.stack([tone(5000, 800, t) for t in range(T)]),
                             {0: params(noise_gain=0.0, band_lp=bl)})
            self.band_lp = bl
        else:
            self.band_lp = 0 if label == "band_lp0" else 21
            super().__init__(np.stack([tone(250, 1500, t) + tone(20000, 900, t) for t in range(T)]),
                             np.stack([tone(1200, 400, t) for t in range(T)]), {0: params(noise_gain=0.5, band_lp=self.band_lp)})

    def check(self, tr_):
        vad, cut, g, sil = tr_["vad"], tr_["cutoff"], tr_["gains"], tr_["silence"][:, 2]
        assert not sil[2:].any()
        if self.label.startswith("noise_gain0"):
            off, on = (vad == 0.0), (vad > 0.0)
            assert off[2:].any() and on[2:].any()
            assert np.all(cut[off] == 0) and np.all(g[off] == -1.0)
            assert np.all(cut[on] == self.band_lp + 1)
            live = g[on][:, :self.band_lp + 1] != -1.0
            assert live.any() and np.all(g[on][:, :self.band_lp + 1][live] == 1.0)   # combined == clean
            assert np.all(g[on][:, self.band_lp + 1:] == -1.0)
        else:
            assert np.all(cut == self.band_lp + 1)
            assert np.all(g[2:, [0, self.band_lp]] != -1.0)   # the 250 Hz and 20 kHz tones: the first and last band kept
            assert np.all(g[:, self.band_lp + 1:] == -1.0)


class ParamsMidRun(Case):
    """Random filters and gains set before frames 0, 8 and 16: the filter memories are nonzero at each change and carry
    over (randomize() replaces the filters, not signal_resp_mem / noise_resp_mem)."""
    name = "params_mid_run"
    AT = (8, 16)

    def __init__(self, rng):
        sig = np.stack([tone(523, 1800, t) + np.round(rng.normal(0, 300, tr.FRAME)) for t in range(T)]).astype(F32)
        noi = np.round(rng.normal(0, 700, (T, tr.FRAME))).astype(F32)
        sched = {t: params(signal_gain=float(F32(10.0) ** F32(rng.integers(-40, 20) / 20.0)),
                           noise_gain=float(F32(10.0) ** F32(rng.integers(-20, 20) / 20.0)),
                           sig=random_filter(rng), noi=random_filter(rng), band_lp=int(rng.integers(0, 22)))
                 for t in (0,) + self.AT}
        super().__init__(sig, noi, sched)

    def check(self, tr_):
        for t in self.AT:
            assert np.all(tr_["resp_mem"][t - 1] != 0.0)
            assert tr_["params"][t].tobytes() != tr_["params"][t - 1].tobytes()


def cases():
    rng = np.random.default_rng(2024)
    return (vad_threshold_cases() + vad_counter_cases() + [GainBeforeEnergy(), EnergyOverflow()]
            + [GainMask("noise_band"), GainMask("cancel"), ClampAtOne(rng), ExactCancel(rng)]
            + [Cutoff("noise_gain0"), Cutoff("noise_gain0_band_lp9"), Cutoff("band_lp0"), Cutoff("band_lp21")]
            + [ParamsMidRun(rng), ParamsMidRun(rng)])


def lay_out(cs, L, shift=0):
    """Lane l runs case (l + shift) % len(cs) -> (lane cases, signal [T][L][480], noise [T][L][480], params {frame: [L]}):
    every frame that changes a lane's parameters sets all lanes (the others to what they already had)."""
    lane = [cs[(l + shift) % len(cs)] for l in range(L)]
    sig = np.stack([c.signal for c in lane], axis=1)
    noi = np.stack([c.noise for c in lane], axis=1)
    cur = tr.default_params(L)
    table = {}
    for t in sorted({t for c in lane for t in c.schedule}):
        for l, c in enumerate(lane):
            if t in c.schedule:
                cur[l] = c.schedule[t]
        table[t] = cur.copy()
    return lane, sig, noi, table


def params_by_frame(table, L):
    """The parameters in force during each frame: [T][L]."""
    cur, out = tr.default_params(L), np.empty((T, L), tr.SIM_PARAMS_DTYPE)
    for t in range(T):
        if t in table:
            cur = table[t]
        out[t] = cur
    return out
