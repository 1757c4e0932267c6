"""A numpy restatement of one training frame (src/training.rs), vectorised over lanes (TEST INFRASTRUCTURE).

FrontRef repeats NoiseSimulator::next_frame (src/training.rs:388-421) and the three feature extractors'
shift_and_filter_input (src/features.rs:97-104) bit for bit: numpy's float32 and float64 operations are IEEE, rounded
once each and never contracted, so the reference's statements are restated in their own order and precision --
  * the frame energy before the gain: a float32 sum over the 480 samples in order (read_signal, :331-339);
  * the gains: float32 products (read_noise :322-328, read_signal);
  * the two random-filter biquads: float64 arithmetic, float32 memory (Biquad::filter_in_place, src/util.rs:109-124);
  * the mix: a float32 sum (:402-404);
  * the three BIQUAD_HP chains (src/util.rs:68-71, 95-107), into each stream's last 1728 high-passed samples;
  * the VAD counter, its clamp and the gain cutoff (:368-386, :406-413).
Every lane carries its parameters, resp_mem (signal m0 m1, noise m0 m1), vad_count, and per stream (clean, noise,
combined) mem_hp_x and the history window.

assemble_rows builds the rest of the 87-float row (src/training.rs:132-159) from a frame's band energies ex and
combined-stream silence flags: the gain columns in float32, the noise levels as float64 log10 of the float32 sum, the
VAD column.  The features are the combined stream's own."""
import numpy as np

F32, F64 = np.float32, np.float64
FRAME = 480
HIST = 1728
NB_BANDS = 22
NB_FEATURES = 42
ROW = NB_FEATURES + 2 * NB_BANDS + 1

SIM_PARAMS_DTYPE = np.dtype([
    ("signal_gain", F32), ("noise_gain", F32),
    ("sig_a", F32, 2), ("sig_b", F32, 2),
    ("noise_a", F32, 2), ("noise_b", F32, 2),
    ("band_lp", np.int32),
])  # RNNoiseSimParams / nno_sim_params
HP_A = (F32(-1.99599), F32(0.99600))  # BIQUAD_HP, src/util.rs:68-71
HP_B = (F32(-2.0), F32(1.0))


def default_params(n):
    """NoiseSimulator::new (src/training.rs:300-320): gains 1, zero filters, band_lp 21."""
    p = np.zeros(n, SIM_PARAMS_DTYPE)
    p["signal_gain"] = 1.0
    p["noise_gain"] = 1.0
    p["band_lp"] = NB_BANDS - 1
    return p


def biquad(x, a, b, mem):
    """Biquad::filter_in_place over x [L][n] float32 with coefficients a, b [L][2] float32 and memory mem [L][2]
    float32 (updated in place) -> y [L][n] float32."""
    a0, a1 = a[:, 0].astype(F64), a[:, 1].astype(F64)
    b0, b1 = b[:, 0].astype(F64), b[:, 1].astype(F64)
    m0, m1 = mem[:, 0].copy(), mem[:, 1].copy()
    y = np.empty_like(x)
    for i in range(x.shape[1]):
        x64 = x[:, i].astype(F64)
        y64 = x64 + m0.astype(F64)
        m0 = (m1.astype(F64) + (b0 * x64 - a0 * y64)).astype(F32)
        m1 = (b1 * x64 - a1 * y64).astype(F32)
        y[:, i] = y64.astype(F32)
    mem[:, 0], mem[:, 1] = m0, m1
    return y


def frame_energy(x):
    """read_signal's energy: float32, sample 0 first. x [L][480] -> [L]."""
    e = np.zeros(x.shape[0], F32)
    for i in range(x.shape[1]):
        e = e + x[:, i] * x[:, i]
    return e


class FrontRef:
    def __init__(self, n_lanes):
        L = self.L = int(n_lanes)
        self.params = default_params(L)
        self.resp_mem = np.zeros((L, 4), F32)
        self.vad_count = np.zeros(L, np.int32)
        self.hp_mem = np.zeros((3, L, 2), F32)   # [clean | noise | combined][lane]
        self.hist = np.zeros((3, L, HIST), F32)

    def set_params(self, params, lanes=None):
        """randomize()'s outcome: the parameters change, every memory carries over."""
        lanes = np.arange(self.L) if lanes is None else np.asarray(lanes)
        self.params[lanes] = params

    def frame(self, signal, noise):
        """signal, noise [L][480] (raw, i16-valued) -> dict(energy, vad_count, vad, cutoff) of the frame; advances
        every memory and the three histories."""
        sig = np.asarray(signal, F32).reshape(self.L, FRAME)
        noi = np.asarray(noise, F32).reshape(self.L, FRAME)
        p = self.params
        with np.errstate(over="ignore", invalid="ignore"):
            energy = frame_energy(sig)
            s = sig * p["signal_gain"][:, None]
            n = noi * p["noise_gain"][:, None]
            s = biquad(s, p["sig_a"], p["sig_b"], self.resp_mem[:, 0:2])
            n = biquad(n, p["noise_a"], p["noise_b"], self.resp_mem[:, 2:4])
            z = s + n
            a = np.broadcast_to(np.array(HP_A, F32), (self.L, 2))
            b = np.broadcast_to(np.array(HP_B, F32), (self.L, 2))
            for k, x in enumerate((s, n, z)):
                m = self.hp_mem[k].copy()
                y = biquad(x, a, b, m)
                self.hp_mem[k] = m
                self.hist[k] = np.concatenate([self.hist[k][:, FRAME:], y], axis=1)
        vc = self.vad_count.astype(np.int64)
        vc = np.where(energy > F32(1e9), 0, np.where(energy > F32(1e8), vc - 5, np.where(energy > F32(1e7), vc + 1, vc + 2)))
        self.vad_count = np.clip(vc, 0, 15).astype(np.int32)
        vad = np.where(self.vad_count >= 10, F32(0.0), np.where(self.vad_count > 0, F32(0.5), F32(1.0))).astype(F32)
        cutoff = np.where((vad == 0.0) & (p["noise_gain"] == 0.0), 0, p["band_lp"] + 1).astype(np.int32)
        return dict(energy=energy, vad_count=self.vad_count.copy(), vad=vad, cutoff=cutoff)


def silence_from_ex(ex):
    """compute_frame_features' silence test (src/features.rs): the float32 sum of the 22 band energies, band 0 first,
    below 0.04.  ex [..][22] -> bool [..]."""
    e = np.zeros(ex.shape[:-1], F32)
    for i in range(NB_BANDS):
        e = e + ex[..., i]
    return e < F32(0.04)


def gains_f32(ce, me, cutoff, silence):
    """The gain columns (src/training.rs:141-151) in float32: min(sqrt((ce + 1e-3) / (me + 1e-3)), 1), -1 where both
    band energies are below 5e-2 and from the cutoff on (0 on a silent combined frame).  ce, me [L][22] float32."""
    ce, me = np.asarray(ce, F32), np.asarray(me, F32)
    g = np.minimum(np.sqrt((ce + F32(1e-3)) / (me + F32(1e-3))), F32(1.0))
    masked = (ce < F32(5e-2)) & (me < F32(5e-2))
    cut = np.where(silence, 0, cutoff)
    masked |= np.arange(NB_BANDS)[None, :] >= cut[:, None]
    return np.where(masked, F32(-1.0), g).astype(F32)


def gains_unclamped_f64(ce, me):
    """The same quotient in float64 without the clamp: the check on gains_f32 and the measure of the clamp."""
    ce, me = np.asarray(ce, F32).astype(F64), np.asarray(me, F32).astype(F64)
    return np.sqrt((ce + F64(F32(1e-3))) / (me + F64(F32(1e-3))))


def noise_levels_f64(ne):
    """log10 of the float32 sum ne + 1e-2 (src/training.rs:152), evaluated in float64."""
    return np.log10((np.asarray(ne, F32) + F32(1e-2)).astype(F64))


def assemble_rows(ex, silence, features, vad, cutoff):
    """ex [3][L][22] (clean, noise, combined), silence [L] of the combined stream, features [L][42] of the combined
    stream, vad [L], cutoff [L] -> (rows [L][87] float32 with the noise levels rounded from float64, noise levels [L][22]
    in float64)."""
    L = ex.shape[1]
    rows = np.empty((L, ROW), F32)
    rows[:, :NB_FEATURES] = features
    rows[:, NB_FEATURES:NB_FEATURES + NB_BANDS] = gains_f32(ex[0], ex[2], cutoff, silence)
    nl = noise_levels_f64(ex[1])
    rows[:, NB_FEATURES + NB_BANDS:ROW - 1] = nl.astype(F32)
    rows[:, ROW - 1] = vad
    return rows, nl
