"""The float64 reference of the spectral stages (tests/spectral_ref.py) against the golden-pinned oracle, without a GPU.

- The float64 FFTs equal the oracle's f64 DFT mode rounded once to f32.
- Driven by the oracle's own states over the signal set of test_spectral_kernels.py, the reference's analysis and
  synthesis agree with the oracle within the spread of the oracle's three FFTs.
- Every output of the reference, the band quantities and features included, lies within what the oracle's three FFTs
  allow: their spread plus the f32 rounding they share, both derived.
- The same frames, with the oracle's f64-DFT order in the GPU's place, pass the checks test_spectral_kernels.py applies
  to the GPU.
"""
import numpy as np
import pytest

import nnnoiseless_b200 as nb
import oracle
import oracle_state as ost
import spectral_ref as sr
import test_spectral_kernels as tk


def _half_ulp(v):
    return 0.5 * np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


def test_float64_fft_against_oracle_f64_dft():
    """np.fft in float64 against the oracle's DFT sums in f64 (nno_set_fft_mode(1)), which round to f32 once: every
    bin and sample within half an f32 ulp plus 1e-12 of the largest magnitude."""
    L = oracle.lib()
    rng = np.random.default_rng(3)
    fr = [rng.standard_normal(960) * 1000, np.cos(2 * np.pi * 240 * np.arange(960) / 960) * 3e4, np.ones(960) * 7.0,
          np.where(np.arange(960) % 2 == 0, 1.0, -1.0) * 1e-5]
    L.nno_set_fft_mode(1)
    try:
        for x in fr:
            x = x.astype(np.float32)
            re, im = np.empty(481, np.float32), np.empty(481, np.float32)
            L.nno_rfft960(x.ctypes.data, re.ctypes.data, im.ctypes.data)
            ref = np.fft.rfft(x.astype(np.float64))
            lim = 1e-12 * np.abs(ref).max()
            assert (np.abs(re - ref.real) <= _half_ulp(ref.real) + lim).all()
            assert (np.abs(im - ref.imag) <= _half_ulp(ref.imag) + lim).all()
            X = (rng.standard_normal(481) + 1j * rng.standard_normal(481)) * np.abs(x).max()
            X[0], X[480] = X[0].real, X[480].real
            Xr, Xi = np.ascontiguousarray(X.real, np.float32), np.ascontiguousarray(X.imag, np.float32)
            out = np.empty(960, np.float32)
            L.nno_irfft960(Xr.ctypes.data, Xi.ctypes.data, out.ctypes.data)
            y = 960.0 * np.fft.irfft(Xr.astype(np.float64) + 1j * Xi.astype(np.float64), n=960)
            assert (np.abs(out - y) <= _half_ulp(y) + 1e-12 * np.abs(y).max()).all()
    finally:
        L.nno_set_fft_mode(0)


def oracle_frames(model: bytes, x, mode=1):
    """The oracle, with FFT `mode`, in the GPU's place: per frame the dict run_frames gives for the GPU."""
    ost.set_fft_mode(mode)
    try:
        return _oracle_frames(model, x)
    finally:
        ost.set_fft_mode(0)


def _oracle_frames(model, x):
    om = ost.Model(model)
    orc = oracle.Model(model)
    widths = nb.gru_widths(model)
    dt = nb.state_dtype(widths)
    nst, nfr = x.shape[:2]
    states = [ost.State(om) for _ in range(nst)]
    prev = np.stack([s.export() for s in states])
    frames = []
    for f in range(nfr):
        a = [ost.analysis_frame(om, prev[s], x[s, f]) for s in range(nst)]
        rb = prev.view(dt).reshape(-1)
        gains = np.zeros((nst, sr.NB_BANDS), np.float32)
        vad = np.zeros(nst, np.float32)
        for s in range(nst):
            if not a[s]["silence"]:
                g = rb["vad_gru"][s], rb["noise_gru"][s], rb["denoise_gru"][s]
                _, _, _, gains[s], vad[s] = oracle.rnn_step(orc, *g, a[s]["features"])
        out = np.empty((nst, 480), np.float32)
        for s in range(nst):
            out[s], _ = states[s].process_frame(x[s, f])
        rec = np.stack([s.export() for s in states])
        st = lambda k: np.stack([o[k] for o in a])  # noqa: E731
        sil = st("silence").astype(np.int32)
        frames.append(dict(before=prev, after=rec, rb=rb, ra=rec.view(dt).reshape(-1), pitch=st("pitch").astype(np.int32),
                           silence=sil, features=st("features"), gains=gains, vad=vad, vad_out=np.where(sil != 0, 0.0, vad),
                           out=out, X=st("X"), P=np.ascontiguousarray(st("P")[:, :sr.NB_BINS_BANDED]), ex=st("ex"),
                           ep=st("ep"), exp=st("exp")))
        prev = rec
    return frames


@pytest.fixture(scope="module")
def driven(builtin_bytes):
    x, _ = tk.spectral_signals()
    return x, oracle_frames(builtin_bytes, x), builtin_bytes


def _modes(fn):
    out = []
    for mode in (0, 1, 2):
        ost.set_fft_mode(mode)
        try:
            out.append(fn())
        finally:
            ost.set_fft_mode(0)
    return out


def test_reference_within_oracle_fft_spread(driven):
    """Every output of the float64 reference, element by element, against the nearest of the oracle's three FFTs
    (pinned f32, f64 DFT, f32 in another radix order) on the same inputs.  The allowance is the part where they differ
    plus the part they share, each derived rather than assumed:
    - FFT: for the spectra the per-stream spread of the three over all bins (FFT rounding is spread over the bins in
      absolute terms); for everything after them the element's own spread, or that spectrum spread propagated to first
      order through the band weights, the normalisation, the logs and DCTs (spectral_ref.analysis_bounds), whichever is
      larger;
    - shared: the rounding of the f32 products window x input before the FFT, propagated the same way, plus the f32
      arithmetic after the FFT that all three do alike (analysis_bounds with arith; synthesis_bounds), plus half an f32
      ulp of the element (the oracle's outputs are f32).
    A float64 reference that were wrong by more than this would be caught here, before it could widen the GPU test's
    yardstick, which is built from the deviation of the oracle's f32 orders from it."""
    x, frames, model = driven
    om = ost.Model(model)
    nst = len(x)
    worst = {}
    cplx = lambda a: np.asarray(a).astype(np.complex128 if np.iscomplexobj(a) else np.float64)  # noqa: E731

    def within(q, r64, os_, allow, live=None):
        os_ = [cplx(o) for o in os_]
        near = np.min([np.abs(o - r64) for o in os_], axis=0)
        lim = allow + 0.5 * np.spacing(np.abs(r64).astype(np.float32)).astype(np.float64)
        if live is not None:
            near, lim = near[live], lim[live]
        worst[q] = max(worst.get(q, 0.0), float(tk._share(near, lim).max(initial=0.0)))
        assert (near <= lim).all(), (q, np.argwhere(near > lim)[:5], float(tk._share(near, lim).max()))

    def spread(os_, per_stream=False):
        os_ = [cplx(o) for o in os_]
        d = np.max([np.abs(a - b) for a in os_ for b in os_], axis=0)
        return d.reshape(len(d), -1).max(axis=1).reshape((-1,) + (1,) * (d.ndim - 1)) if per_stream else d

    for f, fr in enumerate(frames):
        rb, ra = fr["rb"], fr["ra"]
        ref = sr.analysis(ra["input_mem"], fr["pitch"], rb["cepstral_mem"], rb["mem_id"])
        o = _modes(lambda: [ost.analysis_frame(om, fr["before"][s], x[s, f]) for s in range(nst)])
        o = [{k: np.stack([d[k] for d in r]) for k in r[0]} for r in o]
        wX, wP = sr.windowing_bounds(ra["input_mem"], fr["pitch"])
        sX, sP = spread([d["X"] for d in o], True), spread([d["P"][:, :sr.NB_BINS_BANDED] for d in o], True)
        # the spectra: FFT spread + windowing + the wnorm product
        within("X", ref["X"], [d["X"] for d in o], sX + wX + tk.U32 * np.abs(ref["X"]))
        within("P", ref["P"], [d["P"] for d in o], sP + wP + tk.U32 * np.abs(ref["P"]))
        dX, dP = sX + wX + tk.U32 * np.abs(ref["X"]), sP + wP + tk.U32 * np.abs(ref["P"])
        band = {q: spread([d[q] for d in o]) for q in ("ex", "ep", "exp")}
        b = sr.analysis_bounds(ref, dX, dP, band=band, arith=True)
        for q in ("ex", "ep", "exp"):
            within(q, ref[q], [d[q] for d in o], b[q])
        # features and the new row where all three took the reference's (non-silent) branch
        live = ~ref["silence"] & np.all([d["silence"] == 0 for d in o], axis=0)
        rows = np.arange(nst)
        mid = rb["mem_id"]
        within("features", ref["features"], [d["features"] for d in o], np.maximum(spread([d["features"] for d in o]), b["features"]), live)
        within("ceps row", ref["row"], [d["ceps"][rows, mid] for d in o], np.maximum(spread([d["ceps"][rows, mid] for d in o]), b["row"]), live)
        sil = fr["silence"] != 0
        Pf = np.zeros((nst, sr.FREQ_SIZE), np.complex64)
        Pf[:, :sr.NB_BINS_BANDED] = fr["P"]
        args = (fr["X"], fr["P"], fr["ex"], fr["ep"], fr["exp"], fr["gains"], rb["lastg"], rb["synthesis_mem"], sil)
        ref = sr.synthesis(*args)
        o = _modes(lambda: [ost.synthesis_from(fr["X"][s], Pf[s], fr["ex"][s], fr["ep"][s], fr["exp"][s], fr["gains"][s],
                                               rb["lastg"][s], rb["synthesis_mem"][s], sil[s]) for s in range(nst)])
        d_out, d_mem = sr.synthesis_bounds(ref)
        for q, i, dq in (("out", 0, d_out), ("synth_mem", 2, d_mem)):
            os_ = [np.stack([d[i] for d in r]) for r in o]
            within(q, ref[q], os_, spread(os_, True) + dq)
        assert np.array_equal(np.stack([d[1] for d in o[0]]), ra["lastg"])
    print("\nlargest share of the allowance:", ", ".join("%s %.2f" % kv for kv in worst.items()))


def test_kernel_checks_pass_with_the_oracle_in_place_of_the_gpu(driven):
    """The GPU test's checks, with the oracle's f64-DFT order in the GPU's place.  It is not one of the two f32 orders the
    yardstick d32 is built from, so this is a real run of every check: an f32 implementation whose only difference is a
    more accurate FFT must pass with room to spare."""
    x, frames, model = driven
    om = ost.Model(model)
    wa, ws, cov = tk.Worst(), tk.Worst(), tk.new_coverage()
    for f, fr in enumerate(frames):
        tk.check_analysis(fr, tk.oracle_analysis(om, frames, x, f), wa, cov)
        tk.check_synthesis(fr, ws, cov)
    print("\nK3:", wa.line())
    print("K5:", ws.line())
    for w in (wa, ws):
        for q, (_, share) in w.q.items():
            assert share <= 0.5, (q, share)
    assert cov["mem_ids"] == set(range(8)) and cov["near_silent"] and cov["near_live"]
