"""Fit denoise models to training rows on the GPU: the counterpart of the reference's ``train/rnn_train.py`` (Keras)
followed by ``train/dump_rnn.py``.

The arithmetic -- forward pass, backprop through time, loss, Adam, weight clip -- runs in the hand-written kernels of
``csrc/fit.cu`` behind ``rnnoise_fit_*`` (include/rnnoise.h).  This module is the host control plane, as
``training.randomize`` is for the rows: windowing, sample weights, initialisation, the epoch loop and shuffling.

    python -m nnnoiseless_b200.fit rows.npy -o weights.rnn

rows.npy holds the generator's rows, ``[frames][lanes][87]`` (or ``[frames][87]`` for one lane).  There is NO CPU
fallback: without the CUDA library / a GPU, :class:`Fit` raises.
"""
import argparse
import ctypes as C

import numpy as np

from . import NB_BANDS, NB_FEATURES, NnnoiselessError, RnnModel, _np_ptr, last_error, lib

TRAIN_ROW = NB_FEATURES + 2 * NB_BANDS + 1
WIDTHS = (24, 24, 48, 96)  # input_dense, vad_gru, noise_gru, denoise_gru (rnn_train.py:66-73)
LAYERS = ("input_dense", "vad_gru", "noise_gru", "denoise_gru", "denoise_output", "vad_output")


def layer_shapes(widths=WIDTHS):
    """The parameter arrays in the order of the flat vector (the .rnn file's layer order), Keras shapes:
    [(layer, name, shape)] with name kernel / recurrent_kernel / bias."""
    nd, nv, nn, ndn = (int(w) for w in widths)
    spec = [("input_dense", NB_FEATURES, nd, 1), ("vad_gru", nd, nv, 3), ("noise_gru", nd + nv + NB_FEATURES, nn, 3),
            ("denoise_gru", nv + nn + NB_FEATURES, ndn, 3), ("denoise_output", ndn, NB_BANDS, 1), ("vad_output", nv, 1, 1)]
    out = []
    for name, ni, n, gates in spec:
        out.append((name, "kernel", (ni, gates * n)))
        if gates == 3:
            out.append((name, "recurrent_kernel", (n, 3 * n)))
        out.append((name, "bias", (gates * n,)))
    return out


def n_params(widths=WIDTHS) -> int:
    return sum(int(np.prod(s)) for _, _, s in layer_shapes(widths))


def unflatten(params, widths=WIDTHS):
    """Flat vector -> {(layer, name): array view of its Keras shape}."""
    out, p = {}, 0
    for layer, name, shape in layer_shapes(widths):
        k = int(np.prod(shape))
        out[(layer, name)] = params[p:p + k].reshape(shape)
        p += k
    return out


def windows(rows, window: int) -> np.ndarray:
    """Rows [frames][lanes][87] (or [frames][87]) -> sequences [n][window][87]: each lane cut into whole windows in time
    order, lane after lane, so that no window mixes lanes (rnn_train.py:91-105 cuts one stream the same way).  The
    frames past a lane's last whole window are dropped."""
    rows = np.asarray(rows, np.float32)
    if rows.ndim == 2:
        rows = rows[:, None, :]
    if rows.ndim != 3 or rows.shape[2] != TRAIN_ROW:
        raise ValueError("rows must be [frames][lanes][87]")
    frames, lanes, _ = rows.shape
    k = frames // int(window)
    lane_major = np.ascontiguousarray(rows[:k * window].transpose(1, 0, 2))
    return lane_major.reshape(lanes * k, window, TRAIN_ROW)


def sample_weights(rows) -> np.ndarray:
    """rnn_train.py:108-118: each row's weight from the mean of its unmasked gains, so that the hi (> 2/3), med and lo
    (< 1/3) classes carry the same total weight.  rows [..., 87] -> weights [...] (float32).  A row whose gains are all
    masked gets weight 0.  If a class is empty the reference divides by zero and trains on NaN weights; this raises
    ValueError naming the class instead."""
    rows = np.asarray(rows)
    y = rows[..., NB_FEATURES:NB_FEATURES + NB_BANDS].astype(np.float64)
    valid = y != -1
    cnt = valid.sum(axis=-1)
    means = np.where(cnt > 0, np.where(valid, y, 0.0).sum(axis=-1) / np.maximum(cnt, 1), np.nan)
    with np.errstate(invalid="ignore"):
        hi, lo = means > 2 / 3, means < 1 / 3
        med = (means >= 1 / 3) & (means <= 2 / 3)
    total = hi.size
    w = np.zeros(hi.shape)
    for name, cls in (("hi", hi), ("med", med), ("lo", lo)):
        k = int(cls.sum())
        if k == 0:
            raise ValueError("no training row falls in the %s gain class; the reference's weights would be NaN" % name)
        w += cls * (total / k)
    return (w / 3).astype(np.float32)


def init_params(widths=WIDTHS, seed=0) -> np.ndarray:
    """Keras initialisation (tf.keras 2.x defaults of Dense / GRU): kernels glorot_uniform (limit
    sqrt(6 / (fan_in + fan_out)), fan_out = 3n for a GRU kernel), recurrent kernels orthogonal, biases zero; drawn from
    numpy's generator seeded with `seed`.  -> flat float32 vector."""
    rng = np.random.default_rng(seed)
    parts = []
    for _, name, shape in layer_shapes(widths):
        if name == "bias":
            parts.append(np.zeros(shape))
        elif name == "kernel":
            lim = np.sqrt(6.0 / (shape[0] + shape[1]))
            parts.append(rng.uniform(-lim, lim, shape))
        else:  # Orthogonal: QR of a normal [3n][n] matrix, signs fixed by diag(R), transposed to [n][3n]
            q, r = np.linalg.qr(rng.standard_normal((shape[1], shape[0])))
            parts.append((q * np.sign(np.diag(r))).T)
    return np.concatenate([p.reshape(-1) for p in parts]).astype(np.float32)


def export_params(params, widths=WIDTHS) -> bytes:
    """The .rnn bytes of a flat parameter vector (dump_rnn.py), computed by the library on the host."""
    p = np.ascontiguousarray(params, np.float32)
    if p.size != n_params(widths):
        raise ValueError("expected %d parameters" % n_params(widths))
    nd, nv, nn, ndn = (int(w) for w in widths)
    n = lib().rnnoise_fit_export_params(nd, nv, nn, ndn, _np_ptr(p), None, 0)
    if n == 0:
        raise NnnoiselessError(last_error())
    buf = (C.c_ubyte * n)()
    if lib().rnnoise_fit_export_params(nd, nv, nn, ndn, _np_ptr(p), buf, n) != n:
        raise NnnoiselessError(last_error())
    return bytes(buf)


class Fit:
    """One network being fitted on one GPU (rnnoise_fit_*): up to max_sequences windows of `window` frames per call."""

    def __init__(self, widths=WIDTHS, max_sequences=32, window=2000, device=-1):
        self.widths = tuple(int(w) for w in widths)
        self.max_sequences, self.window = int(max_sequences), int(window)
        self._h = lib().rnnoise_fit_create(*self.widths, self.max_sequences, self.window, int(device))
        if not self._h:
            raise NnnoiselessError("rnnoise_fit_create failed: " + last_error())
        self.n_params = int(lib().rnnoise_fit_n_params(self._h))

    def _check(self, rc):
        if rc != 0:
            raise NnnoiselessError(last_error())

    def get_params(self) -> np.ndarray:
        p = np.empty(self.n_params, np.float32)
        self._check(lib().rnnoise_fit_get_params(self._h, _np_ptr(p)))
        return p

    def set_params(self, params):
        """Set the flat parameter vector; resets Adam."""
        p = np.ascontiguousarray(params, np.float32)
        if p.size != self.n_params:
            raise ValueError("expected %d parameters" % self.n_params)
        self._check(lib().rnnoise_fit_set_params(self._h, _np_ptr(p)))

    def set_params_from_model(self, model: RnnModel = None):
        """Start from a model's weights (int8 / 256); None: the built-in model.  Resets Adam."""
        self._check(lib().rnnoise_fit_set_params_from_model(self._h, model._h if model is not None else None))

    def _inputs(self, rows, weights):
        rows = np.ascontiguousarray(rows, np.float32)
        weights = np.ascontiguousarray(weights, np.float32)
        if rows.ndim != 3 or rows.shape[1:] != (self.window, TRAIN_ROW) or weights.shape != rows.shape[:2]:
            raise ValueError("expected rows [n][%d][87] and weights [n][%d]" % (self.window, self.window))
        return rows, weights

    def step(self, rows, weights) -> float:
        """One Adam step on rows [n][window][87] with weights [n][window]; returns the loss before the step."""
        rows, weights = self._inputs(rows, weights)
        loss = C.c_double()
        self._check(lib().rnnoise_fit_step(self._h, _np_ptr(rows), _np_ptr(weights), len(rows), C.byref(loss)))
        return loss.value

    def evaluate(self, rows, weights) -> dict:
        """The loss without a step: dict(loss, mycost, crossentropy, msse)."""
        rows, weights = self._inputs(rows, weights)
        out = (C.c_double * 4)()
        self._check(lib().rnnoise_fit_evaluate(self._h, _np_ptr(rows), _np_ptr(weights), len(rows), out))
        return dict(loss=out[0], mycost=out[1], crossentropy=out[2], msse=out[3])

    def grads(self) -> np.ndarray:
        """Debug tap: the gradient of the most recent step's loss (L2 included), flat."""
        g = np.empty(self.n_params, np.float32)
        self._check(lib().rnnoise_fit_get_grads(self._h, _np_ptr(g)))
        return g

    def activations(self, n_seq: int) -> dict:
        """Debug tap of the most recent forward pass over n_seq sequences: dict(gains, vad, state)."""
        T = self.window
        gains = np.empty((n_seq, T, NB_BANDS), np.float32)
        vad = np.empty((n_seq, T), np.float32)
        state = np.empty((n_seq, T, sum(self.widths[1:])), np.float32)
        self._check(lib().rnnoise_fit_get_activations(self._h, _np_ptr(gains), _np_ptr(vad), _np_ptr(state)))
        return dict(gains=gains, vad=vad, state=state)

    def export(self) -> bytes:
        """The .rnn bytes of the current parameters (dump_rnn.py)."""
        n = lib().rnnoise_fit_export(self._h, None, 0)
        if n == 0:
            raise NnnoiselessError(last_error())
        buf = (C.c_ubyte * n)()
        if lib().rnnoise_fit_export(self._h, buf, n) != n:
            raise NnnoiselessError(last_error())
        return bytes(buf)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib().rnnoise_fit_destroy(h)
            self._h = None


def fit(rows, epochs=20, batch_size=32, window=2000, validation_split=0.1, seed=0, widths=WIDTHS, init_model=None,
        device=-1, verbose=False):
    """rnn_train.py:84-129: windows of `window` frames, sample weights over all of them, the last `validation_split`
    of the windows held out (before any shuffling), the training windows shuffled every epoch, batches of batch_size.
    Returns (RnnModel of the exported weights, history dict(loss, val_loss) per epoch: the mean of the batch losses
    weighted by batch size, as Keras reports them)."""
    seqs = windows(rows, window)
    if len(seqs) == 0:
        raise ValueError("fewer frames than one window")
    wts = sample_weights(seqs)
    split_at = int(np.floor(len(seqs) * (1.0 - validation_split)))
    if split_at < 1:
        raise ValueError("no training windows left after the validation split")
    f = Fit(widths, min(batch_size, len(seqs)), window, device)
    if init_model is not None:
        f.set_params_from_model(init_model)
    else:
        f.set_params(init_params(widths, seed))
    rng = np.random.default_rng(seed)
    history = dict(loss=[], val_loss=[])
    for epoch in range(int(epochs)):
        order = rng.permutation(split_at)
        total = 0.0
        for b0 in range(0, split_at, batch_size):
            idx = order[b0:b0 + batch_size]
            total += f.step(seqs[idx], wts[idx]) * len(idx)
        history["loss"].append(total / split_at)
        if split_at < len(seqs):
            total = 0.0
            for b0 in range(split_at, len(seqs), batch_size):
                sl = slice(b0, min(b0 + batch_size, len(seqs)))
                total += f.evaluate(seqs[sl], wts[sl])["loss"] * (sl.stop - sl.start)
            history["val_loss"].append(total / (len(seqs) - split_at))
        if verbose:
            print("epoch %d: loss %.6f%s" % (epoch + 1, history["loss"][-1],
                                             "  val_loss %.6f" % history["val_loss"][-1] if history["val_loss"] else ""))
    model = RnnModel.from_bytes(f.export())
    if model is None:
        raise NnnoiselessError("the exported model does not parse")
    return model, history


def main(argv=None):
    ap = argparse.ArgumentParser(description="Fit a denoise model to training rows on the GPU and write it as .rnn")
    ap.add_argument("rows", help=".npy of training rows [frames][lanes][87] (or [frames][87])")
    ap.add_argument("-o", "--output", default="weights.rnn")
    ap.add_argument("--epochs", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--window", type=int, default=2000)
    ap.add_argument("--validation-split", type=float, default=0.1)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--widths", type=lambda s: tuple(int(x) for x in s.split(",")), default=WIDTHS,
                    help="input_dense,vad_gru,noise_gru,denoise_gru neurons (default 24,24,48,96)")
    ap.add_argument("--init-model", help="start from this .rnn model (fine-tuning)")
    ap.add_argument("--device", type=int, default=-1)
    a = ap.parse_args(argv)
    init = None
    if a.init_model:
        with open(a.init_model, "rb") as fh:
            init = RnnModel.from_bytes(fh.read())
        if init is None:
            raise SystemExit("%s is not a valid model" % a.init_model)
    model, _ = fit(np.load(a.rows, mmap_mode="r"), a.epochs, a.batch_size, a.window, a.validation_split, a.seed, a.widths,
                   init, a.device, verbose=True)
    with open(a.output, "wb") as fh:
        fh.write(model.to_bytes())
    print("wrote", a.output)


if __name__ == "__main__":
    main()
