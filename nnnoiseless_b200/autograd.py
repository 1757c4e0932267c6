"""Torch autograd through synthesis (DESIGN.md 7i): train a network between ``DenoiseBatch.analyze_device`` and
``DenoiseBatch.synthesize_saving_device`` on a loss of the output samples.

    out = synthesis_grad(gains, out, ctx)   # out now depends on gains in torch's graph
    loss(out, target).backward()            # gains.grad from rnnoise_synthesis_backward_device, on the GPU

``DenoiseNetwork`` is the network the library serves, as a torch module (DESIGN.md 7l): trained through synthesis, it
exports a ``.rnn`` model that ``DenoiseBatch`` runs on the fused path.

``intelligibility`` is STOI and ESTOI as a loss (DESIGN.md 7r): its gradient reaches ``out`` through
rnnoise_intelligibility_backward_device, so a network can train on ``1 - ESTOI`` through ``synthesis_grad``.

This module imports torch; the package itself does not.
"""
import torch

from . import (NB_BANDS, NB_FEATURES, FRAME_SIZE, SYNTH_CONTEXT_BYTES, INTELLIGIBILITY_DTYPE, RnnModel, NnnoiselessError, gru_widths,
               intelligibility_backward_device, intelligibility_backward_workspace_bytes, intelligibility_device,
               intelligibility_workspace_bytes, synthesis_backward_device, synthesis_backward_workspace_bytes)
from . import fit


def _layout(x, batch_first, last):
    """(stream stride, frame stride) of a [B][T][last] (batch_first) or [T][B][last] tensor whose rows are contiguous."""
    if x.dim() != 3 or x.shape[2] != last or x.stride(2) != 1:
        raise ValueError("expected a %s tensor with contiguous rows of %d" % ("[B][T][.]" if batch_first else "[T][B][.]", last))
    return (x.stride(0), x.stride(1)) if batch_first else (x.stride(1), x.stride(0))


class _SynthesisGrad(torch.autograd.Function):
    @staticmethod
    def forward(fctx, gains, out, ctx, batch_first):
        fctx.save_for_backward(ctx)
        fctx.batch_first = batch_first
        fctx.gains_shape = gains.shape
        return out.view_as(out)

    @staticmethod
    def backward(fctx, grad_out):
        (ctx,) = fctx.saved_tensors
        bf = fctx.batch_first
        if grad_out.stride(2) != 1:
            grad_out = grad_out.contiguous()
        B, T = (grad_out.shape[0], grad_out.shape[1]) if bf else (grad_out.shape[1], grad_out.shape[0])
        go_s, go_f = _layout(grad_out, bf, FRAME_SIZE)
        grad = torch.empty(fctx.gains_shape, dtype=torch.float32, device=grad_out.device)
        gg_s, gg_f = _layout(grad, bf, NB_BANDS)
        cs, cf = (ctx.stride(0), ctx.stride(1)) if bf else (ctx.stride(1), ctx.stride(0))
        nbytes = synthesis_backward_workspace_bytes(B, T)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=grad_out.device)
        synthesis_backward_device(ctx.data_ptr(), cs // SYNTH_CONTEXT_BYTES, cf // SYNTH_CONTEXT_BYTES, grad_out.data_ptr(), go_s, go_f,
                                  grad.data_ptr(), gg_s, gg_f, B, T, ws.data_ptr(), nbytes, grad_out.device.index,
                                  torch.cuda.current_stream(grad_out.device).cuda_stream)
        return grad, None, None, None


def synthesis_grad(gains, out, ctx, batch_first=True):
    """Attach the output of a window of saving synthesis calls to the raw gains they used.

    gains: float32 [B][T][22] (batch_first) or [T][B][22], the tensor whose values were passed to the saving calls
    (typically the network's output, requiring grad).  out: float32 [B][T][480] or [T][B][480], what those calls wrote.
    ctx: uint8 [B][T][SYNTH_CONTEXT_BYTES] or [T][B][SYNTH_CONTEXT_BYTES], their context records.  All on one GPU.
    Returns out as a tensor of the graph: its gradient reaches gains through rnnoise_synthesis_backward_device, run on
    the current torch stream.  The gradient's contract (window, kinks, silent frames) is include/rnnoise.h's."""
    for name, x, dt in (("gains", gains, torch.float32), ("out", out, torch.float32), ("ctx", ctx, torch.uint8)):
        if x.dtype != dt or not x.is_cuda:
            raise ValueError("%s must be a %s CUDA tensor" % (name, dt))
    _layout(gains, batch_first, NB_BANDS)
    _layout(out, batch_first, FRAME_SIZE)
    _layout(ctx, batch_first, SYNTH_CONTEXT_BYTES)
    if gains.shape[:2] != out.shape[:2] or ctx.shape[:2] != out.shape[:2]:
        raise ValueError("gains, out and ctx must have the same leading dimensions")
    return _SynthesisGrad.apply(gains, out, ctx, batch_first)


def _strides(x, batch_first):
    """(sequence stride, frame stride) of a [B][T][..] (batch_first) or [T][B][..] tensor."""
    return (x.stride(0), x.stride(1)) if batch_first else (x.stride(1), x.stride(0))


def check_window(features, silence, state, batch_first, window, max_streams, state_width, device):
    """What DenoiseNetwork.forward checks before any library call: dtypes, shapes, layouts and devices.  -> B."""
    if not isinstance(features, torch.Tensor) or features.dtype != torch.float32 or features.dim() != 3:
        raise ValueError("features must be a float32 tensor [B][T][42] (batch_first) or [T][B][42]")
    B, T = (features.shape[0], features.shape[1]) if batch_first else (features.shape[1], features.shape[0])
    if features.shape[2] != NB_FEATURES or features.stride(2) != 1:
        raise ValueError("features must have rows of 42 contiguous floats")
    if T != window:
        raise ValueError("features hold %d frames; this network's window is %d" % (T, window))
    if not 1 <= B <= max_streams:
        raise ValueError("features hold %d streams; this network takes 1..%d" % (B, max_streams))
    if silence is not None and (not isinstance(silence, torch.Tensor) or silence.dtype != torch.int32 or tuple(silence.shape) != (T, B)):
        raise ValueError("silence must be an int32 tensor [T][B] (analyze_window_device's layout)")
    if state is not None and (not isinstance(state, torch.Tensor) or state.dtype != torch.float32
                              or tuple(state.shape) != (B, state_width) or not state.is_contiguous()):
        raise ValueError("state must be a contiguous float32 tensor [B][%d]" % state_width)
    for name, x in (("features", features), ("silence", silence), ("state", state)):
        if x is not None and x.device != device:
            raise ValueError("%s must be on %s, the network's device" % (name, device))
    return B


class _NetworkFunction(torch.autograd.Function):
    @staticmethod
    def forward(fctx, params, features, silence, state, net, batch_first):
        gains, vad, state_out = net._forward(params, features, silence, state, batch_first)
        fctx.net, fctx.generation, fctx.batch_first, fctx.gains_shape = net, net._generation, batch_first, gains.shape
        fctx.save_for_backward(params)
        fctx.mark_non_differentiable(state_out)
        return gains, vad, state_out

    @staticmethod
    def backward(fctx, grad_gains, grad_vad, _):
        (params,) = fctx.saved_tensors
        net = fctx.net
        if net._generation != fctx.generation:
            raise NnnoiselessError("DenoiseNetwork: this forward's activations were overwritten by a later forward of the same "
                                   "network; call backward before the next forward")
        bf = fctx.batch_first
        grad = torch.empty_like(params)
        # the kernels read rows of 22 contiguous gradients; torch may hand over broadcast (stride 0) or other views
        gg = grad_gains.contiguous() if grad_gains is not None else torch.zeros(fctx.gains_shape, device=params.device)
        gv = grad_vad.contiguous() if grad_vad is not None else None
        ggs, ggf = _strides(gg, bf)
        gvs, gvf = _strides(gv, bf) if gv is not None else (0, 0)
        net._fit.backward_device(params.data_ptr(), gg.data_ptr(), ggs, ggf, gv.data_ptr() if gv is not None else 0, gvs, gvf,
                                 grad.data_ptr(), torch.cuda.current_stream(params.device).cuda_stream)
        return grad, None, None, None, None, None


class DenoiseNetwork(torch.nn.Module):
    """The denoiser's own network (dense -> three GRUs -> dense, Keras ``reset_after=False`` cells) as a torch module whose
    forward and backward are the fitting kernels (rnnoise_fit_forward_device / _backward_device).  ``params`` is one flat
    float32 Parameter in the layout of ``fit.layer_shapes``; train it with any torch optimiser, call ``clip_()`` after
    each step as the training script does, and ``to_model()`` gives the ``.rnn`` model ``DenoiseBatch`` serves.

    The handle keeps the activations of one forward: backward a forward before the next forward of the same network
    (a ``no_grad`` evaluation included), or the backward raises."""

    def __init__(self, max_streams: int, window: int, widths=fit.WIDTHS, seed: int = 0, device=None):
        super().__init__()
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise ValueError("DenoiseNetwork runs on a CUDA device")
        dev = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self._fit = fit.Fit(widths, max_streams, window, dev.index)
        self.widths, self.max_streams, self.window = self._fit.widths, self._fit.max_sequences, self._fit.window
        self.params = torch.nn.Parameter(torch.from_numpy(fit.init_params(self.widths, seed)).to(dev))
        self._generation = 0

    @classmethod
    def from_model(cls, model: RnnModel, max_streams: int, window: int, device=None):
        """The network of a model (None: the built-in one): its int8 weights / 256, its widths and its activations."""
        data = (model if model is not None else RnnModel()).to_bytes()
        net = cls(max_streams, window, (data[1],) + gru_widths(data), device=device)
        net._fit.set_params_from_model(model)
        with torch.no_grad():
            net.params.copy_(torch.from_numpy(net._fit.get_params()))
        return net

    @property
    def state_width(self) -> int:
        """Floats of one stream's GRU state: nv + nn + ndn."""
        return sum(self.widths[1:])

    def _forward(self, params, features, silence, state, batch_first):
        B = check_window(features, silence, state, batch_first, self.window, self.max_streams, self.state_width, params.device)
        T = self.window
        gains = torch.empty((B, T, NB_BANDS) if batch_first else (T, B, NB_BANDS), device=params.device)
        vad = torch.empty((B, T) if batch_first else (T, B), device=params.device)
        state_out = torch.empty((B, self.state_width), device=params.device)
        fs, ff = _strides(features, batch_first)
        ss, sf = (silence.stride(1), silence.stride(0)) if silence is not None else (0, 0)
        gs, gf = _strides(gains, batch_first)
        vs, vf = _strides(vad, batch_first)
        self._fit.forward_device(params.data_ptr(), B, features.data_ptr(), fs, ff, silence.data_ptr() if silence is not None else 0, ss, sf,
                                 state.data_ptr() if state is not None else 0, state_out.data_ptr(), gains.data_ptr(), gs, gf,
                                 vad.data_ptr(), vs, vf, torch.cuda.current_stream(params.device).cuda_stream)
        self._generation += 1  # the handle now holds this forward's activations
        return gains, vad, state_out

    def forward(self, features, silence=None, state=None, batch_first=True):
        """features float32 [B][T][42] (batch_first) or [T][B][42], T = window; silence int32 [T][B] as
        analyze_window_device writes it (None: no frame silent); state [B][nv + nn + ndn], the state_out of the previous
        window of the same streams (None: zeros).  -> (gains [B][T][22], vad [B][T], state_out [B][nv + nn + ndn]), or
        [T][B]-first when not batch_first.  gains and vad require grad; state_out is detached.  On silent frames gains
        and vad are 0 and every state is carried.  Runs on the current torch stream."""
        return _NetworkFunction.apply(self.params, features, silence, state, self, batch_first)

    def clip_(self):
        """Clamp every parameter to +-0.499, the training script's constraint that keeps the export within int8."""
        with torch.no_grad():
            self.params.clamp_(-0.499, 0.499)
        return self

    def export(self) -> bytes:
        """The .rnn bytes of the current parameters, with this network's activations (a model's relu GRUs included)."""
        self._fit.set_params(self.params.detach().cpu().numpy())
        return self._fit.export()

    def to_model(self) -> RnnModel:
        model = RnnModel.from_bytes(self.export())
        if model is None:
            raise NnnoiselessError("the exported model does not parse")
        return model


class _Intelligibility(torch.autograd.Function):
    @staticmethod
    def forward(fctx, out, clean, rate):
        B, n = out.shape
        stride = out.stride(0) if B > 1 else n
        nbytes = intelligibility_workspace_bytes(B, n, rate)
        if nbytes == 0:
            raise NnnoiselessError("no workspace size for %d pairs of %d samples at %d Hz" % (B, n, rate))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=out.device)
        rec = torch.empty((B, INTELLIGIBILITY_DTYPE.itemsize // 8), dtype=torch.float64, device=out.device)
        intelligibility_device(out.data_ptr(), clean.data_ptr(), B, n, stride, rate, rec.data_ptr(), ws.data_ptr(), nbytes,
                               out.device.index, torch.cuda.current_stream(out.device).cuda_stream)
        fctx.rec, fctx.ws = rec, ws  # neither is an input or output: held on the context until backward
        fctx.shape, fctx.rate = (B, n), rate
        return rec[:, 0].clone(), rec[:, 1].clone()

    @staticmethod
    @torch.autograd.function.once_differentiable  # the kernels' gradient is not itself a graph: create_graph raises
    def backward(fctx, grad_stoi, grad_estoi):
        rec, ws = fctx.rec, fctx.ws
        (B, n), rate = fctx.shape, fctx.rate
        gs = grad_stoi.to(torch.float64).contiguous() if grad_stoi is not None else None
        ge = grad_estoi.to(torch.float64).contiguous() if grad_estoi is not None else None
        grad = torch.empty((B, n), dtype=torch.float32, device=rec.device)
        nbytes = intelligibility_backward_workspace_bytes(B, n, rate)
        bws = torch.empty(nbytes, dtype=torch.uint8, device=rec.device)
        intelligibility_backward_device(B, n, rate, rec.data_ptr(), ws.data_ptr(), ws.numel(), gs.data_ptr() if gs is not None else 0,
                                        ge.data_ptr() if ge is not None else 0, grad.data_ptr() if grad.numel() else bws.data_ptr(), n,
                                        bws.data_ptr(), nbytes, rec.device.index, torch.cuda.current_stream(rec.device).cuda_stream)
        return grad, None, None


def intelligibility(out, clean, rate: int = 48000):
    """STOI and ESTOI of each row of float32 CUDA tensors out (processed) and clean, [B][n] -> (stoi, estoi), float64
    CUDA tensors [B] (NaN for a row with fewer than 30 STFT frames after silence removal), differentiable with respect
    to out.

    The forward is rnnoise_intelligibility_device on torch's current stream; the backward is
    rnnoise_intelligibility_backward_device, whose contract (what is differentiated, kinks, exact zeros) is
    include/rnnoise.h's.  Until backward (or until the graph is freed) the call holds the forward's workspace,
    intelligibility_workspace_bytes(B, n, rate) bytes (about B (8 n10 + 124 F) for n10 = n * 10000 / rate samples at
    10 kHz and F = n10 / 128 frames: 4.4 GB for 16,384 rows of 3 s), and 32 bytes of records per row; the backward allocates
    intelligibility_backward_workspace_bytes(B, n, rate) more while it runs.  clean takes no gradient: a clean that
    requires grad is refused, since its gradient would be dropped silently.  Rows must not overlap, as for
    nnnoiseless_b200.intelligibility."""
    if not isinstance(out, torch.Tensor) or not isinstance(clean, torch.Tensor) or out.shape != clean.shape or out.dim() != 2:
        raise ValueError("out and clean must be [B][n] tensors of one shape")
    if clean.requires_grad:
        raise ValueError("clean requires grad, but intelligibility gives no gradient for clean; pass clean.detach()")
    B, n = out.shape
    if n > 1 and (out.stride(1) != 1 or clean.stride(1) != 1):
        raise ValueError("out and clean must have unit sample stride")
    if B > 1 and (out.stride(0) != clean.stride(0) or out.stride(0) < n):
        raise ValueError("out and clean must have one row stride of at least n = %d (rows must not overlap); strides %d and %d"
                         % (n, out.stride(0), clean.stride(0)))
    if out.dtype != torch.float32 or clean.dtype != torch.float32 or not out.is_cuda or clean.device != out.device:
        raise ValueError("out and clean must be float32 CUDA tensors on one device")
    return _Intelligibility.apply(out, clean, int(rate))
