"""Torch autograd through synthesis (DESIGN.md 7i): train a network between ``DenoiseBatch.analyze_device`` and
``DenoiseBatch.synthesize_saving_device`` on a loss of the output samples.

    out = synthesis_grad(gains, out, ctx)   # out now depends on gains in torch's graph
    loss(out, target).backward()            # gains.grad from rnnoise_synthesis_backward_device, on the GPU

This module imports torch; the package itself does not.
"""
import torch

from . import NB_BANDS, FRAME_SIZE, SYNTH_CONTEXT_BYTES, synthesis_backward_device, synthesis_backward_workspace_bytes


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
