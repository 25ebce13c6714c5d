"""``TYPE = "pact"`` (sparsebit/quantization/quantizers/pact.py:13-46): activations are clamped to a
learnable [-alpha, alpha] (or [0, alpha]) before the fake-quant op whose qparams follow alpha.

The reference runs ``torch.clamp`` in front of the fake-quant op and lets autograd chain the two.  What that chain
computes depends on the range:

* Unsigned ([0, alpha], the grid's ``scale`` built from ``alpha.detach()``): every clamped value quantises inside
  [qmin, qmax], so the clamp changes neither the forward value nor the straight-through mask.  The forward is the
  native QDQ alone and the backward is ``sb200_clamp_bwd`` (gx = gy inside [0, alpha]; d/d alpha = sum of gy above
  alpha).
* Signed ([-alpha, alpha], SURVEY Q19): ``alpha / scale`` is ``(qmax - qmin) / 2``, a half-integer, so ``+alpha``
  rounds to ``qmax + 1`` for most alphas and the straight-through mask drops every element clamped to it; for the
  others ``-alpha`` rounds to ``qmin + 1`` and the clamp narrows the forward grid.  ``scale`` also depends on alpha
  through the non-detached ``lower = -alpha``.  The forward therefore fake-quantises the clamped tensor, and the
  backward runs the STE backward kernel on it, then ``sb200_clamp_bwd`` on that gradient; the scale gradient returns to
  alpha through the port's own ``calc_qparams_with_minmax`` graph (``-alpha``, the ``maximum`` tie, ``/ span``)."""
import torch
import torch.nn as nn

from ... import ops
from ..common import QuantTarget
from . import Quantizer as BaseQuantizer
from . import register_quantizer
from .quant_tensor import STE, fake_quant_factory


def _f32c(t):
    t = t.detach()
    return (t if t.dtype == torch.float32 else t.float()).contiguous()


class PactSTE(torch.autograd.Function):
    """clamp(x, lower, alpha) -> fake-quant as one op with the reference chain's gradients for x, alpha, lower and
    scale.  On unsigned ranges the clamp is folded into the fake-quant grid and the backward is the clamp's alone (see
    the module docstring)."""

    @staticmethod
    def forward(ctx, x, alpha, lower, signed, scale, zero_point, qdesc, backend):
        ctx.signed, ctx.qdesc = signed, qdesc
        if not signed:
            ctx.save_for_backward(x, alpha, lower)
            return fake_quant_factory[backend](x, scale, zero_point, qdesc)
        xc = torch.clamp(_f32c(x), _f32c(lower).reshape(1), _f32c(alpha).reshape(1))
        ctx.save_for_backward(x, alpha, lower, xc, scale, zero_point)
        return fake_quant_factory[backend](xc, scale, zero_point, qdesc)

    @staticmethod
    def backward(ctx, gout):
        x, alpha, lower = ctx.saved_tensors[:3]
        if not x.is_cuda:
            raise NotImplementedError("We recommended that use cuda to speedup when training")  # like STE, quant_tensor.py:113-116
        lo, hi = _f32c(lower).reshape(1), _f32c(alpha).reshape(1)
        gy = _f32c(gout)
        gs = None
        if ctx.signed:
            xc, scale, zero_point = ctx.saved_tensors[3:]
            qmin, qmax = ctx.qdesc.qrange
            gy, gs, _ = ops.qdq_backward(xc, _f32c(scale).reshape(1), _f32c(zero_point).reshape(1), gy, qmin, qmax,
                                         need_gs=ctx.needs_input_grad[4], need_gzp=False)
            gs = gs.reshape(scale.shape) if ctx.needs_input_grad[4] else None
        gx, g_hi, g_lo = ops.clamp_backward(_f32c(x), gy, lo, hi)
        g_lo = g_lo.reshape(lower.shape) if ctx.needs_input_grad[2] else None
        return gx, g_hi.reshape(alpha.shape), g_lo, None, gs, None, None, None


@register_quantizer
class Quantizer(BaseQuantizer):
    TYPE = "PACT"

    def __init__(self, config):
        super().__init__(config)
        assert self.qdesc.target == QuantTarget.FEATURE, "PACT only support feature quantization"
        assert not self.qdesc.is_perchannel, "PACT no yet supports per-channel"
        self.init_alpha_value = config.QUANTIZER.PACT.ALPHA_VALUE

    def calc_qparams_steps(self):
        if self.fake_fused:
            return self.scale, self.zero_point
        scale, zero_point = yield from super().calc_qparams_steps()
        self.alpha = nn.Parameter(torch.tensor([float(self.init_alpha_value)], device=self.device))
        return scale, zero_point

    def _qparams_preprocess(self, x):
        self.lower = -self.alpha if self.qdesc.qmin < 0 else torch.zeros(1, device=self.alpha.device)
        return self.calc_qparams_with_minmax(self.lower, self.alpha.detach())

    def _forward(self, x, scale, zero_point=None):
        if not x.is_cuda:  # host tensors: the reference op chain shape (clamp -> STE through the host-buffer entry point)
            return STE.apply(torch.clamp(x, self.lower, self.alpha), scale, zero_point, self.qdesc, self.backend)
        return PactSTE.apply(x, self.alpha, self.lower, self.qdesc.qmin < 0, scale, zero_point, self.qdesc, self.backend)
