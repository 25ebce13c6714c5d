"""``TYPE = "lsq"`` -- learned step size quantization (sparsebit/quantization/quantizers/lsq.py:25-76).

scale is an ``nn.Parameter`` initialised from calibration data as 2 * mean(|x|) / sqrt(qmax)
(per tensor or per channel, lsq.py:32-51); the forward is the same fake-quant op as ``uniform`` with
the scale's gradient damped by 1 / sqrt(numel * qmax) (lsq.py:68-76).  Forward and backward run in
the sm_90a kernels through ``STE`` (the scale gradient is the kernels' deterministic ``gs``).
"""
import math
import warnings

import torch
import torch.nn as nn

from ... import distributed as sbdist
from ... import ops
from . import Quantizer as BaseQuantizer
from . import register_quantizer
from .quant_tensor import STE


class GradScale(torch.autograd.Function):
    """identity forward, gradient multiplied by ``ratio`` (lsq.py:13-22 ``gs_scaling``)."""

    @staticmethod
    def forward(ctx, x, ratio):
        ctx.ratio = ratio
        return x

    @staticmethod
    def backward(ctx, grad):
        return grad * ctx.ratio, None


def grad_scale_ratio(x, qdesc):
    n = x.numel() / x.shape[qdesc.ch_axis] if qdesc.is_perchannel else x.numel()
    return 1.0 / math.sqrt(n * qdesc.qmax)


def clamp_qparams(quantizer):
    """lsq.py:53-66 / lsq_plus.py:57-70: |scale| and the zero point clamped to the integer range."""
    qd = quantizer.qdesc
    scale = quantizer.scale.abs()
    zero_point = torch.clamp(quantizer.zero_point, qd.qmin, qd.qmax)
    if quantizer.export_onnx:
        return scale.detach().clone(), zero_point.detach().clone()
    return scale, zero_point


@register_quantizer
class Quantizer(BaseQuantizer):
    TYPE = "LSQ"

    def __init__(self, config):
        super().__init__(config)
        self.init_params = False
        self.observer.keep_data = True  # the step-size initialisation needs the calibration batches themselves

    def calc_qparams_steps(self):
        if self.fake_fused or self.init_params:
            return self.scale, self.zero_point
        cache = self.observer.data_cache
        rows = cache.rows(self.is_perchannel)  # [C, M] per channel, [1, N] per tensor
        # one native pass per cached batch: the running min (negativity test) comes from the streaming MinMax
        # state (observers that keep none -- percentile, moving_average -- get one built from the cached rows),
        # mean |x| from the fp64 row moments (sb200_observe_moments) -- no ATen reductions
        obs = self.observer
        if obs._mm_state is None:
            obs._mm_state = ops.minmax_new(rows[0].shape[0], rows[0].device)
            for r in rows:
                ops.minmax_update(r, obs._mm_state, 0 if self.is_perchannel else None)
        running_min, _ = yield from obs._running_minmax_steps()
        if bool((running_min < 0).any()) and not self.qdesc.is_symmetric:
            warnings.warn("Found data less than 0, reset quantizer scheme as symmetric")
            self.qdesc.set_symmetric(True)
        acc = ops.moments_new(rows[0].shape[0], rows[0].device)
        for r in rows:
            ops.moments_update(r, acc)
        count = torch.tensor([float(sum(r.shape[1] for r in rows))], dtype=torch.float64, device=rows[0].device)
        yield sbdist.Sync.sum([acc, count], local=obs._local)  # sharded calibration: moments of the WHOLE set
        total = acc[:, 2] if self.is_perchannel else acc[0, 2]
        scale = (2 * (total / count) / math.sqrt(self.qdesc.qmax)).to(torch.float32)
        self.observer._reset()
        self.scale = nn.Parameter(self._broadcast_qparams(scale.to(self.device)))
        self.zero_point = self._broadcast_qparams(torch.zeros_like(self.scale.detach()))
        self.init_params = True
        return self.scale, self.zero_point

    def _qparams_preprocess(self, x):
        return clamp_qparams(self)

    def _forward(self, x, scale, zero_point):
        scale = GradScale.apply(scale, grad_scale_ratio(x, self.qdesc))
        return STE.apply(x, scale, zero_point, self.qdesc, self.backend)
