"""The slice of the reference's QuantOpr family that the calibration / AdaRound path drives
(sparsebit/quantization/modules/base.py:9-70, conv.py:8-43, linear.py:7-34, activations.py:9-38):
an operator owning an ``input_quantizer`` (and a ``weight_quantizer`` when it has a weight), built from
the ``config.A`` / ``config.W`` sub-trees, switched by ``set_quant``.  Graph conversion, fusion and the
~40 other operator wrappers of the reference are out of scope (SURVEY §8: control plane); any module
exposing these attributes works with ``tools.CalibrationRunner``."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .common import Backend
from .quantizers import build_quantizer
from .quantizers.quant_tensor import check_trt_symmetric


class QuantOpr(nn.Module):
    def __init__(self):
        super().__init__()
        self.weight = None
        self.input_quantizer = None
        self.weight_quantizer = None

    def build_quantizer(self, a_cfg, w_cfg=None, backend=Backend.VIRTUAL):
        """``a_cfg`` / ``w_cfg``: the per-module config sub-trees with TARGET already set
        (``sparsebit_b200.config.quantizer_config``); modules/base.py:36-45."""
        if self.weight is not None:
            assert w_cfg is not None, "an operator with a weight needs the W config"
            self.weight_quantizer = build_quantizer(w_cfg)
            self.weight_quantizer.set_backend(backend)
        self.input_quantizer = build_quantizer(a_cfg)
        self.input_quantizer.set_backend(backend)
        return self

    def set_quant(self, w_quant=False, a_quant=False):
        for quantizer, on in ((self.weight_quantizer, w_quant), (self.input_quantizer, a_quant)):
            if quantizer is None:
                continue
            if on and not quantizer.fake_fused:
                quantizer.enable_quant()
            else:
                quantizer.disable_quant()


class QConv2d(QuantOpr):
    def __init__(self, org_module):
        assert isinstance(org_module, nn.Conv2d)
        super().__init__()
        self.fwd_kwargs = dict(stride=org_module.stride, padding=org_module.padding, dilation=org_module.dilation,
                               groups=org_module.groups)
        self.weight, self.bias = org_module.weight, org_module.bias

    def forward(self, x_in):
        return F.conv2d(self.input_quantizer(x_in), self.weight_quantizer(self.weight), self.bias, **self.fwd_kwargs)


class QLinear(QuantOpr):
    def __init__(self, org_module):
        assert isinstance(org_module, nn.Linear)
        super().__init__()
        self.weight, self.bias = org_module.weight, org_module.bias

    def forward(self, x_in):
        return F.linear(self.input_quantizer(x_in), self.weight_quantizer(self.weight), self.bias)


_PLAIN_QDQ_TYPES = ("uniform", "lsq", "lsq+", "pact")  # quantizers whose forward is the plain fake-quant op


def _qparams(quantizer, x):
    scale, zero_point = quantizer._qparams_preprocess(x)
    return scale.detach().float().reshape(-1), zero_point.detach().float().reshape(-1)


def int8_ineligibility(qlinear):
    """Why ``QLinearInt8.from_qlinear`` cannot convert ``qlinear`` (None when it can)."""
    if not isinstance(qlinear, QLinear):
        return f"expected a QLinear, got {type(qlinear).__name__}"
    n = qlinear.weight.shape[0]
    for role, q in (("input", qlinear.input_quantizer), ("weight", qlinear.weight_quantizer)):
        if q is None:
            return f"the {role} quantizer is missing"
        if q.fake_fused:
            return f"the {role} quantizer is fake_fused"
        if not q.use_quant:
            return f"the {role} quantizer is not enabled"
        if q.export_onnx:
            return f"the {role} quantizer is in export_onnx mode"
        if q.TYPE.lower() not in _PLAIN_QDQ_TYPES:
            return f"the {role} quantizer is {q.TYPE}, whose forward is not the plain fake-quant op"
        if q.bit > 8:
            return f"the {role} quantizer has {q.bit} bits (at most 8)"
    aq, wq = qlinear.input_quantizer, qlinear.weight_quantizer
    if aq.is_perchannel:
        return "the input quantizer is per-channel (the integer path needs one activation scale)"
    if wq.is_perchannel and wq.qdesc.ch_axis != 0:
        return f"the weight quantizer is per-channel along axis {wq.qdesc.ch_axis} (needs the output channels, axis 0)"
    for role, q, x in (("input", aq, None), ("weight", wq, qlinear.weight)):
        scale, zero_point = _qparams(q, x)
        if scale.numel() not in ((1, n) if role == "weight" else (1,)) or zero_point.numel() != scale.numel():
            return f"the {role} quantizer holds {scale.numel()} scales"
        qmin, qmax = q.qdesc.qrange
        z = torch.round(zero_point)
        if bool(((z < qmin) | (z > qmax) | torch.isnan(z)).any()):
            return f"the {role} zero point lies outside [{qmin}, {qmax}]"
        if q.backend == Backend.TENSORRT:
            try:
                check_trt_symmetric(zero_point)
            except AssertionError as e:
                return f"the {role} quantizer: {e}"
    return None


class QLinearInt8(nn.Module):
    """Inference-only replacement of a calibrated ``QLinear``: the fake-quant linear computed on the integer grid by
    ``ops.int8_linear`` (exact int8 x int8 sums on the tensor cores, zero points removed in int64, then
    s_x s_w[n] I + bias).  Built by ``from_qlinear``; the weights are quantized once at conversion.  fp16 input is
    up-cast and the output is fp32, as in the fake-quant op.  There is no backward: QAT keeps ``QLinear``."""

    def __init__(self, in_features, out_features, device):
        super().__init__()
        self.in_features, self.out_features = int(in_features), int(out_features)
        kp = ops.int8_padded_k(in_features)
        self.register_buffer("w_q", torch.zeros(out_features, kp, dtype=torch.int8, device=device))
        self.register_buffer("w_rowsum", torch.zeros(out_features, dtype=torch.int32, device=device))
        self.register_buffer("w_scale", torch.zeros(out_features, dtype=torch.float32, device=device))
        self.register_buffer("w_zero", torch.zeros(out_features, dtype=torch.int32, device=device))
        self.register_buffer("scale", torch.ones(1, dtype=torch.float32, device=device))
        self.register_buffer("zero_point", torch.zeros(1, dtype=torch.float32, device=device))
        self.register_buffer("bias", None)
        self.qmin, self.qmax = -128, 127

    @classmethod
    def from_qlinear(cls, qlinear):
        reason = int8_ineligibility(qlinear)
        if reason is not None:
            raise ValueError(f"QLinearInt8.from_qlinear: {reason}")
        aq, wq = qlinear.input_quantizer, qlinear.weight_quantizer
        weight = qlinear.weight.detach()
        n, k = weight.shape
        mod = cls(k, n, weight.device)
        with torch.no_grad():
            ws, wz = _qparams(wq, qlinear.weight)
            xs, xz = _qparams(aq, None)
            wqmin, wqmax = wq.qdesc.qrange
            w_q, w_sum, w_nan = ops.int8_quantize_rows(weight.float().contiguous(), ws.contiguous(), wz.contiguous(), wqmin, wqmax)
            mod.w_q.copy_(w_q)
            mod.w_rowsum.copy_(w_sum)
            # a weight row holding a NaN makes its output column NaN, as in the fake-quant matmul
            mod.w_scale.copy_(torch.where(w_nan, torch.full_like(w_sum, float("nan"), dtype=torch.float32), ws.expand(n)))
            mod.w_zero.copy_((torch.round(wz) - ops.int8_grid_offset(wqmin)).to(torch.int32).expand(n))
            mod.scale.copy_(xs.reshape(1))
            mod.zero_point.copy_(xz.reshape(1))
            if qlinear.bias is not None:
                mod.bias = qlinear.bias.detach().float().clone().contiguous()
        mod.qmin, mod.qmax = aq.qdesc.qrange
        return mod

    def forward(self, x_in):
        if torch.is_grad_enabled() and x_in.requires_grad:
            raise RuntimeError("QLinearInt8 is inference-only and has no backward; run it under torch.no_grad() or "
                               "keep QLinear for training")
        x = x_in.float() if x_in.dtype != torch.float32 else x_in
        return ops.int8_linear(x.contiguous(), self.scale, self.zero_point, self.qmin, self.qmax, self.w_q, self.w_rowsum,
                               self.w_scale, self.w_zero, self.bias, k=self.in_features)

    def extra_repr(self):
        return f"in_features={self.in_features}, out_features={self.out_features}, qrange=[{self.qmin}, {self.qmax}]"


class QReLU(QuantOpr):
    def __init__(self, org_module=None):
        super().__init__()
        self.inplace = bool(getattr(org_module, "inplace", False))

    def forward(self, x_in):
        return F.relu(self.input_quantizer(x_in), inplace=self.inplace)


class QIdentity(QuantOpr):
    """Carrier of one input quantizer in front of a multi-input operator (modules/unary.py QIdentity)."""

    def forward(self, x_in):
        return self.input_quantizer(x_in)
