"""The slice of the reference's QuantOpr family that the calibration / AdaRound path drives
(sparsebit/quantization/modules/base.py:9-70, conv.py:8-43, linear.py:7-34, activations.py:9-38):
an operator owning an ``input_quantizer`` (and a ``weight_quantizer`` when it has a weight), built from
the ``config.A`` / ``config.W`` sub-trees, switched by ``set_quant``.  Graph conversion, fusion and the
~40 other operator wrappers of the reference are out of scope (SURVEY §8: control plane); any module
exposing these attributes works with ``tools.CalibrationRunner``."""
import math

import torch
import torch.fx
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..ops import _pair
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


def _int8_plain_qdq_reason(role, q, types=_PLAIN_QDQ_TYPES):
    """Why quantizer ``q`` does not run the plain <= 8-bit fake-quant op that the integer path restates (None if it does);
    ``types``: the quantizer types the caller restates."""
    if q is None:
        return f"the {role} quantizer is missing"
    if q.fake_fused:
        return f"the {role} quantizer is fake_fused"
    if not q.use_quant:
        return f"the {role} quantizer is not enabled"
    if q.export_onnx:
        return f"the {role} quantizer is in export_onnx mode"
    if q.TYPE.lower() not in types:
        return f"the {role} quantizer is {q.TYPE}, whose forward is not the plain fake-quant op"
    if q.bit > 8:
        return f"the {role} quantizer has {q.bit} bits (at most 8)"
    return None


def _int8_qparams_reason(role, q, x, counts):
    """Why the qparams of ``q`` do not fit the integer path: a scale count outside ``counts``, a zero point outside the
    integer range, or a TensorRT backend with a non-zero zero point (None if they fit)."""
    scale, zero_point = _qparams(q, x)
    if scale.numel() not in counts or zero_point.numel() != scale.numel():
        return f"the {role} quantizer holds {scale.numel()} scales"
    qmin, qmax = q.qdesc.qrange
    z = torch.round(zero_point)
    if bool(((z < qmin) | (z > qmax) | torch.isnan(z)).any()):
        return f"the {role} zero point lies outside [{qmin}, {qmax}]"
    if q.TYPE == "PACT" and qmin < 0 and bool(torch.round(q.alpha.detach().reshape(-1) / scale) <= qmax):
        # SURVEY Q19: -alpha then rounds to qmin + 1, so the clamp narrows the grid below the QDQ kernels' [qmin, qmax]
        return f"the {role} quantizer is PACT with alpha on the grid, whose clamp narrows it to [{qmin + 1}, {qmax}]"
    if q.backend == Backend.TENSORRT:
        try:
            check_trt_symmetric(zero_point)
        except AssertionError as e:
            return f"the {role} quantizer: {e}"
    return None


def _int8_quantizer_ineligibility(mod, input_types=_PLAIN_QDQ_TYPES, weight_types=_PLAIN_QDQ_TYPES):
    """The quantizer rules of the integer path, shared by ``QLinear`` and ``QConv2d``: ``mod`` has an input and a
    weight quantizer and a weight whose axis 0 is the output channels."""
    n = mod.weight.shape[0]
    for role, q, types in (("input", mod.input_quantizer, input_types), ("weight", mod.weight_quantizer, weight_types)):
        reason = _int8_plain_qdq_reason(role, q, types)
        if reason is not None:
            return reason
    aq, wq = mod.input_quantizer, mod.weight_quantizer
    if aq.is_perchannel:
        return "the input quantizer is per-channel (the integer path needs one activation scale)"
    if wq.is_perchannel and wq.qdesc.ch_axis != 0:
        return f"the weight quantizer is per-channel along axis {wq.qdesc.ch_axis} (needs the output channels, axis 0)"
    for role, q, x, counts in (("input", aq, None, (1,)), ("weight", wq, mod.weight, (1, n))):
        reason = _int8_qparams_reason(role, q, x, counts)
        if reason is not None:
            return reason
    return None


def int8_ineligibility(qlinear):
    """Why ``QLinearInt8.from_qlinear`` cannot convert ``qlinear`` (None when it can)."""
    if not isinstance(qlinear, QLinear):
        return f"expected a QLinear, got {type(qlinear).__name__}"
    return _int8_quantizer_ineligibility(qlinear)


def _grid_source(wq, weight):
    """The tensor whose plain QDQ grid under ``wq``'s qparams is ``wq``'s grid: the weight itself, DoReFa's normalised
    tanh(w) / max |tanh(w)| (the fake-quant op's own sequence, ``DoReFaSTE``), or AdaRound's eval-mode (hard rounding)
    output RN((q - zp) s), which re-quantizes to q exactly under the preconditions ``dorefa_adaround_ineligibility``
    enforces."""
    kind = wq.TYPE.lower()
    if kind == "dorefa":
        w = weight.detach().float().contiguous()
        return ops.dorefa_forward(w, ops.dorefa_absmax(w))
    if kind == "adaround":
        return wq(weight.detach())
    return weight.detach()


def _int8_weight_rows(wq, weight):
    """The weights on the stored integer grid, one row per output channel (``weight.reshape(N, -1)``):
    ``(w_q, w_rowsum, w_scale, w_zero)`` as ``ops.int8_linear`` / ``ops.int8_conv2d`` take them.  A weight row holding a
    NaN gets ``w_scale = NaN``, which makes its output channel NaN, as in the fake-quant op (a DoReFa weight holding a
    NaN makes every row NaN: its max |tanh| is global)."""
    rows = _grid_source(wq, weight).reshape(weight.shape[0], -1)
    n = rows.shape[0]
    ws, wz = _qparams(wq, weight)
    wqmin, wqmax = wq.qdesc.qrange
    w_q, w_sum, w_nan = ops.int8_quantize_rows(rows.float().contiguous(), ws.contiguous(), wz.contiguous(), wqmin, wqmax)
    w_scale = torch.where(w_nan, torch.full_like(w_sum, float("nan"), dtype=torch.float32), ws.expand(n))
    w_zero = (torch.round(wz) - ops.int8_grid_offset(wqmin)).to(torch.int32).expand(n)
    return w_q, w_sum, w_scale, w_zero


def _check_inference_only(mod, training_cls, *inputs):
    """The integer-grid modules have no backward: an input that needs a gradient is an error, not a silent detach."""
    if torch.is_grad_enabled() and any(x.requires_grad for x in inputs):
        raise RuntimeError(f"{type(mod).__name__} is inference-only and has no backward; run it under torch.no_grad() or "
                           f"keep {training_cls} for training")


class _Int8InputModule(nn.Module):
    """What every weight-carrying integer-grid module holds besides its weight operand: the per-tensor activation
    ``scale`` / ``zero_point`` and integer range ``qmin`` / ``qmax``, and ``bias`` (fp32 or None).  A subclass registers
    its weight buffers, then ``_register_input``."""

    def _x_absmax(self, x):
        """The ``x_absmax`` the ops take for input ``x``: None, the input is quantized as it is (see ``_DoReFaInput``)."""
        return None

    def _register_input(self, device):
        self.register_buffer("scale", torch.ones(1, dtype=torch.float32, device=device))
        self.register_buffer("zero_point", torch.zeros(1, dtype=torch.float32, device=device))
        self.register_buffer("bias", None)
        self.qmin, self.qmax = -128, 127

    @classmethod
    def _check_eligible(cls, reason, method):
        if reason is not None:
            raise ValueError(f"{cls.__name__}.{method}: {reason}")

    def _load_input(self, qmod):
        """Fills the activation qparams and the bias from the calibrated ``qmod``; returns ``self``."""
        aq = qmod.input_quantizer
        with torch.no_grad():
            xs, xz = _qparams(aq, None)
            self.scale.copy_(xs.reshape(1))
            self.zero_point.copy_(xz.reshape(1))
            if qmod.bias is not None:
                self.bias = qmod.bias.detach().float().clone().contiguous()
        self.qmin, self.qmax = aq.qdesc.qrange
        return self


class _Int8WeightModule(_Int8InputModule):
    """The stored weight operand of ``QLinearInt8`` / ``QConv2dInt8``: ``w_q`` int8 [N, Kp] and ``w_rowsum`` /
    ``w_scale`` / ``w_zero`` [N] as ``_int8_weight_rows`` stores them, with the activation qparams and bias of
    ``_Int8InputModule``."""

    def __init__(self, out_features, k, device):
        super().__init__()
        self.register_buffer("w_q", torch.zeros(out_features, ops.int8_padded_k(k), dtype=torch.int8, device=device))
        self.register_buffer("w_rowsum", torch.zeros(out_features, dtype=torch.int32, device=device))
        self.register_buffer("w_scale", torch.zeros(out_features, dtype=torch.float32, device=device))
        self.register_buffer("w_zero", torch.zeros(out_features, dtype=torch.int32, device=device))
        self._register_input(device)

    def _load(self, qmod):
        """Fills the buffers from the calibrated ``qmod`` (a ``QLinear`` or ``QConv2d``); returns ``self``."""
        with torch.no_grad():
            for buf, v in zip((self.w_q, self.w_rowsum, self.w_scale, self.w_zero),
                              _int8_weight_rows(qmod.weight_quantizer, qmod.weight)):
                buf.copy_(v)
        return self._load_input(qmod)


class QLinearInt8(_Int8WeightModule):
    """Inference-only replacement of a calibrated ``QLinear``: the fake-quant linear computed on the integer grid by
    ``ops.int8_linear`` (exact int8 x int8 sums on the tensor cores, zero points removed in int64, then
    s_x s_w[n] I + bias).  Built by ``from_qlinear``; the weights are quantized once at conversion.  fp16 input is
    up-cast and the output is fp32, as in the fake-quant op.  There is no backward: QAT keeps ``QLinear``."""

    def __init__(self, in_features, out_features, device):
        super().__init__(out_features, in_features, device)
        self.in_features, self.out_features = int(in_features), int(out_features)

    @classmethod
    def from_qlinear(cls, qlinear):
        cls._check_eligible(int8_ineligibility(qlinear), "from_qlinear")
        return cls._build(qlinear)

    @classmethod
    def _build(cls, qlinear):
        n, k = qlinear.weight.shape
        return cls(k, n, qlinear.weight.device)._load(qlinear)

    def forward(self, x_in):
        _check_inference_only(self, "QLinear", x_in)
        x = x_in.float() if x_in.dtype != torch.float32 else x_in
        x = x.contiguous()
        return ops.int8_linear(x, self.scale, self.zero_point, self.qmin, self.qmax, self.w_q, self.w_rowsum,
                               self.w_scale, self.w_zero, self.bias, k=self.in_features, x_absmax=self._x_absmax(x))

    def extra_repr(self):
        return f"in_features={self.in_features}, out_features={self.out_features}, qrange=[{self.qmin}, {self.qmax}]"


def _sparse24_operand(qmod):
    """The weight of ``qmod`` (a ``QLinear`` or ``QConv2d``) on the stored grid, rows of ``weight.reshape(C_out, -1)``
    with K = ``weight[0].numel()``, packed by ``ops.int8_sparse24_pack``: ``((vals, meta, dsum, w_scale), reason)``,
    where ``reason`` names the first row and group of 4 that is not 2:4 on the centred grid d = g_w - rint(zp_w), or
    whose d leaves s8 (None when every row packs); k indexes a row of ``weight.reshape(C_out, -1)``."""
    w_q, _, w_scale, w_zero = _int8_weight_rows(qmod.weight_quantizer, qmod.weight)
    k = qmod.weight[0].numel()
    vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero.contiguous(), w_scale.contiguous(), k)
    rows = torch.nonzero(bad).reshape(-1)
    if rows.numel() == 0:
        return (vals, meta, dsum, w_scale.contiguous()), None
    r = int(rows[0])
    d = w_q[r, :k].to(torch.int32) - w_zero[r]
    d = F.pad(d, (0, (-k) % 4)).reshape(-1, 4)
    wrong = ((d != 0).sum(1) > 2) | ((d < -128) | (d > 127)).any(1)
    g = int(torch.nonzero(wrong).reshape(-1)[0])
    if bool(((d[g] < -128) | (d[g] > 127)).any()):
        why = f"the centred weight grid g_w - rint(zp_w) leaves s8 in row {r}, group {g} (k = {4 * g} .. {4 * g + 3})"
    else:
        why = f"the weight is not 2:4 sparse on the grid: row {r}, group {g} (k = {4 * g} .. {4 * g + 3}) has more than two nonzeros"
    return None, why


def _sparse24_checked(qmod, dense_reason):
    """``_sparse24_operand(qmod)`` on top of a dense rule: ``(None, dense_reason)`` when that rule refuses ``qmod``."""
    return (None, dense_reason) if dense_reason is not None else _sparse24_operand(qmod)


def int8_sparse24_ineligibility(qlinear):
    """Why ``QLinearSparse24Int8.from_qlinear`` cannot convert ``qlinear`` (None when it can): a rule of
    ``int8_ineligibility``, a centred weight grid outside s8 (possible for affine 8-bit weights only), or a group of 4
    along a row of the weight grid with more than two nonzeros."""
    return _sparse24_checked(qlinear, int8_ineligibility(qlinear))[1]


class _Sparse24WeightModule(_Int8InputModule):
    """The compressed 2:4 weight operand of ``QLinearSparse24Int8`` / ``QConv2dSparse24Int8``: ``vals`` int8
    [N, K64 / 2] (the kept centred grid values), ``meta`` (their 2-bit indices), ``dsum`` int32 [N] and ``w_scale``
    fp32 [N] as ``_sparse24_operand`` packs them, with the activation qparams and bias of ``_Int8InputModule``."""

    def __init__(self, out_features, k, device):
        super().__init__()
        vshape, mshape = ops.int8_sparse24_shapes(out_features, k)
        self.register_buffer("vals", torch.zeros(vshape, dtype=torch.int8, device=device))
        self.register_buffer("meta", torch.zeros(mshape, dtype=torch.int32, device=device))
        self.register_buffer("dsum", torch.zeros(out_features, dtype=torch.int32, device=device))
        self.register_buffer("w_scale", torch.zeros(out_features, dtype=torch.float32, device=device))
        self._register_input(device)

    @classmethod
    def _eligible_operand(cls, qmod, dense_reason, method):
        """The packed weight of the calibrated ``qmod``; raises the class-named ``ValueError`` when the dense rule's
        ``dense_reason`` or the 2:4 rule refuses it."""
        operand, reason = _sparse24_checked(qmod, dense_reason)
        cls._check_eligible(reason, method)
        return operand

    def _load(self, qmod, operand):
        """Fills the buffers from ``_eligible_operand``'s ``operand`` and the calibrated ``qmod``; returns ``self``."""
        with torch.no_grad():
            for buf, v in zip((self.vals, self.meta, self.dsum, self.w_scale), operand):
                buf.copy_(v)
        return self._load_input(qmod)


class QLinearSparse24Int8(_Sparse24WeightModule):
    """Inference-only replacement of a calibrated ``QLinear`` whose weight is 2:4 sparse on the grid: the linear of
    ``QLinearInt8`` on the sparse int8 tensor cores (``ops.int8_sparse24_linear``), bit-identical to ``QLinearInt8`` on
    the same module.  Only the compressed weight is stored: ``vals`` int8 [N, K64 / 2] (the kept centred grid values),
    ``meta`` (their 2-bit indices), ``dsum`` int32 [N] and ``w_scale`` fp32 [N], about 0.625 byte per weight.  fp16
    input is up-cast and the output is fp32, as in the fake-quant op.  Built by ``from_qlinear``; no backward."""

    def __init__(self, in_features, out_features, device):
        super().__init__(out_features, in_features, device)
        self.in_features, self.out_features = int(in_features), int(out_features)

    @classmethod
    def from_qlinear(cls, qlinear):
        operand = cls._eligible_operand(qlinear, int8_ineligibility(qlinear), "from_qlinear")
        n, k = qlinear.weight.shape
        return cls(k, n, qlinear.weight.device)._load(qlinear, operand)

    def forward(self, x_in):
        _check_inference_only(self, "QLinear", x_in)
        x = x_in.float() if x_in.dtype != torch.float32 else x_in
        return ops.int8_sparse24_linear(x.contiguous(), self.scale, self.zero_point, self.qmin, self.qmax, self.vals,
                                        self.meta, self.dsum, self.w_scale, self.bias, k=self.in_features)

    def extra_repr(self):
        return (f"in_features={self.in_features}, out_features={self.out_features}, qrange=[{self.qmin}, {self.qmax}], "
                f"2:4 sparse")


def resolve_conv_padding(padding, kernel_size, dilation=1, stride=1):
    """The (top, bottom, left, right) zero padding of a conv2d's ``padding`` argument: an int, a (pad_h, pad_w) pair,
    ``'valid'`` or ``'same'`` (total d (k - 1) per dimension, the odd one on the bottom / right, as ``F.conv2d``).
    Raises ``ValueError`` when it does not resolve to four non-negative ints."""
    if isinstance(padding, str):
        if padding == "valid":
            return (0, 0, 0, 0)
        if padding != "same":
            raise ValueError(f"padding {padding!r} is neither 'valid' nor 'same'")
        if any(s != 1 for s in _pair(stride)):
            raise ValueError("padding 'same' needs stride 1")
        pads = []
        for k, d in zip(_pair(kernel_size), _pair(dilation)):
            total = d * (k - 1)
            pads += [total // 2, total - total // 2]
        return tuple(pads)
    try:
        ph, pw = _pair(padding)
    except (TypeError, ValueError):
        raise ValueError(f"padding {padding!r} is not an int or a pair of ints") from None
    if ph < 0 or pw < 0:
        raise ValueError(f"padding {padding!r} is negative")
    return (ph, ph, pw, pw)


def _int8_conv_ineligibility(qconv, groups_rule, quantizer_rule=_int8_quantizer_ineligibility):
    """The conversion rules of a ``QConv2d`` in the order they are reported: the quantizer rules, then
    ``groups_rule(groups, K_g)`` (a reason or None; K_g = C / groups KH KW), then the padding."""
    if not isinstance(qconv, QConv2d):
        return f"expected a QConv2d, got {type(qconv).__name__}"
    reason = quantizer_rule(qconv)
    if reason is not None:
        return reason
    kw = qconv.fwd_kwargs
    c_out, c_g, kh, kwd = qconv.weight.shape
    reason = groups_rule(kw["groups"], c_g * kh * kwd)
    if reason is not None:
        return reason
    try:
        resolve_conv_padding(kw["padding"], (kh, kwd), kw["dilation"], kw["stride"])
    except ValueError as e:
        return f"the conv's {e}"
    return None


def _dense_conv_rule(groups, k_g):
    return None if groups == 1 else f"the conv has groups = {groups} (the integer path runs groups = 1 only)"


def int8_conv_ineligibility(qconv):
    """Why ``QConv2dInt8.from_qconv2d`` cannot convert ``qconv`` (None when it can)."""
    return _int8_conv_ineligibility(qconv, _dense_conv_rule)


class _Int8Conv2dModule:
    """The conv geometry and forward shared by the integer-grid conv modules: ``_set_geometry`` records it, a subclass
    supplies ``_conv(x, nhwc)`` of an fp32 [N, C, H, W] input, contiguous (NCHW) or, with ``nhwc``, channels-last.
    ``forward`` takes [N, C, H, W] or unbatched [C, H, W] and up-casts fp16; the output is fp32.  A batched input that is
    channels-last (and not also NCHW-contiguous) runs the channels-last kernels and gets a channels-last output, as
    ``F.conv2d`` returns; every other input, an unbatched one whatever its strides included, is made contiguous and
    gets a contiguous output, as ``F.conv2d`` returns for it.  The values are the same."""

    def _set_geometry(self, in_channels, out_channels, kernel_size, stride, padding, dilation, groups=1):
        self.in_channels, self.out_channels, self.groups = int(in_channels), int(out_channels), int(groups)
        self.kernel_size, self.stride, self.dilation = tuple(kernel_size), tuple(stride), tuple(dilation)
        self.padding = tuple(padding)  # (top, bottom, left, right)

    @staticmethod
    def _geometry_of(qconv):
        """The constructor arguments of ``qconv``'s geometry: in / out channels, kernel, stride, resolved padding,
        dilation, groups."""
        kw = qconv.fwd_kwargs
        c_out, c_g, kh, kwd = qconv.weight.shape
        groups = int(kw["groups"])
        padding = resolve_conv_padding(kw["padding"], (kh, kwd), kw["dilation"], kw["stride"])
        return c_g * groups, c_out, (kh, kwd), _pair(kw["stride"]), padding, _pair(kw["dilation"]), groups

    def forward(self, x_in):
        _check_inference_only(self, "QConv2d", x_in)
        x = x_in.float() if x_in.dtype != torch.float32 else x_in
        unbatched = x.dim() == 3
        if unbatched:
            x = x.unsqueeze(0)
        if not unbatched and x.dim() == 4 and x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous():
            y = self._conv(x, True)
        else:
            y = self._conv(x.contiguous(), False)
        return y.squeeze(0) if unbatched else y

    def extra_repr(self):
        return (f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, stride={self.stride}, "
                f"padding={self.padding}, dilation={self.dilation}, qrange=[{self.qmin}, {self.qmax}]")


class QConv2dInt8(_Int8Conv2dModule, _Int8WeightModule):
    """Inference-only replacement of a calibrated ``QConv2d`` (groups = 1): the fake-quant conv2d computed on the
    integer grid by ``ops.int8_conv2d`` -- the input lowered to its int8 grid in one pass, exact int8 x int8 sums on the
    tensor cores, zero points removed in int64, then s_x s_w[n] I + bias, written NCHW.  Built by ``from_qconv2d``; the
    weights (``weight.reshape(C_out, -1)``) are quantized once at conversion.  Takes [N, C, H, W] or unbatched
    [C, H, W]; fp16 input is up-cast and the output is fp32, as in the fake-quant op.  There is no backward: QAT keeps
    ``QConv2d``."""

    _ineligibility = staticmethod(int8_conv_ineligibility)

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation, device, groups=1):
        super().__init__(out_channels, in_channels // int(groups) * kernel_size[0] * kernel_size[1], device)
        self._set_geometry(in_channels, out_channels, kernel_size, stride, padding, dilation, groups)

    @classmethod
    def from_qconv2d(cls, qconv):
        cls._check_eligible(cls._ineligibility(qconv), "from_qconv2d")
        return cls._build(qconv)

    @classmethod
    def _build(cls, qconv):
        *geometry, groups = cls._geometry_of(qconv)
        return cls(*geometry, device=qconv.weight.device, groups=groups)._load(qconv)

    def _conv(self, x, nhwc):
        op = ops.int8_conv2d_nhwc if nhwc else ops.int8_conv2d
        return op(x, self.scale, self.zero_point, self.qmin, self.qmax, self.w_q, self.w_rowsum, self.w_scale, self.w_zero,
                  self.kernel_size, self.bias, self.stride, self.padding, self.dilation, x_absmax=self._x_absmax(x))


def int8_sparse24_conv_ineligibility(qconv):
    """Why ``QConv2dSparse24Int8.from_qconv2d`` cannot convert ``qconv`` (None when it can): a rule of
    ``int8_conv_ineligibility`` (groups >= 2 and unresolvable padding included), a centred weight grid outside s8, or a
    group of 4 along a row of ``weight.reshape(C_out, -1)`` on the grid with more than two nonzeros."""
    return _sparse24_checked(qconv, int8_conv_ineligibility(qconv))[1]


class QConv2dSparse24Int8(_Int8Conv2dModule, _Sparse24WeightModule):
    """Inference-only replacement of a calibrated ``QConv2d`` (groups = 1) whose weight is 2:4 sparse on the grid along
    the rows of ``weight.reshape(C_out, -1)``: the conv2d of ``QConv2dInt8`` on the sparse int8 tensor cores
    (``ops.int8_sparse24_conv2d``), bit-identical to ``QConv2dInt8`` on the same module.  Only the compressed weight
    is stored (``vals``, ``meta``, ``dsum``, ``w_scale``, as ``QLinearSparse24Int8``), about 0.625 byte per weight.
    Takes [N, C, H, W] or unbatched [C, H, W]; fp16 input is up-cast and the output is fp32.  Built by
    ``from_qconv2d``; no backward."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation, device):
        super().__init__(out_channels, in_channels * kernel_size[0] * kernel_size[1], device)
        self._set_geometry(in_channels, out_channels, kernel_size, stride, padding, dilation)

    @classmethod
    def from_qconv2d(cls, qconv):
        operand = cls._eligible_operand(qconv, int8_conv_ineligibility(qconv), "from_qconv2d")
        *geometry, _ = cls._geometry_of(qconv)
        return cls(*geometry, device=qconv.weight.device)._load(qconv, operand)

    def _conv(self, x, nhwc):
        op = ops.int8_sparse24_conv2d_nhwc if nhwc else ops.int8_sparse24_conv2d
        return op(x, self.scale, self.zero_point, self.qmin, self.qmax, self.vals, self.meta, self.dsum, self.w_scale,
                  self.kernel_size, self.bias, self.stride, self.padding, self.dilation)

    def extra_repr(self):
        return super().extra_repr() + ", 2:4 sparse"


INT8_MAX_KG = 1 << 17  # sb200_int8_group_conv2d: K_g = C / groups KH KW must stay below 2^17 (exact int32 sums)


def _group_conv_rule(groups, k_g):
    if groups == 1:
        return "groups = 1: use QConv2dInt8 / to_integer_convs"
    if k_g >= INT8_MAX_KG:
        return f"K_g = C / groups KH KW = {k_g} >= 2^17 (the integer sums must stay exact in int32)"
    return None


def int8_group_conv_ineligibility(qconv):
    """Why ``QConv2dGroupInt8.from_qconv2d`` cannot convert ``qconv`` (None when it can)."""
    return _int8_conv_ineligibility(qconv, _group_conv_rule)


class QConv2dGroupInt8(QConv2dInt8):
    """Inference-only replacement of a calibrated grouped or depthwise ``QConv2d`` (groups >= 2): the fake-quant conv2d
    computed on the integer grid by ``ops.int8_group_conv2d`` -- one direct int8 kernel that quantizes its input tile
    on the fly, exact integer sums per group, zero points removed in int64, then s_x s_w[n] I + bias, written NCHW.
    Built by ``from_qconv2d``; the weights (``weight.reshape(C_out, -1)``, C / groups KH KW per row) are quantized
    once at conversion.  Takes [N, C, H, W] or unbatched [C, H, W]; fp16 input is up-cast and the output is fp32, as in
    the fake-quant op.  There is no backward: QAT keeps ``QConv2d``."""

    _ineligibility = staticmethod(int8_group_conv_ineligibility)

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation, groups, device):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, device, groups)

    def _conv(self, x, nhwc):
        op = ops.int8_group_conv2d_nhwc if nhwc else ops.int8_group_conv2d
        return op(x, self.scale, self.zero_point, self.qmin, self.qmax, self.w_q, self.w_rowsum, self.w_scale, self.w_zero,
                  self.kernel_size, self.groups, self.bias, self.stride, self.padding, self.dilation,
                  x_absmax=self._x_absmax(x))

    def extra_repr(self):
        return super().extra_repr() + f", groups={self.groups}"


# ----------------------------------------------------------------------------- DoReFa and AdaRound layers
ADAROUND_SCALE_RANGE = (2.0 ** -126, 2.0 ** 119)  # |s|: (q - zp) s for |q - zp| <= 255 stays normal and finite


def _is(q, *types):
    return q is not None and q.TYPE.lower() in types


def _adaround_reason(wq, weight):
    """Why an AdaRound weight quantizer's eval-mode output does not re-quantize to its grid exactly (None if it does):
    RN((q - zp) s) / s rounds back to q when zp is integral, |q - zp| <= 255 (zp inside the integer range, which the
    shared rules check) and 2^-126 <= |s| <= 2^119."""
    if wq.training:
        return "the weight quantizer is AdaRound in training mode, whose soft rounding lies off the grid"
    if getattr(wq, "v", None) is None:
        return "the weight quantizer is AdaRound without its rounding variables v (run the reconstruction first)"
    scale, zero_point = _qparams(wq, weight)
    if not bool(torch.equal(zero_point, torch.round(zero_point))):
        return "the weight quantizer is AdaRound with a non-integral zero point"
    lo, hi = ADAROUND_SCALE_RANGE
    a = scale.abs()
    if not bool(((a >= lo) & (a <= hi)).all()):
        return "the weight quantizer is AdaRound with a scale outside [2^-126, 2^119] in magnitude"
    return None


def dorefa_adaround_ineligibility(qmod):
    """Why ``from_dorefa_adaround`` cannot convert ``qmod`` (None when it can): a ``QLinear`` or a ``QConv2d`` of any
    ``groups`` whose input quantizer is DoReFa, or whose weight quantizer is DoReFa or AdaRound (a layer with neither
    belongs to ``to_integer_linears`` / ``to_integer_convs`` / ``to_integer_group_convs``), and that meets every other
    rule of the matching plain converter.  DoReFa on a per-channel input and AdaRound on an input are refused; an
    AdaRound weight must be in eval mode with its ``v``, an integral zero point and 2^-126 <= |s| <= 2^119."""
    if not isinstance(qmod, (QLinear, QConv2d)):
        return f"expected a QLinear or a QConv2d, got {type(qmod).__name__}"
    for role, q in (("input", qmod.input_quantizer), ("weight", qmod.weight_quantizer)):
        if q is None:
            return f"the {role} quantizer is missing"
    aq, wq = qmod.input_quantizer, qmod.weight_quantizer
    if not (_is(aq, "dorefa") or _is(wq, "dorefa", "adaround")):
        return ("neither quantizer is DoReFa or AdaRound: use to_integer_linears / to_integer_convs / "
                "to_integer_group_convs")
    rule = lambda m: _int8_quantizer_ineligibility(m, _PLAIN_QDQ_TYPES + ("dorefa",),  # noqa: E731
                                                  _PLAIN_QDQ_TYPES + ("dorefa", "adaround"))
    if isinstance(qmod, QLinear):
        reason = rule(qmod)
    else:
        groups = int(qmod.fwd_kwargs["groups"])
        reason = _int8_conv_ineligibility(qmod, _dense_conv_rule if groups == 1 else _group_conv_rule, rule)
    if reason is None and _is(wq, "adaround"):
        reason = _adaround_reason(wq, qmod.weight)
    return reason


class _DoReFaInput:
    """A layer whose input quantizer is DoReFa: ``forward`` computes m = ``ops.dorefa_absmax`` over the whole input, the
    tensor the fake-quant quantizer sees, and the kernels quantize tanh(x) / m.  Same buffers as the plain layer."""

    def _x_absmax(self, x):
        # max |tanh| does not depend on the order: a channels-last x is read in its NHWC storage order
        return ops.dorefa_absmax(x if x.is_contiguous() else x.permute(0, 2, 3, 1))

    def extra_repr(self):
        return super().extra_repr() + ", input=DoReFa"


class QLinearDoReFaInt8(_DoReFaInput, QLinearInt8):
    """``QLinearInt8`` of a ``QLinear`` whose input quantizer is DoReFa (per-tensor); built by ``from_dorefa_adaround``."""


class QConv2dDoReFaInt8(_DoReFaInput, QConv2dInt8):
    """``QConv2dInt8`` of a ``QConv2d`` (groups = 1) whose input quantizer is DoReFa (per-tensor); built by
    ``from_dorefa_adaround``."""


class QConv2dGroupDoReFaInt8(_DoReFaInput, QConv2dGroupInt8):
    """``QConv2dGroupInt8`` of a grouped or depthwise ``QConv2d`` whose input quantizer is DoReFa (per-tensor); built by
    ``from_dorefa_adaround``."""


def from_dorefa_adaround(qmod):
    """The integer-grid layer of a calibrated ``QLinear`` / ``QConv2d`` that ``dorefa_adaround_ineligibility`` accepts:
    the weights stored on the weight quantizer's grid (``_grid_source``), and ``QLinearDoReFaInt8`` /
    ``QConv2dDoReFaInt8`` / ``QConv2dGroupDoReFaInt8`` when the input quantizer is DoReFa, else the plain
    ``QLinearInt8`` / ``QConv2dInt8`` / ``QConv2dGroupInt8``.  Raises ``ValueError`` with the reason otherwise."""
    reason = dorefa_adaround_ineligibility(qmod)
    if reason is not None:
        raise ValueError(f"from_dorefa_adaround: {reason}")
    dorefa = _is(qmod.input_quantizer, "dorefa")
    if isinstance(qmod, QLinear):
        cls = QLinearDoReFaInt8 if dorefa else QLinearInt8
    elif int(qmod.fwd_kwargs["groups"]) == 1:
        cls = QConv2dDoReFaInt8 if dorefa else QConv2dInt8
    else:
        cls = QConv2dGroupDoReFaInt8 if dorefa else QConv2dGroupInt8
    return cls._build(qmod)


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


class QMatMul(nn.Module):
    """The activation x activation matmul (modules/matmul.py MatMul) together with the two carriers that the reference
    inserts in front of its inputs: ``left`` and ``right`` are ``QIdentity`` operators, each owning the input quantizer
    of one operand.  The module itself has no quantizer attributes, so calibration sees the two carriers."""

    def __init__(self, org_module=None):
        super().__init__()
        self.left, self.right = QIdentity(), QIdentity()

    def build_quantizer(self, a_cfg, backend=Backend.VIRTUAL):
        self.left.build_quantizer(a_cfg, backend=backend)
        self.right.build_quantizer(a_cfg, backend=backend)
        return self

    def set_quant(self, w_quant=False, a_quant=False):
        self.left.set_quant(w_quant, a_quant)
        self.right.set_quant(w_quant, a_quant)

    def forward(self, x_left, x_right):
        return torch.matmul(self.left(x_left), self.right(x_right))


def int8_matmul_ineligibility(qmatmul):
    """Why ``QMatMulInt8.from_qmatmul`` cannot convert ``qmatmul`` (None when it can)."""
    if not isinstance(qmatmul, QMatMul):
        return f"expected a QMatMul, got {type(qmatmul).__name__}"
    for role, q in (("left", qmatmul.left.input_quantizer), ("right", qmatmul.right.input_quantizer)):
        reason = _int8_plain_qdq_reason(role, q)
        if reason is not None:
            return reason
        if q.is_perchannel:
            return f"the {role} quantizer is per-channel (the integer matmul needs one scale per operand)"
        reason = _int8_qparams_reason(role, q, None, (1,))
        if reason is not None:
            return reason
    return None


def _register_operand_qparams(mod, roles, device):
    """One per-tensor ``{role}_scale`` / ``{role}_zero_point`` buffer pair per operand role of ``mod``."""
    for role in roles:
        mod.register_buffer(f"{role}_scale", torch.ones(1, dtype=torch.float32, device=device))
        mod.register_buffer(f"{role}_zero_point", torch.zeros(1, dtype=torch.float32, device=device))


def _from_operand_quantizers(cls, quantizers, *args):
    """``cls(device, *args)`` with the buffers of ``_register_operand_qparams`` holding the qparams of ``quantizers``
    ({role: per-tensor quantizer}), and the integer ranges {role: (qmin, qmax)}."""
    qparams = {role: _qparams(q, None) for role, q in quantizers.items()}
    mod = cls(next(iter(qparams.values()))[0].device, *args)
    with torch.no_grad():
        for role, (s, z) in qparams.items():
            getattr(mod, f"{role}_scale").copy_(s.reshape(1))
            getattr(mod, f"{role}_zero_point").copy_(z.reshape(1))
    return mod, {role: tuple(q.qdesc.qrange) for role, q in quantizers.items()}


class QMatMulInt8(nn.Module):
    """Inference-only replacement of a calibrated ``QMatMul``: the matmul of the two fake-quant operands computed on the
    integer grid by ``ops.int8_matmul`` -- both operands quantized on the fly, exact int8 x int8 sums on the tensor
    cores, zero points removed in int64, then s_left s_right I.  Built by ``from_qmatmul``.  Operands have at least 2
    dimensions and broadcast as in ``torch.matmul``; fp16 input is up-cast and the output is fp32, as in the fake-quant
    op.  There is no backward: QAT keeps ``QMatMul``."""

    def __init__(self, device):
        super().__init__()
        _register_operand_qparams(self, ("left", "right"), device)
        self.left_qrange, self.right_qrange = (-128, 127), (-128, 127)

    @classmethod
    def from_qmatmul(cls, qmatmul):
        reason = int8_matmul_ineligibility(qmatmul)
        if reason is not None:
            raise ValueError(f"QMatMulInt8.from_qmatmul: {reason}")
        mod, qranges = _from_operand_quantizers(cls, {"left": qmatmul.left.input_quantizer,
                                                      "right": qmatmul.right.input_quantizer})
        mod.left_qrange, mod.right_qrange = qranges["left"], qranges["right"]
        return mod

    def forward(self, x_left, x_right):
        _check_inference_only(self, "QMatMul", x_left, x_right)
        if x_left.dim() < 2 or x_right.dim() < 2:
            raise ValueError(f"QMatMulInt8 takes operands with at least 2 dimensions (got {x_left.dim()}-D and "
                             f"{x_right.dim()}-D); 1-D operands are not supported")
        return ops.int8_matmul(x_left.float(), self.left_scale, self.left_zero_point, self.left_qrange,
                               x_right.float(), self.right_scale, self.right_zero_point, self.right_qrange)

    def extra_repr(self):
        return f"left_qrange={list(self.left_qrange)}, right_qrange={list(self.right_qrange)}"


def masked_scores(s, attn_mask=None, causal=False):
    """The scores of ``QAttention`` after its mask: with ``causal`` the keys j > i + (Tk - Tq) of row i become -inf (the
    band aligned bottom-right), then ``attn_mask`` is added in fp32.  A leaf of ``torch.fx`` traces (``fx.wrap``)."""
    if causal:
        tq, tk = s.shape[-2], s.shape[-1]
        i = torch.arange(tq, device=s.device)[:, None]
        j = torch.arange(tk, device=s.device)[None, :]
        s = s.masked_fill(j > i + (tk - tq), float("-inf"))
    if attn_mask is not None:
        s = s + ops.attention_mask_check(attn_mask)
    return s


torch.fx.wrap("masked_scores")


class QAttention(nn.Module):
    """Softmax attention between two ``QMatMul``: ``qk`` (carriers of q and k^T) and ``pv`` (carriers of the softmax
    output p and of v), the reference's MatMul -> Softmax -> MatMul behind its four ``QIdentity`` carriers.
    ``forward(q, k, v, attn_mask=None, causal=False)`` is, in this order::

        s = qk(q, k^T); s = s * scale (when scale is not None)
        causal:    s = where(j <= i + (Tk - Tq), s, -inf)   for query row i and key j
        attn_mask: s = s + attn_mask                         (additive float, broadcastable to [..., Tq, Tk])
        out = pv(softmax(s, -1), v)

    The causal band is aligned bottom-right, as in the reference's GPT-2 example: with Tq < Tk the last query row sees
    every key.  This is not the top-left ``is_causal`` of ``torch.nn.functional.scaled_dot_product_attention`` when
    Tq != Tk.  A query row that sees no key (causal with Tq > Tk, or an all -inf mask row) is NaN, as ``softmax`` gives.
    float16 / bfloat16 masks are up-cast (exact); a bool mask raises ``TypeError``.  Like ``QMatMul`` it is not itself a
    quant operator, so calibration (streaming or the fx replay) sees the four carriers, p after the mask."""

    def __init__(self, scale=None):
        super().__init__()
        self.scale = scale
        self.qk, self.pv = QMatMul(), QMatMul()

    def build_quantizer(self, a_cfg, p_cfg=None, backend=Backend.VIRTUAL):
        """``a_cfg`` builds the carriers of q, k and v; ``p_cfg`` (default ``a_cfg``) that of p, ``pv.left``, so that
        the softmax output can use an unsigned affine range."""
        self.qk.build_quantizer(a_cfg, backend=backend)
        self.pv.build_quantizer(a_cfg, backend=backend)
        if p_cfg is not None:
            self.pv.left.build_quantizer(p_cfg, backend=backend)
        return self

    def set_quant(self, w_quant=False, a_quant=False):
        self.qk.set_quant(w_quant, a_quant)
        self.pv.set_quant(w_quant, a_quant)

    def forward(self, q, k, v, attn_mask=None, causal=False):
        s = self.qk(q, k.transpose(-2, -1))
        if self.scale is not None:
            s = s * self.scale
        if attn_mask is not None or causal:
            s = masked_scores(s, attn_mask, causal)
        return self.pv(s.softmax(-1), v)

    def extra_repr(self):
        return f"scale={self.scale}"


def int8_attention_ineligibility(qattn):
    """Why ``QAttentionInt8.from_qattention`` cannot convert ``qattn`` (None when it can)."""
    if not isinstance(qattn, QAttention):
        return f"expected a QAttention, got {type(qattn).__name__}"
    for role in ("qk", "pv"):
        child = getattr(qattn, role)
        if isinstance(child, QMatMulInt8):
            return (f"the {role} matmul is already a QMatMulInt8: run to_integer_attentions before "
                    "to_integer_matmuls")
        reason = int8_matmul_ineligibility(child)
        if reason is not None:
            return f"the {role} matmul: {reason}"
    if qattn.scale is not None and not math.isfinite(float(qattn.scale)):
        return f"the scale {qattn.scale} is not finite"
    return None


class QAttentionInt8(nn.Module):
    """Inference-only replacement of a calibrated ``QAttention``: ``ops.int8_attention``, one fused kernel on the
    integer grid -- q and k quantized on the fly, exact int8 scores on the tensor cores (bit-identical to
    ``QMatMulInt8``), the softmax in fp32 registers quantized with p's qparams, exact p @ v on the grid; the [Tq, Tk]
    scores never reach memory.  Built by ``from_qattention``.  q, k, v have equal leading dimensions; fp16 input is
    up-cast and the output is fp32, as in the fake-quant op.  ``attn_mask`` and ``causal`` are those of
    ``QAttention.forward``, computed in the kernel (``ops.int8_attention``).  There is no backward: QAT keeps
    ``QAttention``.

    Generation: ``new_cache(lead, capacity, d, dv)`` makes an ``ops.Int8KVCache`` bound to this layer, and
    ``forward(q, k, v, attn_mask, causal, cache=cache)`` appends the new keys and values k, v to it (quantized once)
    and attends q to all ``cache.length`` stored keys: ``forward(q, cat(past_k, k), cat(past_v, v), attn_mask,
    causal)``, bit for bit for Tq > 16; for Tq <= 16 the split-key decode kernels give the same scores and an output
    exact on their own p grid, which can differ from the fused kernel's by one step (``ops.int8_attention_cached``)."""

    ROLES = ("q", "k", "p", "v")

    def __init__(self, device, scale=None):
        super().__init__()
        self.scale = scale
        _register_operand_qparams(self, self.ROLES, device)
        self.qranges = {role: (-128, 127) for role in self.ROLES}

    @classmethod
    def from_qattention(cls, qattn):
        reason = int8_attention_ineligibility(qattn)
        if reason is not None:
            raise ValueError(f"QAttentionInt8.from_qattention: {reason}")
        carriers = (qattn.qk.left, qattn.qk.right, qattn.pv.left, qattn.pv.right)
        mod, qranges = _from_operand_quantizers(cls, {r: c.input_quantizer for r, c in zip(cls.ROLES, carriers)},
                                                None if qattn.scale is None else float(qattn.scale))
        mod.qranges.update(qranges)
        return mod

    def new_cache(self, lead, capacity, d, dv):
        """An empty int8 key/value cache of ``capacity`` keys for q / k / v with leading dimensions ``lead``, on this
        layer's device and bound to this layer (its qparams quantize what is appended)."""
        return ops.Int8KVCache(self, lead, capacity, d, dv, self.q_scale.device)

    def forward(self, q, k, v, attn_mask=None, causal=False, cache=None):
        _check_inference_only(self, "QAttention", q, k, v)
        qp = [(getattr(self, f"{r}_scale"), getattr(self, f"{r}_zero_point"), self.qranges[r]) for r in self.ROLES]
        if cache is None:
            return ops.int8_attention(q.float(), k.float(), v.float(), *qp, scale=self.scale, attn_mask=attn_mask,
                                      causal=causal)
        if not isinstance(cache, ops.Int8KVCache) or cache.layer is not self:
            raise ValueError("QAttentionInt8: the cache was not created by this layer's new_cache")
        lead = tuple(q.shape[:-2])
        if (lead != cache.lead or tuple(k.shape[:-2]) != lead or tuple(v.shape[:-2]) != lead or q.shape[-1] != cache.d
                or k.shape[-1] != cache.d or v.shape[-1] != cache.dv or k.shape[-2] != v.shape[-2]):
            raise ValueError(f"QAttentionInt8: q {tuple(q.shape)}, k {tuple(k.shape)} and v {tuple(v.shape)} do not "
                             f"match the cache's lead {cache.lead}, d = {cache.d} and dv = {cache.dv}")
        # the mask over the keys after the append is checked first, so that a bad mask leaves the cache untouched
        ops._attention_mask("QAttentionInt8", attn_mask, causal, q.device, lead, q.shape[-2],
                            cache.length + k.shape[-2])
        ops.int8_kv_append(cache, k.float(), v.float(), qp[1], qp[3])
        return ops.int8_attention_cached(q.float(), cache, *qp, scale=self.scale, attn_mask=attn_mask, causal=causal)

    def extra_repr(self):
        return f"scale={self.scale}, " + ", ".join(f"{r}_qrange={list(self.qranges[r])}" for r in self.ROLES)
