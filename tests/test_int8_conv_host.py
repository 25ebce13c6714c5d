"""CPU: the fp64 truth of the integer-grid conv2d, the host side of sb200_int8_im2col_quantize / sb200_int8_conv2d and
the eligibility rules of QConv2dInt8.from_qconv2d.

* The truth (the fp64 conv of the oracle's fake-quant tensors, zero-padded after the fake-quant) equals the integer
  form on the lowered rows -- padding taps stored as the zero point -- exactly for power-of-two scales and within the
  stated bound otherwise, for symmetric and affine ranges.
* Padding resolution: int, pair, 'valid', 'same' with odd and even kernels (checked against F.conv2d).
* Every bad argument of the three entry points is rejected on the host, before any CUDA call, with its code.
* Every rule of from_qconv2d gives its reason, and to_integer_convs leaves those layers alone."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from int8_conv_ref import integer_terms, lowered, out_hw, to_nchw, truth
from int8_harness import (BAD_GEOMS, E_INVALID, E_WORKSPACE, buf, check_geometry_rules, conv_geom, refusal,
                          rejector)
from sparsebit_b200 import _lib
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.common import Backend
from sparsebit_b200.quantization.modules import (QConv2d, QConv2dInt8, QLinear, int8_conv_ineligibility,
                                                 resolve_conv_padding)
from sparsebit_b200.quantization.tools import to_integer_convs

GEOMS = [
    # (n, c, h, w, c_out, kh, kw, stride, padding, dilation)
    (2, 3, 7, 6, 5, 3, 3, 1, 1, 1),
    (1, 4, 9, 9, 3, 3, 3, 2, (1, 0, 2, 1), 1),
    (2, 2, 8, 7, 4, 1, 3, 1, (0, 1), 2),
    (1, 3, 11, 10, 2, 7, 7, 2, 3, 1),
]
RANGES = [((-128, 127), (-128, 127)), ((0, 255), (-128, 127)), ((0, 15), (-8, 7)), ((0, 3), (-2, 1))]


def _operands(rng, geom, xrange, wrange, pow2):
    n, c, h, w, c_out, kh, kw = geom[:7]
    x = (rng.standard_normal((n, c, h, w)) * 3 + 1).astype(np.float32)
    wt = (rng.standard_normal((c_out, c, kh, kw)) / np.sqrt(c * kh * kw)).astype(np.float32)
    (xqmin, xqmax), (wqmin, wqmax) = xrange, wrange
    if pow2:
        xs = np.float32(2.0 ** -3)
        ws = (2.0 ** -rng.integers(4, 8, c_out)).astype(np.float32)
    else:
        xs = np.float32(np.abs(x).max() / (xqmax - xqmin) * 1.7)
        ws = (np.abs(wt).reshape(c_out, -1).max(axis=1) / (wqmax - wqmin) * 1.9).astype(np.float32)
    xz = np.float32(0 if xqmin < 0 else rng.integers(xqmin + 1, xqmax))  # the zero point away from 0
    wz = np.zeros(c_out, np.float32)
    return x, xs, xz, xqmin, xqmax, wt, ws, wz, wqmin, wqmax


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("xrange,wrange", RANGES)
@pytest.mark.parametrize("pow2", [True, False])
def test_truth_equals_the_integer_form_on_lowered_rows(geom, xrange, wrange, pow2):
    rng = np.random.default_rng(abs(hash((geom, xrange, wrange, pow2))) % 2**32)
    ops_ = _operands(rng, geom, xrange, wrange, pow2)
    stride, padding, dilation = geom[7:]
    bias = None if pow2 else rng.standard_normal(geom[4]).astype(np.float32)
    t, bound = truth(*ops_, bias=bias, stride=stride, padding=padding, dilation=dilation)
    a, b, zx, zw, i = integer_terms(*ops_, stride=stride, padding=padding, dilation=dilation)
    assert np.array_equal(i, (a - zx) @ (b - zw[:, None]).T)
    if xrange[0] >= 0:
        assert (a == zx).any()  # padding taps hold the zero point (v = 0), not the stored 0
    x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax = ops_
    n = x.shape[0]
    oh, ow = out_hw(x.shape[2], x.shape[3], w.shape[2], w.shape[3], stride, padding, dilation)
    y = to_nchw(float(xs) * ws.astype(np.float64)[None, :] * i.astype(np.float64), n, oh, ow)
    if bias is not None:
        y = y + bias.astype(np.float64)[None, :, None, None]
    assert y.shape == t.shape
    if pow2:
        assert np.array_equal(y, t)
    else:
        assert np.all(np.abs(y - t) <= bound) and np.all(bound > 0)


def test_lowered_rows_flag_exactly_the_windows_holding_a_nan():
    x = np.ones((1, 2, 5, 5), np.float32)
    x[0, 1, 2, 3] = np.nan
    q, row_sum, nan = lowered(x, 3, 0.5, 3, 0, 255, padding=1)
    ih, iw = np.divmod(np.arange(25), 5)
    assert np.array_equal(nan, (np.abs(ih - 2) <= 1) & (np.abs(iw - 3) <= 1))
    assert q.shape == (25, 32) and not q[:, 18:].any()
    assert np.array_equal(row_sum, q.sum(1))


@pytest.mark.parametrize("padding,kernel,dilation", [(0, 3, 1), (2, 3, 1), ((1, 2), (3, 5), 1), ("valid", 3, 1),
                                                     ("same", 3, 1), ("same", 4, 1), ("same", (2, 5), 1),
                                                     ("same", (4, 3), (2, 3)), ("same", 1, 1)])
def test_padding_resolution_matches_conv2d(padding, kernel, dilation):
    kh, kw = (kernel, kernel) if isinstance(kernel, int) else kernel
    x = torch.randn(1, 2, 9, 10, dtype=torch.float64)
    w = torch.randn(3, 2, kh, kw, dtype=torch.float64)
    pt, pb, pl, pr = resolve_conv_padding(padding, (kh, kw), dilation)
    assert min(pt, pb, pl, pr) >= 0
    ref = F.conv2d(x, w, padding=padding, dilation=dilation)
    got = F.conv2d(F.pad(x, (pl, pr, pt, pb)), w, dilation=dilation)
    assert torch.equal(ref, got)


def test_padding_that_does_not_resolve():
    for bad in ("full", (-1, 0), -2, (1, 2, 3)):
        with pytest.raises(ValueError):
            resolve_conv_padding(bad, (3, 3))
    with pytest.raises(ValueError, match="stride 1"):
        resolve_conv_padding("same", (3, 3), 1, 2)


# ---------------------------------------------------------------------------------------------- C-ABI on the host
def test_im2col_quantize_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    g = conv_geom()
    # (x, geom, scale, zp, qmin, qmax, q, row_sum, nan_flag, stream)
    ok = [p, ctypes.byref(g), p, p, 0, 255, p, p, p, None]
    rejected = rejector(lib.sb200_int8_im2col_quantize, ok)
    for i in (0, 1, 2, 3, 6, 7, 8):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    check_geometry_rules(rejected, 1)
    rejected(E_INVALID, b"wider than 8 bits", a4=-200, a5=100)
    rejected(E_INVALID, b"qmin", a4=5, a5=4)
    rejected(E_INVALID, b"neither signed", a4=-1, a5=200)
    rejected(E_INVALID, b"16-byte aligned", a6=p + 4)


def test_conv2d_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    g = conv_geom()
    ws_ok = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    # (x, geom, xs, xz, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, ws, ws_bytes, stream)
    ok = [p, ctypes.byref(g), p, p, -128, 127, p, p, p, p, None, p, 8, p, ws_ok, None]
    rejected = rejector(lib.sb200_int8_conv2d, ok)
    for i in (0, 1, 2, 3, 6, 7, 8, 9, 11, 13):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    rejected(E_INVALID, b"empty operand", a12=0)
    rejected(E_INVALID, b"empty operand", a12=-4)
    rejected(E_INVALID, b"too large", a12=1 << 31)
    check_geometry_rules(rejected, 1)
    rejected(E_INVALID, b"wider than 8 bits", a4=0, a5=256)
    rejected(E_INVALID, b"neither signed", a4=-129, a5=0)
    rejected(E_INVALID, b"16-byte aligned", a6=p + 1)
    rejected(E_WORKSPACE, b"workspace too small", a14=ws_ok - 1)
    rejected(E_WORKSPACE, b"workspace too small", a14=0)


def test_workspace_query_is_pure():
    lib = _lib.load()
    q = lib.sb200_int8_conv2d_workspace_bytes
    lin = lib.sb200_int8_linear_workspace_bytes
    assert q(None) == 0
    for bad in BAD_GEOMS + [dict(kh=11), dict(n=1 << 20, h=64, w=64, c=1)]:
        assert q(ctypes.byref(conv_geom(**bad))) == 0
    for kw in [{}, dict(stride_h=2, stride_w=2), dict(c=3, kh=7, kw=7, pad_top=3, pad_bottom=3, pad_left=3, pad_right=3)]:
        g = conv_geom(**kw)
        first = q(ctypes.byref(g))
        oh = (g.h + g.pad_top + g.pad_bottom - g.dilation_h * (g.kh - 1) - 1) // g.stride_h + 1
        ow = (g.w + g.pad_left + g.pad_right - g.dilation_w * (g.kw - 1) - 1) // g.stride_w + 1
        assert first == lin(g.n * oh * ow, g.c * g.kh * g.kw)
        assert all(q(ctypes.byref(g)) == first for _ in range(3))


# ---------------------------------------------------------------------------------------------- eligibility
def _qconv(a_scheme="per-tensor-affine", a_bit=8, w_scheme="per-channel-symmetric", w_bit=8, w_type="uniform",
           a_type="uniform", backend=Backend.VIRTUAL, a_disable=False, **conv):
    kw = dict(kernel_size=3, padding=1)
    kw.update(conv)
    q = QConv2d(nn.Conv2d(4, 6, **kw)).build_quantizer(
        sbcfg.quantizer_config(a_scheme, a_bit, "feature", qtype=a_type, disable=a_disable),
        sbcfg.quantizer_config(w_scheme, w_bit, "weight", qtype=w_type), backend=backend)
    q.set_quant(w_quant=True, a_quant=True)
    return q


def test_eligible_convs():
    assert int8_conv_ineligibility(_qconv()) is None
    assert int8_conv_ineligibility(_qconv("per-tensor-symmetric", 8, "per-tensor-symmetric", 4)) is None
    assert int8_conv_ineligibility(_qconv(w_type="lsq", a_type="lsq")) is None
    assert int8_conv_ineligibility(_qconv("per-tensor-symmetric", backend=Backend.TENSORRT)) is None
    for padding in (0, (1, 2), "valid", "same"):
        assert int8_conv_ineligibility(_qconv(padding=padding)) is None
    assert int8_conv_ineligibility(_qconv(kernel_size=4, padding="same", dilation=2)) is None


_reason = refusal(int8_conv_ineligibility, QConv2dInt8.from_qconv2d)


def test_every_ineligible_conv_gives_its_reason():
    q = _qconv()
    q.set_quant(w_quant=True, a_quant=False)
    assert "input quantizer is not enabled" in _reason(q)
    q = _qconv()
    q.set_quant(w_quant=False, a_quant=True)
    assert "weight quantizer is not enabled" in _reason(q)
    assert "input quantizer is fake_fused" in _reason(_qconv(a_disable=True))
    q = _qconv()
    q.input_quantizer.enable_export_onnx()
    assert "export_onnx" in _reason(q)
    assert "DoReFa" in _reason(_qconv(w_type="dorefa"))
    assert "adaround" in _reason(_qconv(w_type="adaround"))
    assert "input quantizer is per-channel" in _reason(_qconv(a_scheme="per-channel-affine"))
    assert "9 bits" in _reason(_qconv(a_bit=9))
    assert "16 bits" in _reason(_qconv(w_bit=16))
    q = _qconv()
    q.weight_quantizer.qdesc._ch_axis = 1
    assert "axis 1" in _reason(q)
    q = _qconv()
    q.input_quantizer.zero_point = torch.tensor([-3.0])
    assert "input zero point lies outside [0, 255]" in _reason(q)
    q = _qconv()
    q.weight_quantizer.scale = torch.ones(4, 1, 1, 1)
    q.weight_quantizer.zero_point = torch.zeros(4, 1, 1, 1)
    assert "holds 4 scales" in _reason(q)
    q = _qconv("per-tensor-symmetric", backend=Backend.TENSORRT)
    q.input_quantizer.zero_point = torch.tensor([3.0])
    assert "tensorrt only support symmetric" in _reason(q)
    assert "groups = 2" in _reason(_qconv(groups=2))
    q = _qconv()
    q.fwd_kwargs["padding"] = (-1, 0)
    assert "padding" in _reason(q) and "negative" in _reason(q)
    q = _qconv()
    q.fwd_kwargs["padding"] = "full"
    assert "neither 'valid' nor 'same'" in _reason(q)
    assert "expected a QConv2d" in int8_conv_ineligibility(nn.Conv2d(3, 4, 3))
    lin = QLinear(nn.Linear(3, 4))
    assert "expected a QConv2d" in int8_conv_ineligibility(lin)


def test_to_integer_convs_skips_ineligible_layers():
    model = nn.Sequential(_qconv(w_type="dorefa"), nn.ReLU(), _qconv(groups=2), _qconv(a_bit=9))
    assert to_integer_convs(model) == []
    assert all(isinstance(model[i], QConv2d) for i in (0, 2, 3))


def test_qconv2d_int8_module_contract():
    mod = QConv2dInt8(3, 5, (3, 2), (1, 2), (1, 0, 1, 1), (2, 1), torch.device("cpu"))
    buffers = {name: (b.dtype, tuple(b.shape)) for name, b in mod.named_buffers()}
    assert buffers == {"w_q": (torch.int8, (5, 32)), "w_rowsum": (torch.int32, (5,)), "w_scale": (torch.float32, (5,)),
                       "w_zero": (torch.int32, (5,)), "scale": (torch.float32, (1,)), "zero_point": (torch.float32, (1,))}
    assert set(mod.state_dict()) == set(buffers) and "bias" in mod._buffers and mod.bias is None
    assert (mod.in_channels, mod.out_channels, mod.qmin, mod.qmax) == (3, 5, -128, 127)
    assert (mod.kernel_size, mod.stride, mod.padding, mod.dilation) == ((3, 2), (1, 2), (1, 0, 1, 1), (2, 1))
    assert repr(mod) == ("QConv2dInt8(3, 5, kernel_size=(3, 2), stride=(1, 2), padding=(1, 0, 1, 1), dilation=(2, 1), "
                         "qrange=[-128, 127])")
    for x in (torch.zeros(1, 3, 6, 6, requires_grad=True), torch.zeros(3, 6, 6, requires_grad=True)):
        with pytest.raises(RuntimeError, match=r"^QConv2dInt8 is inference-only and has no backward; .* keep QConv2d for"):
            mod(x)
