"""CPU: the host side of sb200_int8_sparse24_conv2d and the device-free rules of QConv2dSparse24Int8.from_qconv2d.

* Every bad argument is rejected on the host, before any CUDA call, with its code and in sb200_int8_conv2d's order.
* The ineligibility reasons that need no device: not a QConv2d, a missing quantizer, groups >= 2 (the dense conv's
  reason)."""
import ctypes

import torch.nn as nn

from int8_harness import E_INVALID, E_UNSUPPORTED, E_WORKSPACE, buf, cfg, conv_geom, rejector
from sparsebit_b200 import _lib
from sparsebit_b200.quantization.common import Backend
from sparsebit_b200.quantization.modules import QConv2d, int8_conv_ineligibility, int8_sparse24_conv_ineligibility

def test_argument_errors_come_before_any_cuda_call():
    lib = _lib.load()
    keep, p = buf()
    g = conv_geom()
    ws_ok = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    # (x, geom, xs, xz, qmin, qmax, vals, meta, dsum, w_scale, bias, out, c_out, ws, ws_bytes, stream)
    ok = [p, ctypes.byref(g), p, p, -128, 127, p, p, p, p, None, p, 8, p, ws_ok, None]
    rejected = rejector(lib.sb200_int8_sparse24_conv2d, ok)
    for i in (0, 1, 2, 3, 6, 7, 8, 9, 11, 13):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    rejected(E_INVALID, b"empty operand", a12=0)
    rejected(E_INVALID, b"empty operand", a12=-4)
    rejected(E_INVALID, b"too large", a12=1 << 31)
    for bad in (dict(n=0), dict(c=-1), dict(kh=0), dict(stride_w=-1), dict(dilation_h=0), dict(pad_top=-1), dict(h=1 << 31)):
        rejected(E_INVALID, b"non-positive geometry", a1=ctypes.byref(conv_geom(**bad)))
    rejected(E_INVALID, b"empty output", a1=ctypes.byref(conv_geom(kh=11)))
    rejected(E_INVALID, b"too many output pixels", a1=ctypes.byref(conv_geom(n=1 << 20, h=64, w=64, c=1)))
    rejected(E_INVALID, b"wider than 8 bits", a4=0, a5=256)
    rejected(E_INVALID, b"neither signed", a4=-129, a5=0)
    rejected(E_INVALID, b"16-byte aligned", a6=p + 8)
    rejected(E_INVALID, b"16-byte aligned", a7=p + 4)
    for big in (dict(c=1 << 17, kh=1, kw=1, pad_top=0, pad_bottom=0, pad_left=0, pad_right=0),
                dict(c=(1 << 17) // 9 + 1)):
        rejected(E_UNSUPPORTED, b"K < 2^17", a1=ctypes.byref(conv_geom(**big)), a14=1 << 40)
    rejected(E_WORKSPACE, b"workspace too small", a14=ws_ok - 1)
    rejected(E_WORKSPACE, b"workspace too small", a14=0)
    # the order of the rules: a null pointer before the geometry, the geometry before the range, the range before the
    # alignment, the alignment before K, K before the workspace
    rejected(E_INVALID, b"null pointer", a0=None, a1=ctypes.byref(conv_geom(n=0)))
    rejected(E_INVALID, b"non-positive geometry", a1=ctypes.byref(conv_geom(n=0)), a4=0, a5=256)
    rejected(E_INVALID, b"wider than 8 bits", a4=0, a5=256, a6=p + 8)
    rejected(E_INVALID, b"16-byte aligned", a6=p + 8, a1=ctypes.byref(conv_geom(c=1 << 17, kh=1, kw=1)))
    rejected(E_UNSUPPORTED, b"K < 2^17", a1=ctypes.byref(conv_geom(c=(1 << 17) // 9 + 1)), a14=0)


def test_ineligibility_rules_without_a_device():
    assert "expected a QConv2d" in int8_sparse24_conv_ineligibility(nn.Conv2d(4, 4, 3))
    assert "expected a QConv2d" in int8_sparse24_conv_ineligibility(nn.Linear(4, 4))
    q = QConv2d(nn.Conv2d(8, 4, 3))
    assert int8_sparse24_conv_ineligibility(q) == "the input quantizer is missing"
    dw = QConv2d(nn.Conv2d(8, 8, 3, groups=8)).build_quantizer(cfg("per-tensor-affine", "feature"),
                                                               cfg("per-channel-symmetric", "weight"), Backend.VIRTUAL)
    dw.set_quant(w_quant=True, a_quant=True)
    reason = int8_sparse24_conv_ineligibility(dw)
    assert reason == int8_conv_ineligibility(dw) and "groups = 8" in reason
