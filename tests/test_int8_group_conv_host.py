"""The grouped / depthwise integer-grid conv on the host: the fp64 truth equals the per-group integer form, every
C-ABI rejection of sb200_int8_group_conv2d (no kernel launched), the conversion rules of QConv2dGroupInt8, and the
branch coverage of the GPU branch suite."""
import ctypes
import functools

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_group_geometry as geo
from int8_group_conv_ref import group_integer_form, truth
from int8_harness import BAD_GEOMS, E_INVALID, E_UNSUPPORTED, buf, conv_geom, refusal, rejector
from sparsebit_b200 import _lib
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.common import Backend
from sparsebit_b200.quantization.modules import (QConv2d, QConv2dGroupInt8, QLinear, int8_conv_ineligibility,
                                                 int8_group_conv_ineligibility)
from sparsebit_b200.quantization.modules import QConv2dInt8
from sparsebit_b200.quantization.tools import to_integer_convs, to_integer_group_convs
from test_gpu_int8_group_branches import BIG, CASES, case_branches


GEOMS = [
    # (n, c, h, w, c_out, groups, kernel, stride, padding, dilation)
    (2, 6, 9, 8, 6, 6, 3, 1, 1, 1),
    (1, 4, 11, 10, 8, 4, 5, 2, 2, 1),
    (2, 6, 9, 9, 4, 2, 3, 1, (0, 2, 1, 0), 2),
    (1, 12, 7, 7, 6, 3, (1, 3), 1, (0, 1), 1),
    (2, 16, 8, 8, 16, 2, 3, 2, 1, 1),
]
RANGES = [((-128, 127), (-128, 127)), ((0, 255), (-128, 127)), ((0, 15), (-8, 7))]


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("xrange,wrange", RANGES)
def test_truth_equals_the_group_integer_form(geom, xrange, wrange):
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation = geom
    kh, kw = (kernel, kernel) if isinstance(kernel, int) else kernel
    rng = np.random.default_rng(abs(hash((geom, xrange, wrange))) % 2**32)
    (xqmin, xqmax), (wqmin, wqmax) = xrange, wrange
    x = (rng.standard_normal((n, c, h, w)) * 3 + 1).astype(np.float32)
    wt = rng.standard_normal((c_out, c // groups, kh, kw)).astype(np.float32)
    xs, ws = np.float32(2.0 ** -3), (2.0 ** -rng.integers(1, 4, c_out)).astype(np.float32)
    xz = np.float32(0 if xqmin < 0 else rng.integers(xqmin + 1, xqmax))
    wz = np.zeros(c_out, np.float32) if wqmin < 0 else rng.integers(wqmin, wqmax, c_out).astype(np.float32)
    args = (x, xs, xz, xqmin, xqmax, wt, ws, wz, wqmin, wqmax, groups)
    t_, _ = truth(*args, stride=stride, padding=padding, dilation=dilation)
    i, s = group_integer_form(*args, stride=stride, padding=padding, dilation=dilation)
    assert np.array_equal(t_, i * s[None, :, None, None])


# ---------------------------------------------------------------------------------------------- C-ABI on the host
_geom = functools.partial(conv_geom, c=8)


def test_group_conv2d_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    g = _geom()
    # (x, geom, groups, xs, xz, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, stream)
    ok = [p, ctypes.byref(g), 8, p, p, -128, 127, p, p, p, p, None, p, 8, None]
    rejected = rejector(lib.sb200_int8_group_conv2d, ok)
    for i in (0, 1, 3, 4, 7, 8, 9, 10, 12):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    rejected(E_INVALID, b"empty operand", a13=0)
    rejected(E_INVALID, b"empty operand", a13=-8)
    rejected(E_INVALID, b"too large", a13=1 << 31)
    rejected(E_INVALID, b"sb200_int8_conv2d", a2=1)
    rejected(E_INVALID, b"groups = 0", a2=0)
    rejected(E_INVALID, b"groups = -2", a2=-2)
    for bad in BAD_GEOMS:
        rejected(E_INVALID, b"non-positive geometry", a1=ctypes.byref(_geom(**bad)))
    rejected(E_INVALID, b"empty output", a1=ctypes.byref(_geom(kh=11)))
    rejected(E_INVALID, b"too many output pixels", a1=ctypes.byref(_geom(n=1 << 20, h=64, w=64)))
    rejected(E_INVALID, b"does not divide", a2=3)
    rejected(E_INVALID, b"does not divide", a13=12)
    rejected(E_INVALID, b"wider than 8 bits", a5=0, a6=256)
    rejected(E_INVALID, b"qmin", a5=5, a6=4)
    rejected(E_INVALID, b"neither signed", a5=-129, a6=0)
    big = _geom(c=2 << 17, kh=1, kw=1, pad_top=0, pad_bottom=0, pad_left=0, pad_right=0)
    rejected(E_UNSUPPORTED, b"K_g < 2^17", a1=ctypes.byref(big), a2=2, a13=2)
    rejected(E_UNSUPPORTED, b"K_g < 2^17", a1=ctypes.byref(_geom(c=2 * ((1 << 17) // 9 + 1))), a2=2, a13=2)
    # K_g just below the limit passes the checks up to the launch; a geometry the kernel takes needs no workspace query
    assert lib.sb200_int8_group_conv2d.argtypes[2] is ctypes.c_int64


# ---------------------------------------------------------------------------------------------- eligibility
def _qconv(a_scheme="per-tensor-affine", a_bit=8, w_scheme="per-channel-symmetric", w_bit=8, w_type="uniform",
           a_type="uniform", backend=Backend.VIRTUAL, a_disable=False, c_in=8, c_out=8, **conv):
    kw = dict(kernel_size=3, padding=1, groups=4)
    kw.update(conv)
    q = QConv2d(nn.Conv2d(c_in, c_out, **kw)).build_quantizer(
        sbcfg.quantizer_config(a_scheme, a_bit, "feature", qtype=a_type, disable=a_disable),
        sbcfg.quantizer_config(w_scheme, w_bit, "weight", qtype=w_type), backend=backend)
    q.set_quant(w_quant=True, a_quant=True)
    return q


def test_eligible_group_convs():
    assert int8_group_conv_ineligibility(_qconv()) is None
    assert int8_group_conv_ineligibility(_qconv(groups=8)) is None  # depthwise
    assert int8_group_conv_ineligibility(_qconv(c_out=16, groups=8)) is None  # channel multiplier 2
    assert int8_group_conv_ineligibility(_qconv("per-tensor-symmetric", 8, "per-tensor-symmetric", 4)) is None
    assert int8_group_conv_ineligibility(_qconv(w_type="lsq", a_type="lsq")) is None
    for padding in (0, (1, 2), "valid", "same"):
        assert int8_group_conv_ineligibility(_qconv(padding=padding)) is None
    assert int8_group_conv_ineligibility(_qconv(kernel_size=4, padding="same", dilation=2)) is None


_reason = refusal(int8_group_conv_ineligibility, QConv2dGroupInt8.from_qconv2d)


def test_every_ineligible_group_conv_gives_its_reason():
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
    assert _reason(_qconv(groups=1)) == "groups = 1: use QConv2dInt8 / to_integer_convs"
    assert "K_g" in _reason(_qconv(c_in=2 * 1457, c_out=2, groups=2, kernel_size=(9, 10), padding=0))
    q = _qconv()
    q.fwd_kwargs["padding"] = (-1, 0)
    assert "padding" in _reason(q) and "negative" in _reason(q)
    q = _qconv()
    q.fwd_kwargs["padding"] = "full"
    assert "neither 'valid' nor 'same'" in _reason(q)
    assert "expected a QConv2d" in int8_group_conv_ineligibility(nn.Conv2d(3, 4, 3))
    assert "expected a QConv2d" in int8_group_conv_ineligibility(QLinear(nn.Linear(3, 4)))


def test_dense_conv_rules_are_unchanged():
    assert "groups = 4" in int8_conv_ineligibility(_qconv())
    assert int8_conv_ineligibility(_qconv(groups=1)) is None


def test_to_integer_group_convs_skips_dense_and_ineligible_layers():
    model = nn.Sequential(_qconv(groups=1), nn.ReLU(), _qconv(w_type="dorefa"), _qconv(a_bit=9), _qconv(groups=2, a_bit=9))
    assert to_integer_group_convs(model) == []
    assert all(isinstance(model[i], QConv2d) for i in (0, 2, 3, 4))


# ---------------------------------------------------------------------------------------------- branch coverage
def test_branch_cases_reach_every_branch():
    reached = set()
    for case in list(CASES.values()) + [BIG]:
        reached |= case_branches(case)
    assert reached == geo.REQUIRED, (geo.REQUIRED - reached, reached - geo.REQUIRED)


def test_each_branch_case_reaches_its_branch():
    expect = {"dw_vec": "load.vec", "dw_scalar_odd_w": "load.scalar", "dw_multiplier": "dw.multiplier",
              "dw_cb_partial": "dw.cb_partial", "dw_partial_tiles": "tile.partial_h", "dw_shrunk": "tile.shrunk",
              "dw_nan": "nan.rescan", "grp_c4_pad_quad": "grp.quad_partial", "grp_mb_partial": "grp.mb_partial",
              "grp_partial_tiles": "tile.partial_w", "grp_shrunk": "tile.shrunk", "grp_nan": "nan.rescan",
              "direct_dw": "path.direct", "direct_grp_nan": "path.direct", "dw_misaligned_x": "load.scalar"}
    for name, branch in expect.items():
        assert branch in case_branches(CASES[name]), (name, branch, case_branches(CASES[name]))
    assert "grid.loop" in case_branches(BIG)
    assert case_branches(CASES["grp_shrunk"]) >= {"path.grouped"}


def test_qconv2d_group_int8_module_contract():
    mod = QConv2dGroupInt8(8, 16, (3, 3), (2, 1), (1, 1, 0, 2), (1, 2), 4, torch.device("cpu"))
    assert isinstance(mod, QConv2dInt8)
    buffers = {name: (b.dtype, tuple(b.shape)) for name, b in mod.named_buffers()}
    assert buffers == {"w_q": (torch.int8, (16, 32)), "w_rowsum": (torch.int32, (16,)), "w_scale": (torch.float32, (16,)),
                       "w_zero": (torch.int32, (16,)), "scale": (torch.float32, (1,)), "zero_point": (torch.float32, (1,))}
    assert set(mod.state_dict()) == set(buffers) and "bias" in mod._buffers and mod.bias is None
    assert (mod.in_channels, mod.out_channels, mod.groups, mod.qmin, mod.qmax) == (8, 16, 4, -128, 127)
    assert (mod.kernel_size, mod.stride, mod.padding, mod.dilation) == ((3, 3), (2, 1), (1, 1, 0, 2), (1, 2))
    assert repr(mod) == ("QConv2dGroupInt8(8, 16, kernel_size=(3, 3), stride=(2, 1), padding=(1, 1, 0, 2), dilation=(1, 2), "
                         "qrange=[-128, 127], groups=4)")
    for x in (torch.zeros(1, 8, 6, 6, requires_grad=True), torch.zeros(8, 6, 6, requires_grad=True)):
        with pytest.raises(RuntimeError, match=r"^QConv2dGroupInt8 is inference-only and has no backward; .* keep QConv2d "):
            mod(x)
