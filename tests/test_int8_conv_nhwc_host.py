"""The channels-last integer-grid convs on the host: the branch cases of tests/test_gpu_int8_conv_nhwc_branches.py
together reach every launch branch tests/int8_nhwc_geometry.py names, every new C-ABI entry point rejects bad arguments
before any CUDA call (in the order and with the codes of its NCHW counterpart), and the ``_nhwc`` ops refuse tensors
that are not channels-last."""
import ctypes

import pytest
import torch

import int8_nhwc_geometry as geo
import test_gpu_int8_conv_nhwc_branches as suite
from branch_cases import assert_table_covers, check_reach
from sparsebit_b200 import SparsebitB200Error, _lib, ops
from int8_harness import E_INVALID, E_UNSUPPORTED, E_WORKSPACE, buf, check_geometry_rules, conv_geom, rejector


def test_branch_cases_reach_every_branch():
    assert_table_covers(suite.LOWER, geo.LOWER_REQUIRED, lambda c: check_reach(c, suite.reached(c)), suite.__doc__)
    assert_table_covers(suite.GROUP, geo.GROUP_REQUIRED, lambda c: check_reach(c, suite.reached(c)), suite.__doc__)


def test_geometry_restates_the_launch_decisions():
    # a stride-1 unpadded 1x1 conv of c >= 256 is the row quantizer whatever its dilation; padding, stride or a short
    # row takes the lowering
    assert geo.lower_plan(2, 256, 7, 7, 1, dilation=3)["path"] == "rows"
    assert geo.lower_plan(2, 256, 7, 7, 1, padding=1)["path"] == "nhwc"
    assert geo.lower_plan(2, 256, 7, 7, 1, stride=2)["path"] == "nhwc"
    assert geo.lower_plan(2, 255, 7, 7, 1)["path"] == "nhwc"
    assert geo.lower_plan(2, 64, 7, 7, 1)["kc"] == 64
    # chunks: 16 channels of a 3x3 (144 bytes), 128 channels of a 1x1, the whole row of the stem, 640 bytes at most
    assert geo.lower_plan(1, 512, 4, 4, 3, padding=1)["kc"] == 144
    assert geo.lower_plan(1, 512, 8, 8, 1, stride=2)["kc"] == 128
    assert geo.lower_plan(1, 3, 32, 32, 7, stride=2, padding=3)["kc"] == 160
    assert geo.lower_plan(1, 16, 12, 12, 7, padding=3)["kc"] == 640
    # vector loads need c % 4 = 0 and a 16-byte aligned x
    assert geo.lower_plan(1, 64, 8, 8, 3, x_off=4)["vec"] is False
    assert geo.lower_plan(1, 3, 8, 8, 3)["vec"] is False
    # the grouped kernel's paths and tiles
    assert geo.group_plan(2, 32, 8, 8, 32, 32, 3)["mode"] == "dw"
    assert geo.group_plan(2, 6, 8, 8, 12, 6, 3)["mode"] == "any"
    assert geo.group_plan(2, 8, 8, 8, 32, 8, 3)["mode"] == "quad"  # depthwise multiplier 4 shares the quad's channel
    p = geo.group_plan(2, 960, 7, 7, 960, 960, 3)
    assert (p["qb"], p["pix"], p["nblocks"]) == (16, 64, 15)
    assert geo.group_plan(1, 256, 12, 12, 8, 2, 10)["mode"] == "any"  # weights past 48 KB at one quad


def test_each_branch_case_reaches_its_branch():
    for case in suite.CASES:
        check_reach(case, suite.reached(case))


def test_im2col_quantize_nhwc_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    g = conv_geom()
    ok = [p, ctypes.byref(g), p, p, 0, 255, p, p, p, None]
    rejected = rejector(lib.sb200_int8_im2col_quantize_nhwc, ok)
    for i in (0, 1, 2, 3, 6, 7, 8):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    check_geometry_rules(rejected, 1)
    rejected(E_INVALID, b"wider than 8 bits", a4=-200, a5=100)
    rejected(E_INVALID, b"qmin", a4=5, a5=4)
    rejected(E_INVALID, b"neither signed", a4=-1, a5=200)
    rejected(E_INVALID, b"16-byte aligned", a6=p + 4)
    assert b"sb200_int8_im2col_quantize_nhwc" in lib.sb200_last_error()


@pytest.mark.parametrize("fn", ["sb200_int8_conv2d_nhwc", "sb200_int8_sparse24_conv2d_nhwc"])
def test_conv2d_nhwc_rejects_bad_arguments_on_the_host(fn):
    lib = _lib.load()
    keep, p = buf()
    g = conv_geom()
    ws_ok = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    # dense: (x, geom, xs, xz, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, ws, ws_bytes, stream)
    # 2:4:   (x, geom, xs, xz, qmin, qmax, vals, meta, dsum, w_scale, bias, out, c_out, ws, ws_bytes, stream)
    ok = [p, ctypes.byref(g), p, p, -128, 127, p, p, p, p, None, p, 8, p, ws_ok, None]
    rejected = rejector(getattr(lib, fn), ok)
    for i in (0, 1, 2, 3, 6, 7, 8, 9, 11, 13):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    rejected(E_INVALID, b"empty operand", a12=0)
    rejected(E_INVALID, b"too large", a12=1 << 31)
    check_geometry_rules(rejected, 1)
    rejected(E_INVALID, b"wider than 8 bits", a4=0, a5=256)
    rejected(E_INVALID, b"neither signed", a4=-129, a5=0)
    rejected(E_INVALID, b"16-byte aligned", a6=p + 1)
    if "sparse24" in fn:
        rejected(E_INVALID, b"16-byte aligned", a7=p + 4)
    rejected(E_WORKSPACE, b"workspace too small", a14=ws_ok - 1)
    rejected(E_WORKSPACE, b"workspace too small", a14=0)
    assert fn.encode() in lib.sb200_last_error()


def test_group_conv2d_nhwc_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    g = conv_geom(c=8)
    # (x, geom, groups, xs, xz, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, stream)
    ok = [p, ctypes.byref(g), 8, p, p, -128, 127, p, p, p, p, None, p, 8, None]
    rejected = rejector(lib.sb200_int8_group_conv2d_nhwc, ok)
    for i in (0, 1, 3, 4, 7, 8, 9, 10, 12):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    rejected(E_INVALID, b"empty operand", a13=0)
    rejected(E_INVALID, b"too large", a13=1 << 31)
    rejected(E_INVALID, b"sb200_int8_conv2d_nhwc", a2=1)
    rejected(E_INVALID, b"groups = 0", a2=0)
    rejected(E_INVALID, b"empty output", a1=ctypes.byref(conv_geom(c=8, kh=11)))
    rejected(E_INVALID, b"non-positive geometry", a1=ctypes.byref(conv_geom(c=8, stride_h=0)))
    rejected(E_INVALID, b"too many output pixels", a1=ctypes.byref(conv_geom(c=8, n=1 << 20, h=64, w=64)))
    rejected(E_INVALID, b"does not divide", a2=3)
    rejected(E_INVALID, b"does not divide", a13=12)
    rejected(E_INVALID, b"wider than 8 bits", a5=0, a6=256)
    rejected(E_INVALID, b"neither signed", a5=-129, a6=0)
    rejected(E_UNSUPPORTED, b"K_g < 2^17", a1=ctypes.byref(conv_geom(c=2 * ((1 << 17) // 9 + 1))), a2=2, a13=2)


def _nhwc_ops():
    x = torch.zeros(2, 8, 6, 6)
    s = torch.ones(1)
    w = torch.zeros(8, 80, dtype=torch.int8)
    i32 = torch.zeros(8, dtype=torch.int32)
    return [
        lambda x: ops.int8_im2col_quantize_nhwc(x, 3, s, s, -128, 127),
        lambda x: ops.int8_conv2d_nhwc(x, s, s, -128, 127, w, i32, s, i32, 3),
        lambda x: ops.int8_sparse24_conv2d_nhwc(x, s, s, -128, 127, w, i32, i32, s, 3),
        lambda x: ops.int8_group_conv2d_nhwc(x, s, s, -128, 127, w, i32, s, i32, 3, 2),
    ], x


def test_nhwc_ops_refuse_tensors_that_are_not_channels_last():
    calls, x = _nhwc_ops()
    for call in calls:
        with pytest.raises(SparsebitB200Error, match="expected a CUDA tensor"):  # checked before the layout
            call(x.to(memory_format=torch.channels_last))
        with pytest.raises(SparsebitB200Error, match="channels-last"):
            call(x[0])  # 3-D
        with pytest.raises(SparsebitB200Error):
            call(x)  # NCHW-contiguous CPU tensor: refused

