"""Every launch branch of the grouped / depthwise integer-grid conv (csrc/int8_group_conv.cu): one case per branch
named by tests/int8_group_geometry.py, run through the C-ABI into a sentinel-filled output and compared, exactly, with
the per-group integer form (power-of-two scales) -- every element written, none left at the sentinel."""
import ctypes

import numpy as np
import pytest
import torch

import int8_group_geometry as geo
from gpu_util import dev, on_device, t
from int8_group_conv_ref import group_integer_form
from sparsebit_b200 import _lib, ops

F32 = np.float32
SENTINEL = 1234.5

# name -> (n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off, bias, nan)
CASES = {
    "dw_vec": (2, 16, 12, 16, 16, 16, 3, 1, 1, 1, 0, True, False),
    "dw_scalar_odd_w": (2, 12, 11, 13, 12, 12, 3, 2, 1, 1, 0, False, False),
    "dw_misaligned_x": (1, 8, 9, 16, 8, 8, 3, 1, 1, 1, 4, True, False),
    "dw_multiplier": (2, 6, 10, 12, 18, 6, 3, 1, 1, 1, 0, True, False),
    "dw_cb_partial": (1, 45, 7, 7, 45, 45, 3, 1, 1, 1, 0, True, False),
    "dw_partial_tiles": (1, 4, 45, 140, 4, 4, 3, 1, 1, 1, 0, True, False),
    "dw_shrunk": (1, 2, 300, 300, 2, 2, 3, 1, 100, 100, 0, True, False),
    "dw_nan": (2, 8, 10, 12, 8, 8, 3, 1, 1, 1, 0, True, True),
    "grp_c4_pad_quad": (2, 12, 9, 9, 9, 3, 3, 1, 1, 1, 0, True, False),
    "grp_mb_partial": (1, 160, 6, 8, 160, 2, 3, 1, 1, 1, 0, False, False),
    "grp_partial_tiles": (1, 8, 70, 130, 8, 2, 3, 1, 1, 1, 0, True, False),
    "grp_shrunk": (1, 256, 20, 20, 8, 2, 5, 1, 6, 3, 0, True, False),
    "grp_nan": (2, 32, 8, 8, 32, 4, 3, 1, 1, 1, 0, True, True),
    "direct_dw": (1, 2, 250, 250, 2, 2, 3, 1, 0, 120, 0, True, False),
    "direct_grp_nan": (1, 8, 200, 200, 4, 2, 3, 1, 2, 90, 0, True, True),
    "no_pad_valid": (1, 16, 12, 12, 32, 8, 3, 2, 0, 1, 0, True, False),
}
# reached by test_gpu_int8_group_conv.py::test_far_end_past_2_31_elements (1 x 129 x 4096 x 4096, depthwise 3x3)
BIG = (1, 129, 4096, 4096, 129, 129, 3, 1, 1, 1, 0, False, False)


def case_branches(case):
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off, bias, nan = case
    return geo.branches(n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off, bias, nan)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_branch_case(name):
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off, with_bias, with_nan = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    kh = kw = kernel
    xs, ws = F32(2.0 ** -4), (2.0 ** -rng.integers(3, 8, c_out)).astype(F32)
    x = rng.uniform(-6, 6, (n, c, h, w)).astype(F32)
    if with_nan:
        x[0, c // groups, h // 2, w // 2] = np.nan
    wt = (rng.uniform(-0.7, 0.7, (c_out, c // groups, kh, kw)) * 255 * ws[:, None, None, None]).astype(F32)
    bias = (rng.integers(-64, 64, c_out) / 8).astype(F32) if with_bias else None
    i, s = group_integer_form(x, xs, 0, -128, 127, wt, ws, np.zeros(c_out, F32), -128, 127, groups, stride, padding,
                              dilation)
    exp = (i * s[None, :, None, None]).astype(F32)
    if with_bias:
        exp = exp + bias[None, :, None, None]
    plan = geo.plan(n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off)
    assert exp.shape[2:] == (plan["oh"], plan["ow"])
    # x at a byte offset x_off from a 16-byte aligned buffer
    xv = on_device(x, x_off, unit="byte")
    assert (xv.data_ptr() - x_off) % 16 == 0
    out = torch.full(exp.shape, SENTINEL, device=dev())
    w_q, w_sum, w_nan = ops.int8_quantize_rows(t(wt.reshape(c_out, -1)), t(ws), t(np.zeros(c_out, F32)), -128, 127)
    w_zero = torch.zeros(c_out, dtype=torch.int32, device=dev())
    pt, pb, pl, pr = geo._pads(padding)
    g = _lib.Conv2dGeom(n, c, h, w, kh, kw, stride, stride, dilation, dilation, pt, pb, pl, pr)
    lib = _lib.load()
    # every tensor whose address goes to the C-ABI stays referenced until the results are read
    keep = dict(xs=t(np.array([xs], F32)), xz=t(np.zeros(1, F32)), ws=t(ws), bias=t(bias) if with_bias else None)
    rc = lib.sb200_int8_group_conv2d(xv.data_ptr(), ctypes.byref(g), groups, keep["xs"].data_ptr(), keep["xz"].data_ptr(),
                                     -128, 127, w_q.data_ptr(), w_sum.data_ptr(), keep["ws"].data_ptr(), w_zero.data_ptr(),
                                     keep["bias"].data_ptr() if with_bias else None, out.data_ptr(), c_out, None)
    assert rc == 0, lib.sb200_last_error()
    y = out.cpu().numpy()
    del keep
    assert not (y == SENTINEL).any()
    if with_nan:
        c_g, m_g = c // groups, c_out // groups
        nan_group = 1  # channel c_g is the first of group 1
        assert np.isnan(y[0, nan_group * m_g:(nan_group + 1) * m_g]).any()
        assert not np.isnan(np.delete(y, np.s_[nan_group * m_g:(nan_group + 1) * m_g], axis=1)).any()
        assert not np.isnan(y[1:]).any()
        ok = ~np.isnan(y)
        assert np.array_equal(y[ok], exp[ok])
    else:
        assert np.array_equal(y, exp)
