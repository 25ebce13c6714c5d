"""Every launch branch of the channels-last integer-grid convs: one case per branch named by tests/int8_nhwc_geometry.py,
run through the C-ABI into sentinel-filled outputs and compared with the NCHW entry point on the same values -- the
NHWC lowering (q, row sums, NaN flags) byte for byte against sb200_int8_im2col_quantize, the NHWC grouped / depthwise
conv bit for bit against sb200_int8_group_conv2d.  Every element is written, none left at the sentinel.

Lowering cases: rows_1x1, rows_1x1_odd_c, short_1x1, stem_scalar, deep_chunks, chunk_tail, chunk_split, misaligned_nan.
Grouped cases: dw_vec, dw_scalar_partial, dw_nblocks_nan, quad_vec, quad_c4_pad, quad_shrunk, any_multiplier,
any_fallback, grid_loop.

Branches: lower.rows, lower.nhwc, load.vec, load.scalar, nan, kp_tail, pad_taps, m_tail, k_chunks, k_chunk_tail,
k_chunk_split; path.dw, path.quad, path.any, bias, no_bias, store.vec, store.scalar, pix_tail, nblock_partial,
quad_partial, nblocks, grid.loop, quads.shrunk, quad.c4_pad."""
import ctypes

import pytest
import torch

import int8_nhwc_geometry as geo
from branch_cases import C, check_reach, params
from gpu_util import bits_equal, dev, seed
from sparsebit_b200 import _lib, ops

SENTINEL = 1234.5

LOWER = [
    C("rows_1x1", "lower", ["lower.rows", "load.vec"], shape=(2, 256, 9, 9), kernel=1),
    C("rows_1x1_odd_c", "lower", ["lower.rows", "load.scalar", "kp_tail"], shape=(2, 258, 5, 5), kernel=1),
    C("short_1x1", "lower", ["lower.nhwc", "load.vec", "m_tail"], shape=(2, 64, 9, 9), kernel=1),
    C("stem_scalar", "lower", ["lower.nhwc", "load.scalar", "kp_tail", "pad_taps", "m_tail"], shape=(2, 3, 40, 40),
      kernel=7, stride=2, padding=3),
    C("deep_chunks", "lower", ["lower.nhwc", "load.vec", "k_chunks"], shape=(1, 512, 4, 4), kernel=3, padding=1),
    C("chunk_tail", "lower", ["k_chunks", "k_chunk_tail"], shape=(2, 40, 9, 9), kernel=3, padding=1),
    C("chunk_split", "lower", ["k_chunk_split", "k_chunk_tail"], shape=(1, 16, 12, 12), kernel=7, padding=3),
    C("misaligned_nan", "lower", ["load.scalar"], ["nan"], shape=(2, 64, 8, 8), kernel=3, padding=1, x_off=4,
      nan=True),
]
GROUP = [
    C("dw_vec", "group", ["path.dw", "load.vec", "store.vec", "pad_taps", "bias"], shape=(2, 32, 10, 10), c_out=32,
      groups=32, kernel=3, padding=1),
    C("dw_scalar_partial", "group", ["path.dw", "load.scalar", "store.scalar", "quad_partial", "nblock_partial",
                                     "no_bias"], shape=(2, 18, 9, 9), c_out=18, groups=18, kernel=3, padding=1,
      bias=False),
    C("dw_nblocks_nan", "group", ["nblocks", "nblock_partial", "pix_tail"], ["nan"], shape=(2, 144, 8, 8), c_out=144,
      groups=144, kernel=3, stride=2, padding=1, nan=True),
    C("quad_vec", "group", ["path.quad", "load.vec"], shape=(2, 64, 9, 9), c_out=64, groups=8, kernel=3, padding=1),
    C("quad_c4_pad", "group", ["path.quad", "load.scalar", "quad.c4_pad"], ["nan"], shape=(2, 12, 9, 9), c_out=24,
      groups=2, kernel=3, padding=1, nan=True),
    C("quad_shrunk", "group", ["quads.shrunk"], shape=(1, 64, 8, 8), c_out=64, groups=2, kernel=5, padding=2),
    C("any_multiplier", "group", ["path.any"], ["nan"], shape=(2, 6, 10, 12), c_out=18, groups=6, kernel=3, padding=1,
      nan=True),
    C("any_fallback", "group", ["path.any"], shape=(1, 256, 12, 12), c_out=8, groups=2, kernel=10),
    C("grid_loop", "group", ["grid.loop"], shape=(1, 16384, 129, 128), c_out=16384, groups=16384, kernel=3, padding=1),
]
CASES = LOWER + GROUP


def reached(case):
    n, c, h, w = case.get("shape")
    kw = dict(stride=case.get("stride", 1), padding=case.get("padding", 0), dilation=case.get("dilation", 1),
              x_off=case.get("x_off", 0))
    if case.op == "lower":
        return geo.lower_branches(n, c, h, w, case.get("kernel"), nan=case.get("nan", False), **kw)
    return geo.group_branches(n, c, h, w, case.get("c_out"), case.get("groups"), case.get("kernel"),
                              bias=case.get("bias", True), nan=case.get("nan", False), **kw)


def _x_channels_last(case):
    """x as a channels-last tensor whose storage starts x_off bytes past a 16-byte boundary, values from a seeded
    generator, a NaN planted in channel 1 (group 1 of a depthwise / grouped conv) when the case asks for one."""
    n, c, h, w = case.get("shape")
    g = torch.Generator(device=dev()).manual_seed(seed(case.name))
    vals = (torch.rand(n, h, w, c, generator=g, device=dev()) - 0.5) * 12
    if case.get("nan"):
        vals[0, h // 2, w // 2, min(1, c - 1)] = float("nan")
    off = case.get("x_off", 0) // 4
    raw = torch.zeros(off + vals.numel() + 4, device=dev())
    raw[off:off + vals.numel()] = vals.reshape(-1)
    return raw[off:off + vals.numel()].view(n, h, w, c).permute(0, 3, 1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(CASES))
def test_branch_case(case):
    check_reach(case, reached(case))
    x = _x_channels_last(case)
    assert x.is_contiguous(memory_format=torch.channels_last)
    n, c, h, w = case.get("shape")
    kernel, stride, padding = case.get("kernel"), case.get("stride", 1), case.get("padding", 0)
    s = torch.tensor([2.0 ** -4], device=dev())
    z = torch.zeros(1, device=dev())
    lib = _lib.load()
    g = ops.conv2d_geometry((n, c, h, w), kernel, stride, padding, 1)
    oh, ow = ops.conv2d_output_hw(g)
    if case.op == "lower":
        q0, rs0, nan0 = ops.int8_im2col_quantize(x.contiguous(), kernel, s, z, -128, 127, stride, padding)
        q = torch.full_like(q0, 77)
        rs = torch.full_like(rs0, -5)
        nan = torch.full(nan0.shape, 9, dtype=torch.uint8, device=dev())
        rc = lib.sb200_int8_im2col_quantize_nhwc(x.data_ptr(), ctypes.byref(g), s.data_ptr(), z.data_ptr(), -128, 127,
                                                 q.data_ptr(), rs.data_ptr(), nan.data_ptr(), None)
        assert rc == 0, lib.sb200_last_error()
        torch.cuda.synchronize()
        assert torch.equal(q, q0) and torch.equal(rs, rs0) and torch.equal(nan, nan0.to(torch.uint8))
        assert bool(nan.any()) == bool(case.get("nan", False))
        return
    c_out, groups = case.get("c_out"), case.get("groups")
    kh = kernel
    gen = torch.Generator(device=dev()).manual_seed(seed(case.name) + 1)
    ws = torch.full((c_out,), 2.0 ** -6, device=dev())
    wt = (torch.rand(c_out, c // groups * kh * kh, generator=gen, device=dev()) - 0.5) * 255 * 2.0 ** -6
    w_q, w_sum, _ = ops.int8_quantize_rows(wt, ws, torch.zeros_like(ws), -128, 127)
    w_zero = torch.zeros(c_out, dtype=torch.int32, device=dev())
    bias = torch.randn(c_out, generator=gen, device=dev()) if case.get("bias", True) else None
    y0 = ops.int8_group_conv2d(x.contiguous(), s, z, -128, 127, w_q, w_sum, ws, w_zero, kernel, groups, bias, stride,
                               padding)
    out = torch.full((n, c_out, oh, ow), SENTINEL, device=dev()).to(memory_format=torch.channels_last)
    rc = lib.sb200_int8_group_conv2d_nhwc(x.data_ptr(), ctypes.byref(g), groups, s.data_ptr(), z.data_ptr(), -128, 127,
                                          w_q.data_ptr(), w_sum.data_ptr(), ws.data_ptr(), w_zero.data_ptr(),
                                          bias.data_ptr() if bias is not None else None, out.data_ptr(), c_out, None)
    assert rc == 0, lib.sb200_last_error()
    torch.cuda.synchronize()
    assert not bool((out == SENTINEL).any())
    assert bool(torch.isnan(out).any()) == bool(case.get("nan", False))
    if c * h * w < (1 << 24):
        assert bits_equal(out.cpu().numpy(), y0.cpu().numpy())
    else:
        assert torch.equal(torch.nan_to_num(out, nan=7.0), torch.nan_to_num(y0, nan=7.0))
