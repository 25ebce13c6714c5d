"""Every launch branch and epilogue path of sb200_int8_sparse24_conv2d, as tests/int8_sparse24_conv_geometry.py names
them: one case per branch, run through the C-ABI into a sentinel-filled output and compared, bit for bit, with
sb200_int8_conv2d on the same stored weight -- every element written, none left at the sentinel.

Cases: in_image (a tile inside one image, 16-byte stores, one stage, pad steps), stem_k27 (K = 27: 3x3 on 3 channels,
no second box, tiles spanning images at P = 49, the idle second warpgroup), ring (K = 4608: the ring wraps, partial M
and N), p_one (a 1x1 output, P = 1, scalar stores), unsigned_pad (unsigned activations with padding taps, a NaN
window, asymmetric padding, no bias), scalar_out (an output 4 bytes off 16-byte alignment: every store scalar),
multi_stage (three stages, a partial last tile spanning images)."""
import ctypes

import numpy as np
import pytest
import torch

import int8_sparse24_conv_geometry as geo
import int8_sparse24_ref as ref
from branch_cases import C, assert_table_covers, check_reach, params
from gpu_util import dev, on_device, seed, stream, t
from sparsebit_b200 import _lib, ops

F32 = np.float32
SENTINEL = 1234.5


def G(n, c, h, w, c_out, kh, kw, stride=1, padding=0, dilation=1):
    return dict(n=n, c=c, h=h, w=w, c_out=c_out, kh=kh, kw=kw, stride=stride, padding=padding, dilation=dilation)


CASES = [
    C("in_image", "conv", {"nchw_tile_in_image", "nchw_store_vec4", "gemm_one_stage", "gemm_pad_steps", "gemm_bias",
                           "gemm_x_signed", "conv_pad_taps"}, geom=G(2, 16, 16, 16, 128, 3, 3, 1, 1)),
    C("stem_k27", "conv", {"gemm_no_second_box", "nchw_tile_spans_images", "nchw_p_below_tile", "gemm_partial_n",
                           "gemm_idle_warpgroup"}, geom=G(4, 3, 14, 14, 64, 3, 3, 2, 1)),
    C("ring", "conv", {"gemm_ring_wraps", "gemm_multi_stage", "gemm_partial_m", "gemm_partial_n"},
      geom=G(3, 512, 4, 4, 130, 3, 3, 1, 1)),
    C("p_one", "conv", {"nchw_p_one", "nchw_store_scalar"}, geom=G(5, 32, 3, 3, 200, 3, 3)),
    C("unsigned_pad", "conv", {"gemm_x_unsigned", "conv_unsigned_pad_taps", "gemm_no_bias"}, ("(data) conv_nan_window",),
      geom=G(3, 8, 13, 13, 96, 3, 3, 2, (1, 0, 2, 1)), unsigned=True, bias=False),
    C("scalar_out", "conv", {"nchw_store_scalar"}, geom=G(2, 16, 8, 8, 64, 1, 1), out_off=4),
    C("multi_stage", "conv", {"gemm_multi_stage", "gemm_partial_m", "nchw_tile_spans_images"},
      geom=G(2, 64, 14, 14, 256, 3, 3, 1, 1)),
]


def covers(case):
    return check_reach(case, geo.branches(case.get("geom"), case.get("out_off", 0), case.get("bias", True),
                                          case.get("unsigned", False)))


def test_case_table_covers_every_branch():
    assert_table_covers(CASES, geo.REQUIRED, covers, __doc__, doc_branches=False, reject_unknown=True)


def _stored_pruned(rng, c_out, k):
    """2:4-pruned weight rows on the stored grid, per-channel power-of-two scales."""
    ws = (2.0 ** -rng.integers(3, 8, c_out)).astype(F32)
    w = (rng.uniform(-0.45, 0.45, (c_out, k)) * 255 * ws[:, None]).astype(F32)
    w = np.where(ref.mask24(rng.standard_normal((c_out, k)).astype(F32)), w, F32(0))
    z = np.zeros(c_out, F32)
    w_q, w_sum, w_nan = ops.int8_quantize_rows(t(w), t(ws), t(z), -128, 127)
    w_scale = torch.where(w_nan, torch.full_like(t(ws), float("nan")), t(ws))
    return w_q, w_sum, w_scale, t(np.zeros(c_out, np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(CASES))
def test_branch_case(case):
    lib = _lib.load()
    rng = np.random.default_rng(seed(case.name))
    geom = case.get("geom")
    g = geo.conv_plan(**geom)
    unsigned = case.get("unsigned", False)
    qmin, qmax = (0, 255) if unsigned else (-128, 127)
    w_q, w_sum, w_scale, w_zero = _stored_pruned(rng, g["N"], g["K"])
    vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero, w_scale, g["K"])
    assert not bad.any()
    x = (rng.uniform(-6, 6, (geom["n"], geom["c"], geom["h"], geom["w"])) + (8 if unsigned else 0)).astype(F32)
    if unsigned:
        x[1, 2, 5, 6] = np.nan
    xs = t(np.array([2.0 ** -4], F32))
    xz = t(np.array([131 if unsigned else 0], F32))
    bias = t(rng.standard_normal(g["N"]).astype(F32)) if case.get("bias", True) else None
    shape = (geom["n"], g["N"], g["OH"], g["OW"])
    out = on_device(np.full(shape, SENTINEL, F32), case.get("out_off", 0), unit="byte")
    gs = ops.conv2d_geometry((geom["n"], geom["c"], geom["h"], geom["w"]), (geom["kh"], geom["kw"]), geom["stride"],
                             geom["padding"], geom["dilation"])
    ws_bytes = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(gs)))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    xt = t(x)
    _lib.check(lib.sb200_int8_sparse24_conv2d(xt.data_ptr(), ctypes.byref(gs), xs.data_ptr(), xz.data_ptr(), qmin, qmax,
                                              vals.data_ptr(), meta.data_ptr(), dsum.data_ptr(), w_scale.data_ptr(),
                                              bias.data_ptr() if bias is not None else None, out.data_ptr(), g["N"],
                                              ws.data_ptr(), ws_bytes, stream()))
    dense = ops.int8_conv2d(xt, xs, xz, qmin, qmax, w_q, w_sum, w_scale, w_zero, (geom["kh"], geom["kw"]), bias,
                            geom["stride"], geom["padding"], geom["dilation"])
    y = out.cpu().numpy()
    assert not (y == F32(SENTINEL)).any()
    assert np.array_equal(y.view(np.uint32), dense.cpu().numpy().view(np.uint32))
    if unsigned:
        assert np.isnan(y).any() and not np.isnan(y).all()
