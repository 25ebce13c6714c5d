"""The integer-grid convolutions (csrc/int8_linear.cu, int8_sparse24.cu, int8_group_conv.cu), with and without a DoReFa
input, and the DoReFa kernels (csrc/dorefa.cu) on operands of more than 2^31 elements.

Every one of these entry points takes int64 sizes and does its own 64-bit index arithmetic, and ordinary shapes reach
2^31: a 3 x 3 conv of 128 x 64 channels at 514^2 reads 2.16e9 elements of x, a 1 x 1 conv to 520 channels of 64 x 256^2
pixels writes 2.18e9 elements of out, and the integer-grid layers call dorefa_absmax on whole activations.  Each case
below runs one entry point just past its bound and names the launch regime it must reach, as tests/int8_geometry.py,
int8_nhwc_geometry.py, int8_group_geometry.py, int8_sparse24_conv_geometry.py and weight_geometry.py restate it; the
CPU tests check the table against those plans.

  case          entry point                           shape (N, C, H = W; kernel, stride, pad)     past the bound
  conv_out      ops.int8_conv2d                       64, 16, 256; 1x1; C_out 520, bias            out (NCHW epilogue)
  conv_x        ops.int8_conv2d                       128, 64, 514; 3x3 s2 p1; C_out 24            x (lowering), q
  nhwc_out      ops.int8_conv2d_nhwc                  conv_out's, channels-last                    out (row-major)
  nhwc_x        ops.int8_conv2d_nhwc                  conv_x's, channels-last                      x (pix_org), q
  nhwc_rows     ops.int8_conv2d_nhwc (row quantizer)  128, 256, 257; 1x1; C_out 264                x, q, out
  sp24_nchw     ops.int8_sparse24_conv2d              conv_out's, 2:4 weight                       out (NCHW epilogue)
  sp24_nhwc     ops.int8_sparse24_conv2d_nhwc         conv_out's, 2:4 weight                       out (row-major)
  grp_dw        ops.int8_group_conv2d, depthwise      128, 64, 516; 3x3 p1; groups 64              x, out, grid loop
  grp_grouped   ops.int8_group_conv2d, C_g 4          128, 64, 516; 3x3 p1; groups 16              x, out, grid loop
  grp_direct    ops.int8_group_conv2d, kDirect        128, 64, 514; 3x3 p120 d120; groups 64       x, out, grid loop
  nhgrp_dw      ops.int8_group_conv2d_nhwc, kNhDw     128, 64, 516; 3x3 p1; groups 64              x, out
  nhgrp_quad    ops.int8_group_conv2d_nhwc, kNhQuad   128, 64, 516; 3x3 p1; groups 16 (M_g 4)      x, out
  nhgrp_any     ops.int8_group_conv2d_nhwc, kNhAny    128, 48, 594; 3x3 p1; groups 16 (M_g 3)      x, out
  dorefa_conv   ops.int8_conv2d, x_absmax             conv_x's                                     x, q (kDoReFa)
  dorefa_nhwc   ops.int8_conv2d_nhwc, x_absmax        conv_x's, channels-last                      x, q (kDoReFa)
  dorefa_grp    ops.int8_group_conv2d, x_absmax       grp_grouped's                                x, out
  dorefa_nhgrp  ops.int8_group_conv2d_nhwc, x_absmax  nhgrp_any's (its own launch bound)           x, out
  absmax_v4     ops.dorefa_absmax                     2^31 + 2^24 + 2 elements, aligned            x
  absmax_v1     ops.dorefa_absmax                     the same at x + 1 (scalar body)              x
  absmax_2_32   ops.dorefa_absmax                     2^32 + 3 elements                            x, and 2^32
  dorefa_fwd    ops.dorefa_forward, normalise-only    [2080, 4, 260000]                            x, out
                and per-tensor QDQ
  dorefa_fwd_pc ops.dorefa_forward, per-channel QDQ   [2080, 4, 260000], ch_axis 1                 x, out
  dorefa_bwd    ops.dorefa_backward, per-channel      [2080, 4, 260000]                            x, gy, gx

W = 516 keeps the NCHW grouped kernels on their vector loads (W % 4 = 0).  Image sizes are chosen so that a whole
image is at most 2^28 elements in every tensor, which lets the comparison slabs below be cut in whole images.
conv_out's images are 1 x 1 convs of C = 16, so its lowering takes the NHWC route in nhwc_out and sp24_nhwc, and
nhwc_rows is the 1 x 1 conv of C >= 256 that the row quantizer serves.  The DoReFa elementwise cases are cut in rows
of 260000 elements, which the per-channel runs cycle through 4 channels.

How each is checked.  Inputs come from a seeded torch.Generator on the device.  Every output starts as a NaN sentinel
(no element may keep it).  Values are planted in windows of three whole images (convs) or three whole rows (DoReFa) at
the head, around element 2^31 of every operand past its bound, and at the end:
* Convs: +inf, -inf and (but for the DoReFa convs, whose max |tanh(x)| a NaN would make NaN) a NaN in x, one of each in
  every window, and NaN / -inf at elements 2^31 + 1 and 2^31 + 5 of an x past 2^31, so that the per-row NaN flags past
  2^31 are tested.  Scales are powers of two and the bias a multiple of 2^-6, so that the fp64 truth of
  tests/int8_conv_ref.py / int8_group_conv_ref.py is exact: each window equals it bit for bit wherever the truth is
  an fp32 value, and lies within the references' bound everywhere, NaN positions included.  The DoReFa convs are held
  to the same references on ops.dorefa_forward(x, m) of the window, which the integer path equals bit for bit.
* dorefa_absmax: the largest |x| (3.0) planted past 2^31 (past 2^32 for absmax_2_32) and runners-up at the head and
  the end; the result is exactly the kernel's tanh(3.0) and the max over launches on 16-byte aligned sub-ranges of at
  most 2^28 elements.  A second run with a NaN in its place returns NaN.
* DoReFa elementwise: NaN, +-inf, +-0 and 20 in the window rows; each window equals, bit for bit, the oracle
  (oracle/qdq.py: qdq, ste_backward on the normalised value) rebuilt from the kernel's own tanhf of the window, with the
  channel of every row (row % 4), as tests/test_gpu_weight_branches.py rebuilds it.
* The whole output against launches of the same entry point on slabs of whole images (whole [4, 260000] entries for
  DoReFa) of at most 2^28 elements in every tensor, compared on the device bit for bit: convs have no cross-image work
  and DoReFa none across elements, so a slab's result must be identical.  The CPU test checks that every slab takes
  the same kernel as the whole.
Each GPU test states its device-memory need, skips when the device has less free and checks its peak against it.

These cases make three older single-window tests redundant: the far-end lowering tests of test_gpu_int8_conv.py and
test_gpu_int8_conv_nhwc.py (a C = 1 workspace past 2^31, first and last image only), and the far-end window of
test_gpu_int8_group_conv.py (one 10 x 201 window of the last channel).
"""
import contextlib
import ctypes
import dataclasses
import functools
import gc

import numpy as np
import pytest
import torch

import int8_conv_ref as cref
import int8_geometry as igeo
import int8_group_conv_ref as gref
import int8_group_geometry as grgeo
import int8_nhwc_geometry as nhgeo
import int8_sparse24_conv_geometry as scgeo
import int8_sparse24_ref as sref
import weight_geometry as wgeo
from branch_cases import C, assert_table_covers, check_reach, params
from gpu_util import bits_equal, dev, real_sm, seed_of, stream
from int8_harness import stored_rows
from oracle import qdq as oqdq
from sparsebit_b200 import _lib, ops

F32, F64 = np.float32, np.float64
B31, B32 = 1 << 31, 1 << 32
SUB = 1 << 28          # elements per slab launch at most
MARGIN = 1 << 22       # a case is past each 2^31 bound by at least this many elements
SENTINEL = 0x7FA5A5A5  # a NaN no kernel writes
GIB = 1 << 30
MAX_GIB = 28.0         # ~30 GB: the suite shares the card
WIN = 3                # images (rows) per truth window
X_Q = (F32(2.0 ** -4), F32(131.0), 0, 255)    # conv activations: unsigned 8-bit, zero point 131
XD_Q = (F32(2.0 ** -7), F32(128.0), 0, 255)   # a DoReFa input's tanh(x) / m in [-1, 1]
DOREFA_M = F32(0.9)    # the absmax the elementwise cases read: not a power of two, below max |t| = 1
D_Q = (-8, 7)          # their 4-bit grid

_CONV = dict(conv_out=dict(n=64, c=16, hw=256, kernel=1, c_out=520),
             conv_x=dict(n=128, c=64, hw=514, kernel=3, stride=2, padding=1, c_out=24),
             grp_dw=dict(n=128, c=64, hw=516, kernel=3, padding=1, c_out=64, groups=64),
             grp_grouped=dict(n=128, c=64, hw=516, kernel=3, padding=1, c_out=64, groups=16),
             nhgrp_any=dict(n=128, c=48, hw=594, kernel=3, padding=1, c_out=48, groups=16))
_DOREFA = dict(outer=2080, c=4, inner=260000)

# -------------------------------------------------------------------------------------------------- cases
CASES = [
    C("conv_out", "conv", ("gemm.kb1", "gemm.bias", "gemm.tiles", "gemm.n_partial", "low.one_chunk"),
      **_CONV["conv_out"], bounds=("out",), gib=11.0),
    C("conv_x", "conv", ("gemm.kb_lt6", "gemm.n_partial", "low.chunks", "low.stride", "low.pad_taps",
                         "low.tile_spans_images", "nchw.image_in_tile"), **_CONV["conv_x"], bounds=("x", "q"),
      gib=15.0),
    C("nhwc_out", "conv_nhwc", ("lower.nhwc", "load.vec", "gemm.kb1", "gemm.n_partial"), **_CONV["conv_out"],
      bounds=("out",), gib=11.0),
    C("nhwc_x", "conv_nhwc", ("lower.nhwc", "load.vec", "k_chunks", "pad_taps", "gemm.kb_lt6"),
      **_CONV["conv_x"], bounds=("x", "q"), gib=15.0),
    C("nhwc_rows", "conv_nhwc", ("lower.rows", "load.vec", "gemm.kb_lt6", "gemm.n_partial"), n=128, c=256, hw=257,
      kernel=1, c_out=264, bounds=("x", "q", "out"), gib=20.0),
    C("sp24_nchw", "sp24", ("gemm_one_stage", "gemm_pad_steps", "gemm_x_unsigned", "nchw_store_vec4",
                            "nchw_tile_in_image"), **_CONV["conv_out"], bounds=("out",), gib=11.0),
    C("sp24_nhwc", "sp24_nhwc", ("gemm_one_stage", "gemm_store_vec4", "gemm_partial_n", "lower.nhwc"),
      **_CONV["conv_out"], bounds=("out",), gib=11.0),
    C("grp_dw", "group", ("path.depthwise", "load.vec", "grid.loop", "pad_taps", "nan.rescan"), **_CONV["grp_dw"],
      bounds=("x", "out"), gib=19.0),
    C("grp_grouped", "group", ("path.grouped", "load.vec", "grid.loop", "pad_taps", "nan.rescan"),
      **_CONV["grp_grouped"], bounds=("x", "out"), gib=19.0),
    C("grp_direct", "group", ("path.direct", "grid.loop", "pad_taps"), n=128, c=64, hw=514, kernel=3, padding=120,
      dilation=120, c_out=64, groups=64, bounds=("x", "out"), gib=19.0),
    C("nhgrp_dw", "group_nhwc", ("path.dw", "load.vec", "store.vec", "grid.loop", "pad_taps", "nan"),
      **_CONV["grp_dw"], bounds=("x", "out"), gib=19.0),
    C("nhgrp_quad", "group_nhwc", ("path.quad", "load.vec", "store.vec", "grid.loop", "nan"), **_CONV["grp_grouped"],
      bounds=("x", "out"), gib=19.0),
    C("nhgrp_any", "group_nhwc", ("path.any", "store.vec", "grid.loop", "nan"), **_CONV["nhgrp_any"],
      bounds=("x", "out"), gib=19.0),
    C("dorefa_conv", "conv", ("gemm.kb_lt6", "low.chunks", "low.stride"), **_CONV["conv_x"], dorefa=True,
      bounds=("x", "q"), gib=15.0),
    C("dorefa_nhwc", "conv_nhwc", ("lower.nhwc", "load.vec", "k_chunks"), **_CONV["conv_x"], dorefa=True,
      bounds=("x", "q"), gib=15.0),
    C("dorefa_grp", "group", ("path.grouped", "grid.loop"), **_CONV["grp_grouped"], dorefa=True, bounds=("x", "out"),
      gib=19.0),
    C("dorefa_nhgrp", "group_nhwc", ("path.any", "grid.loop"), **_CONV["nhgrp_any"], dorefa=True,
      bounds=("x", "out"), gib=19.0),
    C("absmax_v4", "absmax", ("absmax.vec", "absmax.vec.stride", "absmax.vec.tail", "absmax.cap"),
      n=B31 + (1 << 24) + 2, x_off=0, at=B31 + 7, bounds=("x",), gib=10.0),
    C("absmax_v1", "absmax", ("absmax.scalar", "absmax.scalar.stride", "absmax.cap"), n=B31 + (1 << 24) + 2, x_off=1,
      at=B31 + 6, bounds=("x",), gib=10.0),
    C("absmax_2_32", "absmax", ("absmax.vec", "absmax.vec.stride", "absmax.vec.tail", "absmax.cap"), n=B32 + 3,
      x_off=0, at=B32 + 1, bounds=("x", "x32"), gib=18.0),
    C("dorefa_fwd", "dorefa", ("dorefa.norm.vec", "dorefa.norm.vec.stride", "dorefa.qdq.vec",
                               "dorefa.qdq.vec.stride"), **_DOREFA, runs=("norm", "qdq_pt"), bounds=("x", "out"),
      gib=19.0),
    C("dorefa_fwd_pc", "dorefa", ("dorefa.qdq.vec", "dorefa.qdq.vec.stride.partial", "dorefa.qdq.perchannel"),
      **_DOREFA, runs=("qdq_pc",), bounds=("x", "out"), gib=19.0),
    C("dorefa_bwd", "dorefa", ("dorefa.bwd.vec", "dorefa.bwd.vec.stride.partial", "dorefa.bwd.perchannel"),
      **_DOREFA, runs=("bwd_pc",), bounds=("x", "gy", "out"), gib=27.0),
]
BY_NAME = {c.name: c for c in CASES}
CONV_OPS = ("conv", "conv_nhwc", "sp24", "sp24_nhwc", "group", "group_nhwc")


def _cdiv(a, b):
    return -(-a // b)


def _pad4(case):
    return (case.get("padding", 0),) * 4


def geom(case):
    """N, C, H, W, OH, OW, K (per group), Kp, M of a conv case."""
    g = case.get
    n, c, hw, k, s, p, d = g("n"), g("c"), g("hw"), g("kernel"), g("stride", 1), g("padding", 0), g("dilation", 1)
    oh, ow = cref.out_hw(hw, hw, k, k, s, p, d)
    kk = c // g("groups", 1) * k * k
    return dict(n=n, c=c, h=hw, w=hw, oh=oh, ow=ow, k=kk, kp=igeo.padded_k(kk), m=n * oh * ow)


def units(case):
    """The units windows and slabs are cut in: images for the convs, rows for DoReFa, elements for dorefa_absmax."""
    if case.op in CONV_OPS:
        return case.get("n")
    if case.op == "dorefa":
        return case.get("outer") * case.get("c")
    return case.get("n")


def unit_elems(case):
    """Elements per unit of every tensor the case's call touches."""
    if case.op in CONV_OPS:
        g = geom(case)
        e = dict(x=g["c"] * g["h"] * g["w"], out=case.get("c_out") * g["oh"] * g["ow"])
        if case.op not in ("group", "group_nhwc"):
            e["q"] = g["oh"] * g["ow"] * g["kp"]  # the lowered workspace [M, Kp] (int8)
        return e
    if case.op == "dorefa":
        return dict(x=case.get("inner"), gy=case.get("inner"), out=case.get("inner"))
    return dict(x=1, x32=1)


def crossing(case, bound):
    """How far ``bound`` is taken: (elements, limit)."""
    return units(case) * unit_elems(case)[bound], (B32 if bound == "x32" else B31)


def bound_units(case):
    """The unit holding element 2^31 (2^32 for x32) of each operand past its bound."""
    if case.op == "absmax":
        return [case.get("at")]
    return [(B32 if b == "x32" else B31) // unit_elems(case)[b] for b in case.get("bounds")]


def regime(case, sm, u=None):
    """The launch branches one call on ``u`` units (default: the whole case) reaches, from the geometry mirrors."""
    g = case.get
    u = units(case) if u is None else u
    if case.op == "absmax":
        return wgeo.dorefa_absmax_branches(u, g("x_off"), sm)
    if case.op == "dorefa":
        out = set()
        for run in g("runs"):
            op = run.split("_")[0]
            shape = (u // g("c"), g("c"), g("inner")) if run.endswith("_pc") else (1, 1, u * g("inner"))
            out |= wgeo.chunk_branches("dorefa", op, *shape, {}, sm)
        return out
    k, s, p, d = g("kernel"), g("stride", 1), g("padding", 0), g("dilation", 1)
    hw, c, co = g("hw"), g("c"), g("c_out")
    if case.op == "conv":
        return igeo.conv_branches(u, c, hw, hw, k, k, co, s, p, d)
    if case.op == "group":
        return grgeo.branches(u, c, hw, hw, co, g("groups"), k, s, p, d, nan=not g("dorefa"))
    if case.op == "group_nhwc":
        return nhgeo.group_branches(u, c, hw, hw, co, g("groups"), k, s, p, d, nan=not g("dorefa"))
    low = nhgeo.lower_branches(u, c, hw, hw, k, s, p, d)
    m = u * geom(case)["oh"] * geom(case)["ow"]
    if case.op == "conv_nhwc":
        return low | igeo.gemm_branches(m, c * k * k, co)
    gemm = scgeo.gemm_branches(m, c * k * k, co, unsigned_x=True)
    if case.op == "sp24_nhwc":
        return low | gemm
    # the NCHW epilogue's store decisions: with P % 128 = 0 every tile lies in one image and P % 4 = 0 gives every
    # feature row the same 16-byte phase, so two images and four features show every decision the whole call makes
    pp = geom(case)["oh"] * geom(case)["ow"]
    assert pp % scgeo.TOK == 0
    return (gemm - {"gemm_store_vec4", "gemm_store_scalar"}) | scgeo.nchw_store_branches(min(m, 2 * pp), min(co, 4), pp)


def kernel_ids(case, sm, u=None):
    """The ids that name which kernel (template instance) runs: slabs must reach the same ones as the whole."""
    keep = ("path.", "load.", "lower.", "store.", "gemm.kb", "gemm_one_stage", "gemm_multi_stage", "low.one_chunk",
            "low.chunks", "absmax.vec", "absmax.scalar", "dorefa.")
    return {b for b in regime(case, sm, u) if b.startswith(keep) and
            not any(w in b for w in ("stride", "partial", "tail", "perchannel"))}


def slabs(case):
    """[a, b) unit ranges of at most SUB elements in every tensor, cut evenly so that the last is not a sliver: whole
    [C, inner] entries for DoReFa, and for dorefa_absmax sub-ranges that start 16-byte aligned in memory."""
    n = units(case)
    step = case.get("c") if case.op == "dorefa" else 4 if case.op == "absmax" else 1
    off = case.get("x_off", 0) if case.op == "absmax" else 0
    per = max(SUB // max(unit_elems(case).values()) - step + 1, 1)  # room for the rounding of the cuts below
    k = _cdiv(n, per)
    cuts = [0] + [(n * i // k + off) // step * step - off for i in range(1, k)] + [n]
    return list(zip(cuts[:-1], cuts[1:]))


def windows(case):
    """Unit ranges of WIN units: the head, around each bound unit, and the tail; overlapping ranges merged."""
    n = units(case)
    wins = sorted([(0, WIN), (n - WIN, n)] + [(max(u - WIN // 2, 0), min(u - WIN // 2 + WIN, n))
                                              for u in bound_units(case)])
    merged = [wins[0]]
    for r0, r1 in wins[1:]:
        if r0 <= merged[-1][1]:
            merged[-1] = (merged[-1][0], max(r1, merged[-1][1]))
        else:
            merged.append((r0, r1))
    return merged


def allocations(case):
    """Bytes of every device tensor the GPU test holds while its big call runs (a slab output and its workspace come on
    top, in the stated need's headroom)."""
    if case.op == "absmax":
        return dict(x=4 * (case.get("n") + case.get("x_off")))
    e = unit_elems(case)
    n = units(case)
    if case.op == "dorefa":
        return {k: 4 * n * v for k, v in e.items() if k != "gy" or "bwd_pc" in case.get("runs")}
    g = geom(case)
    out = dict(x=4 * n * e["x"], out=4 * n * e["out"], w=case.get("c_out") * (g["kp"] + 16))
    if "q" in e:
        lib = _lib.load()
        out["ws"] = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(_geom(case))))
    return out


def _geom(case, n=None):
    g = case.get
    return ops.conv2d_geometry((n or g("n"), g("c"), g("hw"), g("hw")), g("kernel"), g("stride", 1), g("padding", 0),
                               g("dilation", 1))


# -------------------------------------------------------------------------------------------------- CPU tests
def _check_case(case, sm):
    """The table's claims about one case (see test_case_table_crosses_its_bounds_and_reaches_its_regimes)."""
    for b in case.get("bounds"):
        value, limit = crossing(case, b)
        assert value > limit and (b == "x32" or value - limit >= MARGIN), (case.name, b, value, limit)
    if case.op in CONV_OPS:
        g = geom(case)
        assert g["m"] < B31 and g["k"] < igeo.MAX_K, case.name
    if case.op == "absmax":
        assert case.get("n") > case.get("at") >= max(crossing(case, b)[1] for b in case.get("bounds")), case.name
    cuts = slabs(case)
    assert cuts[0][0] == 0 and cuts[-1][1] == units(case) and all(p[1] == q[0] for p, q in zip(cuts, cuts[1:]))
    for a, b in cuts:
        assert b > a and (b - a) * max(unit_elems(case).values()) <= SUB, (case.name, a, b)
        assert kernel_ids(case, sm, b - a) == kernel_ids(case, sm), (case.name, a, b)
        if case.op == "dorefa":
            assert a % case.get("c") == 0 == (b - a) % case.get("c")
        if case.op == "absmax" and a:
            assert (a + case.get("x_off")) % 4 == 0
    held = sum(allocations(case).values()) / GIB
    assert held <= case.get("gib") <= held + 3.0 and case.get("gib") <= MAX_GIB, (case.name, held)
    for r0, r1 in windows(case):
        assert 0 <= r0 < r1 <= units(case)
    check_reach(case, regime(case, sm))


def test_case_table_crosses_its_bounds_and_reaches_its_regimes():
    """Every case is past each bound it names by more than a rounding error (4M elements; x32 past 2^32 at all) and
    stays inside the host limits (M = N OH OW < 2^31, K < 2^17); reaches the regime it names at 132 SMs (H100 SXM);
    cuts into slabs that take the same kernel and stay below 2^28 elements; states a memory need that covers its tensors
    with at most 3 GiB of headroom, within ~30 GB; and is named in the docstring."""
    sm = wgeo.SM_COUNT_H100
    for case in CASES:
        _check_case(case, sm)
    assert_table_covers(CASES, set(), lambda c: check_reach(c, regime(c, sm)), __doc__, doc_branches=False)


def test_table_check_fails_below_each_bound():
    """The table check is sensitive to the shapes: each case shrunk until one bound it names is no longer crossed (the
    conv batch, the DoReFa outer dimension, dorefa_absmax's n) fails it."""
    for case in CASES:
        for b in case.get("bounds"):
            spec = dict(case.spec)
            limit = crossing(case, b)[1]
            if case.op in CONV_OPS:
                spec["n"] = limit // unit_elems(case)[b]
            elif case.op == "dorefa":
                spec["outer"] = limit // (spec["c"] * spec["inner"])
            else:
                spec["n"] = limit
            with pytest.raises(AssertionError):
                _check_case(dataclasses.replace(case, spec=spec), wgeo.SM_COUNT_H100)


def test_windows_hold_the_bound_rows():
    """Each bound unit lies inside a window with a unit on either side of it (the last unit excepted), and the planted
    elements 2^31 + 1 and 2^31 + 5 of an x past 2^31 lie in a window."""
    for case in CASES:
        wins = windows(case)
        for u in bound_units(case):
            assert any(r0 < u < r1 - 1 or r1 == units(case) > u >= r0 for r0, r1 in wins), (case.name, u, wins)
        if case.op in CONV_OPS and "x" in case.get("bounds"):
            e = unit_elems(case)["x"]
            for p in (B31 + 1, B31 + 5):
                assert any(r0 * e <= p < r1 * e for r0, r1 in wins), (case.name, p)


# -------------------------------------------------------------------------------------------------- GPU helpers
def _frees_device_memory(test):
    """A failing far-end test would keep its tensors alive through the traceback and starve the cases after it: clear
    the finished frames of the traceback and release the cache before the failure propagates."""
    @functools.wraps(test)
    def run(*args, **kwargs):
        try:
            test(*args, **kwargs)
        except BaseException as e:
            tb = e.__traceback__.tb_next
            while tb is not None:
                try:
                    tb.tb_frame.clear()
                except RuntimeError:  # a frame still running
                    pass
                tb = tb.tb_next
            gc.collect()
            torch.cuda.empty_cache()
            raise
    return run


@contextlib.contextmanager
def _far_end(case):
    """Skip without the case's stated free memory; run it on a stream of its own, so that the ops wrappers' per-stream
    workspaces it grows are dropped afterwards; report the peak and hold it to the stated need."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    need = case.get("gib")
    free, _ = torch.cuda.mem_get_info()
    if free < need * GIB:
        pytest.skip(f"needs {need:.1f} GiB of free device memory, {free / GIB:.1f} GiB free")
    check_reach(case, regime(case, real_sm()))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    side = torch.cuda.Stream()
    try:
        with torch.cuda.stream(side):
            yield
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() / GIB
        print(f"{case.name}: peak {peak:.2f} GiB allocated, {need:.1f} GiB stated")
        assert peak <= need, (case.name, peak, need)
    finally:
        torch.cuda.synchronize()
        for key in [k for k in ops._int8_ws if k[1] == side.cuda_stream]:
            ops._int8_ws.pop(key)
        gc.collect()
        torch.cuda.empty_cache()


def _gen(case, *extra):
    return torch.Generator(device=dev()).manual_seed(seed_of(case.name, *extra))


def _sentinel(n):
    out = torch.empty(n, device=dev())
    out.view(torch.int32).fill_(SENTINEL)
    return out


def _no_sentinel(flat):
    iv = flat.view(torch.int32)
    left = sum(int((iv[a:a + SUB] == SENTINEL).sum()) for a in range(0, iv.numel(), SUB))
    assert left == 0, f"{left} outputs keep the sentinel"


def _memory_order(t):
    """The 1-D view of a contiguous NCHW or channels-last [N, C, H, W] tensor in memory order (no copy)."""
    return (t.permute(0, 2, 3, 1) if not t.is_contiguous() else t).reshape(-1)


def _same_slabs(case, big, run):
    """``run(a, b)`` returns the entry point's output for units [a, b); in memory order it must equal big's elements of
    those units bit for bit."""
    per = big.numel() // units(case)
    for a, b in slabs(case):
        got = _memory_order(run(a, b)).view(torch.int32)
        assert torch.equal(got, big[a * per:b * per].view(torch.int32)), \
            f"{case.name}: units [{a}, {b}) differ from a launch on them alone"
        del got


def _scalar(v):
    return torch.tensor([v], dtype=torch.float32, device=dev())


# -------------------------------------------------------------------------------------------------- GPU: convs
def _conv_tensor(flat, case, nhwc, n, c, h, w):
    """[n, c, h, w] over ``flat``: NCHW, or channels-last when ``nhwc``."""
    return flat.view(n, h, w, c).permute(0, 3, 1, 2) if nhwc else flat.view(n, c, h, w)


def _conv_weights(case, rng):
    """Weights on the grid with power-of-two row scales, a bias of multiples of 2^-6 and, for the 2:4 cases, the
    L1 2:4 mask: (host w, ws, wz, bias) and the device operands the entry point takes."""
    g = geom(case)
    co, kk = case.get("c_out"), case.get("kernel")
    ws = (2.0 ** -rng.integers(3, 8, co)).astype(F32)
    q = rng.integers(-100, 101, (co, g["k"])).astype(F32)
    if case.op.startswith("sp24"):
        q = np.where(sref.mask24(rng.standard_normal((co, g["k"])).astype(F32)), q, F32(0))
    w = (q * ws[:, None]).reshape(co, g["k"] // (kk * kk), kk, kk)
    wz = np.zeros(co, F32)
    bias = (rng.integers(-256, 257, co) / 64.0).astype(F32)
    w_q, w_sum, w_scale, w_zero = stored_rows(w, ws, wz, -128, 127)
    dev_ops = dict(w_q=w_q, w_sum=w_sum, w_scale=w_scale, w_zero=w_zero, bias=torch.from_numpy(bias).to(dev()))
    if case.op.startswith("sp24"):
        vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero, w_scale, g["k"])
        assert not bad.any()
        dev_ops.update(vals=vals, meta=meta, dsum=dsum)
    return (w, ws, wz, bias), dev_ops


def _conv_call(case, x, d, xq, am=None, out=None):
    """One call of the case's entry point on x; into ``out`` (flat, memory order) through the C entry point with a
    workspace of its own, else through the ops wrapper."""
    g = case.get
    s, z, qmin, qmax = xq
    kw = dict(stride=g("stride", 1), padding=g("padding", 0), dilation=g("dilation", 1))
    op, nhwc = case.op.split("_")[0], case.op.endswith("nhwc")
    if out is None:
        dk = {} if am is None else dict(x_absmax=am)
        if op == "conv":
            f = ops.int8_conv2d_nhwc if nhwc else ops.int8_conv2d
            return f(x, s, z, qmin, qmax, d["w_q"], d["w_sum"], d["w_scale"], d["w_zero"], g("kernel"), d["bias"], **kw,
                     **dk)
        if op == "sp24":
            f = ops.int8_sparse24_conv2d_nhwc if nhwc else ops.int8_sparse24_conv2d
            return f(x, s, z, qmin, qmax, d["vals"], d["meta"], d["dsum"], d["w_scale"], g("kernel"), d["bias"], **kw)
        f = ops.int8_group_conv2d_nhwc if nhwc else ops.int8_group_conv2d
        return f(x, s, z, qmin, qmax, d["w_q"], d["w_sum"], d["w_scale"], d["w_zero"], g("kernel"), g("groups"),
                 d["bias"], **kw, **dk)
    lib = _lib.load()
    geo = _geom(case)
    sfx = ("_nhwc" if nhwc else "") + ("_dorefa" if am is not None else "")
    head = [x.data_ptr(), ctypes.byref(geo)]
    amp = [am.data_ptr()] if am is not None else []
    tail = [d["bias"].data_ptr(), out.data_ptr(), g("c_out")]
    if op == "group":
        rc = getattr(lib, "sb200_int8_group_conv2d" + sfx)(*head, g("groups"), s.data_ptr(), z.data_ptr(), *amp, qmin,
                                                          qmax, d["w_q"].data_ptr(), d["w_sum"].data_ptr(),
                                                          d["w_scale"].data_ptr(), d["w_zero"].data_ptr(), *tail,
                                                          stream())
    else:
        nb = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(geo)))
        wsp = torch.empty(nb, dtype=torch.uint8, device=dev())
        if op == "sp24":
            rc = getattr(lib, "sb200_int8_sparse24_conv2d" + sfx)(*head, s.data_ptr(), z.data_ptr(), qmin, qmax,
                                                                  d["vals"].data_ptr(), d["meta"].data_ptr(),
                                                                  d["dsum"].data_ptr(), d["w_scale"].data_ptr(), *tail,
                                                                  wsp.data_ptr(), nb, stream())
        else:
            rc = getattr(lib, "sb200_int8_conv2d" + sfx)(*head, s.data_ptr(), z.data_ptr(), *amp, qmin, qmax,
                                                         d["w_q"].data_ptr(), d["w_sum"].data_ptr(),
                                                         d["w_scale"].data_ptr(), d["w_zero"].data_ptr(), *tail,
                                                         wsp.data_ptr(), nb, stream())
        torch.cuda.current_stream().synchronize()
        del wsp
    assert rc == 0, lib.sb200_last_error()
    return out


def _exact_and_within(y, t, bound, what):
    """y equals the fp64 truth wherever that is an fp32 value, and lies within its bound everywhere; NaN where it is."""
    y = np.asarray(y, F64)
    assert np.array_equal(np.isnan(y), np.isnan(t)), f"{what}: NaN positions differ from the fp64 truth"
    ok = ~np.isnan(t)
    err = np.abs(y[ok] - t[ok])
    assert np.all(err <= bound[ok]), f"{what}: error {err.max():.3g} over the 2^-21 bound"
    with np.errstate(all="ignore"):
        exact = ok & (t.astype(F32).astype(F64) == t)
    assert exact.mean() > 0.9 and np.array_equal(y[exact], t[exact]), f"{what}: not the exact truth"


@pytest.mark.gpu
@pytest.mark.parametrize("case", params([c for c in CASES if c.op in CONV_OPS]))
@_frees_device_memory
def test_conv_far_end(case):
    g = geom(case)
    nhwc, dorefa = case.op.endswith("nhwc"), bool(case.get("dorefa"))
    n, c, h, w, co = g["n"], g["c"], g["h"], g["w"], case.get("c_out")
    rng = np.random.default_rng(seed_of(case.name))
    with _far_end(case):
        xf = torch.empty(n * c * h * w, device=dev()).normal_(generator=_gen(case)).mul_(3).add_(0.5)
        x = _conv_tensor(xf, case, nhwc, n, c, h, w)
        ex = c * h * w
        wins = windows(case)
        fixed = {B31 + 1: np.nan, B31 + 5: -np.inf} if n * ex > B31 and not dorefa else {}
        for r0, r1 in wins:  # +inf in the window's first image, -inf in the middle one, NaN in the last
            hx = xf[r0 * ex:r1 * ex].cpu().numpy().reshape(r1 - r0, ex)
            hx[0, 7], hx[(r1 - r0) // 2, ex // 2] = np.inf, -np.inf
            hx[-1, ex - 9] = 30.0 if dorefa else np.nan
            for p, v in fixed.items():
                if r0 * ex <= p < r1 * ex:
                    hx.reshape(-1)[p - r0 * ex] = v
            xf[r0 * ex:r1 * ex].copy_(torch.from_numpy(hx.reshape(-1)))
        (wh, ws, wz, bias), d = _conv_weights(case, rng)
        xq = (_scalar(XD_Q[0] if dorefa else X_Q[0]), _scalar(XD_Q[1] if dorefa else X_Q[1]), 0, 255)
        am = ops.dorefa_absmax(xf) if dorefa else None
        if dorefa:
            assert float(am) == 1.0  # tanh(+-inf)
        eo = co * g["oh"] * g["ow"]
        of = _sentinel(n * eo)
        _conv_call(case, x, d, xq, am, of)
        _no_sentinel(of)
        out = _conv_tensor(of, case, nhwc, n, co, g["oh"], g["ow"])
        kw = dict(stride=case.get("stride", 1), padding=case.get("padding", 0), dilation=case.get("dilation", 1))
        qx = (float(xq[0]), float(xq[1]), 0, 255)
        for r0, r1 in wins:
            xw = x[r0:r1]
            if dorefa:
                xw = ops.dorefa_forward(xw.contiguous(), am)
            xw = xw.contiguous().cpu().numpy()
            if case.op.startswith("group"):
                t, bound = gref.truth(xw, *qx, wh, ws, wz, -128, 127, case.get("groups"), bias, **kw)
            else:
                t, bound = cref.truth(xw, *qx, wh, ws, wz, -128, 127, bias, **kw)
            y = out[r0:r1].contiguous().cpu().numpy()
            _exact_and_within(y, t, bound, f"{case.name} images [{r0}, {r1})")
            assert dorefa or np.isnan(y[-1]).any()
            del t, bound, y, xw
        _same_slabs(case, of, lambda a, b: _conv_call(case, x[a:b], d, xq, am))


# -------------------------------------------------------------------------------------------------- GPU: DoReFa
def _kernel_tanh(xw):
    """The kernel's own tanhf of a window: normalise-only with absmax = 1 (the quotient t / 1 is t)."""
    return ops.dorefa_forward(xw, torch.ones(1, device=dev())).cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("case", params([c for c in CASES if c.op == "absmax"]))
@_frees_device_memory
def test_dorefa_absmax_far_end(case):
    n, off, at = case.get("n"), case.get("x_off"), case.get("at")
    with _far_end(case):
        raw = torch.empty(n + off, device=dev()).uniform_(-2.0, 2.0, generator=_gen(case))
        x = raw[off:]
        x[0], x[n - 1], x[at] = 2.9, -2.95, 3.0
        want = ops.dorefa_absmax(torch.tensor([3.0, 0.0, 0.0, 0.0], device=dev()))
        runner_up = ops.dorefa_absmax(torch.tensor([2.95, 0.0, 0.0, 0.0], device=dev()))
        assert float(want) > float(runner_up)
        got = ops.dorefa_absmax(x)
        parts = torch.cat([ops.dorefa_absmax(x[a:b]) for a, b in slabs(case)])
        assert torch.equal(got, want), (float(got), float(want))
        assert torch.equal(got, parts.max().reshape(1)), (float(got), float(parts.max()))
        x[at] = float("nan")
        got = ops.dorefa_absmax(x)
        assert torch.isnan(got).all(), float(got)
        assert int(got.view(torch.int32)) == 0x7FC00000


def _dorefa_params(case, rng, run):
    c = case.get("c") if run.endswith("_pc") else 1
    s = rng.uniform(0.1, 0.2, c).astype(F32)
    zp = rng.choice(np.array([0.0, 1.0, -0.5, 0.5], F32), c).astype(F32)
    return s, zp


def _dorefa_run(case, run, x, gy, s, zp, out=None):
    """One launch of the run on x (flat rows of ``inner``): into ``out`` through the C entry point, else through ops."""
    inner, c = case.get("inner"), case.get("c")
    m = _scalar(DOREFA_M)
    op = run.split("_")[0]
    pc = run.endswith("_pc")
    sd, zd = (torch.from_numpy(a).to(dev()) for a in (s, zp))
    if out is None:
        xs = x.view(-1, c, inner) if pc else x
        kw = dict(ch_axis=1) if pc else {}
        if op == "norm":
            return ops.dorefa_forward(xs, m)
        if op == "qdq":
            return ops.dorefa_forward(xs, m, sd, zd, *D_Q, **kw)
        return ops.dorefa_backward(xs, m, sd, zd, gy.view(-1, c, inner), *D_Q, **kw)
    lib = _lib.load()
    shape = (x.numel() // (c * inner), c, inner) if pc else (1, 1, x.numel())
    if op == "bwd":
        rc = lib.sb200_dorefa_bwd(x.data_ptr(), m.data_ptr(), sd.data_ptr(), zd.data_ptr(), gy.data_ptr(),
                                  out.data_ptr(), *shape, *D_Q, stream())
    else:
        rc = lib.sb200_dorefa_fwd(x.data_ptr(), m.data_ptr(), sd.data_ptr() if op == "qdq" else None,
                                  zd.data_ptr() if op == "qdq" else None, out.data_ptr(), *shape, *D_Q,
                                  int(op == "qdq"), stream())
    assert rc == 0, lib.sb200_last_error()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", params([c for c in CASES if c.op == "dorefa"]))
@_frees_device_memory
def test_dorefa_far_end(case):
    inner, c = case.get("inner"), case.get("c")
    rows = units(case)
    n = rows * inner
    with _far_end(case):
        x = torch.empty(n, device=dev()).normal_(generator=_gen(case)).mul_(1.2)
        gy = torch.empty(n, device=dev()).normal_(generator=_gen(case, "gy")) if "bwd_pc" in case.get("runs") else None
        wins = windows(case)
        for r0, r1 in wins:
            hx = x[r0 * inner:r1 * inner].cpu().numpy().reshape(r1 - r0, inner)
            for i, v in enumerate((np.nan, np.inf, -np.inf, 0.0, -0.0, 20.0, -20.0)):
                hx[i % (r1 - r0), (i * 7919) % inner] = v
            x[r0 * inner:r1 * inner].copy_(torch.from_numpy(hx.reshape(-1)))
        for run in case.get("runs"):
            rng = np.random.default_rng(seed_of(case.name, run))
            s, zp = _dorefa_params(case, rng, run)
            op, pc = run.split("_")[0], run.endswith("_pc")
            out = _dorefa_run(case, run, x, gy, s, zp, _sentinel(n))
            torch.cuda.synchronize()
            _no_sentinel(out)
            for r0, r1 in wins:
                sl = slice(r0 * inner, r1 * inner)
                t = _kernel_tanh(x[sl]).reshape(r1 - r0, inner)
                ch = np.arange(r0, r1) % c if pc else np.zeros(r1 - r0, np.int64)
                with np.errstate(all="ignore"):
                    xn = (t / DOREFA_M).astype(F32)
                    if op == "norm":
                        want = xn
                    elif op == "qdq":
                        want = oqdq.qdq(xn, s[ch], zp[ch], *D_Q, ch_axis=0)
                    else:
                        g, _, _ = oqdq.ste_backward(xn, s[ch], zp[ch], gy[sl].cpu().numpy().reshape(r1 - r0, inner),
                                                    *D_Q, ch_axis=0)
                        want = ((g / DOREFA_M).astype(F32) * (F32(1) - (t * t).astype(F32)).astype(F32)).astype(F32)
                got = out[sl].cpu().numpy().reshape(r1 - r0, inner)
                assert bits_equal(got, want), f"{case.name} {run} rows [{r0}, {r1}) differ from the oracle"

            def slab(a, b, run=run, s=s, zp=zp):
                part = slice(a * inner, b * inner)
                return _dorefa_run(case, run, x[part], gy[part] if gy is not None else None, s, zp)
            _same_slabs(case, out, slab)
            del out
            gc.collect()
