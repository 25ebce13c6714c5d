"""Every launch branch of the weight-side kernels: the one-launch multi-tensor QDQ, the structured pruning mask, the
MinMax qparams table and PACT's clamp backward (csrc/multi.cu), AdaRound (csrc/adaround.cu), DoReFa (csrc/dorefa.cu)
and the mask helpers of csrc/qdq.cu, each reached by a named case and compared with a plain reference.

tests/weight_geometry.py restates the host launch formulas; every case below asserts, with the SM count of the device it
runs on, that it reaches the branches it is listed for, and the CPU test at the bottom checks at 132 SMs (H100 SXM) that
the cases together reach every branch in REQUIRED.  Ids marked (data) depend on the values, not the launch: the case
claims them and its data plants them.  Every kernel writes into a buffer pre-filled with a finite sentinel bit pattern
(the caching allocator can hand back a block that still holds a correct result), so an element a kernel skips fails.

Multi-tensor QDQ (sb200_qdq_multi_plan / _run), bit-exact against oracle.qdq.qdq of oracle.sparse.mask_apply.  Data:
values past both clamp ends, half-integer quotients on power-of-two scales (ties), half-integer zero points, NaN, +-inf,
+-0, subnormals, +-inf under a zero mask (inf * 0 = NaN).

  branch                        source              case (why it gets there)
  multi.aligned.mask            multi.cu:41-50      multi_cap_skip2: (3,1000,12) and (1,3,1024) with masks
  multi.aligned.nomask          multi.cu:38-57      multi_cap_skip2: (1,2500,132) at x offset 4, out offset 8
  multi.aligned.two             multi.cu:39, 53-56  multi_cap_skip2: inner 132 and 1024 (more than 32 float4 per row)
  multi.aligned.half            multi.cu:39         multi_cap_skip2: inner 12 and 132 (nv % 64 != 0)
  multi.scalar.mask             multi.cu:59-63      multi_cap_skip2; multi_table_max
  multi.scalar.nomask           multi.cu:59-63      multi_cap_skip2: (1,4000,16) at x offset 1
  multi.scalar.inner_odd        multi.cu:89         multi_cap_skip2: (2,1500,7); multi_table_max (inner 5)
  multi.scalar.x_misaligned     multi.cu:89         multi_cap_skip2: (1,4000,16), inner % 4 == 0 on a misaligned base
  multi.scalar.out_misaligned   multi.cu:90         multi_cap_skip2: (5,800,20), x aligned, out offset 2
  multi.scalar.mask_misaligned  multi.cu:91         multi_cap_skip2: (2,1200,8), x and out aligned, mask offset 1
  multi.channels.cycle          multi.cu:80         multi_cap_skip2 (outer > 1 and C > 1)
  multi.cap                     multi.cu:303-304    multi_cap_skip2: 18903 rows > 8 x 132 x 8 warps
  multi.stride                  multi.cu:76         multi_cap_skip2 (3 rows per warp); multi_table_max
  multi.stride.skip1            multi.cu:77         multi_cap_skip2: the walk resumes from the previous row's tensor
  multi.stride.skip2            multi.cu:77         multi_cap_skip2 (8448-row strides over 2400..4000-row tensors)
  multi.walk.entry_skip2        multi.cu:77         multi_cap_skip2; multi_table_max (first rows deep in the table)
  multi.table_max               multi.cu:69, 220    multi_table_max: 4096 tensors of 3 rows, 32 KB of s_begin

Structured mask (sb200_mask_rows_gt), bit-exact.  Data: score == thresh, NaN, +-inf, -0 against a +0 threshold.

  rows.vec                      multi.cu:109-111    rows_vec_lane_loop: (300,144); rows_cap_stride: (9000,8)
  rows.vec.lane_loop            multi.cu:111        rows_vec_lane_loop (36 float4 per row > 32 lanes)
  rows.scalar.inner_odd         multi.cu:113        rows_inner_odd: (50,9)
  rows.scalar.misaligned        multi.cu:109, 113   rows_misaligned: (40,64) at offset 2
  rows.cap, rows.stride         multi.cu:292-294, 106   rows_cap_stride (1125 CTAs wanted > 1056)

PACT clamp backward (sb200_clamp_bwd): gx bit-exact against oracle.qdq.clamp_backward, g_hi / g_lo within the bound of
_clamp_sum_bound against fp64 sums, two runs bit-identical.  Data: x exactly on lo and hi and one ulp outside, NaN,
+-inf, +-0.

  clamp.vec                     multi.cu:175-181    clamp_vec_stride_tail: n = 1000003; clamp_flush; clamp_tiny_tail
  clamp.vec.stride              multi.cu:175        clamp_vec_stride_tail (2 vector iterations); clamp_flush (67)
  clamp.vec.tail                multi.cu:182        clamp_vec_stride_tail; clamp_flush; clamp_tiny_tail: n = 13
  clamp.vec.flush               multi.cu:180        clamp_flush: n = 36000002, 67 vector iterations per thread
  clamp.vec.flush_then_more     multi.cu:180-183    clamp_flush (3 iterations after the flush)
  clamp.cap                     multi.cu:205        clamp_vec_stride_tail, clamp_flush (> 4 x 132 CTAs wanted)
  clamp.scalar                  multi.cu:182        clamp_x_off1, clamp_gy_off2_null_hi, clamp_gx_off3_null_lo
  clamp.scalar.x_misaligned     multi.cu:173        clamp_x_off1: n = 50001 at x offset 1
  clamp.scalar.gy_misaligned    multi.cu:173        clamp_gy_off2_null_hi: n = 4099 at gy offset 2
  clamp.scalar.gx_misaligned    multi.cu:173        clamp_gx_off3_null_lo: n = 70000 at gx offset 3
  clamp.scalar.stride           multi.cu:182        clamp_x_off1 (4 iterations), clamp_gy_off2_null_hi (5)
  clamp.null_hi, clamp.null_lo  multi.cu:200-201    clamp_gy_off2_null_hi, clamp_gx_off3_null_lo
  test_clamp_workspace_contract: the size query is pure, one byte less is SB200_E_WORKSPACE and launches nothing.

AdaRound (sb200_adaround_fwd / _bwd / _init).  Hard rounding bit-exact against oracle.qdq.adaround_forward; soft, backward
and init must equal the kernel's fp32 op chain (_ada_chain) evaluated at one of the values CUDA's documented error bound
allows for its expf (2 ulp) or logf (1 ulp), and match the oracle's NaN / inf pattern.  Data: v = +-0 (hard rounding's
>= 0), v far beyond the sigmoid's saturation, NaN and +-inf in x and v, subnormals, x on grid points.

  ada.<op>.vec, .vec.stride.partial, .perchannel   adaround.cu:102-119, 96   ada_hard_vec, ada_soft_vec, ada_bwd_vec,
                                                    ada_init_vec: (2,300,1500), 1200 chunks > 1056 CTAs, 476-element last
                                                    chunks, row % 300 wraps
  ada.hard.scalar.x_misaligned  adaround.cu:120-134 ada_hard_x_off1: (1,1,5000) per-tensor at x offset 1
  ada.hard.scalar.inner_odd     adaround.cu:145     ada_hard_inner_odd: (3,5,999)
  ada.soft.scalar.v_misaligned  adaround.cu:145     ada_soft_v_off2_stride: (4,300,1020) at v offset 2
  ada.soft.scalar.stride        adaround.cu:96      ada_soft_v_off2_stride (1200 chunks)
  ada.bwd.scalar.gy_misaligned  adaround.cu:146     ada_bwd_gy_off1: (2,3,2048) at gy offset 1
  ada.init.scalar.out_misaligned  adaround.cu:145   ada_init_out_off3: (1,7,1028) at out offset 3
  ada.<op>.scalar               adaround.cu:120-134 the four cases above

DoReFa (sb200_dorefa_absmax / _fwd / _bwd), bit-exact without numpy's tanh: a normalise-only run with absmax = 1.0 gives
the kernel's own tanhf(x) = t (checked against fp64 tanh within tanhf's documented 2 ulp); from t every output is rebuilt
in numpy fp32 one rounding per op as dorefa.cu:54-62 does.

  dorefa.<op>.vec, .vec.stride.partial, .perchannel  dorefa.cu:83-92, 74   dorefa_norm_vec, dorefa_qdq_vec,
                                                    dorefa_bwd_vec: (2,300,1500)
  dorefa.norm.scalar.x_misaligned   dorefa.cu:110   dorefa_norm_x_off1: (1,1,10000) at x offset 1
  dorefa.qdq.scalar.out_misaligned  dorefa.cu:110   dorefa_qdq_out_off2: (3,4,1000) at out offset 2
  dorefa.qdq.scalar.inner_odd       dorefa.cu:110   dorefa_qdq_inner_odd: (3,4,999)
  dorefa.bwd.scalar.gy_misaligned   dorefa.cu:110   dorefa_bwd_gy_off3: (2,5,2000) at gy offset 3
  dorefa.<op>.scalar                dorefa.cu:93-99 the four cases above
  absmax.vec, absmax.vec.tail   dorefa.cu:32-36     absmax_vec_tail: n = 10003, the largest |tanh| in the last 3
  absmax.vec.stride, absmax.cap dorefa.cu:32, 129-131   absmax_vec_stride: n = 5000001 (1056 CTAs)
  absmax.scalar, absmax.scalar.stride   dorefa.cu:36    absmax_scalar_stride: n = 30001 at x offset 1
  absmax.nan (data)             dorefa.cu:29        absmax_nan: one NaN among 4096

qdq.cu mask helpers, bit-exact.  Data: |w| == thresh, NaN, +-inf, +-0, subnormals; inf * 0 in the float mask.

  gt.vec, gt.vec.stride, gt.vec.tail, gt.cap   qdq.cu:603-610, 505-510   gt_vec_stride_tail: n = 3000003
  gt.scalar.w_misaligned, gt.scalar.stride     qdq.cu:601, 612           gt_w_off1: n = 10001 at w offset 1
  gt.scalar.mask_misaligned     qdq.cu:601          gt_mask_off1: n = 10000 at mask offset 1
  mulf.cap, mulf.stride         qdq.cu:620, 702     mulf_cap_stride: n = 600001
  mulf.misaligned               qdq.cu:616-622      mulf_misaligned: n = 5003 at offsets 1 / 2 / 3

MinMax qparams (sb200_minmax_qparams_multi) bit-exact against oracle.observers.calc_qparams_with_minmax fed with the
decoded state; min / max against the decoded state.

  qparams.chan_loop, qparams.one_pass   multi.cu:137    qp_mixed_table: 300 and 129 channels; 7 and 1
  qparams.sym, qparams.asym, qparams.multi_entry, qparams.mixed_table   multi.cu:141-147   qp_mixed_table
  qparams.data.* (data)         multi.cu:138-147    qp_mixed_table: a never-observed channel, a NaN state, a -inf / +inf
                                                    state, states under the 1e-6 floor, zero points on a .5 tie, all
                                                    beyond channel 128 too

test_multi_equals_per_tensor_calls runs multi_cap_skip2 against the per-tensor qdq_perchannel /
mask_apply_qdq_perchannel entry points, and test_multi_plan_count_limits checks that a plan takes 4096 tensors and
refuses 4097.
"""
import ctypes
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import branch_cases
import weight_geometry as geo
from branch_cases import assert_table_covers, check_reach, fs, params
from gpu_util import bits_equal, dev, on_device, real_sm, seed, stream
from oracle import observers as oobs
from oracle import qdq as oqdq
from oracle import sparse as osp
from sparsebit_b200 import _lib, ops

F32 = np.float32
F64 = np.float64
U32 = np.uint32
SENTINEL = np.array([0x4B5A5A5A], U32).view(F32)[0]  # 14310490.0: finite, so "unwritten" never reads as NaN == NaN
SENTINEL_U8 = 0xA5
E_INVALID, E_WORKSPACE = -1, -4
STRETCH, GAMMA = F32(1.1 - (-0.1)), F32(-0.1)  # adaround.cu:22-23


# -------------------------------------------------------------------------------------------------- helpers
def sentinel(n, offset=0, dtype=torch.float32):
    """`n` elements `offset` into a fresh allocation, filled (with the slack around them) with the sentinel."""
    buf = torch.empty(n + offset + 4, dtype=dtype, device=dev())
    if dtype == torch.uint8:
        buf.fill_(SENTINEL_U8)
    else:
        buf.fill_(float(SENTINEL))
    return buf[offset:offset + n]


def host(t):
    return t.cpu().numpy()


def subnormals(rng, n):
    bits = rng.integers(1, 1 << 23, n, dtype=np.int64).astype(U32)
    bits |= (rng.random(n) < 0.5).astype(U32) << U32(31)
    return bits.view(F32)


def plant(rng, x, specials, frac=0.01):
    """Overwrite a random `frac` of the flat array x (in place) with the given values, cycling."""
    flat = x.reshape(-1)
    k = max(len(specials), int(flat.size * frac))
    idx = rng.choice(flat.size, size=min(k, flat.size), replace=False)
    flat[idx] = np.resize(np.asarray(specials, F32), idx.size)
    return idx


NONFINITE = [np.nan, np.inf, -np.inf, 0.0, -0.0]


def same(a, b):
    """Elementwise: equal values (+0 == -0) or both NaN."""
    return (a == b) | (np.isnan(a) & np.isnan(b))


def ulp_steps(r, k):
    """The fp32 values within k representable steps of r (total order through +-0, clamped at +-inf; NaN stays)."""
    r = np.asarray(r, F32)
    b = r.view(np.int32).astype(np.int64)
    key = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    out = []
    for j in range(-k, k + 1):
        kk = np.clip(key + j, -0x7F800000, 0x7F800000)
        bits = np.where(kk < 0, (-kk) | 0x80000000, kk).astype(np.uint32)
        out.append(np.where(np.isnan(r), r, bits.view(F32)))
    return out


# -------------------------------------------------------------------------------------------------- cases
@dataclass(frozen=True)
class Case(branch_cases.Case):
    """op: multi | rows | clamp | ada | dorefa | absmax | gt | mulf | qp; spec: a tuple, laid out per op below."""

    def branches(self, sm):
        s = self.spec
        if self.op == "multi":
            return geo.multi_branches([t[:6] for t in s], sm) | ({"multi.table_max"} if len(s) == geo.MULTI_MAX_TENSORS else set())
        if self.op == "rows":
            return geo.mask_rows_gt_branches(*s, sm)
        if self.op == "clamp":
            return geo.clamp_bwd_branches(*s[:4], sm, null_hi=s[4], null_lo=s[5])
        if self.op in ("ada", "dorefa"):
            kind, outer, c, inner, offs = s
            return geo.chunk_branches(self.op, kind, outer, c, inner, dict(offs), sm)
        if self.op == "absmax":
            return geo.dorefa_absmax_branches(*s, sm)
        if self.op == "gt":
            return geo.mask_gt_branches(*s, sm)
        if self.op == "mulf":
            n, w_off, m_off, o_off = s
            return geo.mask_apply_f32_branches(n, dict(w=w_off, m=m_off, out=o_off), sm)
        return geo.qparams_branches([(c, sym) for c, sym, _, _ in s])


MULTI_CAP_SKIP2 = (  # (outer, C, inner, x_off, out_off, mask_off or None, qmin, qmax)
    (3, 1000, 12, 0, 0, 0, -128, 127),
    (1, 2500, 132, 4, 8, None, -8, 7),
    (2, 1500, 7, 0, 0, 0, 0, 15),
    (1, 4000, 16, 1, 0, None, -128, 127),
    (5, 800, 20, 0, 2, 0, -128, 127),
    (2, 1200, 8, 0, 0, 1, 0, 255),
    (1, 3, 1024, 0, 0, 0, -128, 127),
)
MULTI_TABLE_MAX = tuple((1, 3, 5, i % 4, (i // 4) % 4, (i % 3) if i % 2 == 0 else None, -8, 7) for i in range(4096))
MULTI_DATA = fs("multi.data.ties", "multi.data.clamp", "multi.data.nonfinite", "multi.data.inf_times_zero")
MULTI_CASES = [
    Case("multi_cap_skip2", "multi", MULTI_CAP_SKIP2,
         fs("multi.aligned.mask", "multi.aligned.nomask", "multi.aligned.two", "multi.aligned.half", "multi.scalar.mask",
            "multi.scalar.nomask", "multi.scalar.inner_odd", "multi.scalar.x_misaligned", "multi.scalar.out_misaligned",
            "multi.scalar.mask_misaligned", "multi.channels.cycle", "multi.cap", "multi.stride", "multi.stride.skip1",
            "multi.stride.skip2", "multi.walk.entry_skip2", *MULTI_DATA), MULTI_DATA),
    Case("multi_table_max", "multi", MULTI_TABLE_MAX,
         fs("multi.table_max", "multi.scalar.mask", "multi.scalar.inner_odd", "multi.stride.skip2", "multi.walk.entry_skip2")),
]
ROWS_DATA = fs("rows.data.score_eq_thresh", "rows.data.nonfinite")
ROWS_CASES = [  # (rows, inner, mask offset)
    Case("rows_vec_lane_loop", "rows", (300, 144, 0), fs("rows.vec", "rows.vec.lane_loop", *ROWS_DATA), ROWS_DATA),
    Case("rows_cap_stride", "rows", (9000, 8, 0), fs("rows.vec", "rows.cap", "rows.stride")),
    Case("rows_inner_odd", "rows", (50, 9, 0), fs("rows.scalar.inner_odd", *ROWS_DATA), ROWS_DATA),
    Case("rows_misaligned", "rows", (40, 64, 2), fs("rows.scalar.misaligned")),
]
CLAMP_DATA = fs("clamp.data.on_bounds", "clamp.data.nonfinite")
CLAMP_CASES = [  # (n, x_off, gy_off, gx_off, null g_hi, null g_lo)
    Case("clamp_vec_stride_tail", "clamp", (1_000_003, 0, 0, 0, False, False),
         fs("clamp.vec", "clamp.vec.stride", "clamp.vec.tail", "clamp.cap", *CLAMP_DATA), CLAMP_DATA),
    Case("clamp_flush", "clamp", (36_000_002, 0, 0, 0, False, False),
         fs("clamp.vec.flush", "clamp.vec.flush_then_more", "clamp.vec.tail", "clamp.cap")),
    Case("clamp_x_off1", "clamp", (50_001, 1, 0, 0, False, False),
         fs("clamp.scalar", "clamp.scalar.x_misaligned", "clamp.scalar.stride", *CLAMP_DATA), CLAMP_DATA),
    Case("clamp_gy_off2_null_hi", "clamp", (4_099, 0, 2, 0, True, False),
         fs("clamp.scalar.gy_misaligned", "clamp.scalar.stride", "clamp.null_hi")),
    Case("clamp_gx_off3_null_lo", "clamp", (70_000, 0, 0, 3, False, True), fs("clamp.scalar.gx_misaligned", "clamp.null_lo")),
    Case("clamp_tiny_tail", "clamp", (13, 0, 0, 0, False, False), fs("clamp.vec", "clamp.vec.tail")),
]
ADA_DATA = fs("ada.data.v_signed_zero", "ada.data.nonfinite")
ADA_CASES = [Case(f"ada_{op}_vec", "ada", (op, 2, 300, 1500, ()),
                  fs(f"ada.{op}.vec", f"ada.{op}.vec.stride.partial", f"ada.{op}.perchannel", *ADA_DATA), ADA_DATA)
             for op in geo.ADA_OPS] + [
    Case("ada_hard_x_off1", "ada", ("hard", 1, 1, 5000, (("x", 1),)), fs("ada.hard.scalar", "ada.hard.scalar.x_misaligned")),
    Case("ada_hard_inner_odd", "ada", ("hard", 3, 5, 999, ()), fs("ada.hard.scalar.inner_odd")),
    Case("ada_soft_v_off2_stride", "ada", ("soft", 4, 300, 1020, (("v", 2),)),
         fs("ada.soft.scalar", "ada.soft.scalar.v_misaligned", "ada.soft.scalar.stride")),
    Case("ada_bwd_gy_off1", "ada", ("bwd", 2, 3, 2048, (("gy", 1),)), fs("ada.bwd.scalar", "ada.bwd.scalar.gy_misaligned")),
    Case("ada_init_out_off3", "ada", ("init", 1, 7, 1028, (("out", 3),)), fs("ada.init.scalar", "ada.init.scalar.out_misaligned")),
]
DOREFA_CASES = [Case(f"dorefa_{op}_vec", "dorefa", (op, 2, 300, 1500, ()),
                     fs(f"dorefa.{op}.vec", f"dorefa.{op}.vec.stride.partial", f"dorefa.{op}.perchannel"))
                for op in geo.DOREFA_OPS] + [
    Case("dorefa_norm_x_off1", "dorefa", ("norm", 1, 1, 10_000, (("x", 1),)),
         fs("dorefa.norm.scalar", "dorefa.norm.scalar.x_misaligned")),
    Case("dorefa_qdq_out_off2", "dorefa", ("qdq", 3, 4, 1000, (("out", 2),)),
         fs("dorefa.qdq.scalar", "dorefa.qdq.scalar.out_misaligned")),
    Case("dorefa_qdq_inner_odd", "dorefa", ("qdq", 3, 4, 999, ()), fs("dorefa.qdq.scalar.inner_odd")),
    Case("dorefa_bwd_gy_off3", "dorefa", ("bwd", 2, 5, 2000, (("gy", 3),)),
         fs("dorefa.bwd.scalar", "dorefa.bwd.scalar.gy_misaligned")),
]
ABSMAX_CASES = [  # (n, x_off)
    Case("absmax_vec_tail", "absmax", (10_003, 0), fs("absmax.vec", "absmax.vec.tail")),
    Case("absmax_vec_stride", "absmax", (5_000_001, 0), fs("absmax.vec.stride", "absmax.cap", "absmax.vec.tail")),
    Case("absmax_scalar_stride", "absmax", (30_001, 1), fs("absmax.scalar", "absmax.scalar.stride")),
    Case("absmax_nan", "absmax", (4_096, 0), fs("absmax.vec", "absmax.nan"), fs("absmax.nan")),
]
GT_DATA = fs("gt.data.on_thresh", "gt.data.nonfinite")
GT_CASES = [  # (n, w_off, mask_off)
    Case("gt_vec_stride_tail", "gt", (3_000_003, 0, 0), fs("gt.vec", "gt.vec.stride", "gt.vec.tail", "gt.cap", *GT_DATA), GT_DATA),
    Case("gt_w_off1", "gt", (10_001, 1, 0), fs("gt.scalar.w_misaligned", "gt.scalar.stride", *GT_DATA), GT_DATA),
    Case("gt_mask_off1", "gt", (10_000, 0, 1), fs("gt.scalar.mask_misaligned", *GT_DATA), GT_DATA),
]
MULF_CASES = [  # (n, w_off, mask_off, out_off)
    Case("mulf_cap_stride", "mulf", (600_001, 0, 0, 0), fs("mulf.cap", "mulf.stride", "mulf.data.inf_times_zero"),
         fs("mulf.data.inf_times_zero")),
    Case("mulf_misaligned", "mulf", (5_003, 1, 2, 3), fs("mulf.misaligned", "mulf.stride")),
]
QP_DATA = fs("qparams.data.empty", "qparams.data.nan", "qparams.data.inf", "qparams.data.floor", "qparams.data.zp_tie")
QP_CASES = [  # ((channels, symmetric, qmin, qmax), ...)
    Case("qp_mixed_table", "qp", ((300, False, 0, 255), (7, True, -128, 127), (129, True, -8, 7), (1, False, -128, 127)),
         fs("qparams.chan_loop", "qparams.one_pass", "qparams.sym", "qparams.asym", "qparams.multi_entry",
            "qparams.mixed_table", *QP_DATA), QP_DATA),
]
ALL_CASES = (MULTI_CASES + ROWS_CASES + CLAMP_CASES + ADA_CASES + DOREFA_CASES + ABSMAX_CASES + GT_CASES + MULF_CASES
             + QP_CASES)

REQUIRED = {
    "multi.aligned.mask", "multi.aligned.nomask", "multi.aligned.two", "multi.aligned.half", "multi.scalar.mask",
    "multi.scalar.nomask", "multi.scalar.inner_odd", "multi.scalar.x_misaligned", "multi.scalar.out_misaligned",
    "multi.scalar.mask_misaligned", "multi.channels.cycle", "multi.cap", "multi.stride", "multi.stride.skip1",
    "multi.stride.skip2", "multi.walk.entry_skip2", "multi.table_max",
    "rows.vec", "rows.vec.lane_loop", "rows.scalar.inner_odd", "rows.scalar.misaligned", "rows.cap", "rows.stride",
    "clamp.vec", "clamp.vec.stride", "clamp.vec.tail", "clamp.vec.flush", "clamp.vec.flush_then_more", "clamp.cap",
    "clamp.scalar", "clamp.scalar.x_misaligned", "clamp.scalar.gy_misaligned", "clamp.scalar.gx_misaligned",
    "clamp.scalar.stride", "clamp.null_hi", "clamp.null_lo",
    *[f"ada.{op}.{b}" for op in geo.ADA_OPS for b in ("vec", "vec.stride.partial", "perchannel", "scalar")],
    "ada.hard.scalar.x_misaligned", "ada.hard.scalar.inner_odd", "ada.soft.scalar.v_misaligned", "ada.soft.scalar.stride",
    "ada.bwd.scalar.gy_misaligned", "ada.init.scalar.out_misaligned",
    *[f"dorefa.{op}.{b}" for op in geo.DOREFA_OPS for b in ("vec", "vec.stride.partial", "perchannel", "scalar")],
    "dorefa.norm.scalar.x_misaligned", "dorefa.qdq.scalar.out_misaligned", "dorefa.qdq.scalar.inner_odd",
    "dorefa.bwd.scalar.gy_misaligned",
    "absmax.vec", "absmax.vec.tail", "absmax.vec.stride", "absmax.cap", "absmax.scalar", "absmax.scalar.stride", "absmax.nan",
    "gt.vec", "gt.vec.stride", "gt.vec.tail", "gt.cap", "gt.scalar.w_misaligned", "gt.scalar.mask_misaligned",
    "gt.scalar.stride", "mulf.cap", "mulf.stride", "mulf.misaligned",
    "qparams.chan_loop", "qparams.one_pass", "qparams.sym", "qparams.asym", "qparams.multi_entry", "qparams.mixed_table",
}
DOC_ALIASES = {  # ids the docstring names through the row "<family>.<op>.vec, .vec.stride.partial, .perchannel"
    f"{fam}.{op}.{b}": f"{fam}.<op>.{'scalar' if b == 'scalar' else 'vec'}"
    for fam, ops_ in (("ada", geo.ADA_OPS), ("dorefa", geo.DOREFA_OPS)) for op in ops_
    for b in ("vec", "vec.stride.partial", "perchannel", "scalar")
}


# -------------------------------------------------------------------------------------------------- CPU tests
def test_case_table_covers_every_branch():
    assert_table_covers(ALL_CASES, REQUIRED, lambda c: check_reach(c, c.branches(geo.SM_COUNT_H100)), __doc__,
                        doc_alias=lambda b: DOC_ALIASES.get(b, b))


def test_geometry_matches_documented_launches():
    """Spot values of the restated formulas, worked by hand from the .cu files at 132 SMs."""
    sm = geo.SM_COUNT_H100
    # multi: ceil(rows / 8) CTAs, capped at 8 x 132 = 1056; 8448 warps
    assert geo.multi_launch(1557, sm) == dict(ctas=195, capped=False, warps=1560, rows_per_warp=1)
    assert geo.multi_launch(18903, sm) == dict(ctas=1056, capped=True, warps=8448, rows_per_warp=3)
    assert geo.multi_launch(8448, sm)["capped"] is False and geo.multi_launch(8449, sm)["capped"] is True
    assert geo.multi_row_aligned(12, 0, 0, 0) and geo.multi_row_aligned(12, 4, 8, None)
    assert not geo.multi_row_aligned(16, 1, 0, None) and not geo.multi_row_aligned(20, 0, 2, 0)
    assert not geo.multi_row_aligned(8, 0, 0, 1) and not geo.multi_row_aligned(7, 0, 0, 0)
    # the old one-launch test: 8 tensors, 1557 rows, no warp takes a second row
    assert "multi.stride" not in geo.multi_branches([(1, 1557, 4, 0, 0, None)], sm)
    # clamp: ceil(floor(n / 4) / 256) CTAs, capped at 4 x 132 = 528 (135168 threads)
    assert geo.clamp_bwd_ctas(12_288, sm) == 12 and geo.clamp_bwd_ctas(3, sm) == 1 and geo.clamp_bwd_ctas(10**9, sm) == 528
    g = geo.clamp_bwd_geometry(36_000_002, 0, 0, 0, sm)
    assert (g["nv"], g["nt"], g["vec_iters"], g["tail"], g["fp32_terms"]) == (9_000_000, 135_168, 67, 2, 257)
    assert geo.clamp_bwd_geometry(34_603_008, 0, 0, 0, sm)["vec_iters"] == 64  # 64 x 135168 x 4: exactly one flush
    g = geo.clamp_bwd_geometry(50_001, 1, 0, 0, sm)
    assert (g["ctas"], g["nv"], g["tail_iters"]) == (49, 0, 4)
    assert geo.clamp_bwd_workspace_bytes(12_288, sm) == 12 * 16 and geo.clamp_bwd_workspace_bytes(0, sm) == 0
    # AdaRound / DoReFa chunks: rows x ceil(inner / 1024), grid capped at 8 x 132 = 1056
    assert geo.chunk_launch(2, 300, 1500, sm) == dict(rows=600, chunks=1200, grid=1056, iters=2)
    assert geo.chunk_launch(1, 1, 1 << 18, sm) == dict(rows=1, chunks=256, grid=256, iters=1)
    assert geo.chunk_vec("ada", "init", 1024, {"v": 1}) == (True, None)  # init reads no v
    assert geo.chunk_vec("ada", "hard", 1024, {"v": 1}) == (False, "v_misaligned")
    assert geo.chunk_vec("dorefa", "qdq", 1024, {"gy": 1}) == (True, None)  # only the backward reads gy
    assert geo.chunk_vec("dorefa", "bwd", 1024, {"gy": 1}) == (False, "gy_misaligned")
    assert geo.chunk_vec("ada", "bwd", 1022, {}) == (False, "inner_odd")
    # the old DoReFa tests: 9408 elements per tensor is 10 chunks, one pass
    assert geo.chunk_launch(1, 1, 9408, sm)["iters"] == 1
    # absmax: floor(n / 4) / 256 rounded up, plus one, capped at 1056
    assert geo.dorefa_absmax_launch(10_003, 0, sm)["grid"] == 11 and geo.dorefa_absmax_launch(5_000_001, 0, sm)["grid"] == 1056
    assert geo.dorefa_absmax_launch(30_001, 1, sm)["nt"] == 31 * 256
    # grid_for: ceil(nvec / 1024), capped at 4 x 132 = 528
    assert geo.grid_for(750_000, sm) == (528, True) and geo.grid_for(2_500, sm) == (3, False) and geo.grid_for(0, sm) == (1, False)
    assert geo.grid_for(600_001, sm) == (528, True) and geo.grid_for(540_672, sm) == (528, False)
    # qparams: 128 threads per entry
    assert geo.qparams_branches([(128, True)]) == {"qparams.sym", "qparams.one_pass"}
    assert "qparams.chan_loop" in geo.qparams_branches([(129, False)])


# -------------------------------------------------------------------------------------------------- multi-tensor QDQ
def _multi_tensor_data(rng, outer, c, inner, qmin, qmax, with_mask):
    """x [outer, C, inner] around the channel's grid with ties, clamp overshoot and non-finite values; channel scales
    alternate powers of two (exact ties) and arbitrary values; zero points include half-integers."""
    s = np.where(np.arange(c) % 2 == 0, 2.0 ** -(3 + np.arange(c) % 5), rng.uniform(0.01, 0.1, c)).astype(F32)
    zp = rng.choice(np.array([0.0, 2.5, 3.5, -1.5, 1.0], F32), c).astype(F32)
    zp = np.clip(zp, qmin, qmax).astype(F32)
    v = rng.uniform(qmin - 12, qmax + 12, (outer, c, inner)).astype(F32)
    v = np.where(rng.random(v.shape) < 0.15, np.rint(v) + F32(0.5), v).astype(F32)  # quotients on a .5 tie
    x = (v - zp[None, :, None]) * s[None, :, None]
    x = x.astype(F32)
    plant(rng, x, NONFINITE + list(subnormals(rng, 4)), frac=0.01)
    mask = None
    if with_mask:
        mask = (rng.random(x.shape) < 0.7).astype(np.uint8)
        flat, mflat = x.reshape(-1), mask.reshape(-1)
        off = np.flatnonzero(mflat == 0)[:8]
        flat[off] = np.resize(np.array([np.inf, -np.inf], F32), off.size)  # inf * 0 = NaN
    return x, s, zp, mask


def _pack(arrays_offs, dtype):
    """One device buffer holding every array at its offset class: array i starts on a 16-byte boundary plus off_i."""
    cursor, starts = 0, []
    for a, off in arrays_offs:
        cursor = (cursor + 3) // 4 * 4 + off % 4
        starts.append(cursor)
        cursor += a.size
    buf = torch.empty(cursor + 4, dtype=dtype, device=dev())
    staged = np.zeros(cursor + 4, dtype=torch.empty(0, dtype=dtype).numpy().dtype)
    for (a, _), st in zip(arrays_offs, starts):
        staged[st:st + a.size] = a.reshape(-1)
    buf.copy_(torch.from_numpy(staged))
    return buf, starts


def _multi_setup(spec, rng):
    data = [_multi_tensor_data(rng, o, c, i, qmin, qmax, m is not None) for o, c, i, _, _, m, qmin, qmax in spec]
    xbuf, xs = _pack([(d[0], t[3]) for d, t in zip(data, spec)], torch.float32)
    obuf = sentinel(sum(d[0].size + 8 for d in data))
    _, os_ = _pack([(d[0], t[4]) for d, t in zip(data, spec)], torch.float32)  # offsets only; out is sentinel-filled
    masked = [(d[3], t[5]) for d, t in zip(data, spec) if d[3] is not None]
    mbuf, ms = _pack(masked, torch.uint8) if masked else (None, [])
    sbuf, ss = _pack([(d[1], 0) for d in data], torch.float32)
    zbuf, zs = _pack([(d[2], 0) for d in data], torch.float32)
    descs, mi = [], 0
    for k, ((x, s, zp, mask), t) in enumerate(zip(data, spec)):
        outer, c, inner, *_ , qmin, qmax = t
        mp = None
        if mask is not None:
            mp = mbuf.data_ptr() + ms[mi]
            mi += 1
        descs.append(ops._QdqTensorDesc(xbuf.data_ptr() + 4 * xs[k], mp, sbuf.data_ptr() + 4 * ss[k],
                                        zbuf.data_ptr() + 4 * zs[k], obuf.data_ptr() + 4 * os_[k], outer, c, inner, qmin, qmax))
    keep = (xbuf, obuf, mbuf, sbuf, zbuf)
    return data, descs, keep, os_


def _multi_plan(descs):
    lib = _lib.load()
    arr = (ops._QdqTensorDesc * len(descs))(*descs)
    table = torch.empty(max(int(lib.sb200_qdq_multi_table_bytes(len(descs))), 64), dtype=torch.uint8, device=dev())
    rows = ctypes.c_int64(0)
    rc = lib.sb200_qdq_multi_plan(arr, len(descs), table.data_ptr(), table.numel(), ctypes.byref(rows), stream())
    return rc, table, rows.value


def _multi_expected(data, spec):
    out = []
    for (x, s, zp, mask), t in zip(data, spec):
        with np.errstate(invalid="ignore"):  # inf * 0 under the mask
            xm = osp.mask_apply(x, mask) if mask is not None else x
        out.append(oqdq.qdq(xm, s, zp, t[6], t[7], ch_axis=1))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(MULTI_CASES))
def test_multi_branch_vs_oracle(case):
    check_reach(case, case.branches(real_sm()))
    rng = np.random.default_rng(seed(case.name))
    data, descs, keep, os_ = _multi_setup(case.spec, rng)
    rc, table, rows = _multi_plan(descs)
    assert rc == 0 and rows == sum(o * c for o, c, *_ in case.spec)
    lib = _lib.load()
    assert lib.sb200_qdq_multi_run(table.data_ptr(), len(descs), rows, stream()) == 0
    got = host(keep[1])
    for k, (e, t) in enumerate(zip(_multi_expected(data, case.spec), case.spec)):
        g = got[os_[k]:os_[k] + e.size].reshape(e.shape)
        assert bits_equal(g, e), f"{case.name}: tensor {k} {t[:6]}: {int(np.sum(~same(g, e)))} elements differ"
    if case.name == "multi_cap_skip2":  # the planted inf * 0 really reached the output as NaN
        x, _, _, mask = data[0]
        assert np.isnan(got[os_[0]:os_[0] + x.size][(mask.reshape(-1) == 0) & np.isinf(x.reshape(-1))]).all()


@pytest.mark.gpu
def test_multi_equals_per_tensor_calls():
    """A plan whose 8448-warp stride crosses two or more tensors computes what one qdq_perchannel /
    mask_apply_qdq_perchannel call per tensor computes."""
    spec = MULTI_CAP_SKIP2
    assert "multi.stride.skip2" in geo.multi_branches([t[:6] for t in spec], real_sm())
    rng = np.random.default_rng(seed("multi_equals_per_tensor_calls"))
    data, descs, keep, os_ = _multi_setup(spec, rng)
    rc, table, rows = _multi_plan(descs)
    assert rc == 0
    assert _lib.load().sb200_qdq_multi_run(table.data_ptr(), len(descs), rows, stream()) == 0
    got = host(keep[1])
    for k, ((x, s, zp, mask), t) in enumerate(zip(data, spec)):
        xd, sd, zd = on_device(x).view(x.shape), on_device(s), on_device(zp)
        out = sentinel(x.size).view(x.shape)
        if mask is None:
            ops.qdq_perchannel(xd, sd, zd, t[6], t[7], ch_axis=1, out=out)
        else:
            ops.mask_apply_qdq_perchannel(xd, on_device(mask).view(torch.bool).view(x.shape), sd, zd, t[6], t[7], ch_axis=1,
                                          out=out)
        assert bits_equal(got[os_[k]:os_[k] + x.size], host(out).reshape(-1)), f"tensor {k} {t[:6]}"


@pytest.mark.gpu
def test_multi_plan_count_limits():
    """sb200_qdq_multi_plan takes 4096 tensors (multi_table_max runs such a plan) and refuses 4097 before any launch."""
    lib = _lib.load()
    x = torch.zeros(8, device=dev())
    d = ops._QdqTensorDesc(x.data_ptr(), None, x.data_ptr(), x.data_ptr(), x.data_ptr(), 1, 1, 1, -8, 7)
    rc, _, rows = _multi_plan([d] * 4096)
    assert rc == 0 and rows == 4096
    before = _lib.launch_count()
    rc, _, _ = _multi_plan([d] * 4097)
    assert rc == E_INVALID and b"count must be in [1, 4096]" in lib.sb200_last_error()
    assert _lib.launch_count() == before


# -------------------------------------------------------------------------------------------------- structured mask
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(ROWS_CASES))
def test_mask_rows_gt_branch_vs_numpy(case):
    check_reach(case, case.branches(real_sm()))
    rows, inner, off = case.spec
    rng = np.random.default_rng(seed(case.name))
    th = F32(0.0)
    score = rng.standard_normal(rows).astype(F32)
    score[::7] = th  # score == thresh: pruned (strict >)
    score[1::11] = np.resize(np.array([np.nan, np.inf, -np.inf, -0.0], F32), score[1::11].size)
    mask = sentinel(rows * inner, off)
    lib = _lib.load()
    assert lib.sb200_mask_rows_gt(on_device(score).data_ptr(), on_device(np.array([th], F32)).data_ptr(), mask.data_ptr(),
                                  rows, inner, stream()) == 0
    want = np.repeat((score > th).astype(F32), inner)
    assert bits_equal(host(mask), want)


# -------------------------------------------------------------------------------------------------- PACT clamp backward
LO, HI = F32(-0.75), F32(1.25)


def _clamp_data(rng, n, positive):
    x = rng.uniform(-1.5, 2.0, n).astype(F32)
    gy = rng.uniform(0.5, 1.5, n).astype(F32) if positive else rng.standard_normal(n).astype(F32)
    if not positive:
        edges = [LO, HI, np.nextafter(LO, F32(-2)), np.nextafter(HI, F32(2)), np.nextafter(LO, F32(0)),
                 np.nextafter(HI, F32(0))] + NONFINITE
        plant(rng, x, edges, frac=0.002)
        x[-3:] = [HI, np.inf, LO]  # edges in the tail too
    return x, gy


def _clamp_sum_bound(gy, sel, terms):
    """Error bound of one of g_hi / g_lo against the fp64 sum.  Each thread adds its selected gy (zeros for the rest,
    which are exact) into an fp32 accumulator; at most `terms` fp32 additions happen before the partial is added to an
    fp64 one (4 per vector iteration, flushed every 64 iterations, plus the tail / scalar iterations, multi.cu:175-183).
    A chain of k fp32 additions errs by at most (k - 1) 2^-24 times the sum of its |terms|, so all chains together err by
    less than terms 2^-24 sum|selected gy|.  The fp64 sums over iterations, warps, CTAs and the finish (at most ~2^20
    additions in all) add less than 2^-32 sum|selected gy|, and the final fp32 rounding 2^-24 |result|."""
    a = np.abs(gy[sel].astype(F64)).sum()
    exact = gy[sel].astype(F64).sum()
    err = terms * 2.0 ** -24 * a + 2.0 ** -32 * a
    return exact, err + 2.0 ** -24 * (abs(exact) + err)


def _clamp_run(x_d, gy_d, gx, g_hi, g_lo, n, ws):
    lib = _lib.load()
    lo, hi = on_device(np.array([LO], F32)), on_device(np.array([HI], F32))
    return lib.sb200_clamp_bwd(x_d.data_ptr(), gy_d.data_ptr(), lo.data_ptr(), hi.data_ptr(), gx.data_ptr(),
                               g_hi.data_ptr() if g_hi is not None else None, g_lo.data_ptr() if g_lo is not None else None,
                               n, ws.data_ptr(), ws.numel(), stream())


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(CLAMP_CASES))
def test_clamp_bwd_branch_vs_oracle(case):
    check_reach(case, case.branches(real_sm()))
    n, x_off, gy_off, gx_off, null_hi, null_lo = case.spec
    rng = np.random.default_rng(seed(case.name))
    x, gy = _clamp_data(rng, n, positive=case.name == "clamp_flush")
    x_d, gy_d = on_device(x, x_off), on_device(gy, gy_off)
    lib = _lib.load()
    ws = torch.empty(int(lib.sb200_clamp_bwd_workspace_bytes(n)), dtype=torch.uint8, device=dev())
    runs = []
    for _ in range(2):
        gx = sentinel(n, gx_off)
        g_hi = None if null_hi else sentinel(1)
        g_lo = None if null_lo else sentinel(1)
        assert _clamp_run(x_d, gy_d, gx, g_hi, g_lo, n, ws) == 0
        runs.append((host(gx), None if g_hi is None else host(g_hi)[0], None if g_lo is None else host(g_lo)[0]))
    (gx, h, l), second = runs[0], runs[1]
    assert np.array_equal(gx.view(U32), second[0].view(U32)) and h == second[1] and l == second[2]  # deterministic
    want_gx, _, _ = oqdq.clamp_backward(x, gy, LO, HI)
    assert bits_equal(gx, want_gx), f"{int(np.sum(~same(gx, want_gx)))} of {n} gx elements differ"
    terms = geo.clamp_bwd_geometry(n, x_off, gy_off, gx_off, real_sm())["fp32_terms"]
    for got, sel in ((h, x > HI), (l, x < LO)):
        if got is None:
            continue
        exact, bound = _clamp_sum_bound(gy, sel, terms)
        assert abs(F64(got) - exact) <= bound, (case.name, float(got), exact, bound)


@pytest.mark.gpu
def test_clamp_workspace_contract():
    """sb200_clamp_bwd_workspace_bytes is a pure function of n matching the restated formula; one byte less than it is
    SB200_E_WORKSPACE before any launch."""
    lib = _lib.load()
    sm = real_sm()
    for n in (1, 13, 12_288, 1_000_003, 36_000_002):
        need = int(lib.sb200_clamp_bwd_workspace_bytes(n))
        assert need == int(lib.sb200_clamp_bwd_workspace_bytes(n)) == geo.clamp_bwd_workspace_bytes(n, sm)
    assert lib.sb200_clamp_bwd_workspace_bytes(0) == 0
    n = 100_003
    need = int(lib.sb200_clamp_bwd_workspace_bytes(n))
    x = on_device(np.ones(n, F32))
    ws = torch.empty(need, dtype=torch.uint8, device=dev())
    gx, g_hi, g_lo = sentinel(n), sentinel(1), sentinel(1)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    lo, hi = on_device(np.array([LO], F32)), on_device(np.array([HI], F32))
    rc = lib.sb200_clamp_bwd(x.data_ptr(), x.data_ptr(), lo.data_ptr(), hi.data_ptr(), gx.data_ptr(), g_hi.data_ptr(),
                             g_lo.data_ptr(), n, ws.data_ptr(), need - 1, stream())
    assert rc == E_WORKSPACE and b"workspace too small" in lib.sb200_last_error()
    assert _lib.launch_count() == before
    assert (host(gx).view(U32) == SENTINEL.view(U32)).all()
    assert lib.sb200_clamp_bwd(x.data_ptr(), x.data_ptr(), lo.data_ptr(), hi.data_ptr(), gx.data_ptr(), g_hi.data_ptr(),
                               g_lo.data_ptr(), n, ws.data_ptr(), need, stream()) == 0
    assert _lib.launch_count() == before + 2
    assert bits_equal(host(gx), np.ones(n, F32)) and host(g_hi)[0] == 0 and host(g_lo)[0] == 0


# -------------------------------------------------------------------------------------------------- AdaRound
def _quot(x, s):
    """adaround.cu:42: RN32(x * RN64(1 / s)) in fp64."""
    with np.errstate(all="ignore"):
        return (x.astype(F64) * (1.0 / s.astype(F64))).astype(F32)


def _exp_candidates(v):
    """CUDA documents expf within 2 ulp; RN32 of the fp64 exp is within 1/2 ulp of the truth, so the kernel's expf(-v) is
    one of the fp32 values within 3 steps of it (4 near a binade edge, where the step below halves)."""
    with np.errstate(all="ignore"):
        e = np.exp(-v.astype(F64)).astype(F32)
    return ulp_steps(e, 4)


def _ada_chain(op, x, v, gy, s, zp, qmin, qmax, e):
    """adaround.cu:25-83 in numpy fp32, one rounding per op, with expf(-v) = e given."""
    with np.errstate(all="ignore"):
        sg = (F32(1) / (F32(1) + e).astype(F32)).astype(F32)
        raw = ((sg * STRETCH).astype(F32) + GAMMA).astype(F32)
        fl = np.floor(_quot(x, s))
        if op == "soft":
            r = np.minimum(np.maximum(raw, F32(0)), F32(1))  # NaN propagates, like torch.clamp
            qr = ((fl + r).astype(F32) + zp).astype(F32)
            q = np.minimum(np.maximum(qr, F32(qmin)), F32(qmax))
            return ((q - zp).astype(F32) * s).astype(F32)
        r = np.fmin(np.fmax(raw, F32(0)), F32(1))  # fminf / fmaxf
        q = ((fl + r).astype(F32) + zp).astype(F32)
        live = (q >= F32(qmin)) & (q <= F32(qmax)) & (raw >= 0) & (raw <= 1)
        g = ((gy * s).astype(F32) * STRETCH).astype(F32)
        return np.where(live, (g * (sg * (F32(1) - sg).astype(F32)).astype(F32)).astype(F32), F32(0)).astype(F32)


def _ada_init_candidates(x, s):
    """adaround.cu:77-83: z = RN(RN(1 / (rest - gamma)) * stretch) - 1 is exact in numpy; logf is documented within 1 ulp,
    so -logf(z) is one of the values within 2 steps of -RN32(log(z))."""
    with np.errstate(all="ignore"):
        qv = _quot(x, s)
        rest = (qv - np.floor(qv)).astype(F32)
        ratio = ((F32(1) / (rest - GAMMA).astype(F32)).astype(F32) * STRETCH).astype(F32)
        z = (ratio - F32(1)).astype(F32)
        lz = np.log(z.astype(F64)).astype(F32)
    return [(-c).astype(F32) for c in ulp_steps(lz, 2)]


def _ada_data(rng, outer, c, inner, qmin, qmax):
    s = rng.uniform(0.01, 0.05, c).astype(F32)
    s[::3] = 2.0 ** -5
    zp = rng.uniform(qmin, qmax, c).astype(F32)  # not rounded by AdaRound
    zp[::4] = np.rint(zp[::4])
    x = (rng.uniform(qmin - 6, qmax + 6, (outer, c, inner)).astype(F32) - zp[None, :, None]) * s[None, :, None]
    x = x.astype(F32)
    x.reshape(outer, c, -1)[:, ::3, : min(inner, 16)] = (np.arange(min(inner, 16), dtype=F32) * F32(2.0 ** -5))  # on grid
    v = rng.normal(0, 3, x.shape).astype(F32)
    plant(rng, v, [0.0, -0.0, 100.0, -100.0, 88.0, -88.0, 1e-30, -1e-30], frac=0.02)
    plant(rng, x, NONFINITE + list(subnormals(rng, 4)), frac=0.002)
    plant(rng, v, NONFINITE, frac=0.002)
    gy = rng.standard_normal(x.shape).astype(F32)
    return x, v, gy, s, zp


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(ADA_CASES))
def test_adaround_branch_vs_oracle(case):
    check_reach(case, case.branches(real_sm()))
    op, outer, c, inner, offs = case.spec
    offs = dict(offs)
    qmin, qmax = -8, 7
    rng = np.random.default_rng(seed(case.name))
    x, v, gy, s, zp = _ada_data(rng, outer, c, inner, qmin, qmax)
    n = x.size
    xd, vd, gyd = on_device(x, offs.get("x", 0)), on_device(v, offs.get("v", 0)), on_device(gy, offs.get("gy", 0))
    sd, zd = on_device(s), on_device(zp)
    out = sentinel(n, offs.get("out", 0))
    lib = _lib.load()
    if op in ("hard", "soft"):
        rc = lib.sb200_adaround_fwd(xd.data_ptr(), vd.data_ptr(), sd.data_ptr(), zd.data_ptr(), out.data_ptr(), outer, c, inner,
                                    qmin, qmax, int(op == "soft"), stream())
    elif op == "bwd":
        rc = lib.sb200_adaround_bwd(xd.data_ptr(), vd.data_ptr(), sd.data_ptr(), zd.data_ptr(), gyd.data_ptr(), out.data_ptr(),
                                    outer, c, inner, qmin, qmax, stream())
    else:
        rc = lib.sb200_adaround_init(xd.data_ptr(), sd.data_ptr(), out.data_ptr(), outer, c, inner, stream())
    assert rc == 0
    got = host(out).reshape(x.shape)
    s3, z3 = s[None, :, None], zp[None, :, None]
    if op == "hard":
        want = oqdq.adaround_forward(x, v, s, zp, qmin, qmax, ch_axis=1, soft=False)
        assert bits_equal(got, want), f"{int(np.sum(~same(got, want)))} elements differ"
        return
    if op == "init":
        cands = _ada_init_candidates(x, s3)
        ref = oqdq.adaround_init(x, s, ch_axis=1)
    else:
        cands = [_ada_chain(op, x, v, gy, s3, z3, qmin, qmax, e) for e in _exp_candidates(v)]
        ref = (oqdq.adaround_forward(x, v, s, zp, qmin, qmax, ch_axis=1, soft=True) if op == "soft"
               else oqdq.adaround_grad_v(x, v, s, zp, gy, qmin, qmax, ch_axis=1))
    ok = np.zeros(x.shape, bool)
    for cnd in cands:
        ok |= same(got, cnd)
    assert ok.all(), f"{int(np.sum(~ok))} elements outside expf / logf's error bound, e.g. {got[~ok][:4]}"
    with np.errstate(all="ignore"):
        ref = np.asarray(ref).astype(F32)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), "NaN pattern differs from the oracle"
    assert np.array_equal(np.isposinf(got), np.isposinf(ref)) and np.array_equal(np.isneginf(got), np.isneginf(ref))


# -------------------------------------------------------------------------------------------------- DoReFa
# The absmax the fwd / bwd cases read: below max|t| (the planted +-inf give |t| = 1), so quotients leave [-1, 1] and reach
# the clamps, and not a power of two, so the division rounds.
DOREFA_M = F32(0.9)


def _dorefa_x(rng, n):
    x = (rng.standard_normal(n) * 1.2).astype(F32)
    plant(rng, x, [np.nan, np.inf, -np.inf, 0.0, -0.0, 20.0, -20.0, 1e-20] + list(subnormals(rng, 4)), frac=0.002)
    return x


def _fwd(lib, xd, md, sd, zd, out, outer, c, inner, qmin, qmax, quantize):
    return lib.sb200_dorefa_fwd(xd.data_ptr(), md.data_ptr(), sd.data_ptr() if sd is not None else None,
                                zd.data_ptr() if zd is not None else None, out.data_ptr(), outer, c, inner, qmin, qmax,
                                quantize, stream())


def _kernel_tanh(x):
    """The kernel's own tanhf(x): normalise-only with absmax = 1.0 (__fdiv_rn(t, 1) is t), checked against fp64 tanh within
    CUDA's documented 2 ulp for tanhf."""
    lib = _lib.load()
    n = x.size
    t = sentinel(n)
    assert _fwd(lib, on_device(x), on_device(np.array([1.0], F32)), None, None, t, 1, 1, n, 0, 0, 0) == 0
    t = host(t)
    with np.errstate(all="ignore"):
        r = np.tanh(x.astype(F64)).astype(F32)
    ok = np.zeros(n, bool)
    for cnd in ulp_steps(r, 2):
        ok |= same(t, cnd)
    assert ok.all(), f"tanhf beyond 2 ulp at x = {x[~ok][:4]}: {t[~ok][:4]} vs {r[~ok][:4]}"
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(DOREFA_CASES))
def test_dorefa_branch_vs_kernel_tanh(case):
    check_reach(case, case.branches(real_sm()))
    op, outer, c, inner, offs = case.spec
    offs = dict(offs)
    qmin, qmax = -8, 7
    rng = np.random.default_rng(seed(case.name))
    n = outer * c * inner
    x = _dorefa_x(rng, n)
    t = _kernel_tanh(x)
    m = DOREFA_M
    s = rng.uniform(0.1, 0.2, c).astype(F32)
    zp = rng.choice(np.array([0.0, 1.0, -0.5, 0.5], F32), c).astype(F32)
    gy = rng.standard_normal(n).astype(F32)
    lib = _lib.load()
    xd, gyd, md = on_device(x, offs.get("x", 0)), on_device(gy, offs.get("gy", 0)), on_device(np.array([m], F32))
    sd, zd = on_device(s), on_device(zp)
    out = sentinel(n, offs.get("out", 0))
    if op == "bwd":
        rc = lib.sb200_dorefa_bwd(xd.data_ptr(), md.data_ptr(), sd.data_ptr(), zd.data_ptr(), gyd.data_ptr(), out.data_ptr(),
                                  outer, c, inner, qmin, qmax, stream())
    else:
        rc = _fwd(lib, xd, md, sd, zd, out, outer, c, inner, qmin, qmax, int(op == "qdq"))
    assert rc == 0
    got = host(out)
    with np.errstate(all="ignore"):
        xn = (t / m).astype(F32)  # dorefa.cu:56
        if op == "norm":
            want = xn
        elif op == "qdq":
            want = oqdq.qdq(xn.reshape(outer, c, inner), s, zp, qmin, qmax, ch_axis=1).reshape(-1)
        else:  # dorefa.cu:59-61: STE mask, / m, * (1 - t t)
            g, _, _ = oqdq.ste_backward(xn.reshape(outer, c, inner), s, zp, gy.reshape(outer, c, inner), qmin, qmax, ch_axis=1)
            want = ((g.reshape(-1) / m).astype(F32) * (F32(1) - (t * t).astype(F32)).astype(F32)).astype(F32)
    assert bits_equal(got, want), f"{int(np.sum(~same(got, want)))} of {n} elements differ"


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(ABSMAX_CASES))
def test_dorefa_absmax_branch_vs_kernel_tanh(case):
    check_reach(case, case.branches(real_sm()))
    n, x_off = case.spec
    rng = np.random.default_rng(seed(case.name))
    x = rng.uniform(-0.5, 0.5, n).astype(F32)
    x[-3:] = [0.1, 0.2, F32(-0.9)]  # the largest |tanh| in the scalar tail
    x[n // 3] = F32(0.85)  # ... and the runner-up in the vector body
    if case.name == "absmax_nan":
        x[n // 2] = np.nan
    t = _kernel_tanh(x)
    m = torch.zeros(1, dtype=torch.float32, device=dev())  # the caller's initial state (ops.dorefa_absmax)
    assert _lib.load().sb200_dorefa_absmax(on_device(x, x_off).data_ptr(), n, m.data_ptr(), stream()) == 0
    want = F32(np.nan) if np.isnan(t).any() else np.abs(t).max()
    assert bits_equal(host(m), np.array([want], F32)), (host(m)[0], want)


# -------------------------------------------------------------------------------------------------- qdq.cu mask helpers
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(GT_CASES))
def test_mask_gt_branch_vs_numpy(case):
    check_reach(case, case.branches(real_sm()))
    n, w_off, m_off = case.spec
    rng = np.random.default_rng(seed(case.name))
    th = F32(0.5)
    w = rng.uniform(-1, 1, n).astype(F32)
    plant(rng, w, [0.5, -0.5, np.nextafter(th, F32(1)), np.nextafter(th, F32(0))] + NONFINITE + list(subnormals(rng, 4)),
          frac=0.01)
    w[-3:] = [-0.5, 0.75, 0.5]
    mask = sentinel(n, m_off, torch.uint8)
    assert _lib.load().sb200_mask_gt(on_device(w, w_off).data_ptr(), on_device(np.array([th], F32)).data_ptr(),
                                     mask.data_ptr(), n, stream()) == 0
    assert np.array_equal(host(mask), (np.abs(w) > th).astype(np.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(MULF_CASES))
def test_mask_apply_f32_branch_vs_oracle(case):
    check_reach(case, case.branches(real_sm()))
    n, w_off, m_off, o_off = case.spec
    rng = np.random.default_rng(seed(case.name))
    w = rng.standard_normal(n).astype(F32)
    plant(rng, w, NONFINITE + list(subnormals(rng, 4)), frac=0.01)
    m = (rng.random(n) < 0.6).astype(F32)
    m[np.flatnonzero(np.isinf(w))[::2]] = 0.0  # inf * 0 = NaN
    out = sentinel(n, o_off)
    assert _lib.load().sb200_mask_apply_f32(on_device(w, w_off).data_ptr(), on_device(m, m_off).data_ptr(), out.data_ptr(),
                                            n, stream()) == 0
    with np.errstate(invalid="ignore"):
        want = osp.mask_apply(w, m)
    assert bits_equal(host(out), want)


# -------------------------------------------------------------------------------------------------- MinMax qparams
def enc(x):
    """enc_f32 (common.cuh:67-74)."""
    b = np.ascontiguousarray(x, dtype=F32).view(U32)
    return np.where(b & U32(0x80000000), ~b, b | U32(0x80000000)).astype(U32)


def dec(k):
    k = np.asarray(k, dtype=U32)
    return np.where(k & U32(0x80000000), k & U32(0x7FFFFFFF), ~k).astype(U32).view(F32)


QP_SPECIAL_STRIDE = 41


def _qp_state(rng, c, qmin, qmax):
    mn = rng.uniform(-3, 0.5, c).astype(F32)
    mx = np.maximum(mn, rng.uniform(-0.5, 3, c).astype(F32))
    keys = np.stack([enc(mn), enc(mx)], 1)
    span = F32(qmax - qmin)
    step = QP_SPECIAL_STRIDE if c > 128 else 1
    for j in range(0, c, step):  # the special channels, beyond channel 128 too
        kind = (j // step) % 6
        if kind == 0:
            keys[j] = (0xFFFFFFFF, 0x00000000)  # never observed (minmax_init)
        elif kind == 1:
            keys[j] = (0xFFFFFFFF, 0xFFFFFFFF)  # a NaN was observed (common.cuh:276-284)
        elif kind == 2:
            keys[j] = enc(np.array([-np.inf, np.inf], F32))
        elif kind == 3:
            keys[j] = enc(np.array([-1e-9, 1e-9], F32))  # under the 1e-6 floor
        elif kind == 4:  # -min / scale = 2.5 exactly: rint -> 2
            sc = F32(1 / 16)
            keys[j] = enc(np.array([-2.5 * sc, (span - 2.5) * sc], F32))
        else:  # 3.5 -> 4
            sc = F32(1 / 16)
            keys[j] = enc(np.array([-3.5 * sc, (span - 3.5) * sc], F32))
    return keys.reshape(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(QP_CASES))
def test_minmax_qparams_branch_vs_oracle(case):
    check_reach(case, case.branches(real_sm()))
    rng = np.random.default_rng(seed(case.name))
    lib = _lib.load()
    states, outs, descs = [], [], []
    for c, sym, qmin, qmax in case.spec:
        keys = _qp_state(rng, c, qmin, qmax)
        st = on_device(keys.view(np.int32))
        o = [sentinel(c) for _ in range(4)]
        states.append((keys, st))
        outs.append(o)
        descs.append(ops._QparamsDesc(st.data_ptr(), *[t.data_ptr() for t in o], c, qmin, qmax, int(sym)))
    arr = (ops._QparamsDesc * len(descs))(*descs)
    table = torch.empty(64 * len(descs), dtype=torch.uint8, device=dev())
    assert lib.sb200_minmax_qparams_multi(arr, len(descs), table.data_ptr(), table.numel(), stream()) == 0
    for (c, sym, qmin, qmax), (keys, _), o in zip(case.spec, states, outs):
        mn, mx = dec(keys[0::2]), dec(keys[1::2])
        with np.errstate(all="ignore"):
            scale, zp = oobs.calc_qparams_with_minmax(mn, mx, qmin, qmax, sym)
        got = [host(t) for t in o]
        for name, g, w in zip(("min", "max", "scale", "zero_point"), got, (mn, mx, scale, zp)):
            assert bits_equal(g, w), f"{case.name} entry ({c}, {sym}): {name} differs at {np.flatnonzero(~same(g, w))[:8]}"
        if c > 128:  # the planted edges really are there, beyond the first 128 channels too
            for j in range(0, c, QP_SPECIAL_STRIDE):
                kind = (j // QP_SPECIAL_STRIDE) % 6
                assert kind > 1 or np.isnan(got[2][j])
                assert kind != 3 or got[2][j] == F32(1e-6)
                assert sym or kind < 4 or got[3][j] == (2 if kind == 4 else 4)
