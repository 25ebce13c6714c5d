"""Every launch branch of the observer calibration kernels (csrc/observe.cu, and the per-tensor MinMax that qdq.cu runs
through its streaming kernel), each reached by a named case and compared with a numpy reference: MinMax states, sign
counts, histograms and selected values bit-exact, MSE losses within an error bound derived from the kernel's arithmetic,
row moments against fp64 sums.

tests/observe_geometry.py restates the host launch formulas; every case below asserts, with the SM count of the device
it runs on, that it reaches the branches it is listed for, and the CPU test at the bottom checks at 132 SMs (H100 SXM)
that the cases together reach every branch in REQUIRED.  Ids marked (data) depend on the values, not the launch: the
case claims them and its GPU run checks the claim on the data it feeds.

MinMax (sb200_observe_minmax_perchannel / sb200_observe_minmax).  Each row gets planted extremes at its head, its last
elements and its middle, cycling with the row, so a dropped head, tail or row changes some channel; the column cases
plant them in the first, second, third and last row of every row block and in its 1-wide tail.  Special channels (every
case with C >= 7): a NaN at the head of one row of one channel only, -inf at a row head and +inf at a row tail, a channel of
equal values, subnormals of both signs, +-0, all -0 (the reference orders floats like enc_f32: -0 < +0, NaN poisons the
channel).  Every case updates the state twice and compares the raw state after each; the per-tensor cases update it three
times: finite extremes at the head and the scalar tail, then -inf / +inf there, then a NaN in the tail.

  branch                          source                  case: shape, ch_axis, offset (why it gets there)
  mm.cols.v4.loop4                observe.cu:149-156      mm_cols_v4_loop4: (3000,768) ch 1, 6 rows per block
  mm.cols.v4.tail                 observe.cu:157-160      mm_cols_v4_loop4; mm_cols_gy_outer (1 row per block)
  mm.cols.gy_sm                   observe.cu:674          mm_cols_v4_loop4 (want_y 528 < outer 3000; grid.y 500)
  mm.cols.gy_outer                observe.cu:675          mm_cols_gy_outer: (37,768) ch 1 (want_y capped by outer)
  mm.cols.v1                      observe.cu:162          mm_cols_v1_odd: (300,75) ch 1; mm_cols_v1_off1: x offset 1
  mm.rows.cta.tpr1                observe.cu:45-61        mm_cta_4096: (3,7,4096) ch 1 (inner == 4096, one tile)
  mm.rows.cta.tpr_gt1.partial     observe.cu:52-54        mm_cta_8193: (2,7,8193) ch 1
  mm.rows.cta.span.head           observe.cu:28-30        mm_cta_8193 (odd rows start off a 16-byte boundary)
  mm.rows.cta.gridstride          observe.cu:51           mm_cta_gridstride: (2,530,4096) ch 1, 1060 tiles > 8 x 132
  mm.rows.warp.vec                observe.cu:76-83        mm_warp_vec_tail: (15,128) ch 0; mm_warp_gridstride
  mm.rows.warp.vec.tail_rows      observe.cu:84-88        mm_warp_vec_tail (15 % 4 rows take span_minmax)
  mm.rows.warp.scalar             observe.cu:84-88        mm_warp_inner65: (28,65) ch 0; mm_warp_inner4095; mm_warp_off2
  mm.rows.warp.gridstride         observe.cu:72           mm_warp_gridstride: (1000,35,68) ch 1, 35000 rows
  mm.rows.tiny.stage.v4           observe.cu:111-114      mm_tiny_inner64: (8,40,64) ch 1
  mm.rows.tiny.rot                observe.cu:123-126      mm_tiny_inner64 (inner 64 is even)
  mm.rows.tiny.stage.scalar       observe.cu:115-117      mm_tiny_odd_ragged: (21,7,7) ch 0; mm_tiny_off3: x offset 3
  mm.rows.tiny.norot              observe.cu:123          mm_tiny_odd_ragged (inner 49)
  mm.rows.tiny.last_group_lt32    observe.cu:108          mm_tiny_odd_ragged (21 rows)
  mm.rows.tiny.gridstride         observe.cu:107          mm_tiny_gridstride: (1024,100,2) ch 1, 400 CTAs > 3 x 132
  mm.tensor.v4                    qdq.cu:108-208          mmt_v4_tail: n = 4099
  mm.tensor.v4.scalar_tail        qdq.cu:211-228          mmt_v4_tail (4099 % 4 = 3 elements)
  mm.tensor.v1.off1               qdq.cu:433              mmt_off1: n = 5000 at x offset 1 (VEC = 1 body)
  mm.tensor.v1.off2               qdq.cu:433              mmt_off2: x offset 2
  mm.tensor.v1.off3               qdq.cu:433              mmt_off3: x offset 3
  mm.tensor.gridstride            qdq.cu:108              mmt_gridstride: n = 2200003, two grid-stride passes

Histogram (sb200_observe_hist) against oracle.observers.histc, bit-exact, accumulated over two calls.  Data: lo, hi and
one ulp either side, every edge lo + k (hi - lo) / bins (a sample of them for 8192 bins) and +-1, 2 ulp around it, NaN,
+-inf, both at the ends of the buffer (scalar tail) and scattered.

  hist.v4.loop4                   observe.cu:202-208      hist_loop4_tail: n = 1000003, 4 or 3 vectors per thread
  hist.v4.loop1                   observe.cu:209-212      hist_loop4_tail (the threads with 3 vectors)
  hist.v4.tail                    observe.cu:213          hist_loop4_tail (1000003 % 4 = 3)
  hist.bins2048                   observe.cu:177-193      hist_loop4_tail; hist_empty_range
  hist.scalar                     observe.cu:214-216      hist_scalar_bins7: x offset 1
  hist.bins7                      observe.cu:177-193      hist_scalar_bins7; hist_empty_const
  hist.gridstride                 observe.cu:188, 707     hist_gridstride_8192: n = 4400001 (1075 CTAs > 8 x 132)
  hist.bins8192                   observe.cu:177-193      hist_gridstride_8192 (32 KB of shared counters)
  hist.bins1                      observe.cu:193          hist_bins1
  hist.empty_range                observe.cu:181-184      hist_empty_range: all +-0 in [-0, +0]; hist_empty_const: 0.3

MSE sweep (sb200_observe_mse_sweep): per row and candidate sum (x - qdq_oracle(x; s_i, rint(z_i)))^2 in fp64 from
oracle.qdq, with arbitrary per-row candidate tables; bound derived in _mse_reference; += into a non-zero sse; two runs
bit-identical.

  mse.nonbulk, mse.reload         observe.cu:275-286      mse_reload_pad9: (600,243), 600 tiles > 4 x 132 CTAs
  mse.cand_pad                    observe.cu:300          mse_reload_pad9 (9 candidates); mse_mixed_unroll4 (7)
  mse.bulk, mse.tpr_gt1           observe.cu:269-273      mse_bulk_80: (3,16384), 80 candidates; mse_off2: (5,9000) x offset 2
  mse.mixed                       observe.cu:269          mse_mixed_unroll4: (1,327675), 39 TMA tiles + 1 odd-length tile
  mse.ncand1, mse.ncand128        observe.cu:292-317      mse_ncand1: (2,5000); mse_ncand128: (4,1000)
  mse.finish.S1                   observe.cu:630-652      mse_bulk_80, mse_ncand128 (S = 1 slice)
  mse.finish.S_gt1                observe.cu:630-652      mse_reload_pad9 (S = 3), mse_ncand1
  mse.finish.unroll4              observe.cu:639-642      mse_mixed_unroll4 (40 tiles, S = 13)

Radix select (ops.RadixSelect driven directly, both targets per row) against np.sort under the enc_f32 order, bit-exact:

  sel.hist.p0.ntpr2,              observe.cu:342-433      every sel_ case but sel_ntpr1_key1; pct_rows, pct_large
    sel.hist.p1.ntpr2, sel.hist.p2.ntpr2
  sel.hist.p0.ntpr1,              observe.cu:342-433      sel_ntpr1_key1: (3,9001) key_mode 1, x offset 1
    sel.hist.p1.ntpr1, sel.hist.p2.ntpr1
  sel.hist.key_mode1              observe.cu:335          sel_ntpr1_key1
  sel.hist.seg16384               observe.cu:570-575      sel_seg16384_head: (5,20001), 10 tiles
  sel.hist.head                   observe.cu:379-381      sel_seg16384_head (odd rows start off a 16-byte boundary)
  sel.hist.loop4                  observe.cu:385-392      sel_seg16384_head (16384-element segments); pct_large
  sel.hist.tail                   observe.cu:397          sel_seg16384_head
  sel.hist.seg65536               observe.cu:570-575      sel_seg65536_gridstride: (800,100), 800 rows >= 6 x 132
  sel.hist.gridstride             observe.cu:355          sel_seg65536_gridstride (800 tiles > 6 x 132 CTAs)
  sel.hist.seg32768               observe.cu:570-575      sel_seg32768: (396,32769)
  sel.hist.head (extremes)        observe.cu:379-381      sel_extremes: (6,4099) x offset 3; NaN, +-inf, +-0, subnormals,
                                                          ranks at the -0 / +0 / inf / NaN boundaries
  sel.scan.found                  observe.cu:470-477      every select case
  sel.scan.same_bucket (data)     observe.cu:445-494      sel_dups: runs of equal keys spanning both ranks
  sel.hist.p0.counts              observe.cu:369-370, 411-418      pct_rows, pct_large: sign counts from pass 0
  sel.ranks.tie_half_even (data)  observe.cu:529-531      pct_rows: alpha 0.25 with 10 / 26 / 18 elements of a sign
  sel.ranks.kmin_clamp_lo (data)  observe.cu:530          pct_rows: alpha 0, rows without negatives
  sel.ranks.kmax_clamp (data)     observe.cu:534          pct_rows: alpha 1, a row without negatives
  sel.ranks.kmin_clamp_total      observe.cu:535          pct_rows: alpha 2, a row of negatives only
    (data)
  count_sign.multirow,            observe.cu:540-563      cs_gridstride: (1100,50), 1100 tiles > 8 x 132; cs_rows3
    count_sign.gridstride

Row moments (sb200_observe_moments) against fp64 numpy:

  moments.tpr_gt1                 observe.cu:591-598      mom_tpr3_centre: (3,40000), 3 tiles per row
  moments.centre                  observe.cu:599-600      mom_tpr3_centre (a centre per row)
  moments.nocentre                observe.cu:599-600      mom_tpr3_nocentre
  moments.finish.S_gt1            observe.cu:630-652      mom_tpr3_centre (S = 6)
  moments.finish.unroll4          observe.cu:639-642      mom_unroll4: (1,1638407), 101 tiles, S = 32

The finish never runs with one slice for the moments (nval = 5): its block has at least 32 threads, so S >= 6
(test_finish_has_several_slices_below_17_values).  mse.finish.S1 needs ncand >= 17.

The percentile path is also run end to end (hist_pass(0, with_counts) -> percentile_ranks -> scans) and compared with
oracle.observers.percentile(per_channel=True) for the alphas where the reference's kthvalue is defined.  select_scan's
"rank beyond the population" arm (observe.cu:482-491) cannot be reached through sb200_percentile_ranks
(test_percentile_ranks_stay_in_range); a rank set directly to >= n reads out NaN (test_select_rank_beyond_population).
"""
import ctypes
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import branch_cases
import observe_geometry as geo
import qdq_geometry as qgeo
from branch_cases import assert_table_covers, check_reach, fs, params
from gpu_util import bits_equal, dev, on_device, real_sm, seed_of, stream
from oracle import observers as oobs
from oracle import qdq as oqdq
from sparsebit_b200 import _lib, ops

F32 = np.float32
U32 = np.uint32
NAN_KEY = 0xFFFFFFFF


# -------------------------------------------------------------------------------------------------- helpers
def enc(x):
    """enc_f32 (common.cuh:67-74): the total order -0 < +0, as uint32 keys."""
    b = np.ascontiguousarray(x, dtype=F32).view(U32)
    return np.where(b & U32(0x80000000), ~b, b | U32(0x80000000)).astype(U32)


def dec(k):
    k = np.asarray(k, dtype=U32)
    return np.where(k & U32(0x80000000), k & U32(0x7FFFFFFF), ~k).astype(U32).view(F32)


def subnormals(rng, n):
    bits = rng.integers(1, 1 << 23, n, dtype=np.int64).astype(U32)
    bits |= (rng.random(n) < 0.5).astype(U32) << U32(31)
    return bits.view(F32)


def signed_zeros(rng, n):
    return np.where(rng.random(n) < 0.5, F32(-0.0), F32(0.0)).astype(F32)


# -------------------------------------------------------------------------------------------------- cases
@dataclass(frozen=True)
class Case(branch_cases.Case):
    """op: mm | mmt | hist | mse | sel | pct | cs | mom; spec: the input shape."""
    x_off: int = 0
    arg: tuple = ()

    def branches(self, sm):
        n = int(np.prod(self.spec))
        if self.op == "mm":
            outer, c, inner = qgeo.channel_geometry(self.spec, self.arg[0])
            return geo.minmax_branches(outer, c, inner, sm, self.x_off)
        if self.op == "mmt":
            return geo.minmax_tensor_branches(n, sm, self.x_off)
        if self.op == "hist":
            bins, lo, hi = self.arg
            return geo.hist_branches(n, sm, self.x_off) | {f"hist.bins{bins}"} | ({"hist.empty_range"} if lo == hi else set())
        rows, row_len = self.spec
        if self.op == "mse":
            return geo.mse_branches(rows, row_len, self.arg[0], sm, self.x_off)
        if self.op == "sel":
            ntpr, key_mode = self.arg
            return geo.select_hist_branches(rows, row_len, ntpr, (0, 1, 2), sm, self.x_off, key_mode) | {"sel.scan.found"}
        if self.op == "pct":
            return (geo.select_hist_branches(rows, row_len, 2, (0, 1, 2), sm, self.x_off)
                    | {"sel.scan.found", "sel.hist.p0.counts"})
        if self.op == "cs":
            return geo.count_sign_branches(rows, row_len, sm)
        return geo.moments_branches(rows, row_len, self.arg[0], sm)


MM_CASES = [
    Case("mm_cols_v4_loop4", "mm", (3000, 768), fs("mm.cols.v4.loop4", "mm.cols.v4.tail", "mm.cols.gy_sm"), arg=(1,)),
    Case("mm_cols_gy_outer", "mm", (37, 768), fs("mm.cols.v4.tail", "mm.cols.gy_outer"), arg=(1,)),
    Case("mm_cols_v1_odd", "mm", (300, 75), fs("mm.cols.v1"), arg=(1,)),
    Case("mm_cols_v1_off1", "mm", (300, 768), fs("mm.cols.v1"), x_off=1, arg=(1,)),
    Case("mm_cta_4096", "mm", (3, 7, 4096), fs("mm.rows.cta.tpr1"), arg=(1,)),
    Case("mm_cta_8193", "mm", (2, 7, 8193), fs("mm.rows.cta.tpr_gt1.partial", "mm.rows.cta.span.head"), arg=(1,)),
    Case("mm_cta_gridstride", "mm", (2, 530, 4096), fs("mm.rows.cta.gridstride"), arg=(1,)),
    Case("mm_warp_vec_tail", "mm", (15, 128), fs("mm.rows.warp.vec", "mm.rows.warp.vec.tail_rows"), arg=(0,)),
    Case("mm_warp_inner65", "mm", (28, 65), fs("mm.rows.warp.scalar"), arg=(0,)),
    Case("mm_warp_inner4095", "mm", (6, 4095), fs("mm.rows.warp.scalar"), arg=(0,)),
    Case("mm_warp_off2", "mm", (32, 128), fs("mm.rows.warp.scalar"), x_off=2, arg=(0,)),
    Case("mm_warp_gridstride", "mm", (1000, 35, 68), fs("mm.rows.warp.gridstride", "mm.rows.warp.vec"), arg=(1,)),
    Case("mm_tiny_inner64", "mm", (8, 40, 64), fs("mm.rows.tiny.stage.v4", "mm.rows.tiny.rot"), arg=(1,)),
    Case("mm_tiny_odd_ragged", "mm", (21, 7, 7), fs("mm.rows.tiny.stage.scalar", "mm.rows.tiny.norot",
                                                    "mm.rows.tiny.last_group_lt32"), arg=(0,)),
    Case("mm_tiny_off3", "mm", (64, 8), fs("mm.rows.tiny.stage.scalar"), x_off=3, arg=(0,)),
    Case("mm_tiny_gridstride", "mm", (1024, 100, 2), fs("mm.rows.tiny.gridstride"), arg=(1,)),
    Case("mmt_v4_tail", "mmt", (4099,), fs("mm.tensor.v4", "mm.tensor.v4.scalar_tail")),
    Case("mmt_off1", "mmt", (5000,), fs("mm.tensor.v1.off1"), x_off=1),
    Case("mmt_off2", "mmt", (5000,), fs("mm.tensor.v1.off2"), x_off=2),
    Case("mmt_off3", "mmt", (5000,), fs("mm.tensor.v1.off3"), x_off=3),
    Case("mmt_gridstride", "mmt", (2_200_003,), fs("mm.tensor.gridstride")),
]
HIST_CASES = [
    Case("hist_loop4_tail", "hist", (1_000_003,), fs("hist.v4.loop4", "hist.v4.loop1", "hist.v4.tail", "hist.bins2048"),
         arg=(2048, -2.5, 4.25)),
    Case("hist_scalar_bins7", "hist", (50_001,), fs("hist.scalar", "hist.bins7"), x_off=1, arg=(7, -3.17, 3.17)),
    Case("hist_gridstride_8192", "hist", (4_400_001,), fs("hist.gridstride", "hist.bins8192"), arg=(8192, -3.17, 3.17)),
    Case("hist_bins1", "hist", (4099,), fs("hist.bins1"), arg=(1, -1.5, 0.75)),
    Case("hist_empty_range", "hist", (1001,), fs("hist.empty_range"), arg=(2048, -0.0, 0.0)),
    Case("hist_empty_const", "hist", (4097,), fs("hist.empty_range"), x_off=2, arg=(7, 0.3, 0.3)),
]
MSE_CASES = [  # arg: (ncand, qmin, qmax)
    Case("mse_reload_pad9", "mse", (600, 243), fs("mse.nonbulk", "mse.reload", "mse.cand_pad", "mse.finish.S_gt1"),
         arg=(9, -8, 7)),
    Case("mse_bulk_80", "mse", (3, 16384), fs("mse.bulk", "mse.tpr_gt1", "mse.finish.S1"), arg=(80, -8, 7)),
    Case("mse_mixed_unroll4", "mse", (1, 327_675), fs("mse.mixed", "mse.cand_pad", "mse.finish.unroll4"), arg=(7, 0, 15)),
    Case("mse_ncand1", "mse", (2, 5000), fs("mse.ncand1", "mse.bulk", "mse.finish.S_gt1"), arg=(1, -8, 7)),
    Case("mse_ncand128", "mse", (4, 1000), fs("mse.ncand128", "mse.finish.S1"), arg=(128, 0, 15)),
    Case("mse_off2", "mse", (5, 9000), fs("mse.nonbulk", "mse.tpr_gt1"), x_off=2, arg=(16, -8, 7)),
]
_P = ("sel.hist.p0.ntpr2", "sel.hist.p1.ntpr2", "sel.hist.p2.ntpr2")
SEL_CASES = [  # arg: (ntpr, key_mode)
    Case("sel_seg16384_head", "sel", (5, 20001), fs(*_P, "sel.hist.seg16384", "sel.hist.head", "sel.hist.loop4",
                                                    "sel.hist.tail", "sel.scan.found"), arg=(2, 0)),
    Case("sel_seg65536_gridstride", "sel", (800, 100), fs(*_P, "sel.hist.seg65536", "sel.hist.gridstride"), arg=(2, 0)),
    Case("sel_seg32768", "sel", (396, 32769), fs(*_P, "sel.hist.seg32768"), arg=(2, 0)),
    Case("sel_ntpr1_key1", "sel", (3, 9001), fs("sel.hist.p0.ntpr1", "sel.hist.p1.ntpr1", "sel.hist.p2.ntpr1",
                                                "sel.hist.key_mode1"), x_off=1, arg=(1, 1)),
    Case("sel_dups", "sel", (4, 70000), fs(*_P, "sel.scan.same_bucket"), arg=(2, 0), claims=fs("sel.scan.same_bucket")),
    Case("sel_extremes", "sel", (6, 4099), fs(*_P, "sel.hist.head"), x_off=3, arg=(2, 0)),
]
PCT_ALPHAS = (0.25, 0.5, 0.0, 1.0, 2.0)
PCT_CASES = [
    Case("pct_rows", "pct", (4, 40), fs(*_P, "sel.hist.p0.counts", "sel.ranks.tie_half_even", "sel.ranks.kmin_clamp_lo",
                                        "sel.ranks.kmax_clamp", "sel.ranks.kmin_clamp_total"), arg=PCT_ALPHAS,
         claims=fs("sel.ranks.tie_half_even", "sel.ranks.kmin_clamp_lo", "sel.ranks.kmax_clamp",
                   "sel.ranks.kmin_clamp_total")),
    Case("pct_large", "pct", (3, 100_003), fs("sel.hist.p0.counts", "sel.hist.loop4"), arg=(1e-3,)),
]
CS_CASES = [
    Case("cs_gridstride", "cs", (1100, 50), fs("count_sign.gridstride", "count_sign.multirow")),
    Case("cs_rows3", "cs", (3, 100_003), fs("count_sign.multirow")),
]
MOM_CASES = [  # arg: (centre,)
    Case("mom_tpr3_centre", "mom", (3, 40000), fs("moments.tpr_gt1", "moments.centre", "moments.finish.S_gt1"), arg=(True,)),
    Case("mom_tpr3_nocentre", "mom", (3, 40000), fs("moments.tpr_gt1", "moments.nocentre"), arg=(False,)),
    Case("mom_unroll4", "mom", (1, 1_638_407), fs("moments.finish.unroll4"), arg=(True,)),
]
ALL_CASES = MM_CASES + HIST_CASES + MSE_CASES + SEL_CASES + PCT_CASES + CS_CASES + MOM_CASES

REQUIRED = {
    "mm.cols.v4.loop4", "mm.cols.v4.tail", "mm.cols.v1", "mm.cols.gy_outer", "mm.cols.gy_sm",
    "mm.rows.cta.tpr1", "mm.rows.cta.tpr_gt1.partial", "mm.rows.cta.span.head", "mm.rows.cta.gridstride",
    "mm.rows.warp.vec", "mm.rows.warp.vec.tail_rows", "mm.rows.warp.scalar", "mm.rows.warp.gridstride",
    "mm.rows.tiny.stage.v4", "mm.rows.tiny.stage.scalar", "mm.rows.tiny.rot", "mm.rows.tiny.norot",
    "mm.rows.tiny.last_group_lt32", "mm.rows.tiny.gridstride",
    "mm.tensor.v4", "mm.tensor.v4.scalar_tail", "mm.tensor.v1.off1", "mm.tensor.v1.off2", "mm.tensor.v1.off3",
    "mm.tensor.gridstride",
    "hist.v4.loop4", "hist.v4.loop1", "hist.v4.tail", "hist.scalar", "hist.gridstride",
    "hist.bins1", "hist.bins7", "hist.bins2048", "hist.bins8192", "hist.empty_range",
    "mse.bulk", "mse.nonbulk", "mse.mixed", "mse.tpr_gt1", "mse.reload", "mse.cand_pad", "mse.ncand1", "mse.ncand128",
    "mse.finish.S1", "mse.finish.S_gt1", "mse.finish.unroll4", "moments.finish.S_gt1", "moments.finish.unroll4",
    *[f"sel.hist.p{p}.ntpr{t}" for p in range(3) for t in (1, 2)],
    "sel.hist.head", "sel.hist.loop4", "sel.hist.tail", "sel.hist.gridstride",
    "sel.hist.seg65536", "sel.hist.seg32768", "sel.hist.seg16384", "sel.hist.key_mode1", "sel.hist.p0.counts",
    "sel.scan.found", "sel.scan.same_bucket",
    "sel.ranks.kmin_clamp_lo", "sel.ranks.kmin_clamp_total", "sel.ranks.kmax_clamp", "sel.ranks.tie_half_even",
    "count_sign.gridstride", "count_sign.multirow",
    "moments.tpr_gt1", "moments.centre", "moments.nocentre",
}


# -------------------------------------------------------------------------------------------------- CPU tests
def test_case_table_covers_every_branch():
    assert_table_covers(ALL_CASES, REQUIRED, lambda c: check_reach(c, c.branches(geo.SM_COUNT_H100)), __doc__,
                        reject_unknown=True)


def test_geometry_matches_documented_launches():
    """Spot values of the restated formulas, worked by hand from observe.cu / common.cuh at 132 SMs."""
    sm = geo.SM_COUNT_H100
    assert [geo.minmax_regime(i) for i in (1, 2, 64, 65, 4095, 4096, 8193)] == \
        ["cols", "tiny", "tiny", "warp", "warp", "cta", "cta"]
    # sel_seg: 6 x 132 = 792 tiles wanted; halve 65536 -> 32768 -> 16384 while rows * segments < 792
    assert geo.sel_seg(800, 100, sm) == 65536 and geo.sel_seg(792, 65536, sm) == 65536
    assert geo.sel_seg(396, 32769, sm) == 32768  # 396 x 1 < 792 <= 396 x 2
    assert geo.sel_seg(395, 32769, sm) == 16384  # 395 x 2 < 792: down to the floor
    assert geo.sel_seg(1, 10**9, sm) == 65536 and geo.sel_seg(1, 100, sm) == 16384
    # strided_finish_threads: ceil(tpr / 4) slices x nval, at most 1024, rounded up to whole warps
    assert geo.strided_finish_threads(1, 5) == 32 and 32 // 5 == 6
    assert geo.strided_finish_threads(101, 5) == 160 and 160 // 5 == 32 and 3 * 32 < 101
    assert geo.strided_finish_threads(40, 7) == 96 and 96 // 7 == 13 and 3 * 13 < 40
    assert geo.strided_finish_threads(2, 80) == 96 and 96 // 80 == 1
    assert geo.strided_finish_threads(1, 128) == 128 and geo.strided_finish_threads(1, 1) == 32
    assert geo.strided_finish_threads(10**6, 5) == 1024 and geo.strided_finish_threads(10**6, 80) == 960
    # MinMax columns: 768 channels -> 192 float4 columns, 2 x 128-thread blocks, want_y = 528
    g = geo.minmax_cols(3000, 768, True, sm)
    assert (g["gx"], g["want_y"], g["rpb"], g["grid_y"]) == (2, 528, 6, 500)
    assert geo.minmax_cols(37, 768, True, sm)["rpb"] == 1
    assert geo.hist_geometry(4_400_001, sm)["grid"] == 1056 and geo.hist_geometry(1_000_003, sm)["grid"] == 245
    assert geo.mse_workspace_bytes(600, 243, 9) == 600 * 9 * 8 and geo.mse_workspace_bytes(1, 327_675, 7) == 40 * 7 * 8


def test_finish_has_several_slices_below_17_values():
    """strided_finish_threads (common.cuh:312-319) rounds the block up to whole warps, so it never launches fewer than 32
    threads and S = blockDim / nval >= 2 for nval <= 16: with the moments' 5 values S >= 6, so moments.finish.S1 cannot
    run.  Exhaustive over the tile counts up to 2^17 and a spread of larger ones."""
    tprs = list(range(1, 1 << 17)) + [10**6, 10**9, 10**12]
    for nval in range(1, 17):
        for tpr in tprs:
            ft = geo.strided_finish_threads(tpr, nval)
            assert ft >= 32 and ft // nval >= 2, (nval, tpr, ft)
            if nval == geo.K_MOM_VALS:
                assert ft // nval >= 6 and "moments.finish.S1" not in geo.finish_branches(tpr, nval, "moments")
    assert geo.strided_finish_threads(1, 17) // 17 == 1  # the first nval with a single slice


def test_percentile_ranks_stay_in_range():
    """sb200_percentile_ranks never asks for a rank outside [0, total): kmin is clamped into [1, total] and kmax into
    [1, total] since kpos >= 0.  So select_scan's "rank beyond the population" arm (observe.cu:482-491) is reached only by
    a rank set directly.  Exhaustive over small rows (neg + pos + NaN = total) and a spread of alphas, including > 1."""
    alphas = [0.0, 1e-3, 0.1, 0.125, 0.25, 0.3, 0.5, 0.75, 0.999, 1.0, 1.5, 2.0, 10.0]
    for total in range(1, 24):
        for neg in range(total + 1):
            for pos in range(total - neg + 1):
                for a in alphas:
                    lo, hi, _ = geo.percentile_ranks(neg, pos, total, a)
                    assert 0 <= lo < total and 0 <= hi < total, (neg, pos, total, a)
    # the restated rule is Python's round(): half to even on the double product
    assert geo.percentile_ranks(10, 26, 40, 0.25)[:2] == (1, 40 - 6 - 1)
    assert geo.percentile_ranks(18, 22, 40, 0.25)[:2] == (3, 40 - 6 - 1)


# -------------------------------------------------------------------------------------------------- MinMax
def _plant_rows(x3, rng):
    """Per row of x3 [outer, C, inner] (inner > 1): the row's max and min at a head, tail or middle position that cycles
    with the row, with a magnitude drawn per row (so each channel's extreme sits in one pseudo-random row)."""
    outer, c, inner = x3.shape
    xr = x3.reshape(-1, inner)
    rows = xr.shape[0]
    d = np.array(sorted({0, 1, 2, inner // 2, inner - 3, inner - 2, inner - 1} & set(range(inner))))
    r = np.arange(rows)
    pmax = d[r % d.size]
    pmin = d[(r + 1 + d.size // 2) % d.size]
    pmin = np.where(pmin == pmax, d[(r + 1) % d.size], pmin)
    xr[r, pmax] = (8 + 4 * rng.random(rows)).astype(F32)
    xr[r, pmin] = (-8 - 4 * rng.random(rows)).astype(F32)


def _plant_cols(x3, rng, blocks):
    """inner == 1: each channel's max and min in a row that some block of the column kernel handles at a risky place:
    its first, second, third or last row, or its 1-wide tail."""
    outer, c, _ = x3.shape
    danger = sorted({r for r0, r1 in blocks for r in (r0, r0 + 1, r0 + 2, r1 - 1, r1 - (r1 - r0) % 4) if r0 <= r < r1})
    danger = np.array(danger)
    ch = np.arange(c)
    omax = danger[rng.integers(0, danger.size, c)]
    omin = danger[rng.integers(0, danger.size, c)]
    x3[omax, ch, 0] = (8 + 4 * rng.random(c)).astype(F32)
    x3[omin, ch, 0] = (-8 - 4 * rng.random(c)).astype(F32)


def _specials(x3, rng):
    """Channels 1..6 (mod C): one NaN in one row; +inf and -inf; all equal; subnormals of both signs; +-0; all -0."""
    outer, c, inner = x3.shape
    if c < 7:
        return
    x3[0, 1, 0] = np.nan  # row 1: off a 16-byte boundary whenever inner % 4 != 0 (the span head)
    x3[rng.integers(outer), 2, inner - 1] = np.inf
    x3[rng.integers(outer), 2, 0] = -np.inf
    x3[:, 3, :] = F32(0.625)
    x3[:, 4, :] = subnormals(rng, outer * inner).reshape(outer, inner)
    x3[:, 5, :] = signed_zeros(rng, outer * inner).reshape(outer, inner)
    x3[:, 6, :] = F32(-0.0)


def _mm_data(case, rng, sm, update):
    n = int(np.prod(case.spec))
    if case.op == "mmt":
        x = rng.standard_normal(n).astype(F32)
        x[n // 2] = subnormals(rng, 1)[0]
        x[1] = F32(-0.0)
        if update == 0:
            x[[0, n - 1]] = [F32(9.5), F32(-9.5)]  # head and scalar tail
        elif update == 1:
            x[[0, n - 1]] = [-np.inf, np.inf]
        else:
            x[n - 1] = np.nan
        return x
    outer, c, inner = qgeo.channel_geometry(case.spec, case.arg[0])
    x3 = rng.standard_normal((outer, c, inner)).astype(F32)
    if inner == 1:
        vec = c % 4 == 0 and case.x_off % 4 == 0
        _plant_cols(x3, rng, geo.minmax_blocks(outer, c, vec, sm))
    else:
        _plant_rows(x3, rng)
    _specials(x3, rng)
    # view [outer, C, inner] back in the case's shape with the channel on its axis
    ch_axis = case.arg[0] % len(case.spec)
    pre, post = case.spec[:ch_axis], case.spec[ch_axis + 1:]
    return x3.reshape(pre + (c,) + post)


def _mm_expected(x, ch_axis):
    """{enc(min), enc(max)} per channel, NaN poisoning the channel as {0, 0xFFFFFFFF}."""
    if ch_axis is None:
        x2 = x.reshape(1, -1)
    else:
        outer, c, inner = qgeo.channel_geometry(x.shape, ch_axis)
        x2 = x.reshape(outer, c, inner).transpose(1, 0, 2).reshape(c, -1)
    k = enc(x2)
    kmin, kmax = k.min(axis=1), k.max(axis=1)
    nan = np.isnan(x2).any(axis=1)
    kmin[nan], kmax[nan] = 0, NAN_KEY
    return np.stack([kmin, kmax], axis=1).reshape(-1).astype(U32)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(MM_CASES))
def test_minmax_branch_vs_total_order(case):
    sm = real_sm()
    check_reach(case, case.branches(sm))
    rng = np.random.default_rng(seed_of(case.name))
    ch_axis = case.arg[0] if case.op == "mm" else None
    c = 1 if ch_axis is None else case.spec[ch_axis]
    st = ops.minmax_new(c, dev())
    exp = np.full(2 * c, 0, U32)
    exp[0::2] = NAN_KEY
    for update in range(3 if case.op == "mmt" else 2):  # updates into one state == the min / max of the concatenation
        x = _mm_data(case, rng, sm, update)
        ops.minmax_update(on_device(x, case.x_off), st, ch_axis)
        e = _mm_expected(x, ch_axis)
        exp = np.stack([np.minimum(exp[0::2], e[0::2]), np.maximum(exp[1::2], e[1::2])], axis=1).reshape(-1)
        got = st.cpu().numpy().view(U32)
        bad = np.flatnonzero(got != exp)
        assert bad.size == 0, (f"{case.name}: {bad.size} state words differ; first channel {bad[0] // 2}: "
                               f"got {dec(got[bad[0]])!r} expected {dec(exp[bad[0]])!r}")
    mn, mx = ops.minmax_read(st)
    assert bits_equal(mn.cpu().numpy(), dec(exp[0::2])) and bits_equal(mx.cpu().numpy(), dec(exp[1::2]))


# -------------------------------------------------------------------------------------------------- histogram
def _hist_data(n, bins, lo, hi, rng):
    lo, hi = F32(lo), F32(hi)
    if lo == hi:
        return (signed_zeros(rng, n) if lo == 0 else np.full(n, lo, F32))
    w = float(hi) - float(lo)
    x = rng.uniform(float(lo) - 0.1 * w, float(hi) + 0.1 * w, n).astype(F32)
    edges = (lo + np.arange(bins + 1, dtype=np.float64) * (w / bins)).astype(F32)
    edges = np.concatenate([edges, (lo + (np.arange(bins + 1, dtype=F32) * ((hi - lo) / F32(bins))).astype(F32))])
    if edges.size > 4096:
        edges = rng.choice(edges, 4096, replace=False)
    near = [edges.view(np.int32) + d for d in (-2, -1, 0, 1, 2)]
    special = np.concatenate([np.concatenate(near).view(F32),
                              [lo, hi, np.nextafter(lo, -np.inf), np.nextafter(lo, np.inf),
                               np.nextafter(hi, -np.inf), np.nextafter(hi, np.inf), np.nan, np.inf, -np.inf]]).astype(F32)
    special = special[: n // 2]
    x[rng.choice(n, special.size, replace=False)] = special
    x[[0, n - 1, n - 2]] = [hi, lo, np.nan]  # the scalar head / tail elements too
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(HIST_CASES))
def test_hist_branch_vs_histc(case):
    check_reach(case, case.branches(real_sm()))
    bins, lo, hi = case.arg
    n = case.spec[0]
    rng = np.random.default_rng(seed_of(case.name))
    rg = on_device(np.float32([lo, hi]))
    counts = torch.zeros(bins, dtype=torch.int64, device=dev())
    exp = np.zeros(bins, np.int64)
    for m in (n, n // 3 + 1):  # accumulation over two calls
        x = _hist_data(m, bins, lo, hi, rng)
        ops.hist_update(on_device(x, case.x_off), rg, counts)
        exp += oobs.histc(x, bins, lo, hi)
        got = counts.cpu().numpy()
        bad = np.flatnonzero(got != exp)
        assert bad.size == 0, (case.name, m, bad[:8], got[bad[:8]], exp[bad[:8]])


# -------------------------------------------------------------------------------------------------- MSE sweep
U = 2.0 ** -24
PER_THREAD_TERMS = geo.K_MSE_TILE // geo.K_THREADS  # 32 fp32 additions per thread and tile at most


def _mse_reference(x2d, cs, cz, qmin, qmax):
    """exp[r, i] = sum_j (x - xdq_i)^2 in fp64 with xdq from oracle.qdq, and a bound on |kernel - exp| derived from the
    kernel's arithmetic (mse_err2, observe.cu:234-242, and the fp32 per-thread sums, :293-303):
      d = x - (v - zp) * s in fp32, with or without FMA contraction: |d_k - d| <= delta = e_p (1 + u) + u |d|, where
        e_p = |RN32(t s) - t s| is the rounding of the product that the oracle's xdq carries (exact in fp64);
      d_k^2 <= (|d| + delta)^2 and |d_k^2 - d^2| <= 2 |d| delta + delta^2; squaring rounds once more (u);
      each thread adds at most 32 terms in fp32: gamma_31 = 31 u / (1 - 31 u) of their sum; fp64 after that.
    So |got - exp| <= sum(2 |d| delta + delta^2) + 33 u sum((|d| + delta)^2)  (u = 2^-24)."""
    x64 = x2d.astype(np.float64)
    rows, ncand = cs.shape
    exp = np.zeros((rows, ncand))
    tol = np.zeros((rows, ncand))
    for i in range(ncand):
        xdq = oqdq.qdq(x2d, cs[:, i], cz[:, i], qmin, qmax, ch_axis=0).astype(np.float64)
        xq = oqdq.quantize_int(x2d, cs[:, i], cz[:, i], qmin, qmax, ch_axis=0).astype(np.float64)
        prod = (xq - np.rint(cz[:, i]).astype(np.float64)[:, None]) * cs[:, i].astype(np.float64)[:, None]
        ep = np.abs(xdq - prod)
        d = np.abs(x64 - xdq)
        delta = ep * (1 + U) + U * d
        exp[:, i] = (d * d).sum(axis=1)
        tol[:, i] = (2 * d * delta + delta * delta).sum(axis=1) + (PER_THREAD_TERMS + 1) * U * ((d + delta) ** 2).sum(axis=1)
    return exp, tol


def _mse_data(case, rng):
    rows, row_len = case.spec
    ncand, qmin, qmax = case.arg
    scale = rng.uniform(0.5, 3.0, rows).astype(F32)
    x = (rng.standard_normal((rows, row_len)) * scale[:, None]).astype(F32)
    cs = (scale[:, None] * rng.uniform(0.05, 0.5, (rows, ncand))).astype(F32)  # arbitrary, not powers of two
    mid = (qmin + qmax) / 2
    cz = rng.uniform(mid - 3.5, mid + 3.5, (rows, ncand)).astype(F32)       # rint'ed by the kernel, ties included
    cz[:, ::3] = np.floor(cz[:, ::3]) + F32(0.5)
    return x, cs, cz


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(MSE_CASES))
def test_mse_sweep_branch_vs_oracle(case):
    check_reach(case, case.branches(real_sm()))
    ncand, qmin, qmax = case.arg
    rng = np.random.default_rng(seed_of(case.name))
    x, cs, cz = _mse_data(case, rng)
    exp, tol = _mse_reference(x, cs, cz, qmin, qmax)
    assert np.all(tol <= 1e-5 * exp), "the derived bound must be no looser than rtol = 1e-5"
    xd, csd, czd = on_device(x, case.x_off), on_device(cs), on_device(cz)
    sse = torch.zeros(x.shape[0], ncand, dtype=torch.float64, device=dev())
    ops.mse_sweep(xd, csd, czd, qmin, qmax, sse)
    got = sse.cpu().numpy()
    err = np.abs(got - exp)
    bad = np.argwhere(err > tol)
    assert bad.size == 0, (case.name, bad[:4], got[tuple(bad[0])], exp[tuple(bad[0])], tol[tuple(bad[0])])
    again = torch.zeros_like(sse)
    ops.mse_sweep(xd, csd, czd, qmin, qmax, again)
    assert torch.equal(again, sse)  # fixed-order reduction: the same bits run to run
    base = rng.uniform(1.0, 1e3, got.shape)
    acc = torch.from_numpy(base).to(dev())
    ops.mse_sweep(xd, csd, czd, qmin, qmax, acc)  # accumulates into a non-zero sse
    assert np.array_equal(acc.cpu().numpy(), base + got)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,row_len,ncand", [(600, 243, 9), (1, 327_675, 7)])
def test_mse_workspace_contract(rows, row_len, ncand):
    """sb200_observe_mse_sweep accepts exactly sb200_mse_workspace_bytes and returns SB200_E_WORKSPACE for one byte less;
    the size matches the restated formula."""
    lib = _lib.load()
    need = int(lib.sb200_mse_workspace_bytes(rows, row_len, ncand))
    assert need == geo.mse_workspace_bytes(rows, row_len, ncand) > 0
    x = on_device(np.ones((rows, row_len), F32))
    cs, cz = on_device(np.full((rows, ncand), 0.1, F32)), on_device(np.zeros((rows, ncand), F32))
    sse = torch.zeros(rows, ncand, dtype=torch.float64, device=dev())
    ws = torch.empty(need, dtype=torch.uint8, device=dev())

    def call(nbytes):
        return lib.sb200_observe_mse_sweep(x.data_ptr(), rows, row_len, cs.data_ptr(), cz.data_ptr(), ncand, -8, 7,
                                           sse.data_ptr(), ws.data_ptr(), ctypes.c_size_t(nbytes), stream())

    assert call(need) == 0
    torch.cuda.synchronize()
    assert call(need - 1) == -4  # SB200_E_WORKSPACE
    assert b"workspace too small" in lib.sb200_last_error()


# -------------------------------------------------------------------------------------------------- radix select
def sel_keys(x, key_mode):
    """sel_key (observe.cu:333-336): NaN sorts last, key_mode 1 orders |x|."""
    k = enc(np.abs(x) if key_mode else x)
    return np.where(np.isnan(x), U32(NAN_KEY), k).astype(U32)


def key_value_bits(k):
    """select_read (observe.cu:511-518): the float of a key, the canonical NaN for the NaN key."""
    return np.where(k == NAN_KEY, U32(0x7FC00000), dec(k).view(U32)).astype(U32)


def _sel_data(case, rng):
    rows, n = case.spec
    x = (rng.standard_normal((rows, n)) * rng.uniform(0.01, 100, (rows, 1))).astype(F32)
    ranks = rng.integers(0, n, (rows, 2))
    ranks[0] = [0, n - 1]
    if rows > 1:
        ranks[1] = [n - 1, 0]
    if case.name == "sel_dups":
        for r in range(rows):  # a run of equal keys covering both ranks, and runs next to it
            a = rng.integers(0, n // 4)
            x[r, a:a + n // 2] = F32(0.37 * (r + 1))
            x[r, :n // 8] = F32(-0.37 * (r + 1))
            k = np.sort(sel_keys(x[r], 0))
            lo = int(np.searchsorted(k, enc(np.float32([0.37 * (r + 1)]))[0]))
            ranks[r] = [lo, lo + n // 2 - 1] if r % 2 else [lo + 3, lo + n // 3]
    if case.name == "sel_extremes":
        for r in range(rows):
            m = n // 10
            pos = rng.choice(n, 6 * m, replace=False).reshape(6, m)
            x[r, pos[0]] = np.nan
            x[r, pos[1]] = signed_zeros(rng, m)
            x[r, pos[2]] = subnormals(rng, m)
            x[r, pos[3]] = np.where(rng.random(m) < 0.5, np.inf, -np.inf)
            x[r, pos[4]] = F32(-0.0)
            x[r, [0, n - 1]] = [np.nan, F32(-0.0)]
            k = np.sort(sel_keys(x[r], 0))
            marks = [int(np.searchsorted(k, enc(np.float32([v]))[0], side=s))
                     for v, s in ((0.0, "left"), (-0.0, "right"), (0.0, "right"), (np.inf, "left"))]
            marks += [int(np.searchsorted(k, NAN_KEY)), n - 1, 0]
            marks = [min(max(m_, 0), n - 1) for m_ in marks]
            ranks[r] = [marks[r % len(marks)], marks[(r + 3) % len(marks)]]
    return x, np.clip(ranks, 0, n - 1)[:, : case.arg[0]]


def _run_select(x, ranks, case):
    rows, n = x.shape
    ntpr, key_mode = case.arg
    rs = ops.RadixSelect(rows, ntpr, dev(), key_mode)
    rs.set_ranks(torch.from_numpy(np.ascontiguousarray(ranks.reshape(-1))).to(dev()))
    xd = on_device(x, case.x_off)
    for p in range(3):
        rs.hist_pass(p, xd)
        rs.scan(p)
    return rs.values().cpu().numpy().view(U32).reshape(rows, ntpr)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(SEL_CASES))
def test_select_branch_vs_sort(case):
    check_reach(case, case.branches(real_sm()))
    rng = np.random.default_rng(seed_of(case.name))
    x, ranks = _sel_data(case, rng)
    ntpr, key_mode = case.arg
    keys = np.sort(sel_keys(x, key_mode), axis=1)
    kk = np.take_along_axis(keys, ranks, axis=1)
    if "sel.scan.same_bucket" in case.claims:  # (data): both targets of some row in one pass-0 bucket
        assert np.any((kk[:, 0] >> 21) == (kk[:, 1] >> 21))
    exp = key_value_bits(kk)
    got = _run_select(x, ranks, case)
    bad = np.argwhere(got != exp)
    assert bad.size == 0, (case.name, bad[:4], got[tuple(bad[0])], exp[tuple(bad[0])], ranks[bad[0][0]])


def _pct_rows(rng):
    """Rows of 40: (10 neg, 26 pos, 4 NaN), (no negatives, several +-0), (negatives only, -inf), (18 neg incl. a
    subnormal, 22 pos incl. +inf, +0 and a subnormal)."""
    def dist(k, sign):
        return (sign * rng.permutation(np.arange(1, k + 1)) * F32(0.173)).astype(F32)
    a = np.concatenate([dist(10, -1), dist(26, 1), [np.nan] * 4])
    b = np.concatenate([dist(34, 1), signed_zeros(rng, 6)])
    c = np.concatenate([dist(39, -1), [-np.inf]])
    d = np.concatenate([dist(16, -1), [F32(-1e-40), F32(-0.5e-40)], dist(19, 1), [np.inf, F32(0.0), F32(3e-41)]])
    x = np.stack([rng.permutation(v) for v in (a, b, c, d)]).astype(F32)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(PCT_CASES))
def test_percentile_path_vs_oracle(case):
    """hist_pass(0, with_counts) -> percentile_ranks -> scans, as the percentile observer runs it on one batch."""
    check_reach(case, case.branches(real_sm()))
    rng = np.random.default_rng(seed_of(case.name))
    rows, n = case.spec
    x = _pct_rows(rng) if case.name == "pct_rows" else (rng.standard_normal((rows, n)) * (1 + np.arange(rows)[:, None])).astype(F32)
    xd = on_device(x, case.x_off)
    neg, pos = (x < 0).sum(axis=1), (x >= 0).sum(axis=1)
    keys = np.sort(sel_keys(x, 0), axis=1)
    hit = set()
    for alpha in case.arg:
        rs = ops.RadixSelect(rows, 2, dev(), 0)
        rs.hist_pass(0, xd, with_counts=True)
        counts = rs.counts.cpu().numpy().reshape(rows, 2)
        assert np.array_equal(counts, np.stack([neg, pos], axis=1)), (case.name, counts)
        rs.percentile_ranks(torch.full((rows,), n, dtype=torch.int64, device=dev()), alpha)
        rs.scan(0)
        for p in (1, 2):
            rs.hist_pass(p, xd)
            rs.scan(p)
        got = rs.values().cpu().numpy().view(U32).reshape(rows, 2)
        ranks = np.zeros((rows, 2), np.int64)
        for r in range(rows):
            lo, hi, h = geo.percentile_ranks(int(neg[r]), int(pos[r]), n, alpha)
            ranks[r] = [lo, hi]
            hit |= h
        exp = key_value_bits(np.take_along_axis(keys, ranks, axis=1))
        assert np.array_equal(got, exp), (case.name, alpha, got, exp, ranks)
        if alpha <= 0.5:  # where the reference's kthvalue(k) has 1 <= k <= n
            mn = np.where(neg > 0, got[:, 0].view(F32), F32(0))
            mx = np.where(pos > 0, got[:, 1].view(F32), F32(0))
            emn, emx = oobs.percentile([x], alpha, per_channel=True)
            assert bits_equal(mn, emn) and bits_equal(mx, emx), (case.name, alpha, mn, emn, mx, emx)
    assert case.claims <= hit, (case.name, sorted(case.claims - hit))


@pytest.mark.gpu
def test_select_rank_beyond_population():
    """A rank >= n (only possible through a direct set_ranks) finds no bucket in any pass: bucket 0 is taken each time
    and the read-out is NaN (observe.cu:482-491).  Rank n - 1 in the same launch still reads the maximum."""
    x = np.float32([3.0, -1.0, 2.0, 0.5, 7.0])
    rs = ops.RadixSelect(1, 2, dev(), 0)
    rs.set_ranks(torch.tensor([5, 4], dtype=torch.int64, device=dev()))
    xd = on_device(x)
    for p in range(3):
        rs.hist_pass(p, xd.reshape(1, -1))
        rs.scan(p)
    v = rs.values().cpu().numpy()
    assert np.isnan(v[0]) and v[1] == 7.0


def _count_sign_data(rows, n, rng):
    x = rng.standard_normal((rows, n)).astype(F32)
    m = max(n // 20, 1)
    for r in range(rows):
        pos = rng.choice(n, 5 * m, replace=False).reshape(5, m)
        x[r, pos[0]] = signed_zeros(rng, m)
        x[r, pos[1]] = subnormals(rng, m)
        x[r, pos[2]] = np.where(rng.random(m) < 0.5, np.inf, -np.inf)
        x[r, pos[3]] = np.nan
        x[r, pos[4]] = F32(-0.0)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(CS_CASES))
def test_count_sign_branch_vs_numpy(case):
    """sb200_count_sign: #(x < 0) and #(x >= 0) per row (-0 counts as >= 0, NaN as neither), accumulated."""
    check_reach(case, case.branches(real_sm()))
    rng = np.random.default_rng(seed_of(case.name))
    rows, n = case.spec
    x = _count_sign_data(rows, n, rng)
    exp = np.stack([(x < 0).sum(axis=1), (x >= 0).sum(axis=1)], axis=1).reshape(-1)
    lib = _lib.load()
    xd = on_device(x)
    counts = torch.zeros(rows * 2, dtype=torch.int64, device=dev())
    assert lib.sb200_count_sign(xd.data_ptr(), rows, n, counts.data_ptr(), stream()) == 0
    assert np.array_equal(counts.cpu().numpy(), exp)
    assert lib.sb200_count_sign(xd.data_ptr(), rows, n, counts.data_ptr(), stream()) == 0
    assert np.array_equal(counts.cpu().numpy(), 2 * exp)


# -------------------------------------------------------------------------------------------------- moments
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(MOM_CASES))
def test_moments_branch_vs_fp64(case):
    check_reach(case, case.branches(real_sm()))
    rng = np.random.default_rng(seed_of(case.name))
    rows, n = case.spec
    x = (rng.standard_normal((rows, n)) * 3 + 0.5).astype(F32)
    centre = rng.standard_normal(rows) if case.arg[0] else None
    ct = torch.from_numpy(centre).to(dev()) if centre is not None else None
    out = ops.moments_update(on_device(x), ops.moments_new(rows, dev()), centre=ct)
    x64 = x.astype(np.float64)
    d = x64 - (centre[:, None] if centre is not None else 0.0)
    exp = np.stack([x64.sum(1), (x64 * x64).sum(1), np.abs(x64).sum(1), np.abs(d).sum(1), (d * d).sum(1)], axis=1)
    got = out.cpu().numpy()
    np.testing.assert_allclose(got, exp, rtol=1e-12, atol=1e-9)
    again = ops.moments_update(on_device(x), ops.moments_new(rows, dev()), centre=ct)
    assert torch.equal(again, out)


# -------------------------------------------------------------------------------------------------- KL, empty range
@pytest.mark.gpu
def test_kl_perchannel_with_all_zero_channel():
    """A pruned (all-zero) filter gives the KL observer the range [-0, +0]; its histogram takes ATen's widened range and
    every channel's min / max equals the per-tensor oracle on that channel."""
    from sparsebit_b200 import config as sbcfg
    from sparsebit_b200.quantization import build_quantizer
    from sparsebit_b200.quantization.common import Backend

    rng = np.random.default_rng(5)
    w = (rng.standard_normal((4, 3, 3, 3)) * rng.uniform(0.2, 2, (4, 1, 1, 1))).astype(F32)
    w[2] = 0.0
    w[2, 0, 0, :2] = -0.0
    q = build_quantizer(sbcfg.quantizer_config("per-channel-symmetric", 4, "weight", "kl_histogram"))
    q.set_backend(Backend.VIRTUAL)
    q.update_observer(on_device(w))
    q.calc_qparams()
    mn = q.observer.min_val.reshape(-1).cpu().numpy()
    mx = q.observer.max_val.reshape(-1).cpu().numpy()
    for c in range(4):
        emn, emx = oobs.kl_histogram([w[c]], 4)
        assert bits_equal(mn[c], emn) and bits_equal(mx[c], emx), (c, mn[c], emn, mx[c], emx)
    counts = torch.zeros(2048, dtype=torch.int64, device=dev())
    ops.hist_update(on_device(w[2].reshape(-1)), on_device(np.float32([-0.0, 0.0])), counts)
    assert counts[1024].item() == 27 and counts.sum().item() == 27  # [-1, 1]: zero lands in the middle bin
