"""Every launch branch of the fake-quant forward (csrc/qdq.cu) and STE backward (csrc/bwd.cu) kernels, each reached by
a named case and compared with the numpy oracle (oracle/qdq.py): outputs and gx bit-exact, gs / gzp against fp64 sums.

The host picks one of many kernel bodies per call from the geometry, the pointer alignment, the channel count and the
rounding mode.  tests/qdq_geometry.py restates those formulas; every case below asserts, with the SM count of the device
it runs on, that it reaches the branches it is listed for, and the CPU test at the bottom checks at 132 SMs (H100 SXM)
that the cases together reach every branch in REQUIRED.  "R-1@" marks the ROUNDING = -1 template instantiation
(rounding 1 and 2), "<tag>@" a kind of data the case feeds to that branch.

Forward, through ops.qdq_perchannel / mask_apply_qdq_perchannel / qdq_pertensor / qdq_stats_pertensor:

  branch                                  source                  case: shape, ch_axis, offsets (why it gets there)
  fwd.cols.v4.loop4                       qdq.cu:393-405          cols_v4_loop4: (16,197,768) ch 2, 6 rows per block
  fwd.cols.v4.tail                        qdq.cu:406-413          cols_v4_loop4
  fwd.cols.v1                             qdq.cu:415-416          cols_v1_odd_c: (64,197,75) ch 2; cols_v1_x_off1; cols_v1_out_off2
  fwd.chan.notab.v4.fast                  qdq.cu:170-176          notab_c4096_carry: (4096,512,3,3) ch 0, C > 2048
  fwd.chan.notab.v4.carry                 qdq.cu:198-206          notab_c4096_carry: 19 M elements, 9 grid-stride passes
  fwd.chan.notab.v4.straddle              qdq.cu:177-191          notab_straddle: (3,4099,5) ch 1
  fwd.chan.notab.v4.straddle.inner_lt4    qdq.cu:182-185          notab_inner3: (2,2500,3) ch 1
  fwd.chan.notab.v1                       qdq.cu:170-191, VEC=1   notab_v1: (3,4099,5) ch 1, x offset 3
  fwd.chan.tab.v4.nocross                 qdq.cu:142-146          tab_nocross_carry: (64,64,56,56) ch 1
  fwd.chan.tab.v4.cross1                  qdq.cu:147-155          tab_cross1_carry: (1024,64,7,7) ch 1; tab_cross1_small
  fwd.chan.tab.v4.inner_lt4               qdq.cu:156-168          tab_inner3_carry: (300000,4,3) ch 1; mask_inner1
  fwd.chan.tab.v4.carry                   qdq.cu:198-206          tab_nocross_carry, tab_cross1_carry, tab_inner3_carry (> 2.2 M)
  fwd.chan.tab.v1                         qdq.cu:142-146, VEC=1   tab_v1: (8,64,7,7) ch 1, x offset 1, out offset 2
  fwd.mask.v1                             qdq.cu:433-434          mask_misaligned: (64,32,3,3) ch 0, mask at byte offset 1
  fwd.mask.v4, fwd.mask.notab             qdq.cu:443              mask_notab: (2304,64) ch 0
  fwd.mask.inner1                         qdq.cu:501              mask_inner1: (64,96) ch 1 (the stream kernel, not cols)
  fwd.tensor.v4.scalar_tail               qdq.cu:361, 211-228     tma_16383: n = 4*4096 - 1 under variant 2 (LDG)
  fwd.tma                                 qdq.cu:251-324          tma_16384, tma_16387 under variant 2
  fwd.tma.tail                            qdq.cu:326-330          tma_16387
  R-1@<each branch above>                 ROUNDING = -1 bodies    rounding 1 and 2 on each case
  edge_scales@, ties@, zp_edges@,         common.cuh:126-190      |s| = 2^-60, 2^60 and their float neighbours, 1e-30,
  nan_inf@, qranges@ on tab, notab          (QP.fast, the exact     a subnormal, 0, a negative scale, mixed per channel;
  and cols                                  and LAZY fallbacks)     x = (k + 0.5) s +- 0..3 ulp with s not a power of two;
                                                                    zp 0.5, 1.5, 2.5, +-1000; NaN, +-inf; qmin == qmax, (0, 1)

Backward, through ops.qdq_backward.  Every case runs both zero-point rules, runs twice and must give bit-identical
gs / gzp, and runs with need_gs and need_gzp set separately:

  bwd.cols.v4.drain                       bwd.cu:242-246          cols_v4_drain: (560000,4) ch 1, 266 rows per block
  bwd.cols.v4.loop4, bwd.cols.v4.loop2    bwd.cu:233-267          cols_v4_drain; cols_bt128
  bwd.cols.v1.drain                       bwd.cu:278-282          cols_v1_drain: (560000,5) ch 1
  bwd.cols.bt64, bwd.cols.v4.tail         bwd.cu:329-333, 268-276 cols_bt64: (3000,768) ch 1
  bwd.cols.bt128                          bwd.cu:329-333          cols_bt128: (3000,512) ch 1
  bwd.cols.v1                             bwd.cu:372              cols_v1_misaligned: (3000,768) ch 1, x offset 1, gy offset 2
  bwd.finish.cols                         bwd.cu:294-319          every cols case
  bwd.finish.rows.tpr_gt1.multichannel    bwd.cu:164-170          rows_tpr3: (2,3,130,130) ch 1, 3 tiles per row; rows_inner8193
  bwd.finish.rows.tpr_gt1                 bwd.cu:164-170          pertensor: (2000003,), one channel
  bwd.finish.rows.tpr1                    bwd.cu:158-163          rows_inner8192: (3,5,8192) ch 1
  bwd.rows.inner_eq_ktile                 bwd.cu:105, 113         rows_inner8192
  bwd.rows.partial_last_tile              bwd.cu:113              rows_inner8193: (3,5,8193) ch 1
  bwd.span.head                           bwd.cu:60-62            rows_inner8193 (odd rows start off a 16-byte boundary)
  bwd.span.scalar                         bwd.cu:56-59            rows_scalar_span: (4,6,40,40) ch 1, x 1 / gy 2; rows_warp_scalar
  bwd.rows.cta                            bwd.cu:396              rows_tpr3, rows_scalar_span, pertensor
  bwd.rows.warp                           bwd.cu:108              rows_warp: (16,8,7,7) ch 1; rows_warp_scalar
  R-1@, ties@, qedges@, nan_inf@          bwd.cu:32-46            rounding 1 / 2, x = (k + 0.5) s +- ulps, vq exactly on
                                                                    qmin / qmax, NaN and +-inf in x

The two-row loop's drain (bwd.cu:262-266) cannot run: the four-row loop leaves k a multiple of four below 256, and the
two-row loop runs at most once after it (test_bwd_cols_two_row_drain_is_unreachable).
"""
import ctypes
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import qdq_geometry as geo
from branch_cases import assert_table_covers, fs
from gpu_util import bits_equal, dev, on_device, real_sm, seed_of
from oracle import qdq as oqdq
from oracle import sparse as osparse
from sparsebit_b200 import _lib, ops

F32 = np.float32

# -------------------------------------------------------------------------------------------------- data
# |s| in [2^-60, 2^60] takes the fp32 fast path (QP.fast, common.cuh:132); its float neighbours on both sides, tiny,
# subnormal, zero and negative scales do not, or stress it.  Mixed into one tensor, so table entries disagree on `fast`.
EDGE_SCALES = np.array([
    2.0 ** -60, np.nextafter(F32(2.0 ** -60), F32(0)), np.nextafter(F32(2.0 ** -60), F32(1)),
    2.0 ** 60, np.nextafter(F32(2.0 ** 60), F32(0)), np.nextafter(F32(2.0 ** 60), F32(np.inf)),
    1e-30, 1e-40, 0.0, -0.037, 0.25, 1.0 / 3.0,
], dtype=F32)
EDGE_ZPS = np.array([0.5, 1.5, 2.5, -0.5, -1.5, 1000.0, -1000.0], dtype=F32)  # rint ties, far outside the range


def _spread(c, values, shift):
    """Channel indices for len(values) special entries, spread over c channels (fewer if c is small)."""
    k = min(len(values), max(c // 2, 1))
    return (np.linspace(0, c - 1, k).astype(np.int64) + shift) % c, values[:k]


def make_qparams(c, rng, data):
    s = rng.uniform(0.004, 0.06, c).astype(F32)  # not powers of two: the fast quotient is inexact
    z = np.rint(rng.uniform(-3, 3, c)).astype(F32)
    if "edge_scales" in data:
        idx, v = _spread(c, EDGE_SCALES, 0)
        s[idx] = v
    if "zp_edges" in data:
        idx, v = _spread(c, EDGE_ZPS, 1)
        z[idx] = v
    return s, z


def make_x(shape, ch_axis, s, z, rng, data, qmin=-128, qmax=127):
    """x = (k + f) * s_c with k spanning past [qmin, qmax]; 'ties': a quarter of the elements at (k + 0.5) * s_c moved by
    -3..3 ulp; 'qedges': vq exactly qmin / qmax; 'nan_inf': NaN and +-inf sprinkled in."""
    n = int(np.prod(shape))
    if ch_axis is None:
        sc, zc = np.full(n, s[0], F32), np.full(n, np.rint(z[0]), F32)
    else:
        outer, c, inner = geo.channel_geometry(shape, ch_axis)
        ch = (np.arange(n, dtype=np.int64) // inner) % c
        sc, zc = s[ch], np.rint(z)[ch]
    k = rng.integers(qmin - 8, qmax + 8, n, dtype=np.int32).astype(F32) - zc
    x = ((k + rng.uniform(-0.5, 0.5, n).astype(F32)) * sc).astype(F32)
    if "ties" in data:
        sel = rng.random(n) < 0.25
        xt = ((k[sel] + F32(0.5)) * sc[sel]).astype(F32)
        d = rng.integers(-3, 4, xt.size, dtype=np.int32)
        d[np.abs(xt) == 0] = 0
        x[sel] = (xt.view(np.int32) + d).view(F32)
    if "qedges" in data:
        sel = np.flatnonzero(rng.random(n) < 0.02)
        lo = rng.random(sel.size) < 0.5
        x[sel] = (np.where(lo, F32(qmin) - zc[sel], F32(qmax) - zc[sel]) * sc[sel]).astype(F32)
    zero = sc == 0
    x[zero] = rng.standard_normal(int(zero.sum())).astype(F32)
    if "nan_inf" in data:
        sel = rng.choice(n, size=max(3, n // 5000), replace=False)
        x[sel] = np.array([np.nan, np.inf, -np.inf], F32)[np.arange(sel.size) % 3]
    return x.reshape(shape)


def empty_at(shape, offset):
    n = int(np.prod(shape))
    return torch.empty(n + offset, dtype=torch.float32, device=dev())[offset:].view(shape)


# -------------------------------------------------------------------------------------------------- case tables
ALL_FWD_DATA = ("edge_scales", "ties", "zp_edges", "nan_inf")
BWD_DATA = ("ties", "qedges", "nan_inf", "gzp_rules", "determinism", "need_split")


@dataclass(frozen=True)
class FwdCase:
    name: str
    op: str  # perchannel | mask | pertensor
    shape: tuple
    ch_axis: object
    targets: frozenset
    roundings: tuple = (0, 1, 2)
    data: tuple = ALL_FWD_DATA
    x_off: int = 0
    out_off: int = 0
    mask_off: int = 0
    variant: int = 0

    def branches(self, sm):
        return geo.fwd_branches(self.op, self.shape, self.ch_axis, sm, self.x_off, self.out_off, self.mask_off, self.variant)


@dataclass(frozen=True)
class BwdCase:
    name: str
    shape: tuple
    ch_axis: object
    targets: frozenset
    roundings: tuple = (0, 1, 2)
    data: tuple = BWD_DATA
    x_off: int = 0
    gy_off: int = 0

    def branches(self, sm):
        return geo.bwd_branches(self.shape, self.ch_axis, sm, self.x_off, self.gy_off)


FWD_CASES = [
    FwdCase("cols_v4_loop4", "perchannel", (16, 197, 768), 2, fs("fwd.cols.v4.loop4", "fwd.cols.v4.tail")),
    FwdCase("cols_v1_odd_c", "perchannel", (64, 197, 75), 2, fs("fwd.cols.v1")),
    FwdCase("cols_v1_x_off1", "perchannel", (16, 197, 768), 2, fs("fwd.cols.v1"), (0, 1), x_off=1),
    FwdCase("cols_v1_out_off2", "perchannel", (16, 197, 768), 2, fs("fwd.cols.v1"), (2,), out_off=2),
    FwdCase("notab_c4096_carry", "perchannel", (4096, 512, 3, 3), 0, fs("fwd.chan.notab.v4.fast", "fwd.chan.notab.v4.carry")),
    FwdCase("notab_straddle", "perchannel", (3, 4099, 5), 1, fs("fwd.chan.notab.v4.straddle", "fwd.chan.v4.scalar_tail")),
    FwdCase("notab_inner3", "perchannel", (2, 2500, 3), 1, fs("fwd.chan.notab.v4.straddle.inner_lt4")),
    FwdCase("notab_v1", "perchannel", (3, 4099, 5), 1, fs("fwd.chan.notab.v1"), x_off=3),
    FwdCase("tab_nocross_carry", "perchannel", (64, 64, 56, 56), 1, fs("fwd.chan.tab.v4.nocross", "fwd.chan.tab.v4.carry")),
    FwdCase("tab_cross1_carry", "perchannel", (1024, 64, 7, 7), 1, fs("fwd.chan.tab.v4.cross1", "fwd.chan.tab.v4.carry")),
    FwdCase("tab_inner3_carry", "perchannel", (300_000, 4, 3), 1, fs("fwd.chan.tab.v4.inner_lt4", "fwd.chan.tab.v4.carry")),
    FwdCase("tab_cross1_small", "perchannel", (8, 64, 7, 7), 1, fs("fwd.chan.tab.v4.cross1")),
    FwdCase("tab_v1", "perchannel", (8, 64, 7, 7), 1, fs("fwd.chan.tab.v1"), x_off=1, out_off=2),
    FwdCase("mask_misaligned", "mask", (64, 32, 3, 3), 0, fs("fwd.mask.v1", "fwd.mask.tab"), mask_off=1),
    FwdCase("mask_notab", "mask", (2304, 64), 0, fs("fwd.mask.v4", "fwd.mask.notab"), (0, 1)),
    FwdCase("mask_inner1", "mask", (64, 96), 1, fs("fwd.mask.v4", "fwd.mask.inner1", "fwd.chan.tab.v4.inner_lt4"), (0, 2)),
    FwdCase("tma_16383", "pertensor", (4 * 4096 - 1,), None, fs("fwd.tensor.v4.scalar_tail"), (1, 2), ("ties",), variant=2),
    FwdCase("tma_16384", "pertensor", (4 * 4096,), None, fs("fwd.tma"), data=("ties", "nan_inf"), variant=2),
    FwdCase("tma_16387", "pertensor", (4 * 4096 + 3,), None, fs("fwd.tma", "fwd.tma.tail"), data=("ties", "nan_inf"), variant=2),
]
QRANGE_CASES = ["cols_v4_loop4", "notab_straddle", "tab_cross1_small"]
QRANGES = [(3, 3), (0, 1)]

BWD_CASES = [
    BwdCase("cols_v4_drain", (560_000, 4), 1, fs("bwd.cols.v4.drain", "bwd.cols.v4.loop4", "bwd.cols.v4.loop2", "bwd.finish.cols")),
    BwdCase("cols_v1_drain", (560_000, 5), 1, fs("bwd.cols.v1.drain", "bwd.finish.cols")),
    BwdCase("cols_bt64", (3000, 768), 1, fs("bwd.cols.bt64", "bwd.cols.v4.loop4", "bwd.cols.v4.tail"), (0, 1)),
    BwdCase("cols_bt128", (3000, 512), 1, fs("bwd.cols.bt128", "bwd.cols.v4.loop2", "bwd.cols.v4.tail"), (0, 2)),
    BwdCase("cols_v1_misaligned", (3000, 768), 1, fs("bwd.cols.v1"), (0, 1), x_off=1, gy_off=2),
    BwdCase("rows_tpr3", (2, 3, 130, 130), 1, fs("bwd.rows.cta", "bwd.finish.rows.tpr_gt1.multichannel")),
    BwdCase("rows_inner8192", (3, 5, 8192), 1, fs("bwd.rows.inner_eq_ktile", "bwd.finish.rows.tpr1"), (0, 1)),
    BwdCase("rows_inner8193", (3, 5, 8193), 1, fs("bwd.rows.partial_last_tile", "bwd.span.head",
                                                  "bwd.finish.rows.tpr_gt1.multichannel"), (0, 2)),
    BwdCase("rows_warp", (16, 8, 7, 7), 1, fs("bwd.rows.warp")),
    BwdCase("rows_scalar_span", (4, 6, 40, 40), 1, fs("bwd.rows.cta", "bwd.span.scalar"), (0, 1), x_off=1, gy_off=2),
    BwdCase("rows_warp_scalar", (16, 8, 7, 7), 1, fs("bwd.rows.warp", "bwd.span.scalar"), (0, 2), gy_off=3),
    BwdCase("pertensor", (2_000_003,), None, fs("bwd.rows.cta", "bwd.finish.rows.tpr_gt1"), (1, 2)),
]

# Every branch the suite must reach (see the docstring for where each lives).
_FWD_CORE = ["fwd.cols.v4.loop4", "fwd.cols.v4.tail", "fwd.cols.v1",
             "fwd.chan.notab.v4.fast", "fwd.chan.notab.v4.carry", "fwd.chan.notab.v4.straddle",
             "fwd.chan.notab.v4.straddle.inner_lt4", "fwd.chan.notab.v1",
             "fwd.chan.tab.v4.nocross", "fwd.chan.tab.v4.cross1", "fwd.chan.tab.v4.inner_lt4", "fwd.chan.tab.v4.carry",
             "fwd.chan.tab.v1", "fwd.mask.v1", "fwd.mask.v4", "fwd.mask.notab", "fwd.mask.inner1",
             "fwd.tensor.v4.scalar_tail", "fwd.tma", "fwd.tma.tail"]
_FWD_DATA_AT = ["fwd.chan.tab.v4.nocross", "fwd.chan.notab.v4.fast", "fwd.cols.v4.loop4"]
_BWD_CORE = ["bwd.cols.v4.drain", "bwd.cols.v1.drain", "bwd.cols.v4.loop4", "bwd.cols.v4.loop2", "bwd.cols.v4.tail",
             "bwd.cols.bt64", "bwd.cols.bt128", "bwd.cols.v1", "bwd.finish.cols",
             "bwd.finish.rows.tpr_gt1.multichannel", "bwd.finish.rows.tpr_gt1", "bwd.finish.rows.tpr1",
             "bwd.rows.inner_eq_ktile", "bwd.rows.partial_last_tile", "bwd.rows.cta", "bwd.rows.warp",
             "bwd.span.scalar", "bwd.span.head"]
_BWD_KERNELS = ["bwd.rows.cta", "bwd.rows.warp", "bwd.cols.v4.drain", "bwd.cols.v1.drain"]
REQUIRED = set(_FWD_CORE) | set(_BWD_CORE)
REQUIRED |= {"R-1@" + b for b in _FWD_CORE if b not in ("fwd.tensor.v4.scalar_tail",)} | {"R-1@" + b for b in _BWD_KERNELS}
REQUIRED |= {f"{d}@{b}" for d in ALL_FWD_DATA for b in _FWD_DATA_AT}
REQUIRED |= {f"qranges@{b}" for b in ("fwd.cols.v4.loop4", "fwd.chan.notab.v4.straddle", "fwd.chan.tab.v4.cross1")}
REQUIRED |= {f"ties@{b}" for b in ("fwd.chan.tab.v4.cross1", "fwd.chan.tab.v4.inner_lt4", "fwd.chan.notab.v4.straddle",
                                   "fwd.cols.v1", "fwd.tma")}
REQUIRED |= {f"{d}@{b}" for d in BWD_DATA for b in _BWD_KERNELS}
REQUIRED |= {f"{d}@bwd.finish.rows.tpr_gt1.multichannel" for d in ("determinism", "need_split")}


def case_coverage(case, sm):
    """The ids a case stands for: its targets (which must be among the branches it reaches), their R-1@ forms when it
    runs rounding 1 or 2, and <data>@ forms for the data it feeds them."""
    reached = case.branches(sm)
    assert case.targets <= reached, f"{case.name} at {sm} SMs reaches {sorted(reached)}, not {sorted(case.targets - reached)}"
    out = set()
    for r in case.roundings:
        out |= geo.with_rounding(case.targets, r)
    data = case.data + (("qranges",) if case.name in QRANGE_CASES else ())
    out |= {f"{d}@{b}" for d in data for b in case.targets}
    return out


# -------------------------------------------------------------------------------------------------- CPU: coverage
def test_case_table_covers_every_branch():
    # the docstring table names every case and every branch; R-1@ and <data>@ ids through the branch they qualify
    assert_table_covers(FWD_CASES + BWD_CASES, REQUIRED, lambda c: case_coverage(c, geo.SM_COUNT_H100), __doc__,
                        doc_alias=lambda b: b.split("@")[-1])


def test_bwd_cols_two_row_drain_is_unreachable():
    """bwd.cu:262-266 never fires: after the four-row loop k is a multiple of 4 below 256 and the two-row loop runs at most
    once, so k + 2 < 256.  Exhaustive over the row-block sizes the grid can produce."""
    for rows in range(1, 4 * geo.BWD_DRAIN_ROWS + 8):
        assert "loop2.drain" not in geo.bwd_cols_row_loop(rows, True)
    assert "drain" in geo.bwd_cols_row_loop(256, True) and "drain" not in geo.bwd_cols_row_loop(255, True)
    assert "drain" in geo.bwd_cols_row_loop(256, False) and "drain" not in geo.bwd_cols_row_loop(255, False)


def test_geometry_matches_documented_launches():
    """Spot values of the restated formulas, worked by hand from qdq.cu / bwd.cu at 132 SMs."""
    sm = geo.SM_COUNT_H100
    assert geo.launch_cols(16 * 197, 768, True, sm)["rpb"] == 6
    assert geo.launch_cols(4 * 197, 768, True, sm)["rpb"] == 2
    g = geo.launch_stream(4096 * 512 * 9, 4096, 512 * 9, True, sm, True)
    assert (g["grid"], g["use_tab"], g["iterations"]) == (528, False, 9)
    assert geo.cols_block_threads(768) == 64 and geo.cols_block_threads(512) == 128
    nb = geo.cols_row_blocks(560_000, 4, sm)
    assert -(-560_000 // nb) == 266
    assert -(-560_000 // geo.cols_row_blocks(560_000, 5, sm)) >= 256


# -------------------------------------------------------------------------------------------------- GPU: forward
def _fwd_params():
    return [pytest.param(c, r, id=f"{c.name}-r{r}") for c in FWD_CASES for r in c.roundings]


def _run_fwd(case, rounding, qmin=-128, qmax=127):
    assert case.targets <= case.branches(real_sm()), (case.name, sorted(case.branches(real_sm())))
    rng = np.random.default_rng(seed_of(case.name, rounding, qmin, qmax))
    if case.op == "pertensor":
        s = np.float32([0.0173])
        z = np.float32([2.5])
    else:
        s, z = make_qparams(case.shape[case.ch_axis], rng, case.data)
    x = make_x(case.shape, case.ch_axis, s, z, rng, case.data, qmin, qmax)
    xd = on_device(x, case.x_off)
    out = empty_at(case.shape, case.out_off)
    sd, zd = on_device(s), on_device(z)
    if case.op == "perchannel":
        y = ops.qdq_perchannel(xd, sd, zd, qmin, qmax, case.ch_axis, rounding, out=out)
        exp = oqdq.qdq(x, s, z, qmin, qmax, case.ch_axis, rounding)
    elif case.op == "mask":
        m = rng.random(case.shape) < 0.6
        md = on_device(m.astype(np.uint8), case.mask_off)
        y = ops.mask_apply_qdq_perchannel(xd, md, sd, zd, qmin, qmax, case.ch_axis, rounding, out=out)
        with np.errstate(invalid="ignore"):  # inf * 0 for masked-out infinities is NaN, as on the device
            exp = oqdq.qdq(osparse.mask_apply(x, m), s, z, qmin, qmax, case.ch_axis, rounding)
    else:
        lib = _lib.load()
        assert lib.sb200_set_variant(case.variant) == 0
        try:
            y = ops.qdq_pertensor(xd, sd, zd, qmin, qmax, rounding, out=out)
            st = ops.minmax_new(1, dev())
            y2 = ops.qdq_stats_pertensor(xd, sd, zd, qmin, qmax, st, rounding, out=empty_at(case.shape, case.out_off))
            mn, mx = ops.minmax_read(st)
        finally:
            lib.sb200_set_variant(0)
        assert bits_equal(y2.cpu().numpy(), y.cpu().numpy())
        with np.errstate(invalid="ignore"):
            emn, emx = (np.nan, np.nan) if np.isnan(x).any() else (x.min(), x.max())
        assert bits_equal(np.float32([float(mn), float(mx)]), np.float32([emn, emx]))
        exp = oqdq.qdq(x, s, z, qmin, qmax, 0, rounding)
    got = y.cpu().numpy()
    if not bits_equal(got, exp):
        bad = np.flatnonzero(~((got == exp) | (np.isnan(got) & np.isnan(exp))).reshape(-1))
        i = bad[0]
        raise AssertionError(f"{case.name} r{rounding}: {bad.size} of {got.size} differ; first at flat {i}: "
                             f"x={x.reshape(-1)[i]!r} got={got.reshape(-1)[i]!r} expected={exp.reshape(-1)[i]!r}")


@pytest.mark.gpu
@pytest.mark.parametrize("case,rounding", _fwd_params())
def test_forward_branch_vs_oracle(case, rounding):
    _run_fwd(case, rounding)


@pytest.mark.gpu
@pytest.mark.parametrize("name", QRANGE_CASES)
@pytest.mark.parametrize("qrange", QRANGES, ids=lambda q: f"q{q[0]}_{q[1]}")
def test_forward_degenerate_ranges(name, qrange):
    """qmin == qmax (every element clamps to one grid point) and the 1-bit range (0, 1)."""
    case = next(c for c in FWD_CASES if c.name == name)
    _run_fwd(case, 0, *qrange)
    _run_fwd(case, 1, *qrange)


# -------------------------------------------------------------------------------------------------- GPU: backward
def _bwd_params():
    return [pytest.param(c, r, id=f"{c.name}-r{r}") for c in BWD_CASES for r in c.roundings]


def _l1_bounds(x, s, z, gy, qmin, qmax, ch_axis):
    """Per-channel L1 norms bounding the summed terms (test_gpu_reference_ext.py::_close): gs terms are at most
    max(|qmin - zp|, |qmax - zp|, 1) |gy|, gzp terms |s| |gy|."""
    g = np.abs(gy).astype(np.float64)
    zr = np.rint(z).astype(np.float64)
    w = np.maximum(np.maximum(np.abs(qmin - zr), np.abs(qmax - zr)), 1.0)
    if ch_axis is None:
        l1g = np.array([g.sum()])
    else:
        l1g = g.sum(axis=tuple(a for a in range(x.ndim) if a != ch_axis))
    return l1g * w, l1g * np.abs(s.astype(np.float64))


def _close(got, exp, l1):
    got = np.asarray(got, np.float64).reshape(-1)
    exp = np.asarray(exp, np.float64).reshape(-1)
    ok = np.abs(got - exp) <= 1e-6 * (l1 + 1e-30)
    return bool(np.all(ok)), np.flatnonzero(~ok)[:8]


@pytest.mark.gpu
@pytest.mark.parametrize("case,rounding", _bwd_params())
def test_backward_branch_vs_oracle(case, rounding):
    assert case.targets <= case.branches(real_sm()), (case.name, sorted(case.branches(real_sm())))
    qmin, qmax = -16, 15
    rng = np.random.default_rng(seed_of(case.name, rounding))
    c = 1 if case.ch_axis is None else case.shape[case.ch_axis]
    s = rng.uniform(0.01, 0.05, c).astype(F32)
    z = np.rint(rng.uniform(-3, 3, c)).astype(F32)
    x = make_x(case.shape, case.ch_axis, s, z, rng, case.data, qmin, qmax)
    gy = rng.standard_normal(case.shape).astype(F32)
    xd, gyd, sd, zd = on_device(x, case.x_off), on_device(gy, case.gy_off), on_device(s), on_device(z)
    l1s, l1z = _l1_bounds(x, s, z, gy, qmin, qmax, case.ch_axis)
    for closed in (False, True):
        # per-tensor: closed interval always (sb200_qdq_pertensor_bwd); per-channel: the flag picks the rule
        open_top = (not closed) and case.ch_axis is not None
        with np.errstate(invalid="ignore"):  # inf - inf for the +-inf inputs, discarded by the oracle's own mask
            egx, egs, egz = oqdq.ste_backward(x, s, z, gy, qmin, qmax, case.ch_axis or 0, rounding, gzp_open_top=open_top)
        kw = dict(ch_axis=case.ch_axis, rounding=rounding, gzp_closed=closed)
        gx, gs, gz = ops.qdq_backward(xd, sd, zd, gyd, qmin, qmax, **kw)
        gx2, gs2, gz2 = ops.qdq_backward(xd, sd, zd, gyd, qmin, qmax, **kw)
        assert bits_equal(gx.cpu().numpy(), egx), (case.name, closed)
        ok, bad = _close(gs.cpu().numpy(), egs, l1s)
        assert ok, (case.name, closed, "gs", bad, gs.cpu().numpy().reshape(-1)[bad], egs.reshape(-1)[bad])
        ok, bad = _close(gz.cpu().numpy(), egz, l1z)
        assert ok, (case.name, closed, "gzp", bad, gz.cpu().numpy().reshape(-1)[bad], egz.reshape(-1)[bad])
        # fixed-order reductions: a second run gives the same bits
        assert torch.equal(gx, gx2) and torch.equal(gs, gs2) and torch.equal(gz, gz2), (case.name, closed)
        # only the requested gradient is written, and it equals the full run bit for bit
        _, gs_only, gz_none = ops.qdq_backward(xd, sd, zd, gyd, qmin, qmax, need_gzp=False, **kw)
        _, gs_none, gz_only = ops.qdq_backward(xd, sd, zd, gyd, qmin, qmax, need_gs=False, **kw)
        assert torch.equal(gs_only, gs) and torch.equal(gz_only, gz), (case.name, closed)
        assert not gz_none.any() and not gs_none.any(), (case.name, closed)
    assert np.any(egx == 0) and np.any(egx != 0)  # the data clips and passes


@pytest.mark.gpu
@pytest.mark.parametrize("shape,ch_axis", [((3000, 768), 1), ((2, 3, 130, 130), 1)], ids=["cols", "rows"])
def test_backward_workspace_contract(shape, ch_axis):
    """sb200_qdq_perchannel_bwd accepts exactly sb200_qdq_bwd_workspace_bytes and returns SB200_E_WORKSPACE for one byte
    less; the size matches the restated formula."""
    lib = _lib.load()
    outer, c, inner = geo.channel_geometry(shape, ch_axis)
    need = int(lib.sb200_qdq_bwd_workspace_bytes(outer, c, inner))
    assert need == geo.bwd_ws_bytes(outer, c, inner, real_sm()) > 0
    rng = np.random.default_rng(1)
    x = on_device(rng.standard_normal(shape).astype(F32))
    gy = on_device(rng.standard_normal(shape).astype(F32))
    s, z = on_device(np.full(c, 0.02, F32)), on_device(np.zeros(c, F32))
    gx, gs, gz = torch.empty_like(x), torch.empty(c, device=dev()), torch.empty(c, device=dev())
    ws = torch.empty(need, dtype=torch.uint8, device=dev())
    stream = torch.cuda.current_stream().cuda_stream

    def call(nbytes):
        return lib.sb200_qdq_perchannel_bwd(x.data_ptr(), s.data_ptr(), z.data_ptr(), gy.data_ptr(), gx.data_ptr(),
                                            gs.data_ptr(), gz.data_ptr(), outer, c, inner, -128, 127, 0, ws.data_ptr(),
                                            ctypes.c_size_t(nbytes), stream)

    assert call(need) == 0
    torch.cuda.synchronize()
    assert call(need - 1) == -4  # SB200_E_WORKSPACE
    assert b"workspace too small" in lib.sb200_last_error()
