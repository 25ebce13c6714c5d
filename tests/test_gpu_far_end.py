"""The fake-quant forward (csrc/qdq.cu), STE and PACT clamp backward (csrc/bwd.cu, csrc/multi.cu) and observer
(csrc/observe.cu) kernels on tensors of more than 2^31 elements, and the observers on more than 2^32.

The C-ABI gives these kernels int64 sizes, and activations reach that size: the fp32 logits of 8 x 4096 tokens over a
128256-word vocabulary are 4.2e9 elements.  The code that only matters there is the index arithmetic past 2^31: the
per-channel cursor of stream_kernel (advanced once per grid step), the chunk grid of the per-tensor kernel, the TMA
ring's tile offsets, the row blocks of the channel-last kernels, the per-CTA 32-bit shared-memory counters of the
histogram and radix-select kernels flushed into 64-bit counts, the fp32-then-fp64 sums of gs / gzp, and the ranks of the
percentile path.  Each case below runs one entry point just past the bound and names the launch regime it must reach,
as tests/qdq_geometry.py and tests/observe_geometry.py restate it; the CPU test checks the table.

  case            entry point                          shape (ch_axis)            regime
  pt_v4           ops.qdq_pertensor                    2^31 + 6147                LDG chunks, VEC 4, n % 4 tail
  pt_v1           ops.qdq_pertensor                    2^31 + 6147, x / out + 1   LDG chunks, VEC 1
  pt_tma          ops.qdq_pertensor, variant 2         2^31 + 6147                TMA ring and its tail
  stats_v4        ops.qdq_stats_pertensor              2^31 + 6147                fused MinMax, VEC 4
  stats_v1        ops.qdq_stats_pertensor              2^31 + 6147, x / out + 1   fused MinMax, VEC 1
  chan_tab        ops.qdq_perchannel                   (10701, 64, 56, 56) (1)    channel table, VEC 4, cursor carry
  chan_notab      ops.qdq_perchannel                   (74845, 4099, 7) (1)       C > 2048, straddling vectors
  chan_inner3     ops.qdq_perchannel                   (238609295, 3, 3) (1)      inner < 4: the per-element loop
  cols_v4         ops.qdq_perchannel                   (524289, 4096) (-1)        channel-last, VEC 4
  cols_v1         ops.qdq_perchannel                   (523905, 4099) (-1)        channel-last, scalar
  bwd_pt          sb200_qdq_pertensor_bwd              2^31 + 6147                CTA tiles, 262145 tiles
  bwd_rows_cta    sb200_qdq_perchannel_bwd_ex          (65, 13, 2541401) (1)      CTA tiles; both zero-point rules
  bwd_rows_warp   sb200_qdq_perchannel_bwd_ex          (695655, 63, 7, 7) (1)     warp tiles
  bwd_cols_v4     sb200_qdq_perchannel_bwd_ex          (524289, 4096) (-1)        channel-last, VEC 4, 256-row drains
  bwd_cols_v1     sb200_qdq_perchannel_bwd_ex          (523905, 4099) (-1)        channel-last, scalar
  clamp           sb200_clamp_bwd (PACT)               2^31 + 6147                VEC 4, fp32 flushes every 64 steps
  mm_tensor       ops.minmax_update                    2^32 + 3                   stream kernel, VEC 4
  mm_cta          ops.minmax_update                    (3, 7, 102261127) (1)      minmax regime cta
  mm_warp         ops.minmax_update                    (33257, 63, 1025) (1)      minmax regime warp
  mm_tiny         ops.minmax_update                    (695655, 63, 7, 7) (1)     minmax regime tiny
  mm_cols         ops.minmax_update                    (524289, 4096) (-1)        minmax regime cols
  hist_random     ops.hist_update, 2048 bins           2^32 + 3                   VEC 4, grid stride
  hist_const      ops.hist_update, range [0.5, 0.5]    2^32 + 3                   every element in bin 1024
  mse_tensor      ops.mse_sweep, 80 candidates         (1, 2^31 + 6147)           one row, 262145 tiles
  mse_rows        ops.mse_sweep, 80 candidates         (4101, 524161)             64 tiles per row, 4 rows past 2^31
  kth_key0        ops.kth_value, key mode 0            2^31 + 6147                one target, 65536-element segments
  kth_key1        ops.kth_value, key mode 1            2^31 + 6147                the same on |x|
  pct             percentile observer, per tensor      2^31 + 6147                two targets, a rank past 2^31

How each is checked.  Inputs come from a seeded torch.Generator on the device; outputs start as a sentinel NaN.  Ties
(k + 1/2) s and values outside the clamp range are planted in windows of whole channel rows (inner elements of one
channel): the head, the rows around element 2^31 and the last rows with the n % 4 tail; -inf at 2^31 + 5, +inf at
n - 1 and, but for the fused MinMax cases, a NaN at 2^31 + 1.
* Elementwise outputs (y, gx): each window bit for bit against oracle/qdq.py with its true channel indices, and the
  whole tensor against launches of the same entry point on consecutive 16-byte aligned sub-ranges of whole slabs of at
  most 2^28 elements, far below the index ranges under test, compared on the device.
* MinMax: the global extremes past 2^31 (2^31 + 5 and n - 1), per channel in the last slab; exact against chunked
  torch.aminmax.
* Histogram: the counts equal the sum of the sub-range launches' counts and add up to the in-range element count; the
  constant tensor gives counts[1024] == n > 2^32.
* k-th value and percentile: by counting in the kernel's key order, #(key < v) <= k < #(key <= v); the percentile
  observer's qparams equal oracle.observers.calc_qparams_with_minmax of the order statistics so found.
* fp64 reductions (gs, gzp, PACT's g_hi / g_lo, MSE losses): tests/far_end_ref.py restates the oracle's terms in torch
  and sums them in chunks; gs / gzp / g_hi / g_lo within 1e-5 of the terms' L1 norm, MSE losses within 1e-5 relative
  with the same best candidate.  The elements past 2^31 are a few thousand of 2^31, so they are made heavy enough to
  move these sums past the bar: gy past 2^31 is scaled by 4096, the one-row MSE case holds +-12 there (outside every
  clip range, >= 1e-3 of every candidate's loss), and the many-row MSE case has whole rows past 2^31.  Each
  restatement equals its numpy oracle on a small tensor (CPU tests below).

The 65535 cap on gridDim.y of the channel-last kernels cannot bind on an H100: they want ceil(8 SMs / gridDim.x) <= 1056
row blocks.  Each GPU test states its device-memory need and skips when the device has less free; the largest, the
backward cases, hold x, gy and gx (25.8 GB) plus one chunk of the fp64 reference.  The host refusal of a per-tensor QDQ
that needs more than 2^31 - 1 chunk CTAs is checked on the CPU with fake pointers.
"""
import functools
import gc

import numpy as np
import pytest
import torch

import far_end_ref as ref
import observe_geometry as ogeo
import qdq_geometry as qgeo
import weight_geometry as wgeo
from branch_cases import C, assert_table_covers, check_reach, params
from gpu_util import bits_equal, dev, real_sm, seed_of, stream
from int8_harness import E_INVALID, buf
from oracle import observers as oobs
from oracle import qdq as oqdq
from sparsebit_b200 import _lib, ops

F32 = np.float32
B31, B32 = 1 << 31, 1 << 32
N31 = B31 + 6147
N32 = B32 + 3
SUB = 1 << 28          # elements per sub-range launch at most
WIN = 1 << 16          # elements per oracle window, about
SENTINEL = 0x7FA5A5A5  # a NaN no kernel writes
GIB = 1 << 30
# gy past element 2^31 is scaled by this, so that those few thousand elements move gs / gzp / g_hi / g_lo by far more
# than the 1e-5-of-L1 bar (at unit scale they would be below it)
TAIL_GY = 4096.0
MSE_TAIL = 12.0  # |x| past 2^31 in the one-row MSE case: clipped by every candidate


# -------------------------------------------------------------------------------------------------- cases
def _fwd(name, op, shape, ch, targets, **kw):
    return C(name, op, targets, shape=shape, ch=ch, **kw)


FWD_CASES = [
    _fwd("pt_v4", "pertensor", (N31,), None, ("fwd.tensor.v4", "fwd.tensor.v4.scalar_tail")),
    _fwd("pt_v1", "pertensor", (N31,), None, ("fwd.tensor.v1",), x_off=1),
    _fwd("pt_tma", "pertensor", (N31,), None, ("fwd.tma", "fwd.tma.tail"), variant=2),
    _fwd("stats_v4", "stats", (N31,), None, ("fwd.tensor.v4", "fwd.tensor.v4.scalar_tail")),
    _fwd("stats_v1", "stats", (N31,), None, ("fwd.tensor.v1",), x_off=1),
    _fwd("chan_tab", "perchannel", (10701, 64, 56, 56), 1,
         ("fwd.chan.tab.v4", "fwd.chan.tab.v4.nocross", "fwd.chan.tab.v4.carry")),
    _fwd("chan_notab", "perchannel", (74845, 4099, 7), 1,
         ("fwd.chan.notab.v4", "fwd.chan.notab.v4.straddle", "fwd.chan.notab.v4.fast", "fwd.chan.notab.v4.carry",
          "fwd.chan.v4.scalar_tail")),
    _fwd("chan_inner3", "perchannel", (238609295, 3, 3), 1,
         ("fwd.chan.tab.v4.inner_lt4", "fwd.chan.tab.v4.carry", "fwd.chan.v4.scalar_tail")),
    _fwd("cols_v4", "perchannel", (524289, 4096), -1, ("fwd.cols.v4", "fwd.cols.v4.loop4", "fwd.cols.v4.tail")),
    _fwd("cols_v1", "perchannel", (523905, 4099), -1, ("fwd.cols.v1",)),
]
BWD_CASES = [
    _fwd("bwd_pt", "bwd", (N31,), None, ("bwd.rows.cta", "bwd.rows.cta.grid_stride", "bwd.rows.partial_last_tile",
                                         "bwd.finish.rows.tpr_gt1")),
    _fwd("bwd_rows_cta", "bwd", (65, 13, 2541401), 1,
         ("bwd.rows.cta", "bwd.rows.partial_last_tile", "bwd.span.head", "bwd.finish.rows.tpr_gt1.multichannel"),
         closed=True),
    _fwd("bwd_rows_warp", "bwd", (695655, 63, 7, 7), 1, ("bwd.rows.warp", "bwd.rows.warp.grid_stride",
                                                         "bwd.finish.rows.tpr1")),
    _fwd("bwd_cols_v4", "bwd", (524289, 4096), -1, ("bwd.cols.v4", "bwd.cols.v4.loop4", "bwd.cols.v4.drain",
                                                    "bwd.cols.v4.tail", "bwd.finish.cols")),
    _fwd("bwd_cols_v1", "bwd", (523905, 4099), -1, ("bwd.cols.v1", "bwd.cols.v1.drain", "bwd.finish.cols")),
]
CLAMP_CASES = [_fwd("clamp", "clamp", (N31,), None, ("clamp.vec", "clamp.vec.flush_then_more", "clamp.vec.tail"))]
MM_CASES = [
    _fwd("mm_tensor", "minmax", (N32,), None, ("mm.tensor.v4", "mm.tensor.v4.scalar_tail", "mm.tensor.gridstride"),
         bound=32),
    _fwd("mm_cta", "minmax", (3, 7, 102261127), 1, ("mm.rows.cta", "mm.rows.cta.tpr_gt1.partial",
                                                     "mm.rows.cta.gridstride")),
    _fwd("mm_warp", "minmax", (33257, 63, 1025), 1, ("mm.rows.warp", "mm.rows.warp.gridstride")),
    _fwd("mm_tiny", "minmax", (695655, 63, 7, 7), 1, ("mm.rows.tiny", "mm.rows.tiny.gridstride",
                                                       "mm.rows.tiny.last_group_lt32")),
    _fwd("mm_cols", "minmax", (524289, 4096), -1, ("mm.cols.v4", "mm.cols.v4.loop4", "mm.cols.v4.tail")),
]
HIST_CASES = [
    _fwd("hist_random", "hist", (N32,), None, ("hist.v4.loop4", "hist.v4.tail", "hist.gridstride"), bound=32,
         range=(-2.5, 4.25)),
    _fwd("hist_const", "hist", (N32,), None, ("hist.v4.loop4", "hist.v4.tail", "hist.gridstride"), bound=32,
         range=(0.5, 0.5)),
]
MSE_CASES = [
    _fwd("mse_tensor", "mse", (1, N31), None, ("mse.bulk", "mse.nonbulk", "mse.mixed", "mse.tpr_gt1",
                                               "mse.finish.unroll4"), qrange=(-128, 127)),
    _fwd("mse_rows", "mse", (4101, 524161), None, ("mse.bulk", "mse.nonbulk", "mse.tpr_gt1", "mse.reload"),
         qrange=(0, 15)),
]
SEL_CASES = [
    _fwd("kth_key0", "kth", (N31,), None, ("sel.hist.p0.ntpr1", "sel.hist.p2.ntpr1", "sel.hist.seg65536",
                                           "sel.hist.gridstride", "sel.hist.tail"), key_mode=0),
    _fwd("kth_key1", "kth", (N31,), None, ("sel.hist.p0.ntpr1", "sel.hist.key_mode1", "sel.hist.tail"), key_mode=1),
    _fwd("pct", "pct", (N31,), None, ("sel.hist.p0.ntpr2", "sel.hist.p2.ntpr2", "sel.hist.gridstride")),
]
ALL_CASES = FWD_CASES + BWD_CASES + CLAMP_CASES + MM_CASES + HIST_CASES + MSE_CASES + SEL_CASES
NCAND = 80


def _n(case):
    return int(np.prod(case.get("shape"), dtype=np.int64))


def _geometry(case):
    """[outer, C, inner]: per-tensor cases are [n, 1, 1], so that a slab is one element."""
    shape, ch = case.get("shape"), case.get("ch")
    if case.op in ("mse",):
        return shape[0], 1, shape[1]
    return (_n(case), 1, 1) if ch is None else qgeo.channel_geometry(shape, ch)


def regime(case, sm):
    """The launch branches the case reaches, from the geometry mirrors."""
    n, (outer, c, inner) = _n(case), _geometry(case)
    off = case.get("x_off", 0)
    if case.op in ("pertensor", "stats"):
        return qgeo.fwd_branches(case.op, case.get("shape"), 0, sm, off, off, variant=case.get("variant", 0))
    if case.op == "perchannel":
        return qgeo.fwd_branches("perchannel", case.get("shape"), case.get("ch"), sm)
    if case.op == "bwd":
        return qgeo.bwd_branches(case.get("shape"), case.get("ch"), sm)
    if case.op == "clamp":
        return wgeo.clamp_bwd_branches(n, 0, 0, 0, sm)
    if case.op == "minmax":
        if case.get("ch") is None:
            return ogeo.minmax_tensor_branches(n, sm)
        return ogeo.minmax_branches(outer, c, inner, sm) | {"mm.rows." + ogeo.minmax_regime(inner)}
    if case.op == "hist":
        return ogeo.hist_branches(n, sm)
    if case.op == "mse":
        return ogeo.mse_branches(outer, inner, NCAND, sm)
    ntpr = 2 if case.op == "pct" else 1
    return ogeo.select_hist_branches(1, n, ntpr, (0, 1, 2), sm, 0, case.get("key_mode", 0))


def partial_last(case, sm):
    """Whether the last chunk, tile, row block, grid step or segment of the launch is partial."""
    n, (outer, c, inner) = _n(case), _geometry(case)
    vec = case.get("x_off", 0) % 4 == 0
    if case.op in ("pertensor", "stats"):
        if case.get("variant", 0) == 2:
            return (n & ~3) % qgeo.K_TMA_TILE != 0
        return ((n >> 2) if vec else n) % (4 * qgeo.K_THREADS) != 0
    if case.op == "minmax" and case.get("ch") is None:
        g = qgeo.launch_stream(n, 1, n, True, sm, per_channel=False)
        return g["nvec"] % (qgeo.K_UNROLL * g["grid"] * qgeo.K_THREADS) != 0
    if case.op in ("perchannel", "minmax") and inner == 1:
        g = (qgeo.launch_cols(outer, c, c % 4 == 0, sm) if case.op == "perchannel"
             else ogeo.minmax_cols(outer, c, c % 4 == 0, sm))
        return outer % g["rpb"] != 0
    if case.op == "perchannel":
        g = qgeo.launch_stream(n, c, inner, True, sm, per_channel=True)
        return g["nvec"] % (qgeo.K_UNROLL * g["grid"] * qgeo.K_THREADS) != 0
    if case.op == "bwd":
        if case.get("ch") is None:  # sb200_qdq_pertensor_bwd: bwd_rows over one row of n elements
            return n % qgeo.BWD_K_TILE != 0
        if inner == 1:
            return outer % -(-outer // qgeo.cols_row_blocks(outer, c, sm)) != 0
        return inner % qgeo.BWD_K_TILE != 0 or (inner < qgeo.BWD_CTA_TILE_MIN_INNER and (outer * c) % 8 != 0)
    if case.op == "clamp":
        return (n >> 2) % wgeo.clamp_bwd_geometry(n, 0, 0, 0, sm)["nt"] != 0
    if case.op == "minmax":
        reg = ogeo.minmax_regime(inner)
        return {"cta": inner % ogeo.K_ROW_TILE != 0, "warp": (outer * c) % 4 != 0, "tiny": (outer * c) % 32 != 0}[reg]
    if case.op == "hist":
        return (n >> 2) % ogeo.hist_geometry(n, sm)["T"] != 0
    if case.op == "mse":
        return inner % ogeo.K_MSE_TILE != 0
    return n % ogeo.select_geometry(1, n, sm)["seg"] != 0


# -------------------------------------------------------------------------------------------------- CPU tests
def test_case_table_covers_every_branch():
    """Every case is past its bound, has an n % 4 tail unless C % 4 == 0 makes one impossible (a vectorised
    channel-last or channel-table layout), has a partial last chunk, tile, row block, grid step or segment, reaches
    the regime it names at 132 SMs (H100 SXM) and is named in the docstring."""
    sm = qgeo.SM_COUNT_H100
    for case in ALL_CASES:
        n, (_, c, _) = _n(case), _geometry(case)
        bound = B32 if case.get("bound", 31) == 32 else B31
        assert n > bound, (case.name, n)
        assert n % 4 or (c > 1 and c % 4 == 0), (case.name, "no n % 4 tail")
        assert partial_last(case, sm), (case.name, "the last chunk is whole")
    assert_table_covers(ALL_CASES, set(), lambda c: check_reach(c, regime(c, sm)), __doc__, doc_branches=False)


def test_channel_last_grid_y_cap_cannot_bind():
    """launch_cols / cols_row_blocks / the MinMax column launch cap gridDim.y at 65535, but want ceil(8 SM / gx) row
    blocks first, at most 8 x 132 = 1056 on an H100, so the cap never applies there."""
    sm = qgeo.SM_COUNT_H100
    for outer, c in ((524289, 4096), (523905, 4099), (1 << 40, 1), (1 << 40, 4)):
        assert qgeo.launch_cols(outer, c, c % 4 == 0, sm)["want_y"] <= 8 * sm
        assert ogeo.minmax_cols(outer, c, c % 4 == 0, sm)["want_y"] <= 8 * sm
        assert qgeo.cols_row_blocks(outer, c, sm) <= 8 * sm * 2


def test_pertensor_refuses_more_than_2_31_chunks_on_the_host():
    """launch_chunks (qdq.cu) refuses a per-tensor QDQ whose chunk grid would pass 2^31 - 1 CTAs with SB200_E_INVALID,
    before any CUDA call (there is no device here): check_common, use_tma and launch_chunks read only the arguments and
    the variant switch up to that check.  At the boundary: 4 x 1024 elements per CTA on the 128-bit path, 1024 on the
    scalar one (a pointer off 16-byte alignment)."""
    lib = _lib.load()
    keep, p = buf()
    refused = [(p, 1 << 43), (p, (1 << 43) - 4092), (p + 4, (1 << 41) - 1023), (p + 4, 1 << 43)]
    try:
        for variant in (0, 1):
            assert lib.sb200_set_variant(variant) == 0
            for ptr, n in refused:
                assert lib.sb200_qdq_pertensor_fwd(ptr, p, p, ptr, n, -128, 127, 0, None) == E_INVALID, (variant, n)
                assert f"{n} elements exceed the launch limit".encode() in lib.sb200_last_error()
                assert lib.sb200_qdq_stats_pertensor_fwd(ptr, p, p, ptr, p, n, -128, 127, 0, None) == E_INVALID
                assert f"{n} elements exceed the launch limit".encode() in lib.sb200_last_error()
    finally:
        lib.sb200_set_variant(0)


def _small_inputs(rng, n=4099, c=5):
    x = (rng.standard_normal((3, c, n // 3)) * 0.4).astype(F32)
    s = rng.uniform(0.01, 0.05, c).astype(F32)
    z = np.rint(rng.uniform(-3, 3, c)).astype(F32)
    k = rng.integers(-20, 20, x.shape).astype(F32)
    tie = rng.random(x.shape) < 0.2
    x[tie] = ((k + F32(0.5)) * s[None, :, None] * np.ones_like(x))[tie].astype(F32)
    flat = x.reshape(-1)
    flat[[0, 5, 9, 17]] = [np.nan, np.inf, -np.inf, (F32(15) - z[0]) * s[0]]
    return x, s, z, rng.standard_normal(x.shape).astype(F32)


@pytest.mark.parametrize("open_top", [False, True])
def test_ste_restatement_is_the_oracle(open_top):
    rng = np.random.default_rng(3)
    x, s, z, gy = _small_inputs(rng)
    with np.errstate(invalid="ignore"):
        egx, egs, egz = oqdq._ste_terms(x, s, z, gy, -16, 15, 1, 0, open_top)
    gx, gs, gs1, gz, gz1 = ref.ste_sums(*(torch.from_numpy(a) for a in (x, gy, s, z)), -16, 15, open_top)
    assert bits_equal(gx.numpy(), egx)
    np.testing.assert_allclose(gs.numpy(), egs.sum(axis=(0, 2)), rtol=1e-12)
    np.testing.assert_allclose(gz.numpy(), egz.sum(axis=(0, 2)), rtol=1e-12)
    np.testing.assert_allclose(gs1.numpy(), np.abs(egs).sum(axis=(0, 2)), rtol=1e-12)
    np.testing.assert_allclose(gz1.numpy(), np.abs(egz).sum(axis=(0, 2)), rtol=1e-12)


def test_clamp_restatement_is_the_oracle():
    rng = np.random.default_rng(4)
    x, _, _, gy = _small_inputs(rng)
    x = x.reshape(-1) * F32(8)
    x[[1, 2]] = [F32(-1.5), F32(2.25)]
    egx, ehi, elo = oqdq.clamp_backward(x, gy.reshape(-1), -1.5, 2.25)
    gx, ghi, glo, _, _ = ref.clamp_sums(torch.from_numpy(x), torch.from_numpy(gy.reshape(-1)), torch.tensor(-1.5),
                                        torch.tensor(2.25))
    assert bits_equal(gx.numpy(), egx)
    np.testing.assert_allclose([ghi.item(), glo.item()], [ehi, elo], rtol=1e-12)


def test_mse_restatement_is_the_oracle():
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((3, 5000)) * [[0.5], [1.0], [2.0]]).astype(F32)
    cs = rng.uniform(0.01, 0.4, (3, 9)).astype(F32)
    cz = rng.uniform(5, 10, (3, 9)).astype(F32)
    cz[:, ::3] = np.floor(cz[:, ::3]) + F32(0.5)
    exp = np.stack([((x.astype(np.float64) - oqdq.qdq(x, cs[:, i], cz[:, i], 0, 15, ch_axis=0)) ** 2).sum(1)
                    for i in range(9)], axis=1)
    got = ref.mse_sums(*(torch.from_numpy(a) for a in (x, cs, cz)), 0, 15)
    np.testing.assert_allclose(got.numpy(), exp, rtol=1e-12)


def test_select_keys_are_the_kernel_order():
    """sel_keys sorts like enc_f32: -NaN and NaN last, -inf < ... < -0 < +0 < ... < +inf; key mode 1 orders |x|."""
    x = np.float32([np.nan, -np.inf, -2.0, -1e-45, -0.0, 0.0, 1e-45, 3.0, np.inf, -np.nan])
    k0 = ref.sel_keys(torch.from_numpy(x), 0).numpy()
    assert list(np.argsort(k0[1:-1], kind="stable") + 1) == list(range(1, 9))
    assert k0[0] == k0[-1] == 0xFFFFFFFF and k0[1:-1].max() < 0xFFFFFFFF and k0.min() >= 0
    k1 = ref.sel_keys(torch.from_numpy(x), 1).numpy()
    assert k1[4] == k1[5] and k1[2] < k1[7] and k1[1] == k1[8] and k1[-1] == 0xFFFFFFFF


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


def _need(gib):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    free, _ = torch.cuda.mem_get_info()
    if free < gib * GIB:
        pytest.skip(f"needs {gib:.1f} GiB of free device memory, {free / GIB:.1f} GiB free")
    torch.cuda.reset_peak_memory_stats()


def _release(name):
    torch.cuda.synchronize()
    print(f"{name}: peak {torch.cuda.max_memory_allocated() / GIB:.2f} GiB allocated")
    gc.collect()
    torch.cuda.empty_cache()


def _gen(case, *extra):
    return torch.Generator(device=dev()).manual_seed(seed_of(case.name, *extra))


def _randn(n, gen, off=0):
    """n standard normal floats starting ``off`` floats into a fresh (16-byte aligned) allocation."""
    x = torch.empty(n + off, device=dev())[off:]
    return x.normal_(generator=gen)


def _sentinel(n, off=0):
    out = torch.empty(n + off, device=dev())[off:]
    out.view(torch.int32).fill_(SENTINEL)
    return out


def _windows(rows, inner):
    """[r0, r1) ranges of channel rows (``inner`` elements of one channel): the head, the rows around elements 2^31 to
    2^31 + 5 and the last rows, which hold the n % 4 tail."""
    k = max(WIN // inner, 2)
    wins = [(0, k), (max((B31 - WIN // 2) // inner, 0), min((B31 + 6 + WIN // 2) // inner + 1, rows)), (rows - k, rows)]
    merged = [wins[0]]
    for r0, r1 in wins[1:]:  # just past 2^31 the middle and the last window meet
        if r0 <= merged[-1][1]:
            merged[-1] = (merged[-1][0], max(r1, merged[-1][1]))
        else:
            merged.append((r0, r1))
    return merged


def _sub_ranges(units, slab, head=0):
    """Consecutive [a, b) ranges of whole slabs, at most SUB elements each; every range after the first ``head`` units
    starts a multiple of 4 units after ``head``, so on a 16-byte boundary when unit ``head`` is on one."""
    per = max(SUB // slab // 4 * 4, 4)
    cuts = sorted({0, units, *range(head, units, per)})
    return list(zip(cuts[:-1], cuts[1:]))


def _bits_eq(a, b):
    return torch.equal(a.reshape(-1).view(torch.int32), b.reshape(-1).view(torch.int32))


def _row_channels(r0, r1, c):
    return np.arange(r0, r1, dtype=np.int64) % c


def _plant(x3, windows, fixed, make):
    """Plant values in the channel-row windows of x3 [outer, C, inner] (``make(flat, channel_of_each)`` edits a
    window's host copy) and at the global flat positions ``fixed``; return the host copies, [rows, inner] each."""
    outer, c, inner = x3.shape
    xr = x3.view(outer * c, inner)
    host = []
    for r0, r1 in windows:
        w = xr[r0:r1].cpu().numpy()
        flat = w.reshape(-1)
        make(flat, np.repeat(_row_channels(r0, r1, c), inner))
        for p, v in fixed.items():
            if r0 * inner <= p < r1 * inner:
                flat[p - r0 * inner] = v
        xr[r0:r1].copy_(torch.from_numpy(w))
        host.append(w)
    return host


def _grid_values(rng, s, z, qmin, qmax):
    """Ties (k + 1/2) s and values far outside [qmin, qmax] on an eighth and a hundredth of a window."""
    zr = np.rint(z)

    def make(flat, ch):
        m = flat.size
        tie = rng.random(m) < 0.125
        k = rng.integers(qmin - 6, qmax + 6, m).astype(F32) - zr[ch]
        flat[tie] = ((k[tie] + F32(0.5)) * s[ch][tie]).astype(F32)
        far = rng.random(m) < 0.01
        q = np.where(rng.random(m) < 0.5, F32(qmin - 1000), F32(qmax + 1000)) - zr[ch]
        flat[far] = (q[far] * s[ch][far]).astype(F32)
    return make


def _qparams(case, rng, lo, hi):
    c = _geometry(case)[1]
    if c == 1:
        return np.float32([0.5 * (lo + hi)]), np.float32([2.5])
    s = rng.uniform(lo, hi, c).astype(F32)
    z = np.rint(rng.uniform(-3, 3, c)).astype(F32)
    z[::5] += F32(0.5)  # rint ties
    return s, z


def _check_windows(name, got3, windows, host, expect):
    """``expect(i, w, ch)``: the oracle's output for window i (host copy w [rows, inner], ch the row's channels)."""
    outer, c, inner = got3.shape
    gr = got3.view(outer * c, inner)
    for i, ((r0, r1), w) in enumerate(zip(windows, host)):
        got = gr[r0:r1].cpu().numpy()
        exp = expect(i, w, _row_channels(r0, r1, c))
        if not bits_equal(got, exp):
            bad = np.flatnonzero(~((got == exp) | (np.isnan(got) & np.isnan(exp))).reshape(-1))
            j = bad[0]
            raise AssertionError(f"{name}: window of rows [{r0}, {r1}): {bad.size} differ; first at element "
                                 f"{r0 * inner + j}: x={w.reshape(-1)[j]!r} got={got.reshape(-1)[j]!r} "
                                 f"expected={exp.reshape(-1)[j]!r}")


def _oracle_rows(fn, w, ch, s, z, *args):
    """An oracle/qdq.py function on window rows [rows, inner] whose channels are ``ch``: one channel per row."""
    return fn(w.reshape(1, *w.shape), s[ch], z[ch], *args).reshape(w.shape)


def _check_sub_launches(name, x3, big3, head, run):
    """``run(a, b, out)`` writes the entry point's output for slabs [a, b) of x3 into ``out``; every range must equal
    the big launch's output there, bit for bit."""
    outer, c, inner = x3.shape
    scratch = torch.empty(SUB + 4, device=dev())
    for a, b in _sub_ranges(outer, c * inner, head):
        out = scratch[:(b - a) * c * inner].view(b - a, c, inner)
        out.view(torch.int32).fill_(SENTINEL)
        run(a, b, out)
        assert _bits_eq(out, big3[a:b]), f"{name}: slabs [{a}, {b}) differ from a launch on them alone"


# -------------------------------------------------------------------------------------------------- GPU: forward
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(FWD_CASES))
@_frees_device_memory
def test_forward_far_end(case):
    n = _n(case)
    _need(2 * 4 * n / GIB + 2.5)
    check_reach(case, regime(case, real_sm()))
    outer, c, inner = _geometry(case)
    off, qmin, qmax = case.get("x_off", 0), -128, 127
    rng = np.random.default_rng(seed_of(case.name))
    s, z = _qparams(case, rng, 0.02, 0.06)
    sd, zd = torch.from_numpy(s).to(dev()), torch.from_numpy(z).to(dev())
    x = _randn(n, _gen(case), off)
    x3 = x.view(outer, c, inner)
    x3.mul_(sd.view(1, -1, 1) * 50)
    stats = case.op == "stats"
    fixed = {B31 + 5: -np.inf, n - 1: np.inf} if stats else {B31 + 1: np.nan, B31 + 5: -np.inf, n - 1: np.inf}
    windows = _windows(outer * c, inner)
    host = _plant(x3, windows, fixed, _grid_values(rng, s, z, qmin, qmax))
    out = _sentinel(n, off)
    xs, ys = x.view(case.get("shape")), out.view(case.get("shape"))
    lib = _lib.load()
    if case.op == "perchannel":
        ops.qdq_perchannel(xs, sd, zd, qmin, qmax, case.get("ch"), out=ys)
    else:
        assert lib.sb200_set_variant(case.get("variant", 0)) == 0
        try:
            if stats:
                st = ops.minmax_new(1, dev())
                ops.qdq_stats_pertensor(xs, sd, zd, qmin, qmax, st, out=ys)
            else:
                ops.qdq_pertensor(xs, sd, zd, qmin, qmax, out=ys)
        finally:
            lib.sb200_set_variant(0)
    out3 = out.view(outer, c, inner)
    _check_windows(case.name, out3, windows, host,
                   lambda i, w, ch: _oracle_rows(oqdq.qdq, w, ch, s, z, qmin, qmax, 1))
    if stats:
        mn, mx = ops.minmax_read(st)
        assert float(mn) == -np.inf and float(mx) == np.inf, (case.name, float(mn), float(mx))
        st2 = ops.minmax_new(1, dev())

    def run(a, b, o):
        if case.op == "perchannel":
            ops.qdq_perchannel(x3[a:b], sd, zd, qmin, qmax, 1, out=o)
        elif stats:
            ops.qdq_stats_pertensor(x[a:b], sd, zd, qmin, qmax, st2, out=o.reshape(-1))
        else:
            ops.qdq_pertensor(x[a:b], sd, zd, qmin, qmax, out=o.reshape(-1))
    _check_sub_launches(case.name, x3, out3, (-off) % 4 if c == 1 else 0, run)
    if stats:
        assert torch.equal(st, st2), case.name  # the fused MinMax of the pieces is the one of the whole
        del st, st2
    del x, x3, xs, out, out3, ys
    _release(case.name)


# -------------------------------------------------------------------------------------------------- GPU: backward
def _qdq_backward_into(x, s, z, gy, gx, qmin, qmax, ch_axis, gzp_closed=False):
    """sb200_qdq_pertensor_bwd / sb200_qdq_perchannel_bwd_ex as ops.qdq_backward calls them, into a caller-owned gx
    (the wrapper allocates its own, which cannot hold a sentinel)."""
    lib = _lib.load()
    outer, c, inner = (1, 1, x.numel()) if ch_axis is None else ops.channel_geometry(x.shape, ch_axis)
    gs, gz = torch.zeros_like(s), torch.zeros_like(z)
    nb = int(lib.sb200_qdq_bwd_workspace_bytes(outer, c, inner))
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=x.device)
    ptrs = (x.data_ptr(), s.data_ptr(), z.data_ptr(), gy.data_ptr(), gx.data_ptr(), gs.data_ptr(), gz.data_ptr())
    if ch_axis is None:
        rc = lib.sb200_qdq_pertensor_bwd(*ptrs, x.numel(), qmin, qmax, 0, ws.data_ptr(), nb, stream())
    else:
        rc = lib.sb200_qdq_perchannel_bwd_ex(*ptrs, outer, c, inner, qmin, qmax, 0,
                                             ops.BWD_GZP_CLOSED if gzp_closed else 0, ws.data_ptr(), nb, stream())
    assert rc == 0, lib.sb200_last_error()
    return gs, gz


def _within_l1(got, exp, l1, tol=1e-5):
    got = got.double().cpu().reshape(-1)
    bad = torch.nonzero((got - exp.cpu()).abs() > tol * l1.cpu() + 1e-30).reshape(-1)
    return bad.numel() == 0, bad[:8].tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(BWD_CASES))
@_frees_device_memory
def test_backward_far_end(case):
    n = _n(case)
    _need(3 * 4 * n / GIB + 3.5)
    check_reach(case, regime(case, real_sm()))
    outer, c, inner = _geometry(case)
    qmin, qmax, ch = -16, 15, case.get("ch")
    rng = np.random.default_rng(seed_of(case.name))
    s, z = _qparams(case, rng, 0.02, 0.3)
    if c == 1:
        s, z = np.float32([0.07]), np.float32([2.0])
    sd, zd = torch.from_numpy(s).to(dev()), torch.from_numpy(z).to(dev())
    gen = _gen(case)
    x, gy = _randn(n, gen), _randn(n, gen)
    gy[B31:] *= TAIL_GY
    x3, gy3 = x.view(outer, c, inner), gy.view(outer, c, inner)
    windows = _windows(outer * c, inner)
    host = _plant(x3, windows, {B31 + 1: np.nan, B31 + 5: -np.inf, n - 1: np.inf}, _grid_values(rng, s, z, qmin, qmax))
    gyr = gy.view(outer * c, inner)
    gyh = [gyr[r0:r1].cpu().numpy().reshape(1, r1 - r0, inner) for r0, r1 in windows]
    shape = case.get("shape")
    gx = torch.empty(n, device=dev())
    gx3 = gx.view(outer, c, inner)

    def run(a, b, o):  # the ops wrapper, which allocates its own gx
        if ch is None:
            got = ops.qdq_backward(x[a:b], sd, zd, gy[a:b], qmin, qmax, need_gs=False, need_gzp=False)[0]
        else:
            got = ops.qdq_backward(x3[a:b], sd, zd, gy3[a:b], qmin, qmax, 1, need_gs=False, need_gzp=False)[0]
        o.copy_(got.view_as(o))
    # the per-channel default counts vq == qmax as clipped for gzp (open top); per tensor it does not
    rules = [(False, ch is not None)] + ([(True, False)] if case.get("closed") else [])
    for closed, open_top in rules:
        gx.view(torch.int32).fill_(SENTINEL)
        gs, gz = _qdq_backward_into(x.view(shape), sd, zd, gy.view(shape), gx.view(shape), qmin, qmax, ch,
                                    gzp_closed=closed)
        with np.errstate(invalid="ignore"):
            _check_windows(case.name, gx3, windows, host, lambda i, w, ch: oqdq.ste_backward(
                w.reshape(gyh[i].shape), s[ch], z[ch], gyh[i], qmin, qmax, 1)[0].reshape(w.shape))
        _check_sub_launches(case.name, x3, gx3, 0, run)
        sums = [torch.zeros(c, dtype=torch.float64, device=dev()) for _ in range(4)]
        for o0, o1 in ref.slab_chunks(outer, c * inner):
            part = ref.ste_sums(x3[o0:o1], gy3[o0:o1], sd, zd, qmin, qmax, open_top)[1:]
            for acc, v in zip(sums, part):
                acc += v
        egs, egs1, egz, egz1 = sums
        ok, bad = _within_l1(gs, egs, egs1)
        assert ok, (case.name, "gs", closed, bad, gs.cpu()[bad], egs.cpu()[bad])
        ok, bad = _within_l1(gz, egz, egz1)
        assert ok, (case.name, "gzp", closed, bad, gz.cpu()[bad], egz.cpu()[bad])
    del x, gy, x3, gy3, gyr, gx, gx3
    _release(case.name)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(CLAMP_CASES))
@_frees_device_memory
def test_clamp_backward_far_end(case):
    n = _n(case)
    _need(3 * 4 * n / GIB + 3.5)
    check_reach(case, regime(case, real_sm()))
    rng = np.random.default_rng(seed_of(case.name))
    lo, hi = F32(-1.5), F32(2.25)
    lod, hid = torch.tensor([lo], device=dev()), torch.tensor([hi], device=dev())
    gen = _gen(case)
    x, gy = _randn(n, gen).mul_(2), _randn(n, gen)
    gy[B31:] *= TAIL_GY
    x3 = x.view(n, 1, 1)
    edges = np.float32([lo, hi, np.nextafter(lo, F32(-9)), np.nextafter(hi, F32(9)), np.nextafter(lo, F32(9))])

    def make(flat, ch):
        sel = rng.random(flat.size) < 0.05
        flat[sel] = rng.choice(edges, int(sel.sum()))
    windows = _windows(n, 1)
    host = _plant(x3, windows, {B31 + 1: np.nan, B31 + 5: -np.inf, n - 1: np.inf}, make)
    gx = _sentinel(n)
    lib = _lib.load()
    nb = int(lib.sb200_clamp_bwd_workspace_bytes(n))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev())
    g_hi, g_lo = torch.zeros(1, device=dev()), torch.zeros(1, device=dev())
    assert lib.sb200_clamp_bwd(x.data_ptr(), gy.data_ptr(), lod.data_ptr(), hid.data_ptr(), gx.data_ptr(),
                               g_hi.data_ptr(), g_lo.data_ptr(), n, ws.data_ptr(), nb, stream()) == 0
    gyh = [gy[r0:r1].cpu().numpy() for r0, r1 in windows]
    _check_windows(case.name, gx.view(n, 1, 1), windows, host,
                   lambda i, w, ch: oqdq.clamp_backward(w.reshape(-1), gyh[i], lo, hi)[0].reshape(w.shape))
    sums = [torch.zeros((), dtype=torch.float64, device=dev()) for _ in range(4)]
    for a in range(0, n, ref.CHUNK):
        for acc, v in zip(sums, ref.clamp_sums(x[a:a + ref.CHUNK], gy[a:a + ref.CHUNK], lod, hid)[1:]):
            acc += v
    ehi, elo, ehi1, elo1 = sums
    for name, got, exp, l1 in (("g_hi", g_hi, ehi, ehi1), ("g_lo", g_lo, elo, elo1)):
        ok, _ = _within_l1(got, exp.reshape(1), l1.reshape(1))
        assert ok, (case.name, name, float(got), float(exp))
    _check_sub_launches(case.name, x3, gx.view(n, 1, 1), 0,
                        lambda a, b, o: o.copy_(ops.clamp_backward(x[a:b], gy[a:b], lod, hid)[0].view_as(o)))
    del x, gy, x3, gx, ws
    _release(case.name)


# -------------------------------------------------------------------------------------------------- GPU: MinMax
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(MM_CASES))
@_frees_device_memory
def test_minmax_far_end(case):
    n = _n(case)
    _need(4 * n / GIB + 1.5)
    check_reach(case, regime(case, real_sm()))
    outer, c, inner = _geometry(case)
    x = _randn(n, _gen(case))
    x3 = x.view(outer, c, inner)
    ch = case.get("ch")
    if ch is None:
        x[B31 + 5], x[n - 1] = -1234.5, 4321.25
        planted = torch.tensor([-1234.5]), torch.tensor([4321.25])
    else:  # each channel's extremes in the last slab (the last two rows for channel-last tensors)
        cc = torch.arange(c, device=dev())
        vmin, vmax = -(1000 + 0.5 * cc.float()), 1000 + 0.25 * cc.float()
        pos = torch.randint(0, max(inner - 1, 1), (c,), device=dev(), generator=_gen(case, "pos"))
        x3[-1, cc, inner - 1] = vmax
        x3[-1 if inner > 1 else -2, cc, pos] = vmin
        planted = vmin.cpu(), vmax.cpu()
    st = ops.minmax_new(c, dev())
    ops.minmax_update(x.view(case.get("shape")), st, ch)
    mn, mx = ops.minmax_read(st)
    emn = torch.full((c,), np.inf, device=dev())
    emx = torch.full((c,), -np.inf, device=dev())
    for o0, o1 in ref.slab_chunks(outer, c * inner, 1 << 27):
        lo_, hi_ = torch.aminmax(x3[o0:o1].transpose(0, 1).reshape(c, -1), dim=1)
        emn, emx = torch.minimum(emn, lo_), torch.maximum(emx, hi_)
    assert torch.equal(emn.cpu(), planted[0]) and torch.equal(emx.cpu(), planted[1])
    assert torch.equal(mn, emn) and torch.equal(mx, emx), (case.name, (mn != emn).nonzero()[:4],
                                                           (mx != emx).nonzero()[:4])
    del x, x3, st
    _release(case.name)


# -------------------------------------------------------------------------------------------------- GPU: histogram
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(HIST_CASES))
@_frees_device_memory
def test_hist_far_end(case):
    n = _n(case)
    _need(4 * n / GIB + 1.5)
    check_reach(case, regime(case, real_sm()))
    lo, hi = (F32(v) for v in case.get("range"))
    rg = torch.tensor([lo, hi], device=dev())
    counts = torch.zeros(2048, dtype=torch.int64, device=dev())
    if lo == hi:  # widened to [lo - 1, hi + 1]: 0.5 lands in bin 1024 of [-0.5, 1.5]
        x = torch.full((n,), float(lo), device=dev())
        ops.hist_update(x, rg, counts)
        assert counts[1024].item() == n and counts.sum().item() == n, (counts[1024].item(), counts.sum().item())
    else:
        x = _randn(n, _gen(case)).mul_(1.5)
        specials = torch.tensor([np.nan, np.inf, -np.inf, lo, hi, np.nextafter(lo, F32(-9)), np.nextafter(hi, F32(9))],
                                device=dev())
        for base in (B31 - 3, B32 - 4, n - specials.numel()):
            x[base:base + specials.numel()] = specials
        ops.hist_update(x, rg, counts)
        pieces = torch.zeros_like(counts)
        for a, b in _sub_ranges(n, 1):
            ops.hist_update(x[a:b], rg, pieces)
        inside = sum(int(((x[a:a + (1 << 28)] >= lo) & (x[a:a + (1 << 28)] <= hi)).sum()) for a in range(0, n, 1 << 28))
        assert torch.equal(counts, pieces), (counts - pieces).nonzero()[:8]
        assert counts.sum().item() == inside
    del x
    _release(case.name)


# -------------------------------------------------------------------------------------------------- GPU: MSE sweep
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(MSE_CASES))
@_frees_device_memory
def test_mse_sweep_far_end(case):
    n = _n(case)
    _need(4 * n / GIB + 2.5)
    check_reach(case, regime(case, real_sm()))
    rows, row_len = case.get("shape")
    qmin, qmax = case.get("qrange")
    rng = np.random.default_rng(seed_of(case.name))
    f = np.ones(rows, F32) if rows == 1 else rng.uniform(0.5, 3.0, rows).astype(F32)
    x2 = _randn(n, _gen(case)).view(rows, row_len)
    if rows > 1:
        x2.mul_(torch.from_numpy(f).to(dev()).view(-1, 1))
    span = 6.3 * 2 / (qmax - qmin)
    cs = (f[:, None] * span * np.linspace(0.15, 1.0, NCAND)[None, :]).astype(F32)
    mid = (qmin + qmax + 1) / 2
    cz = np.broadcast_to(np.float32(0 if qmin < 0 else mid), cs.shape).copy()
    if qmin >= 0:
        cz += rng.uniform(-1.5, 1.5, cs.shape).astype(F32)
        cz[:, ::3] = np.floor(cz[:, ::3]) + F32(0.5)
    csd, czd = torch.from_numpy(cs).to(dev()), torch.from_numpy(cz).to(dev())
    if rows == 1:
        # The one tile past 2^31 holds 6147 of 2^31 + 6147 elements: at N(0, 1) they would weigh 3e-6 of each loss,
        # below the 1e-5 bar.  At +-12, outside every candidate's clip range, they weigh >= 2e-3 of the smallest
        # candidate's loss and most of the best one's, and the best candidate stays inside the sweep.
        sign = torch.randint(0, 2, (n - B31,), device=dev(), generator=_gen(case, "tail")).float() * 2 - 1
        x2[0, B31:] = sign * MSE_TAIL
    else:
        assert rows - -(-B31 // row_len) >= 2  # whole rows past 2^31, each with losses of its own
    sse = torch.zeros(rows, NCAND, dtype=torch.float64, device=dev())
    ops.mse_sweep(x2, csd, czd, qmin, qmax, sse)
    exp = torch.zeros_like(sse)
    if rows == 1:
        for a in range(0, row_len, ref.CHUNK):
            exp += ref.mse_sums(x2[:, a:a + ref.CHUNK], csd, czd, qmin, qmax)
        tail = ref.mse_sums(x2[:, B31:], csd, czd, qmin, qmax)
        assert bool((tail >= 1e-3 * exp).all()), (tail / exp).min().item()
    else:
        for r0, r1 in ref.slab_chunks(rows, row_len):
            exp[r0:r1] = ref.mse_sums(x2[r0:r1], csd[r0:r1], czd[r0:r1], qmin, qmax)
    got, exp = sse.cpu().numpy(), exp.cpu().numpy()
    bad = np.argwhere(np.abs(got - exp) > 1e-5 * exp)
    assert bad.size == 0, (case.name, bad[:4], got[tuple(bad[0])], exp[tuple(bad[0])])
    # the same winner: the kernel's best candidate is the reference's wherever the runner-up trails by more than the
    # tolerance, and within the tolerance of it elsewhere
    best, second = np.sort(exp, axis=1)[:, :2].T
    win = np.take_along_axis(exp, got.argmin(1)[:, None], 1)[:, 0]
    clear = second - best > 2e-5 * best
    assert np.array_equal(got.argmin(1)[clear], exp.argmin(1)[clear]) and np.all(win <= best * (1 + 2e-5)), case.name
    assert np.all((exp.argmin(1) > 0) & (exp.argmin(1) < NCAND - 1)), "the best candidate is inside the sweep"
    del x2, sse
    _release(case.name)


# -------------------------------------------------------------------------------------------------- GPU: radix select
def _select_input(case):
    """The tensor of the select and percentile cases: N(0, 1) with 257 NaNs and +-inf past 2^31."""
    x = _randn(N31, torch.Generator(device=dev()).manual_seed(seed_of("select far end")))
    x[B31 + 1000:B31 + 1257] = np.nan
    x[B31 + 7], x[N31 - 2] = np.inf, -np.inf
    return x


def _rank_bounds(x, values, key_mode):
    """For each value v: (#(key < key(v)), #(key <= key(v))) over x, counted in chunks in the kernel's key order."""
    kv = ref.sel_keys(values.reshape(-1), key_mode)
    lt = torch.zeros_like(kv)
    le = torch.zeros_like(kv)
    for a in range(0, x.numel(), 1 << 26):
        k = ref.sel_keys(x[a:a + (1 << 26)], key_mode).unsqueeze(1)
        lt += (k < kv).sum(0)
        le += (k <= kv).sum(0)
    return lt.tolist(), le.tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("case", params([c for c in SEL_CASES if c.op == "kth"]))
@_frees_device_memory
def test_kth_value_far_end(case):
    _need(4 * N31 / GIB + 2)
    check_reach(case, regime(case, real_sm()))
    x = _select_input(case)
    key_mode = case.get("key_mode")
    ks = [0, B31 - 1, B31 + 1, N31 - 1]
    vals = torch.cat([ops.kth_value(x, k, key_mode) for k in ks])
    lt, le = _rank_bounds(x, vals, key_mode)
    for k, v, a, b in zip(ks, vals.tolist(), lt, le):
        assert a <= k < b, (case.name, k, v, a, b)
    assert np.isnan(vals[-1].item())  # the NaNs rank last
    del x
    _release(case.name)


@pytest.mark.gpu
@_frees_device_memory
def test_percentile_observer_far_end():
    """The percentile observer on one tensor of 2^31 + 6147 elements: its max side asks for a rank past 2^31."""
    from sparsebit_b200 import config as sbcfg
    from sparsebit_b200.quantization import build_quantizer
    from sparsebit_b200.quantization.common import Backend

    case = next(c for c in SEL_CASES if c.op == "pct")
    _need(2 * 4 * N31 / GIB + 2.5)
    check_reach(case, regime(case, real_sm()))
    alpha = 1e-6
    x = _select_input(case)
    q = build_quantizer(sbcfg.quantizer_config("per-tensor-affine", 8, "feature", "percentile", alpha=alpha))
    q.set_backend(Backend.VIRTUAL)
    q.update_observer(x.view(1, -1))
    scale, zp = q.calc_qparams()
    mn, mx = q.observer.min_val.reshape(-1), q.observer.max_val.reshape(-1)
    neg = sum(int((x[a:a + (1 << 28)] < 0).sum()) for a in range(0, N31, 1 << 28))
    pos = sum(int((x[a:a + (1 << 28)] >= 0).sum()) for a in range(0, N31, 1 << 28))
    kmin, kmax, _ = ogeo.percentile_ranks(neg, pos, N31, alpha)
    assert neg > 0 and pos > 0 and kmax > B31, (neg, pos, kmax)
    lt, le = _rank_bounds(x, torch.cat([mn, mx]), 0)
    assert lt[0] <= kmin < le[0] and lt[1] <= kmax < le[1], (kmin, kmax, lt, le, float(mn), float(mx))
    qmin, qmax = q.qdesc.qrange
    es, ez = oobs.calc_qparams_with_minmax(mn.cpu().numpy(), mx.cpu().numpy(), qmin, qmax, q.qdesc.is_symmetric)
    assert bits_equal(scale.reshape(-1).cpu().numpy(), es.reshape(-1))
    assert bits_equal(zp.reshape(-1).cpu().numpy(), ez.reshape(-1))
    del x, q, mn, mx
    _release(case.name)
