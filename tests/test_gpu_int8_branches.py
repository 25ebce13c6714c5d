"""Every launch branch of the integer-grid kernels (csrc/int8_linear.cu): the row quantizer, the column quantizer, the
conv2d lowering, the linear / conv GEMM and the batched matmul GEMM, each reached by a named case through its C entry
point (pointer offsets under control) and through its ops wrapper, and compared with the numpy integer form bit for bit.

tests/int8_geometry.py restates the launch decisions and in-kernel branches; the CPU test at the bottom checks that the
cases together reach every branch in int8_geometry.REQUIRED.  gemm.nan_row is (data): the case plants a NaN row and
the GPU test checks it is there.

  case                 entry    why it is there
  rows_per_row         rows     per-row qparams, K = 1001: scalar loads, two lane-loop trips, last CTA partial
  rows_k16_full        rows     K = 16: vector loads of full chunks only, idle lanes
  rows_k768_misaligned rows     K = 768 with x 4 bytes past a 16-byte boundary: the scalar path with K % 4 == 0
  cols_vec             cols     batch 3, K = 300 (3 chunks, the last 48 K), N = 200 (N tile partial), vector loads
  cols_scalar          cols     batch 2, K = 77 (K % 4 != 0 inside a group), N = 131 (a partial column quad)
  cols_misaligned      cols     K = 128, N = 64, x 4 bytes past a 16-byte boundary: the scalar loads
  low_all_pad          im2col   3x3 with padding 3 (whole windows in the padding), unsigned zp = 0: pad tap -128
  low_chunks           im2col   C = 20, stride 2, dilation 2: K = 180 in two chunks, the last one short
  lin_k20              linear   K = 20 (vector + scalar tail), M = 37 (warpgroup 1 idle), num_kb 1
  lin_k100             linear   K = 100, 2 x 3 tiles, no bias, unsigned x at zp = qmin
  lin_k1004            linear   K = 1004 (two lane trips, 8 k-blocks: one ring wrap), M = 200 (both warpgroups)
  lin_k768_misaligned  linear   K = 768 (6 k-blocks) with x 4 bytes past a 16-byte boundary
  lin_k512             linear   K = 512: full vector chunks, 4 k-blocks, M = 129
  lin_k3000            linear   K = 3000: 24 k-blocks, the ring phase back to 0
  conv_pad_u0          conv     unsigned x at zp = 0: pad tap -128, 3x3 padding 3, P < 128 spanning images
  conv_pad_u255        conv     unsigned x at zp = 255: pad tap 127
  conv_pad_s_m128      conv     signed x at zp = -128: pad tap -128; stride 2, dilation 2, K in two chunks
  conv_ring            conv     K = 1800 (15 k-blocks), C_out = 130: 3 x 2 tiles, an image boundary inside a tile
  conv_far_end         conv     M Kp >= 2^31 (700 x 1 x 224^2, 7x7): the first and the last image
  mm_k1665_rows        matmul   batch 3, K = 1665 (14 k-blocks), b K-major, partial tiles, 8-byte stores
  mm_k3000_cols        matmul   batch 3, K = 3000 (24 k-blocks), b N-major, N = 131 (scalar stores, odd N)
  mm_n130_out4         matmul   N = 130 with out 4 bytes past an 8-byte boundary: scalar stores with even N
  mm_n131_out4         matmul   N = 131 with out at +4 bytes, b K-major, one k-block
  mm_kb6               matmul   K = 700: exactly 6 k-blocks, N-major b with vector loads
  mm_k1000             matmul   K = 1000: 8 k-blocks, b K-major, full tiles

Contract of every GPU case.  Each output buffer and its slack start as a finite sentinel (0x7B bytes), also q / sum /
nan of the quantizer-only entry points; afterwards the slack still holds it.  The workspace is filled with 0xA5 and
passed at base offsets of 0, 16 and 1008 bytes with exactly sb200_int8_*_workspace_bytes bytes and guard bytes behind
it, which stay untouched.  The three calls and the ops wrapper agree bit for bit.  Quantizer outputs equal the oracle
grid (oracle.qdq.quantize_int, int8_matmul_ref.quantize_cols, int8_conv_ref.lowered) bit for bit, K padding, sums
and NaN flags included.  GEMM outputs equal the numpy integer form y = fp32(fp64(I) (fp64 s_x fp64 s_w)) (+ bias in
fp32; NaN rows and columns) at every element, and meet |y - T| <= 2^-21 (|fx| |fw| + |bias|) against the fp64
fake-quant truth.  Data hold ties, +-inf, +-0, subnormals and a NaN; zero points sit at qmin, qmax and mid-range of
signed and unsigned 8-, 4- and 2-bit ranges.

test_graph_keeps_its_workspace_when_a_later_call_grows_it: a graph captured at a small M keeps writing the workspace it
was captured with; an eager call that outgrows that workspace must not hand its memory to later allocations.
"""
import ctypes
from fractions import Fraction

import numpy as np
import pytest
import torch

import int8_geometry as geo
from branch_cases import C, assert_table_covers, check_reach, params
from gpu_util import dev, no_tf32, on_device, seed, stream  # noqa: F401 -- no_tf32: a fixture
from int8_conv_ref import integer_terms as conv_integer_terms
from int8_conv_ref import lowered, to_nchw
from int8_conv_ref import truth as conv_truth
from int8_linear_ref import grid_offset
from int8_linear_ref import integer_terms as linear_integer_terms
from int8_linear_ref import truth as linear_truth
from int8_matmul_ref import integer_form, quantize_cols
from int8_matmul_ref import truth as matmul_truth
from oracle import qdq as oqdq
from sparsebit_b200 import _lib, ops

F32, F64 = np.float32, np.float64
SENTINEL = 0x7B      # 0x7B7B7B7B = 1.3e36 as fp32: finite
WS_FILL = 0xA5
WS_OFFSETS = (0, 16, 1008)
SLACK = 256          # guard bytes behind every output and workspace
RANGES = {"s8": (-128, 127), "u8": (0, 255), "s4": (-8, 7), "u4": (0, 15), "s2": (-2, 1), "u2": (0, 3)}


# -------------------------------------------------------------------------------------------------- cases
# op: rows | cols | im2col | linear | conv | matmul; the spec's offsets (x_off, a_off, b_off, out_off) are in bytes
_GEOMETRY_KEYS = {"rows", "k", "x_off", "per_row", "batch", "n", "c", "h", "w", "kh", "kw", "stride", "pad", "dilation",
                  "m", "bias", "c_out", "b_k_major", "a_off", "b_off", "out_off"}


def branches(case):
    return geo.branches(case.op, **{k: v for k, v in case.spec.items() if k in _GEOMETRY_KEYS})


def _covers(case):
    """Everything the case reaches, not only its targets: REQUIRED must name every id the geometry produces."""
    reached = branches(case) | case.claims
    check_reach(case, reached)
    return reached


CASES = [
    C("rows_per_row", "rows", ["rows.per_row", "rows.scalar", "rows.trips", "rows.last_cta_partial", "rows.kpad"],
      rows=37, k=1001, per_row=True, xr="s8", zp="mid"),
    C("rows_k16_full", "rows", ["rows.vec", "rows.vec.full", "rows.one_trip", "rows.idle_lanes", "rows.per_tensor"],
      rows=16, k=16, xr="u4", zp="max"),
    C("rows_k768_misaligned", "rows", ["rows.scalar", "rows.scalar.misaligned", "rows.trips"],
      rows=24, k=768, x_off=4, xr="u8", zp="min"),
    C("cols_vec", "cols", ["cols.vec", "cols.n_tile_partial", "cols.chunks", "cols.short_chunk", "cols.batch"],
      batch=3, k=300, n=200, xr="u8", zp="mid"),
    C("cols_scalar", "cols", ["cols.scalar", "cols.quad_partial", "cols.one_chunk", "cols.short_chunk", "cols.k4_partial",
                              "cols.batch"], batch=2, k=77, n=131, xr="s2", zp="min"),
    C("cols_misaligned", "cols", ["cols.scalar", "cols.one_chunk"], batch=1, k=128, n=64, x_off=4, xr="s4", zp="max"),
    C("low_all_pad", "im2col", ["low.tile_partial", "low.tile_spans_images", "low.one_chunk", "low.pad_taps",
                                "low.window_all_pad", "low.kpad"],
      n=2, c=3, h=5, w=6, kh=3, kw=3, pad=3, xr="u8", zp="min"),
    C("low_chunks", "im2col", ["low.chunks", "low.short_chunk", "low.stride", "low.dilation", "low.pad_taps", "low.kpad"],
      n=3, c=20, h=13, w=11, kh=3, kw=3, stride=2, pad=1, dilation=2, xr="s4", zp="mid"),
    C("lin_k20", "linear", ["gemm.kb1", "gemm.m_partial_wg1_idle", "gemm.n_partial", "gemm.bias", "rows.vec.tail",
                            "rows.idle_lanes"], ["gemm.nan_row"], m=37, k=20, n=200, xr="s8", zp="mid"),
    C("lin_k100", "linear", ["gemm.kb1", "gemm.tiles", "gemm.no_bias", "gemm.m_partial_wg1_idle", "rows.vec.tail"],
      ["gemm.nan_row"], m=150, k=100, n=260, bias=False, xr="u8", zp="min", wr="u8"),
    C("lin_k1004", "linear", ["gemm.kb_wrap1", "gemm.m_partial_both", "gemm.n_partial", "rows.vec.tail", "rows.trips"],
      ["gemm.nan_row"], m=200, k=1004, n=130, xr="u4", zp="max"),
    C("lin_k768_misaligned", "linear", ["gemm.kb6", "rows.scalar.misaligned"], ["gemm.nan_row"],
      m=64, k=768, n=128, x_off=4, xr="s2", zp="max"),
    C("lin_k512", "linear", ["gemm.kb_lt6", "rows.vec.full", "rows.one_trip"], m=129, k=512, n=128, xr="u2", zp="mid"),
    C("lin_k3000", "linear", ["gemm.kb_wrap2", "gemm.tiles", "gemm.m_partial_wg1_idle"], ["gemm.nan_row"],
      m=300, k=3000, n=136, xr="s8", zp="min"),
    C("conv_pad_u0", "conv", ["low.window_all_pad", "nchw.p_lt_128", "nchw.image_in_tile", "gemm.kb1", "gemm.bias"],
      n=2, c=3, h=5, w=6, kh=3, kw=3, pad=3, c_out=20, xr="u8", zp="min"),
    C("conv_pad_u255", "conv", ["low.window_all_pad", "nchw.p_lt_128", "gemm.no_bias"],
      n=3, c=2, h=4, w=7, kh=3, kw=3, pad=3, c_out=9, bias=False, xr="u8", zp="max"),
    C("conv_pad_s_m128", "conv", ["low.chunks", "low.short_chunk", "low.stride", "low.dilation", "gemm.kb_lt6"],
      n=3, c=20, h=13, w=11, kh=3, kw=3, stride=2, pad=1, dilation=2, c_out=33, xr="s8", zp="min"),
    C("conv_ring", "conv", ["gemm.kb_wrap2", "gemm.tiles", "gemm.n_partial", "nchw.image_in_tile",
                            "gemm.m_partial_wg1_idle"], n=2, c=200, h=12, w=12, kh=3, kw=3, pad=1, c_out=130, xr="u4",
      zp="mid"),
    C("conv_far_end", "conv", ["gemm.kb1", "low.pad_taps"], n=700, c=1, h=224, w=224, kh=7, kw=7, pad=3, c_out=8,
      xr="u8", zp="mid"),
    C("mm_k1665_rows", "matmul", ["mm.b_rows", "mm.kb_wrap2", "mm.store.vec2", "mm.batch_partial", "mm.m_partial_both",
                                  "mm.n_partial"], batch=3, m=200, k=1665, n=150, b_k_major=True, xr="s8", zp="mid",
      br="u8", bzp="max"),
    C("mm_k3000_cols", "matmul", ["mm.b_cols", "mm.kb_wrap2", "mm.store.scalar_odd", "mm.batch_partial",
                                  "mm.m_partial_wg1_idle", "cols.chunks", "cols.short_chunk", "cols.quad_partial"],
      batch=3, m=60, k=3000, n=131, b_k_major=False, xr="u8", zp="min", br="s4", bzp="min"),
    C("mm_n130_out4", "matmul", ["mm.store.scalar_even_misaligned", "mm.b_cols", "mm.kb_lt6", "mm.batch_partial"],
      batch=2, m=70, k=300, n=130, b_k_major=False, out_off=4, xr="s2", zp="mid", br="u2", bzp="mid"),
    C("mm_n131_out4", "matmul", ["mm.store.scalar_odd", "mm.b_rows", "mm.kb1", "mm.m_partial_wg1_idle"],
      batch=1, m=129, k=64, n=131, b_k_major=True, out_off=4, xr="u4", zp="max", br="s8", bzp="max"),
    C("mm_kb6", "matmul", ["mm.kb6", "mm.b_cols", "cols.vec", "mm.store.vec2"], batch=2, m=128, k=700, n=128,
      b_k_major=False, xr="s8", zp="max", br="u8", bzp="min"),
    C("mm_k1000", "matmul", ["mm.kb_wrap1", "mm.b_rows", "mm.store.vec2"], batch=1, m=256, k=1000, n=256, b_k_major=True,
      xr="u8", zp="mid", br="s8", bzp="mid"),
]


# -------------------------------------------------------------------------------------------------- CPU tests
def test_case_table_covers_every_branch():
    assert_table_covers(CASES, geo.REQUIRED, _covers, __doc__, reject_unknown=True, doc_branches=False)


def test_geometry_matches_hand_worked_launches():
    """Launch values worked by hand from int8_linear.cu."""
    # rows: 37 rows -> 5 CTAs of 8 warps; K = 1001 is not a multiple of 4 -> scalar; Kp = 1008 -> 2 lane trips
    assert geo.rows_plan(37, 1001) == dict(grid=5, kp=1008, vec=False, trips=2)
    assert geo.rows_plan(24, 768, x_off=4)["vec"] is False and geo.rows_plan(24, 768)["vec"] is True
    assert geo.rows_branches(1, 20) >= {"rows.vec.tail"} and geo.rows_branches(1, 32) >= {"rows.vec.full"}
    # cols: N = 200 -> 4 tiles of 64 per batch entry; K = 300 -> Kp 304 = 128 + 128 + 48
    assert geo.cols_plan(3, 300, 200) == dict(grid=12, tiles_n=4, kp=304, vec=True, chunks=3, last_kc=48)
    assert geo.cols_plan(2, 77, 131)["vec"] is False
    # lowering: 2 x 3 x 5 x 6, 3x3 pad 3 -> OH 9, OW 10, M = 180 -> 2 CTAs; K = 27 -> Kp 32
    p = geo.low_plan(2, 3, 5, 6, 3, 3, 1, 3, 1)
    assert (p["oh"], p["ow"], p["m"], p["grid"], p["k"], p["kp"], p["chunks"]) == (9, 10, 180, 2, 27, 32, 1)
    # ... output row 0 sits at ih = -3: all three kernel rows (-3, -2, -1) in the padding
    assert geo._taps_out(5, 9, 3, 1, 3, 1)[:3] == [3, 2, 1]
    # stride 2, dilation 2, 13 x 11, pad 1: OH = (13 + 2 - 4 - 1) // 2 + 1 = 6, OW = 5; K = 180 -> Kp 192 = 128 + 64
    p = geo.low_plan(3, 20, 13, 11, 3, 3, 2, 1, 2)
    assert (p["oh"], p["ow"], p["kp"], p["chunks"], p["last_kc"]) == (6, 5, 192, 2, 64)
    # the far-end conv: M Kp = 700 224^2 64 >= 2^31
    p = geo.low_plan(700, 1, 224, 224, 7, 7, 1, 3, 1)
    assert p["m"] == 700 * 224 * 224 and p["m"] * p["kp"] >= 2 ** 31
    # GEMM: M 300 x N 136 -> 3 x 2 tiles; K 3000 -> 24 k-blocks; K 768 -> 6
    assert geo.gemm_plan(300, 3000, 136) == dict(tiles_m=3, tiles_n=2, grid=6, num_kb=24)
    assert geo.gemm_plan(100, 3000, 131, batch=3)["grid"] == 6
    assert [geo.ring_branch(geo.gemm_plan(1, k, 1)["num_kb"], "") for k in (128, 129, 768, 769, 1536, 1537)] == [
        "kb1", "kb_lt6", "kb6", "kb_wrap1", "kb_wrap1", "kb_wrap2"]
    assert geo._m_tail(64, "") == {"m_partial_wg1_idle"} and geo._m_tail(65, "") == {"m_partial_both"}
    assert geo._m_tail(256, "") == set()
    # matmul stores: even N, out 8-byte aligned -> float2; out at +4 -> scalar
    assert geo.vec2(130) and not geo.vec2(130, 4) and not geo.vec2(131)


def _linear_y(i, sx, sw, bias=None, nan_rows=None):
    """The linear / conv epilogue, :486-489: fp32(fp64(I) * (fp64 s_x * fp64 s_w)) (+ bias in fp32), NaN rows."""
    with np.errstate(all="ignore"):
        y = (np.asarray(i).astype(F64) * (F64(F32(sx)) * np.asarray(sw, F32).astype(F64))[None, :]).astype(F32)
        if bias is not None:
            y = (y + np.asarray(bias, F32)[None, :]).astype(F32)
    if nan_rows is not None:
        y[np.asarray(nan_rows)] = np.nan
    return y


def test_references_reproduce_hand_worked_outputs():
    # linear, signed x (zp 0) and unsigned w (zp 130, stored 2): x = [1, -2, 3] s_x, w = [3, -2, 1] s_w -> grid
    # [133, 128, 131], stored b = [5, 0, 3]; I = sum a b - Z_w sum a = 14 - 2 * 2 = 10 = 3 + 4 + 3; y = 10 * 0.5 * 0.25 + 1
    x = np.array([[1, -2, 3]], F32) * F32(0.5)
    w = np.array([[3, -2, 1]], F32) * F32(0.25)
    a, b, zx, zw, i = linear_integer_terms(x, 0.5, 0, -128, 127, w, 0.25, 130, 0, 255)
    assert a.tolist() == [[1, -2, 3]] and b.tolist() == [[5, 0, 3]] and zx == 0 and zw.tolist() == [2] and i.tolist() == [[10]]
    assert _linear_y(i, 0.5, [0.25], [1.0]).tolist() == [[2.25]]
    # double rounding: I = 1547893691 (94475 products (-128)(-128), (-128)(-119) and 59 * 1), s_x = 1 and
    # s_w = 12358003 2^-23.  I s_w lies 2^-23 of an fp32 ulp (= 256) above the midpoint between two fp32 numbers, within
    # half an fp64 ulp of it: fp64 rounds onto the midpoint, fp32 breaks the tie to even (0x1.0fd670p+31), while the
    # exact product rounds once to 0x1.0fd672p+31.  The kernel rounds twice (:487); the reference must too.
    sw = F32(12358003 * 2.0 ** -23)
    xa = np.array([-128] * 94476 + [59], F32)
    wa = (np.array([-128] * 94475 + [-119, 1], F32) * sw).astype(F32)
    _, _, _, _, i = linear_integer_terms(xa[None], 1.0, 0, -128, 127, wa[None], sw, 0, -128, 127)
    assert i.tolist() == [[1547893691]]
    y = _linear_y(i, 1.0, [sw])
    assert float(y[0, 0]).hex() == "0x1.0fd6700000000p+31"
    single = Fraction(1547893691) * Fraction(float(sw))
    assert abs(Fraction(float.fromhex("0x1.0fd6720000000p+31")) - single) < abs(Fraction(float(y[0, 0])) - single)
    # matmul: a [1, 2] at zp 1 (signed), b [2, 2] with a NaN in column 1; I = sum (a - 1)(b - 0)
    ea = (np.array([[[3.0, -1.0]]], F32), F32(1.0), F32(1.0), -128, 127)
    eb = (np.array([[[2.0, np.nan], [5.0, 1.0]]], F32), F32(0.5), F32(0.0), -8, 7)
    qa, qb, za, zb, i, y = integer_form(ea, eb)
    # grid a = [4, 0], v_a = [3, -1]; v_b col 0 = [4, 7] (5 / 0.5 = 10 clamps to 7) -> I = 12 - 7 = 5, y = 5 * 0.5
    assert qa.tolist() == [[[4, 0]]] and za == 1 and zb == 0 and i[0, 0, 0] == 5 and y[0, 0, 0] == 2.5
    assert np.isnan(y[0, 0, 1])
    # conv: one pixel 1 x 1 x 1 x 1, 3x3 padding 1, unsigned zp 255: eight padding taps store 255 - 128 = 127
    q, s, nan = lowered(np.array([[[[0.5]]]], F32), 3, 0.25, 255, 0, 255, 1, 1, 1)
    # the centre tap: clamp(round(2) + 255, 0, 255) - 128 = 127 too; the K padding 9..15 is zero
    assert q.tolist() == [[127] * 9 + [0] * 7] and s.tolist() == [9 * 127] and not nan.any()
    q, s, _ = lowered(np.array([[[[0.5]]]], F32), 3, 0.25, 0, 0, 255, 1, 1, 1)
    assert q.tolist() == [[-128] * 4 + [2 - 128] + [-128] * 4 + [0] * 7] and s.tolist() == [8 * -128 - 126]


# -------------------------------------------------------------------------------------------------- data
def _zp(qr, at):
    qmin, qmax = RANGES[qr]
    return F32({"min": qmin, "max": qmax, "mid": (qmin + qmax) // 2 + 0.5 * (qmax - qmin > 8)}[at])


def activations(rng, shape, s, z, qr, nan_at=None):
    """Values over the whole grid and past both clamps, 1 in 4 a tie (j + 1/2) s, +-inf, +-0, subnormals, and a NaN at
    ``nan_at`` (an index tuple) if given.  Conv cases plant it at an odd row and column, which stride 2 with dilation 2
    and padding 1 reach too."""
    qmin, qmax = RANGES[qr]
    x = (rng.uniform(qmin - z - 2, qmax - z + 2, shape) * float(s)).astype(F32)
    ties = ((rng.integers(qmin, qmax + 1, shape) - z + 0.5) * float(s)).astype(F32)
    x = np.where(rng.random(shape) < 0.25, ties, x)
    flat = x.reshape(-1)
    special = np.array([np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39], F32)
    flat[rng.choice(flat.size, size=min(flat.size, special.size), replace=False)] = special[:flat.size]
    x = flat.reshape(shape)
    if nan_at is not None:
        x[nan_at] = np.nan
    return x


def weights(rng, n, k, wr):
    """Per-channel weights on ``wr``: signed ranges at zp 0, unsigned ones mid-range."""
    qmin, qmax = RANGES[wr]
    ws = rng.uniform(0.004, 0.02, n).astype(F32)
    wz = np.full(n, 0 if qmin < 0 else (qmin + qmax) // 2, F32)
    w = (rng.uniform(qmin - 1, qmax + 1, (n, k)) - wz[:, None]) * ws[:, None]
    return w.astype(F32), ws, wz


def scalar(v):
    return torch.tensor([float(v)], dtype=torch.float32, device=dev())


class Guarded:
    """``nbytes`` bytes at ``off`` into a buffer filled with ``fill``, with SLACK guard bytes behind them."""

    def __init__(self, nbytes, off=0, fill=SENTINEL):
        self.off, self.n, self.fill = off, int(nbytes), fill
        self.raw = torch.full((off + self.n + SLACK,), fill, dtype=torch.uint8, device=dev())

    def ptr(self):
        return self.raw.data_ptr() + self.off

    def view(self, dtype, shape):
        return self.raw[self.off:self.off + self.n].view(dtype).view(shape)

    def intact(self):
        return bool((self.raw[:self.off] == self.fill).all() and (self.raw[self.off + self.n:] == self.fill).all())


def _check(rc):
    assert rc == 0, _lib.load().sb200_last_error()


def bytes_equal(a, b):
    """The same shape and the same bytes: unlike gpu_util.bits_equal, +0 and -0 differ and so do NaN payloads."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def same_floats(a, b):
    """Bit for bit, any NaN equal to any NaN."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and bytes_equal(a[~na], b[~nb])


def within_truth(y, t, bound):
    y = np.asarray(y, F64)
    assert np.array_equal(np.isnan(y), np.isnan(t)), "NaN positions differ from the fp64 truth"
    ok = ~np.isnan(t)
    err = np.abs(y[ok] - t[ok])
    assert np.all(err <= bound[ok]), f"max error {err.max():.3g} over the 2^-21 bound"


# -------------------------------------------------------------------------------------------------- quantizers
def _run_quantizer(call, outs):
    """Three calls into fresh sentinel-filled outputs; they must agree and leave the slack alone."""
    runs = []
    for _ in range(3):
        bufs = [Guarded(nb) for nb, _, _ in outs]
        _check(call(*[b.ptr() for b in bufs]))
        torch.cuda.synchronize()
        assert all(b.intact() for b in bufs), "a quantizer wrote past its output"
        runs.append([b.view(dt, sh).cpu().numpy() for b, (_, dt, sh) in zip(bufs, outs)])
    for r in runs[1:]:
        assert all(bytes_equal(u, v) for u, v in zip(runs[0], r))
    return runs[0]


QUANT_CASES = [c for c in CASES if c.op in ("rows", "cols", "im2col")]


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(QUANT_CASES))
def test_quantizer_branch_is_the_oracle_grid(case, no_tf32):
    check_reach(case, branches(case))
    rng = np.random.default_rng(seed(case.name))
    qr, lib = case.get("xr"), _lib.load()
    qmin, qmax = RANGES[qr]
    s, z = F32(0.0371), _zp(qr, case.get("zp"))
    x_off = case.get("x_off", 0)
    if case.op == "rows":
        rows, k = case.get("rows"), case.get("k")
        kp = geo.padded_k(k)
        if case.get("per_row"):
            s = rng.uniform(0.01, 0.05, rows).astype(F32)
            z = rng.integers(qmin, qmax + 1, rows).astype(F32)
            z[:3] = [qmin, qmax, F32(qmin + 0.5)]
        sv, zv = np.broadcast_to(s, (rows,)) if case.get("per_row") else np.array([s], F32), \
            np.broadcast_to(z, (rows,)) if case.get("per_row") else np.array([z], F32)
        x = activations(rng, (rows, k), float(np.max(s)), float(np.min(z)), qr, (1, k // 2))
        x_d, s_d, z_d = on_device(x, x_off, unit="byte"), on_device(sv), on_device(zv)
        q, rsum, nan = _run_quantizer(
            lambda pq, ps, pn: lib.sb200_int8_quantize_rows(x_d.data_ptr(), s_d.data_ptr(), z_d.data_ptr(),
                                                            int(bool(case.get("per_row"))), qmin, qmax, pq, ps, pn, rows, k,
                                                            stream()),
            [(rows * kp, torch.int8, (rows, kp)), (rows * 4, torch.int32, (rows,)), (rows, torch.uint8, (rows,))])
        g = oqdq.quantize_int(x, sv if case.get("per_row") else s, zv if case.get("per_row") else z, qmin, qmax)
        en = np.isnan(g)
        stored = np.where(en, 0, np.nan_to_num(g) - grid_offset(qmin)).astype(np.int64)
        eq = np.zeros((rows, kp), np.int64)
        eq[:, :k] = stored
        esum, enan = stored.sum(1), en.any(1)
        wrapped = ops.int8_quantize_rows(x_d, s_d, z_d, qmin, qmax)
    elif case.op == "cols":
        batch, k, n = case.get("batch"), case.get("k"), case.get("n")
        kp = geo.padded_k(k)
        x = activations(rng, (batch, k, n), s, z, qr, (0, k // 3, n - 1))
        x_d, s_d, z_d = on_device(x, x_off, unit="byte"), scalar(s), scalar(z)
        q, rsum, nan = _run_quantizer(
            lambda pq, ps, pn: lib.sb200_int8_quantize_cols(x_d.data_ptr(), s_d.data_ptr(), z_d.data_ptr(), qmin, qmax, pq,
                                                            ps, pn, batch, k, n, stream()),
            [(batch * n * kp, torch.int8, (batch, n, kp)), (batch * n * 4, torch.int32, (batch, n)),
             (batch * n, torch.uint8, (batch, n))])
        eq, esum, enan = quantize_cols(x, s, z, qmin, qmax)
        wrapped = ops.int8_quantize_cols(x_d, s_d, z_d, qmin, qmax)
    else:
        n, c, h, w, kh, kw = (case.get(key) for key in ("n", "c", "h", "w", "kh", "kw"))
        stride, pad, dil = case.get("stride", 1), case.get("pad", 0), case.get("dilation", 1)
        p = geo.low_plan(n, c, h, w, kh, kw, stride, pad, dil)
        m, kp = p["m"], p["kp"]
        x = activations(rng, (n, c, h, w), s, z, qr, (n - 1, c - 1, h // 2 | 1, w // 2 | 1))
        x_d, s_d, z_d = on_device(x), scalar(s), scalar(z)
        g = ops.conv2d_geometry(x.shape, (kh, kw), stride, pad, dil)
        q, rsum, nan = _run_quantizer(
            lambda pq, ps, pn: lib.sb200_int8_im2col_quantize(x_d.data_ptr(), ctypes.byref(g), s_d.data_ptr(),
                                                              z_d.data_ptr(), qmin, qmax, pq, ps, pn, stream()),
            [(m * kp, torch.int8, (m, kp)), (m * 4, torch.int32, (m,)), (m, torch.uint8, (m,))])
        eq, esum, enan = lowered(x, (kh, kw), s, z, qmin, qmax, stride, pad, dil)
        wrapped = ops.int8_im2col_quantize(x_d, (kh, kw), s_d, z_d, qmin, qmax, stride, pad, dil)
        if "low.window_all_pad" in case.targets:
            assert (eq[:, :p["k"]] == int(np.rint(z)) - grid_offset(qmin)).all(axis=1).any(), "no window in the padding"
    assert np.array_equal(q.astype(np.int64), eq), "q differs from the oracle grid"
    assert np.array_equal(rsum.astype(np.int64), esum), "sums differ"
    assert np.array_equal(nan.astype(bool), enan) and enan.any() and not enan.all()
    assert nan.max() <= 1
    wq, wsum, wnan = (t.cpu().numpy() for t in wrapped)
    assert bytes_equal(wq, q) and bytes_equal(wsum, rsum) and np.array_equal(wnan, nan.astype(bool))


# -------------------------------------------------------------------------------------------------- GEMMs
def _run_gemm(call, out_bytes, ws_bytes, out_off=0, offsets=WS_OFFSETS):
    """One call per workspace base offset, each into a fresh sentinel-filled output: they must agree bit for bit and
    leave the output slack and the workspace guard bytes alone."""
    runs = []
    for off in offsets:
        out = Guarded(out_bytes, out_off)
        ws = Guarded(ws_bytes, off, WS_FILL)
        _check(call(out.ptr(), ws.ptr(), ws_bytes))
        torch.cuda.synchronize()
        assert out.intact(), f"the GEMM wrote past its output (workspace at +{off})"
        assert ws.intact(), f"a kernel wrote past the workspace (base at +{off})"
        runs.append(out.view(torch.float32, (out_bytes // 4,)).cpu().numpy())
        del out, ws
    for r in runs[1:]:
        assert bytes_equal(runs[0], r), "the calls differ"
    return runs[0]


def _w_device(w, ws, wz, wr):
    qmin, qmax = RANGES[wr]
    w_q, w_sum, w_nan = ops.int8_quantize_rows(on_device(w), on_device(ws), on_device(wz), qmin, qmax)
    assert not w_nan.any()
    return w_q, w_sum, on_device(ws), on_device((np.rint(wz) - grid_offset(qmin)).astype(np.int32))


def _linear_case(case, rng, lib):
    m, k, n, x_off = case.get("m"), case.get("k"), case.get("n"), case.get("x_off", 0)
    xr, wr = case.get("xr"), case.get("wr", "s8")
    qmin, qmax = RANGES[xr]
    s, z = F32(0.0371), _zp(xr, case.get("zp"))
    x = activations(rng, (m, k), s, z, xr, (m // 2, k - 1))
    w, ws, wz = weights(rng, n, k, wr)
    bias = rng.standard_normal(n).astype(F32) if case.get("bias", True) else None
    x_d, s_d, z_d = on_device(x, x_off, unit="byte"), scalar(s), scalar(z)
    w_q, w_sum, ws_d, wz_d = _w_device(w, ws, wz, wr)
    b_d = on_device(bias) if bias is not None else None
    need = int(lib.sb200_int8_linear_workspace_bytes(m, k))
    y = _run_gemm(lambda po, pw, nb: lib.sb200_int8_linear(
        x_d.data_ptr(), s_d.data_ptr(), z_d.data_ptr(), qmin, qmax, w_q.data_ptr(), w_sum.data_ptr(), ws_d.data_ptr(),
        wz_d.data_ptr(), b_d.data_ptr() if b_d is not None else None, po, m, k, n, pw, nb, stream()), m * n * 4, need)
    y = y.reshape(m, n)
    wrapped = ops.int8_linear(x_d, s_d, z_d, qmin, qmax, w_q, w_sum, ws_d, wz_d, b_d).cpu().numpy()
    nan_rows = np.isnan(oqdq.quantize_int(x, s, z, qmin, qmax)).any(1)
    with np.errstate(all="ignore"):
        i = linear_integer_terms(x, s, z, qmin, qmax, w, ws, wz, *RANGES[wr])[4]
    exact = _linear_y(i, s, ws, bias, nan_rows)
    t, bound = linear_truth(x, s, z, qmin, qmax, w, ws, wz, *RANGES[wr], bias)
    return y, wrapped, exact, t, bound, nan_rows


def _conv_case(case, rng, lib, images=None):
    n, c, h, w_, kh, kw, c_out = (case.get(key) for key in ("n", "c", "h", "w", "kh", "kw", "c_out"))
    stride, pad, dil = case.get("stride", 1), case.get("pad", 0), case.get("dilation", 1)
    xr, wr = case.get("xr"), case.get("wr", "s8")
    qmin, qmax = RANGES[xr]
    s, z = F32(0.0371), _zp(xr, case.get("zp"))
    p = geo.low_plan(n, c, h, w_, kh, kw, stride, pad, dil)
    w, ws, wz = weights(rng, c_out, c * kh * kw, wr)
    w = w.reshape(c_out, c, kh, kw)
    bias = rng.standard_normal(c_out).astype(F32) if case.get("bias", True) else None
    if images is None:
        x = activations(rng, (n, c, h, w_), s, z, xr, (n - 1, c - 1, h // 2 | 1, w_ // 2 | 1))
        x_d = on_device(x)
    else:  # the far end: random data on the device, the oracle's images planted first and last
        x = activations(rng, (2, c, h, w_), s, z, xr, (1, c - 1, h // 2 | 1, w_ // 2 | 1))
        x_d = torch.randn(n, c, h, w_, device=dev()) * float(s) * 40
        x_d[0], x_d[-1] = torch.from_numpy(x[0]).to(dev()), torch.from_numpy(x[1]).to(dev())
    s_d, z_d = scalar(s), scalar(z)
    w_q, w_sum, ws_d, wz_d = _w_device(w.reshape(c_out, -1), ws, wz, wr)
    b_d = on_device(bias) if bias is not None else None
    g = ops.conv2d_geometry((n, c, h, w_), (kh, kw), stride, pad, dil)
    need = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    out_n = n * c_out * p["p"]
    y = _run_gemm(lambda po, pw, nb: lib.sb200_int8_conv2d(
        x_d.data_ptr(), ctypes.byref(g), s_d.data_ptr(), z_d.data_ptr(), qmin, qmax, w_q.data_ptr(), w_sum.data_ptr(),
        ws_d.data_ptr(), wz_d.data_ptr(), b_d.data_ptr() if b_d is not None else None, po, c_out, pw, nb, stream()),
        out_n * 4, need, offsets=WS_OFFSETS if images is None else (0, 16))
    y = y.reshape(n, c_out, p["oh"], p["ow"])
    wrapped = ops.int8_conv2d(x_d, s_d, z_d, qmin, qmax, w_q, w_sum, ws_d, wz_d, (kh, kw), b_d, stride, pad, dil)
    if images is not None:
        y, wrapped = y[[0, -1]], wrapped[[0, -1]].cpu().numpy()
    else:
        wrapped = wrapped.cpu().numpy()
    del x_d
    nx = x.shape[0]
    _, _, nan = lowered(x, (kh, kw), s, z, qmin, qmax, stride, pad, dil)
    with np.errstate(all="ignore"):
        i = conv_integer_terms(x, s, z, qmin, qmax, w, ws, wz, *RANGES[wr], stride, pad, dil)[4]
    exact = to_nchw(_linear_y(i, s, ws, bias, nan), nx, p["oh"], p["ow"])
    t, bound = conv_truth(x, s, z, qmin, qmax, w, ws, wz, *RANGES[wr], bias, stride, pad, dil)
    pad_tap = int(np.rint(z)) - grid_offset(qmin)
    return y, wrapped, exact, t, bound, pad_tap


def _matmul_case(case, rng, lib):
    batch, m, k, n = (case.get(key) for key in ("batch", "m", "k", "n"))
    kmaj, out_off = case.get("b_k_major"), case.get("out_off", 0)
    ar, br = case.get("xr"), case.get("br")
    sa, za, sb, zb = F32(0.0371), _zp(ar, case.get("zp")), F32(0.0213), _zp(br, case.get("bzp"))
    xa = activations(rng, (batch, m, k), sa, za, ar, (batch - 1, m // 2, k // 3))
    xb = activations(rng, (batch, k, n), sb, zb, br, (0, k // 2, n - 2))
    a_d = on_device(xa, case.get("a_off", 0), unit="byte")
    b_host = np.ascontiguousarray(np.swapaxes(xb, -1, -2)) if kmaj else xb
    b_d = on_device(b_host, case.get("b_off", 0), unit="byte")
    pa = (scalar(sa), scalar(za), *RANGES[ar])
    pb = (scalar(sb), scalar(zb), *RANGES[br])
    need = int(lib.sb200_int8_matmul_workspace_bytes(batch, m, k, n))
    y = _run_gemm(lambda po, pw, nb: lib.sb200_int8_matmul(
        a_d.data_ptr(), b_d.data_ptr(), int(kmaj), pa[0].data_ptr(), pa[1].data_ptr(), pa[2], pa[3], pb[0].data_ptr(),
        pb[1].data_ptr(), pb[2], pb[3], po, batch, m, k, n, pw, nb, stream()), batch * m * n * 4, need, out_off)
    y = y.reshape(batch, m, n)
    bt = b_d.transpose(-2, -1) if kmaj else b_d
    wrapped = ops.int8_matmul(a_d, pa[0], pa[1], pa[2:], bt, pb[0], pb[1], pb[2:]).cpu().numpy()
    ea, eb = (xa, sa, za, *RANGES[ar]), (xb, sb, zb, *RANGES[br])
    with np.errstate(all="ignore"):
        exact = integer_form(ea, eb)[-1].astype(F32)
    t, bound = matmul_truth(ea, eb)
    return y, wrapped, exact, t, bound


GEMM_CASES = [c for c in CASES if c.op in ("linear", "conv", "matmul") and c.name != "conv_far_end"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(GEMM_CASES))
def test_gemm_branch_is_the_integer_form(case, no_tf32):
    check_reach(case, branches(case))
    rng = np.random.default_rng(seed(case.name))
    lib = _lib.load()
    if case.op == "linear":
        y, wrapped, exact, t, bound, nan_rows = _linear_case(case, rng, lib)
        if "gemm.nan_row" in case.claims:
            assert nan_rows.any() and not nan_rows.all()
    elif case.op == "conv":
        y, wrapped, exact, t, bound, pad_tap = _conv_case(case, rng, lib)
        if case.name.startswith("conv_pad_"):
            assert pad_tap in (-128, 127)
        assert np.isnan(exact).any() and not np.isnan(exact).all()
    else:
        y, wrapped, exact, t, bound = _matmul_case(case, rng, lib)
    assert same_floats(wrapped, y), "the ops wrapper and the C entry point differ"
    assert same_floats(y, exact), f"{np.count_nonzero(~np.isclose(y, exact, equal_nan=True, rtol=0, atol=0))} outputs " \
                                  "differ from the integer form"
    within_truth(y, t, bound)


@pytest.mark.gpu
def test_conv_gemm_far_end_of_a_workspace_past_2_31(no_tf32):
    """M Kp >= 2^31 through the GEMM as well as the lowering: 700 x 1 x 224^2, 7x7, padding 3, C_out = 8.  The first and
    the last image are the oracle's; both equal the integer form bit for bit."""
    case = next(c for c in CASES if c.name == "conv_far_end")
    check_reach(case, branches(case))
    p = geo.low_plan(700, 1, 224, 224, 7, 7, 1, 3, 1)
    need = p["m"] * p["kp"] + 5 * p["m"] + 700 * 224 * 224 * 4 + 2 * p["m"] * 8 * 4 + (1 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs about {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    try:
        with torch.cuda.stream(side):  # the ops wrapper's 2.3 GB workspace is this stream's, dropped below
            y, wrapped, exact, t, bound, _ = _conv_case(case, np.random.default_rng(seed(case.name)), _lib.load(), images=True)
        torch.cuda.synchronize()
        assert same_floats(wrapped, y) and same_floats(y, exact)
        assert np.isnan(y[1]).any() and not np.isnan(y[0]).any()
        within_truth(y, t, bound)
    finally:
        ops._int8_ws.pop((dev(), side.cuda_stream), None)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


# -------------------------------------------------------------------------------------------------- captured graphs
def _graph_calls(which, rng):
    """(small, big, bytes of the small call's workspace): ops calls whose workspaces differ in size."""
    lib = _lib.load()
    if which == "gptq4":
        from oracle import gptq as ogptq

        k, n = 512, 256
        wq = (rng.standard_normal((n, k)) / 16).astype(F32)
        s4, z4 = ogptq.find_params_int4(wq, 128)
        qw, sc, zr = (torch.from_numpy(v).to(dev()) for v in ogptq.pack_int4(ogptq.quantize_weight(wq, s4, z4, 128), s4, z4))
        xs, xb = torch.randn(64, k, device=dev()), torch.randn(4096, k, device=dev())
        out = torch.zeros(64, n, device=dev())

        def small():
            out.zero_()
            return ops.gptq4_matmul(xs, qw, out, sc, zr, 128)

        return small, lambda: ops.gptq4_matmul(xb, qw, torch.zeros(4096, n, device=dev()), sc, zr, 128), \
            int(lib.sb200_gptq4_workspace_bytes(64, k, n, 128))
    if which == "matmul":
        a1, b1 = torch.randn(2, 1, 64, device=dev()), torch.randn(2, 64, 96, device=dev())
        a2 = torch.randn(2, 4096, 64, device=dev())
        one, zero = scalar(0.02), scalar(0)
        f = lambda a: ops.int8_matmul(a, one, zero, (-128, 127), b1, one, zero, (-128, 127))
        return lambda: f(a1), lambda: f(a2), int(lib.sb200_int8_matmul_workspace_bytes(2, 1, 64, 96))
    k = 576 if which == "linear" else 64
    w = (rng.standard_normal((96, k)) / 8).astype(F32)
    ws, wz = np.full(96, 0.01, F32), np.zeros(96, F32)
    w_q, w_sum, ws_d, wz_d = _w_device(w, ws, wz, "s8")
    sx, zx = scalar(0.03), scalar(3)
    if which == "linear":
        x1, x2 = torch.randn(1, k, device=dev()), torch.randn(4096, k, device=dev())
        f = lambda x: ops.int8_linear(x, sx, zx, -128, 127, w_q, w_sum, ws_d, wz_d)
        return lambda: f(x1), lambda: f(x2), int(lib.sb200_int8_linear_workspace_bytes(1, k))
    x1, x2 = torch.randn(1, 4, 3, 3, device=dev()), torch.randn(64, 4, 32, 32, device=dev())
    f = lambda x: ops.int8_conv2d(x, sx, zx, -128, 127, w_q, w_sum, ws_d, wz_d, 4, None, 1, 1)
    small_ws = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(ops.conv2d_geometry(x1.shape, 4, 1, 1))))
    return lambda: f(x1), lambda: f(x2), small_ws


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["linear", "conv", "matmul", "gptq4"])
def test_graph_keeps_its_workspace_when_a_later_call_grows_it(which):
    """Capture at a small M on a side stream, run a larger call eagerly on that stream (it outgrows the workspace), then
    allocate a dozen tensors of the old workspace's size there and replay: the tensors keep their pattern and the replay
    still gives the eager result."""
    rng = np.random.default_rng(seed(which))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        small, big, old_bytes = _graph_calls(which, rng)
        want = small().clone()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            got = small()
        big()
        side.synchronize()
        held = [torch.full((old_bytes,), 0x3C, dtype=torch.uint8, device=dev()) for _ in range(12)]
        graph.replay()
        side.synchronize()
        intact = [bool((h == 0x3C).all()) for h in held]
    torch.cuda.current_stream().wait_stream(side)
    assert all(intact), f"the replay wrote into {intact.count(False)} of 12 later allocations"
    assert torch.equal(got, want)
    del graph
