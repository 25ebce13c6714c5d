"""The integer-grid GEMMs (csrc/int8_linear.cu, int8_sparse24.cu, int8_attention.cu) and the GPTQ matmul and input-gradient
kernels (csrc/gptq_simt.cu, gptq_tc.cu, gptq.cu, gptq_dgrad.cu) on operands of more than 2^31 elements, and the SIMT
input gradient on more than 262,140 rows.

Every one of these entry points takes int64 sizes and does its own 64-bit index arithmetic, and ordinary shapes reach
2^31: the q k^T scores of 64 x 12 heads at T = 2048 are 3.2e9 elements, and a QLoRA step at 64 x 4096 tokens gives a
grad_in of 2.9e9 elements on an 11008-wide down_proj.  Each case below runs one entry point just past its bound and names
the launch regime it must reach, as tests/int8_geometry.py, int8_sparse24_geometry.py, int8_attention_geometry.py and
gptq_geometry.py restate it; the CPU test checks the table against those plans.

  case           entry point                             shape                          past the bound
  i8_linear_x    ops.int8_linear                         M 524300, K 4100, N 136        x (row K), its row grid q (row Kp)
  i8_linear_out  ops.int8_linear                         M 195100, K 64, N 11008        out (m N + n)
  i8_mm_scores   ops.int8_matmul, K-major b (k^T)        513 x [2048, 64] @ [64, 2048]  out ((b M + m) N), the scores
  i8_mm_pv       ops.int8_matmul, N-major b              16400 x [64, 2056] @ [2056, 64]  a (p, rows) and b (v, b K N)
  sp24_out       ops.int8_sparse24_linear                M 262200, K 64, N 8192         the sparse GEMM's out
  attn_out       ops.int8_attention                      8200 x Tq 2048, Tk 16, d 16, dv 128   out [B, Tq, dv]
  gptq_simt_out  ops.gptq_matmul, 3-bit (SIMT)           M 16390, K 32, N 131072        out (atomicAdd at (m0 + m) N + n)
  gptq_simt_x    ops.gptq_matmul, 3-bit (SIMT)           M 32800, K 65536, N 64         x ((m0 + m) K): 512 K slices
  gptq_tc_out    ops.gptq4_matmul, impl 2 (wgmma)        M 8390000, K 256, N 256        out, and x's a_hi / a_lo planes
  gptq_f16_out   ops.gptq4_linear_f16, prefill M         M 524400, K 128, N 4096        the fp16 out
  dg_simt_rows   ops.gptq_matmul_dgrad, 3-bit and 4-bit impl 1   M 600001, K 64, N 256   the 65535 cap on gridDim.y
  dg_simt_max_m  ops.gptq_matmul_dgrad, 3-bit (SIMT)     M 2^31 - 1, K 1, N 1          the row-tile count M + 3 > INT_MAX
  dg_simt_in     ops.gptq_matmul_dgrad, 2-bit (SIMT)     M 131000, K 16400, N 128       grad_in ((m0 + m) K + k)
  dg_tc          ops.gptq_matmul_dgrad, impl 2 (wgmma)   M 8390000, K 256, N 256        grad_out, g_hi / g_lo, grad_in

p of i8_mm_pv is [B, Tq, Tk] with Tq = dv = 64 rather than Tq = Tk: with both operands past 2^31 a square p would make
the output as large as p, and the case would need more than 30 GB.  dg_simt_rows stays far below 2^31 elements
(K and N small): it is the row count alone that matters, since the SIMT input gradient wants ceil(M / 4) row tiles and
CUDA allows 65535 in y; the kernel walks its row tiles in a loop from there on.  Its slab launches keep below that, so
they never loop.  dg_simt_max_m takes the largest M the argument check accepts, where the kernel's tile count
ceil(M / 4) must be formed without M + 3 overflowing 32 bits (the Python restatement cannot overflow, so only this case
can see it).  With K = N = 1 every output is one product, (g s) q - g z added to the prefill, so instead of slab
launches, which would loop as well, the whole grad_in is compared with that product computed in the same fp32
operations, bit for bit.  The SIMT gradient's split-N path (partial sums plus dgrad_finish_kernel) has no case: it is taken only
when the grid has fewer than 1024 base CTAs, which bounds M K far below 2^31 (a CPU test checks this).

How each is checked.  Inputs come from a seeded torch.Generator on the device.  Outputs written by plain stores start
as a NaN sentinel (no element may keep it); outputs that are accumulated into (GPTQ out, grad_in) start as a seeded
pattern of multiples of 1/16, which is subtracted back out exactly (in fp64) before comparing.  Values are planted in
windows of whole rows (batch entries for the batched cases) at the head, around element 2^31 of every operand past the
bound (around row 262,140 for dg_simt_rows) and at the end: NaN and +-inf in the activations of the integer paths,
whose NaN rules are documented, and for GPTQ rows scaled by 2^-60 and 2^40 (2^-8 and 2^6 in fp16).
* Windows against an fp64 truth: the integer paths against tests/int8_linear_ref.py, int8_matmul_ref.py (the 2:4 linear
  against the dense linear's truth, which it equals bit for bit) and int8_attention_ref.py with their bounds; GPTQ and
  the input gradient against tests/gptq_dgrad_ref.py's dequantised weights at rtol = atol = 1e-5 elementwise, each
  scaled row divided by its power-of-two factor first (the fp16 output: half an fp16 ulp + 1e-5, as the branch suite).
* The whole output against launches of the same entry point on row slabs of at most 2^28 elements, far below the index
  ranges under test, compared on the device: bit for bit for every kernel but the SIMT forward, whose K slices add into
  out with atomics in no fixed order (within 2e-5 relative and absolute, a scaled row's absolute bar scaled with it:
  two results within 1e-5 of the truth).  The CPU test checks that every slab takes the same kernel as the whole.
Each GPU test states its device-memory need, skips when the device has less free and checks its peak against it.
"""
import contextlib
import functools
import gc

import numpy as np
import pytest
import torch

import gptq_geometry as ggeo
import int8_attention_geometry as ageo
import int8_attention_ref as aref
import int8_geometry as igeo
import int8_linear_ref as lref
import int8_matmul_ref as mref
import int8_sparse24_geometry as sgeo
import int8_sparse24_ref as sref
from branch_cases import C, assert_table_covers, check_reach, params
from gpu_util import dev, real_sm, seed_of, stream
from gptq_dgrad_ref import dequant_weight
from sparsebit_b200 import _lib, ops

F32, F64 = np.float32, np.float64
B31 = 1 << 31
SUB = 1 << 28          # elements per slab launch at most
WIN = 1 << 16          # elements per truth window, about
SENTINEL = 0x7FA5A5A5  # a NaN no kernel writes
SENTINEL16 = 0x7DA5    # the same in fp16
GIB = 1 << 30
MAX_GIB = 28.0         # ~30 GB: the suite shares the card
TINY, HUGE = 2.0 ** -60, 2.0 ** 40
TINY16, HUGE16 = 2.0 ** -8, 2.0 ** 6
GS = 128

# -------------------------------------------------------------------------------------------------- cases
CASES = [
    C("i8_linear_x", "linear", ("rows.vec", "rows.vec.tail", "rows.trips", "gemm.kb_wrap2", "gemm.n_partial",
                                "gemm.m_partial_wg1_idle"), m=524300, k=4100, n=136, bounds=("x", "q"), gib=12.5),
    C("i8_linear_out", "linear", ("rows.vec", "rows.one_trip", "gemm.kb1", "gemm.tiles", "gemm.m_partial_wg1_idle"),
      m=195100, k=64, n=11008, bounds=("out",), gib=11.0),
    C("i8_mm_scores", "matmul", ("mm.b_rows", "mm.kb1", "mm.store.vec2"), batch=513, m=2048, k=64, n=2048,
      b_k_major=True, bounds=("out",), gib=11.5),
    C("i8_mm_pv", "matmul", ("mm.b_cols", "cols.vec", "cols.chunks", "cols.batch", "mm.kb_wrap2", "rows.kpad"),
      batch=16400, m=64, k=2056, n=64, b_k_major=False, bounds=("a", "qa", "b", "qb"), gib=22.5),
    C("sp24_out", "sparse24", ("gemm_store_vec4", "gemm_one_stage", "gemm_pad_steps", "gemm_no_second_box",
                               "gemm_partial_m"), m=262200, k=64, n=8192, bounds=("out",), gib=10.5),
    C("attn_out", "attention", ("q_many_tiles", "one_key_block", "key_tail", "d_steps_lt4", "dv_full", "p_q_on",
                                "scale_on", "nan_q", "nan_v"), batch=8200, tq=2048, tk=16, d=16, dv=128,
      bounds=("out",), gib=12.0),
    C("gptq_simt_out", "gptq", ("simt3.mt8", "simt3.mpass", "simt3.k_tail"), bits=3, m=16390, k=32, n=131072,
      impl=0, bounds=("out",), gib=10.5),
    C("gptq_simt_x", "gptq", ("simt3.mt8", "simt3.mpass", "simt3.s_free", "simt3.n_tail"), bits=3, m=32800, k=65536,
      n=64, impl=0, bounds=("x",), gib=10.5),
    C("gptq_tc_out", "gptq", ("dispatch.impl2.tc", "tc.f32", "tc.m_tail"), bits=4, m=8390000, k=256, n=256, impl=2,
      bounds=("x", "out", "a_hi"), gib=26.5),
    C("gptq_f16_out", "f16", ("f16.tc", "tc.f16_out", "tc.f16_out.bias", "tc.m_tail"), bits=4, m=524400, k=128,
      n=4096, bounds=("out",), gib=14.5),
    C("dg_simt_rows", "dgrad", ("dg.simt.m_loop", "dg.simt.one_slice", "dg.simt.mt4", "dg.simt.b3", "dg.simt.b4",
                                "dg.auto.unsupported", "dg.impl1"), runs=((3, 0), (4, 1)), m=600001, k=64, n=256,
      bounds=("grid_y",), slab=131072, gib=3.0),
    C("dg_simt_in", "dgrad", ("dg.simt.b2", "dg.simt.one_slice", "dg.simt.k_tail"), runs=((2, 0),), m=131000,
      k=16400, n=128, bounds=("grad_in",), gib=11.0),
    C("dg_simt_max_m", "dgrad", ("dg.simt.m_loop", "dg.simt.one_slice", "dg.simt.mt4", "dg.simt.b3"),
      runs=((3, 0),), m=(1 << 31) - 1, k=1, n=1, bounds=("grid_y", "m_int"), whole="exact", gib=18.5),
    C("dg_tc", "dgrad", ("dg.impl2", "dg.tc", "dg.tc.m_tail"), runs=((4, 2),), m=8390000, k=256, n=256,
      bounds=("grad_out", "g_hi", "grad_in"), gib=26.5),
]
BY_NAME = {c.name: c for c in CASES}


def _cdiv(a, b):
    return -(-a // b)


def units(case):
    """The rows the windows and slabs are cut in: batch entries for the batched cases, else rows."""
    return case.get("batch") if case.op in ("matmul", "attention") else case.get("m")


def unit_elems(case, m=None):
    """Elements per unit of every tensor the case's call touches, from the geometry modules' plans."""
    g = case.get
    if case.op in ("linear", "sparse24"):
        return dict(x=g("k"), q=igeo.rows_plan(g("m"), g("k"))["kp"], out=g("n"))
    if case.op == "matmul":
        kp_b = (igeo.rows_plan(g("n"), g("k")) if g("b_k_major") else igeo.cols_plan(1, g("k"), g("n")))["kp"]
        return dict(a=g("m") * g("k"), qa=g("m") * igeo.rows_plan(g("m"), g("k"))["kp"], b=g("k") * g("n"),
                    qb=g("n") * kp_b, out=g("m") * g("n"))
    if case.op == "attention":
        return dict(q=g("tq") * g("d"), p_q=g("tq") * aref.padded(g("tk")), out=g("tq") * g("dv"))
    if case.op in ("gptq", "f16"):
        e = dict(x=g("k"), out=g("n"))
        if case.op == "f16" or g("impl") == 2:
            e["a_hi"] = g("k")  # the split kernel's fp16 planes of x [M, K]
        return e
    e = dict(grad_out=g("n"), grad_in=g("k"))
    if any(impl == 2 for _, impl in g("runs")):
        e["g_hi"] = g("n")
    return e


def crossing(case, bound):
    """How far past its bound the case takes ``bound``: (value, limit)."""
    if bound == "grid_y":
        return ggeo.dgrad_simt_plan(case.get("m"), case.get("k"), case.get("n"))["m_tiles"], ggeo.DG_MAX_GRID_Y
    if bound == "m_int":  # M + MT - 1 in the kernel's ceil(M / MT)
        return case.get("m") + ggeo.dgrad_simt_plan(case.get("m"), case.get("k"), case.get("n"))["mt"] - 1, B31 - 1
    return units(case) * unit_elems(case)[bound], B31


def bound_units(case):
    """The unit holding element 2^31 of each tensor past the bound (for the grid case the first row tile that a CTA
    reaches on its second trip, 65535 tiles in)."""
    out = []
    for b in case.get("bounds"):
        if b == "grid_y":
            out.append(ggeo.DG_MAX_GRID_Y * ggeo.dgrad_simt_plan(case.get("m"), case.get("k"), case.get("n"))["mt"])
        elif b == "m_int":
            out.append(case.get("m") - 1)
        else:
            out.append(B31 // unit_elems(case)[b])
    return out


def _kw(case, bits=None):
    return ggeo.packed_rows(bits or case.get("bits"), case.get("k"))


def regime(case, sm, u=None):
    """The launch branches one call reaches, from the geometry mirrors; ``u``: the call on u units instead."""
    g = case.get
    u = units(case) if u is None else u
    if case.op == "linear":
        return igeo.linear_branches(u, g("k"), g("n"))
    if case.op == "sparse24":
        return sgeo.gemm_branches(u, g("k"), g("n"))
    if case.op == "matmul":
        return igeo.matmul_branches(u, g("m"), g("k"), g("n"), g("b_k_major"))
    if case.op == "attention":
        return ageo.branches(u, g("tq"), g("tk"), g("d"), g("dv"), True, 0.25, nan=("q", "v"))
    if case.op == "gptq":
        if g("impl") == 2:
            return ggeo.dispatch(u, g("k"), g("n"), GS, 2)[1] | ggeo.tc_branches(u, g("k"), g("n"), _kw(case), GS)
        return ggeo.simt_branches(g("bits"), u, g("k"), g("n"), _kw(case), sm)
    if case.op == "f16":
        return ggeo.f16_branches(u, g("k"), g("n"), _kw(case), GS, False, True, sm)
    out = set()
    for bits, impl in g("runs"):
        out |= ggeo.dgrad_branches(bits, u, g("k"), g("n"), _kw(case, bits), _dg_gs(case, bits), impl)
    return out


def kernel_ids(case, sm, u=None):
    """The ids that name which kernel runs: slabs must reach the same ones as the whole."""
    keep = ("dispatch.", "f16.tc", "dg.tc", "dg.simt.b", "dg.simt.mt", "dg.simt.one_slice", "dg.simt.slices",
            "simt3.mt", "simt3.s_", "mm.b_", "cols.vec", "rows.vec", "rows.scalar", "gemm_store", "gemm.kb", "mm.kb",
            "p_q_", "d_steps", "one_key_block", "many_key_blocks")
    return {b for b in regime(case, sm, u) if b.startswith(keep)}


def _dg_gs(case, bits):
    return 1024 if bits == 2 else GS


def slabs(case):
    """[a, b) unit ranges of at most SUB elements in every tensor (and ``slab`` units when the case sets it), cut
    evenly so that the last is not a sliver.  None for a case checked whole against its exact product."""
    if case.get("whole") == "exact":
        return []
    n = units(case)
    per = max(SUB // max(unit_elems(case).values()), 1)
    per = min(per, case.get("slab", per))
    k = _cdiv(n, per)
    cuts = [n * i // k for i in range(k + 1)]
    return list(zip(cuts[:-1], cuts[1:]))


def windows(case):
    """Unit ranges: the head, around each bound unit, and the tail; overlapping ranges merged."""
    n = units(case)
    w = max(WIN // max(unit_elems(case).values()), 3)
    wins = sorted([(0, w), (n - w, n)] + [(max(u - w // 2, 0), min(u + w - w // 2, n)) for u in bound_units(case)])
    merged = [wins[0]]
    for r0, r1 in wins[1:]:
        if r0 <= merged[-1][1]:
            merged[-1] = (merged[-1][0], max(r1, merged[-1][1]))
        else:
            merged.append((r0, r1))
    return merged


def allocations(case):
    """Bytes of every device tensor the GPU test holds while its big call runs (the slab launches and the truth
    windows come on top: at most one slab output and its workspace, held in the stated need's headroom)."""
    lib = _lib.load()
    g = case.get
    if case.op in ("linear", "sparse24"):
        m, k, n = g("m"), g("k"), g("n")
        wt = n * igeo.padded_k(k) if case.op == "linear" else n * sref.k64(k)  # w_q, or vals + meta
        return dict(x=4 * m * k, out=4 * m * n, ws=int(lib.sb200_int8_linear_workspace_bytes(m, k)), w=wt + 16 * n)
    if case.op == "matmul":
        b, m, k, n = g("batch"), g("m"), g("k"), g("n")
        return dict(a=4 * b * m * k, b=4 * b * k * n, out=4 * b * m * n,
                    ws=int(lib.sb200_int8_matmul_workspace_bytes(b, m, k, n)))
    if case.op == "attention":
        b, tq, tk, d, dv = (g(x) for x in ("batch", "tq", "tk", "d", "dv"))
        return dict(q=4 * b * tq * d, k=4 * b * tk * d, v=4 * b * tk * dv, out=4 * b * tq * dv,
                    p_q=b * tq * aref.padded(tk), ws=int(lib.sb200_int8_attention_workspace_bytes(b, tq, tk, d, dv)))
    m, k, n = g("m"), g("k"), g("n")
    w = 4 * (_kw(case, 4 if case.op == "f16" else None) if case.op != "dgrad" else
             max(_kw(case, bits) for bits, _ in g("runs"))) * n + 8 * n * _cdiv(k, GS)
    if case.op == "gptq":
        ws = int(lib.sb200_gptq4_workspace_bytes(m, k, n, GS)) if g("bits") == 4 else 0
        return dict(x=4 * m * k, out=4 * m * n, w=w, ws=ws)
    if case.op == "f16":
        return dict(x=2 * m * k, out=2 * m * n, w=w, bias=4 * n,
                    ws=int(lib.sb200_gptq4_linear_f16_workspace_bytes(m, k, n, GS)))
    ws = max(int(lib.sb200_gptq_dgrad_workspace_bytes(m, k, n, bits, _dg_gs(case, bits))) for bits, _ in g("runs"))
    return dict(grad_out=4 * m * n, grad_in=4 * m * k, w=w, ws=ws)


# -------------------------------------------------------------------------------------------------- CPU tests
def test_case_table_crosses_its_bounds_and_reaches_its_regimes():
    """Every case is past each bound it names, by the geometry modules' plans; reaches the regime it names at 132 SMs
    (H100 SXM); cuts into slabs that take the same kernel and stay below 2^28 elements; states a memory need that covers
    its tensors with at most 3 GiB of headroom for the slabs and the truth windows, within ~30 GB; and is named in the
    docstring."""
    sm = ggeo.SM_COUNT_H100
    for case in CASES:
        for b in case.get("bounds"):
            value, limit = crossing(case, b)
            assert value > limit, (case.name, b, value, limit)
        for a, b in slabs(case):
            assert b - a >= 1 and (b - a) * max(unit_elems(case).values()) <= SUB, (case.name, a, b)
            assert kernel_ids(case, sm, b - a) == kernel_ids(case, sm), (case.name, a, b)
            for bound in case.get("bounds"):
                if bound == "grid_y":
                    assert ggeo.dgrad_simt_plan(b - a, case.get("k"), case.get("n"))["m_passes"] == 1
        held = sum(allocations(case).values()) / GIB
        assert held <= case.get("gib") <= held + 3.0 and case.get("gib") <= MAX_GIB, (case.name, held)
        for r0, r1 in windows(case):
            assert 0 <= r0 < r1 <= units(case)
    assert_table_covers(CASES, set(), lambda c: check_reach(c, regime(c, sm)), __doc__, doc_branches=False)


def test_windows_hold_the_bound_rows():
    """Each bound unit lies inside a window with a unit on either side of it (the last unit excepted)."""
    for case in CASES:
        wins = windows(case)
        for u in bound_units(case):
            assert any(r0 < u < r1 - 1 or r1 == units(case) > u >= r0 for r0, r1 in wins), (case.name, u, wins)


@pytest.mark.parametrize("m", [1, 2, 3, 262140, 262141, 600001, 1 << 24, (1 << 31) - 1])
def test_dgrad_simt_grid_stays_within_cuda_limits(m):
    """The SIMT input gradient's grid (gptq_dgrad.cu launch_simt) stays within CUDA's limits (x < 2^31, y and z <=
    65535) for every M the argument check accepts; past 262,140 rows (65535 tiles of 4) its CTAs loop."""
    for k, n in ((32, 61), (64, 256), (6661, 2516), (16400, 128), ((1 << 31) - 1, 8), (11008, 4096)):
        p = ggeo.dgrad_simt_plan(m, k, n)
        gx, gy, gz = p["grid"]
        assert 1 <= gx < B31 and 1 <= gy <= 65535 and 1 <= gz <= 65535, (m, k, n, p)
        assert gy * p["m_passes"] >= p["m_tiles"] > gy * (p["m_passes"] - 1)
        assert (p["m_passes"] > 1) == (m > 4 * 65535)


def test_dgrad_split_n_path_cannot_reach_2_31_elements():
    """slices > 1 needs fewer than 1024 base CTAs (ceil(K / 32) ceil(M / mt) < 1024), so M K < 32 mt 1024 <= 2^17: the
    partial buffer and dgrad_finish_kernel never index past 2^31 and need no far-end case."""
    for m in (1, 2, 3, 4, 5, 100, 255, 1023, 1024, 4092, 4096, 5000):
        for k in (1, 31, 32, 33, 1000, 4096, 32736, 32768, 1 << 20):
            p = ggeo.dgrad_simt_plan(m, k, 1 << 20)
            if p["slices"] > 1:
                assert _cdiv(k, ggeo.DG_UNIT_K) * p["m_tiles"] < ggeo.DG_TARGET_CTAS
                assert m * k < 32 * p["mt"] * ggeo.DG_TARGET_CTAS <= 1 << 17, (m, k)
    assert ggeo.dgrad_simt_plan(4092, 32, 1 << 20)["slices"] > 1  # the path exists


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
        for live in (ops._int8_ws, ops._gptq_ws):
            for key in [k for k in live if k[1] == side.cuda_stream]:
                live.pop(key)
        gc.collect()
        torch.cuda.empty_cache()


def _gen(case, *extra):
    return torch.Generator(device=dev()).manual_seed(seed_of(case.name, *extra))


def _sentinel(shape, dtype=torch.float32):
    out = torch.empty(shape, dtype=dtype, device=dev())
    if dtype == torch.float16:
        out.view(torch.int16).fill_(SENTINEL16)
    else:
        out.view(torch.int32).fill_(SENTINEL)
    return out


def _no_sentinel(out):
    iv = out.reshape(-1).view(torch.int16 if out.dtype == torch.float16 else torch.int32)
    s = SENTINEL16 if out.dtype == torch.float16 else SENTINEL
    left = sum(int((iv[a:a + SUB] == s).sum()) for a in range(0, iv.numel(), SUB))
    assert left == 0, f"{left} outputs keep the sentinel"


def _bits_eq(a, b):
    it = torch.int16 if a.dtype == torch.float16 else torch.int32
    return torch.equal(a.reshape(-1).view(it), b.reshape(-1).view(it))


def _plant(t2, wins, make, fixed=None):
    """Edit the window units of t2 [units, elems] on the host (``make(w)`` on each window's copy [rows, elems]) and the
    flat positions ``fixed``; write them back and return the host copies."""
    host = []
    e = t2.shape[1]
    for r0, r1 in wins:
        w = t2[r0:r1].cpu().numpy()
        make(w)
        for p, v in (fixed or {}).items():
            if r0 * e <= p < r1 * e:
                w.reshape(-1)[p - r0 * e] = v
        t2[r0:r1].copy_(torch.from_numpy(w))
        host.append(w)
    return host


def _specials(nan=True):
    """+inf in a window's first row, -inf in the middle one and, with ``nan``, a NaN in the last."""
    def make(w):
        w[0, 0], w[len(w) // 2, -1] = np.inf, -np.inf
        if nan:
            w[-1, w.shape[1] // 2] = np.nan
    return make


def _within(y, t, bound, what):
    y = np.asarray(y, F64)
    assert np.array_equal(np.isnan(y), np.isnan(t)), f"{what}: NaN positions differ from the fp64 truth"
    ok = ~np.isnan(t)
    err = np.abs(y[ok] - t[ok])
    assert np.all(err <= bound[ok]), f"{what}: error {err.max():.3g} over the 2^-21 bound"


def _same_slabs(case, big, run, tol=None, fac=None):
    """``run(a, b)`` returns the entry point's output for units [a, b); it must equal big[a:b] bit for bit, or with
    ``tol``: |got - big| <= tol (f + |big|) on a row scaled by the factor f (``fac``, else 1)."""
    for a, b in slabs(case):
        got = run(a, b)
        ref = big[a:b].reshape(got.shape)
        if tol is None:
            assert _bits_eq(got, ref), f"{case.name}: units [{a}, {b}) differ from a launch on them alone"
        else:
            f = torch.tensor([(fac or {}).get(r, 1.0) for r in range(a, b)], device=dev())[:, None]
            step = max(SUB // 8 // got.shape[1], 1)
            bad = sum(int(((got[i:i + step] - ref[i:i + step]).abs() > tol * (f[i:i + step] + ref[i:i + step].abs()))
                          .sum()) for i in range(0, b - a, step))
            assert bad == 0, f"{case.name}: {bad} outputs of units [{a}, {b}) off a launch on them alone"
        del got


def _scalar(v):
    return torch.tensor([v], dtype=torch.float32, device=dev())


# -------------------------------------------------------------------------------------------------- GPU: integer grid
X_Q = (F32(0.04), F32(131.0), 0, 255)    # activations: unsigned 8-bit, zero point 131
B_Q = (F32(0.03), F32(0.0), -128, 127)   # the second matmul operand: signed


def _lin_weights(rng, n, k, sparse):
    ws = (2.0 ** -rng.integers(3, 8, n)).astype(F32)
    w = (rng.uniform(-0.45, 0.45, (n, k)) * 255 * ws[:, None]).astype(F32)
    if sparse:
        w = np.where(sref.mask24(rng.standard_normal((n, k)).astype(F32)), w, F32(0))
    return w, ws, np.zeros(n, F32)


def _linear(case):
    m, k, n, sparse = case.get("m"), case.get("k"), case.get("n"), case.op == "sparse24"
    rng = np.random.default_rng(seed_of(case.name))
    lib = _lib.load()
    x = torch.empty(m, k, device=dev()).normal_(generator=_gen(case)).mul_(3).add_(0.5)
    wins = windows(case)
    host = _plant(x, wins, _specials(), {B31 + 1: np.nan, B31 + 5: -np.inf, m * k - 1: np.inf} if m * k > B31 else {})
    w, ws, wz = _lin_weights(rng, n, k, sparse)
    bias = rng.standard_normal(n).astype(F32)
    xs, xz = _scalar(X_Q[0]), _scalar(X_Q[1])
    ws_d, wz_d, b_d = (torch.from_numpy(a).to(dev()) for a in (ws, np.zeros(n, np.int32), bias))
    w_q, w_sum, w_nan = ops.int8_quantize_rows(torch.from_numpy(w).to(dev()), ws_d, torch.from_numpy(wz).to(dev()),
                                               -128, 127)
    assert not w_nan.any()
    if sparse:
        vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, wz_d, ws_d, k)
        assert not bad.any()
        del w_q, w_sum
    out = _sentinel((m, n))
    nb = int(lib.sb200_int8_linear_workspace_bytes(m, k))
    wsp = torch.empty(nb, dtype=torch.uint8, device=dev())
    head = (x.data_ptr(), xs.data_ptr(), xz.data_ptr(), X_Q[2], X_Q[3])
    tail = (b_d.data_ptr(), out.data_ptr(), m, k, n, wsp.data_ptr(), nb, stream())
    if sparse:
        rc = lib.sb200_int8_sparse24_linear(*head, vals.data_ptr(), meta.data_ptr(), dsum.data_ptr(), ws_d.data_ptr(),
                                            *tail)
    else:
        rc = lib.sb200_int8_linear(*head, w_q.data_ptr(), w_sum.data_ptr(), ws_d.data_ptr(), wz_d.data_ptr(), *tail)
    assert rc == 0, lib.sb200_last_error()
    del wsp
    _no_sentinel(out)
    for (r0, r1), xh in zip(wins, host):
        t, bound = lref.truth(xh, X_Q[0], X_Q[1], X_Q[2], X_Q[3], w, ws, wz, -128, 127, bias)
        _within(out[r0:r1].cpu().numpy(), t, bound, f"{case.name} rows [{r0}, {r1})")
    assert np.isnan(out[wins[0][1] - 1].cpu().numpy()).all()  # a NaN in x makes its row NaN

    def run(a, b):
        if sparse:
            return ops.int8_sparse24_linear(x[a:b], xs, xz, X_Q[2], X_Q[3], vals, meta, dsum, ws_d, b_d)
        return ops.int8_linear(x[a:b], xs, xz, X_Q[2], X_Q[3], w_q, w_sum, ws_d, wz_d, b_d)
    _same_slabs(case, out, run)


def _matmul(case):
    bt, m, k, n, kmaj = (case.get(x) for x in ("batch", "m", "k", "n", "b_k_major"))
    lib = _lib.load()
    gen = _gen(case)
    a = torch.empty(bt, m, k, device=dev()).normal_(generator=gen).mul_(3).add_(0.5)
    b_store = torch.empty((bt, n, k) if kmaj else (bt, k, n), device=dev()).normal_(generator=gen).mul_(2)
    wins = windows(case)
    a2, b2 = a.view(bt, m * k), b_store.view(bt, -1)
    ha = _plant(a2, wins, _specials(), {B31 + 1: np.nan, B31 + 5: -np.inf} if bt * m * k > B31 else {})
    hb = _plant(b2, wins, _specials(nan=False), {B31 + 1: np.nan, B31 + 5: -np.inf} if bt * k * n > B31 else {})
    if B31 + 1 >= bt * k * n:  # a NaN column in the last entry of b all the same
        b2[-1, (k // 2) * n + n // 3 if not kmaj else (n // 3) * k + k // 2] = np.nan
        hb[-1][-1, (k // 2) * n + n // 3 if not kmaj else (n // 3) * k + k // 2] = np.nan
    pa = (_scalar(X_Q[0]), _scalar(X_Q[1]), X_Q[2:])
    pb = (_scalar(B_Q[0]), _scalar(B_Q[1]), B_Q[2:])
    out = _sentinel((bt, m, n))
    nb = int(lib.sb200_int8_matmul_workspace_bytes(bt, m, k, n))
    wsp = torch.empty(nb, dtype=torch.uint8, device=dev())
    rc = lib.sb200_int8_matmul(a.data_ptr(), b_store.data_ptr(), int(kmaj), pa[0].data_ptr(), pa[1].data_ptr(), *X_Q[2:],
                               pb[0].data_ptr(), pb[1].data_ptr(), *B_Q[2:], out.data_ptr(), bt, m, k, n, wsp.data_ptr(),
                               nb, stream())
    assert rc == 0, lib.sb200_last_error()
    del wsp
    _no_sentinel(out)
    nan_seen = False
    for (r0, r1), xa, xb in zip(wins, ha, hb):
        xb = xb.reshape(r1 - r0, n, k).transpose(0, 2, 1) if kmaj else xb.reshape(r1 - r0, k, n)
        t, bound = mref.truth((xa.reshape(r1 - r0, m, k), *X_Q), (xb, *B_Q))
        y = out[r0:r1].cpu().numpy()
        _within(y, t, bound, f"{case.name} entries [{r0}, {r1})")
        nan_seen |= bool(np.isnan(y).any())
    assert nan_seen

    def bview(x):
        return x.transpose(-2, -1) if kmaj else x
    _same_slabs(case, out, lambda s, e: ops.int8_matmul(a[s:e], pa[0], pa[1], pa[2], bview(b_store[s:e]), pb[0], pb[1],
                                                        pb[2]))


A_Q = (F32(4 / 127), F32(0), -128, 127)   # q and k of the attention
V_Q = (F32(8 / 255), F32(7), 0, 255)
P_Q = (F32(1 / 255), F32(0), 0, 255)
SCALE = 0.25


def _attention(case):
    bt, tq, tk, d, dv = (case.get(x) for x in ("batch", "tq", "tk", "d", "dv"))
    lib = _lib.load()
    gen = _gen(case)
    q = torch.empty(bt, tq, d, device=dev()).normal_(generator=gen)
    k = torch.empty(bt, tk, d, device=dev()).normal_(generator=gen)
    v = torch.empty(bt, tk, dv, device=dev()).normal_(generator=gen)
    wins = windows(case)
    hq = _plant(q.view(bt, -1), wins, _specials())
    hk = _plant(k.view(bt, -1), wins, _specials(nan=False))
    hv = _plant(v.view(bt, -1), wins, lambda w: w.__setitem__((-1, 3 * dv + 5), np.nan))  # a NaN column of out
    qp = [(_scalar(o[0]), _scalar(o[1]), o[2:]) for o in (A_Q, A_Q)] + [(_scalar(P_Q[0]), _scalar(P_Q[1]), P_Q[2:])] + \
         [(_scalar(V_Q[0]), _scalar(V_Q[1]), V_Q[2:])]
    out = _sentinel((bt, tq, dv))
    tkp = aref.padded(tk)
    pq = torch.full((bt, tq, tkp), 0x5A, dtype=torch.int8, device=dev())
    nb = int(lib.sb200_int8_attention_workspace_bytes(bt, tq, tk, d, dv))
    wsp = torch.empty(nb, dtype=torch.uint8, device=dev())
    args = [q.data_ptr(), k.data_ptr(), v.data_ptr()]
    for s, z, (lo, hi) in qp:
        args += [s.data_ptr(), z.data_ptr(), lo, hi]
    rc = lib.sb200_int8_attention(*args, 1, SCALE, out.data_ptr(), pq.data_ptr(), bt, tq, tk, d, dv, wsp.data_ptr(), nb,
                                  stream())
    assert rc == 0, lib.sb200_last_error()
    del wsp
    _no_sentinel(out)
    for (r0, r1), xq, xk, xv in zip(wins, hq, hk, hv):
        nw = r1 - r0
        oq, ok_, ov = (xq.reshape(nw, tq, d), *A_Q), (xk.reshape(nw, tk, d), *A_Q), (xv.reshape(nw, tk, dv), *V_Q)
        g = pq[r0:r1].cpu().numpy()
        assert not g[..., tk:].any()
        y = out[r0:r1].cpu().numpy()
        assert np.array_equal(y, aref.expected(g, oq, ok_, ov, P_Q, SCALE), equal_nan=True), (case.name, r0, r1)
        s, bad = aref.scores(oq, ok_, SCALE)
        lo, hi = aref.admissible_range(aref.softmax64(s), P_Q)
        gg = g[..., :tk].astype(np.int64)
        assert np.all(((gg >= lo) & (gg <= hi))[~bad]), (case.name, r0, r1)
        assert bad.any() and np.isnan(y).any() and not np.isnan(y).all()

    def run(a, b):
        y, p = ops.int8_attention(q[a:b], k[a:b], v[a:b], *qp, scale=SCALE, return_p=True)
        assert torch.equal(p, pq[a:b]), f"{case.name}: p of entries [{a}, {b}) differs"
        return y
    _same_slabs(case, out, run)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params([c for c in CASES if c.op in ("linear", "sparse24", "matmul", "attention")]))
@_frees_device_memory
def test_integer_grid_far_end(case):
    with _far_end(case):
        {"linear": _linear, "sparse24": _linear, "matmul": _matmul, "attention": _attention}[case.op](case)


# -------------------------------------------------------------------------------------------------- GPU: GPTQ
def _gptq_weights(rng, bits, k, n, gs, red):
    """Random packed words (every bit pattern is a valid packing), integer zero points near the middle of the grid and
    scales that put |W| near 1 / sqrt(red), as a layer's weights are scaled for its reduction length ``red`` (the
    existing suites quantize randn / sqrt(K)), so that outputs are O(1) and 1e-5 elementwise is a relative bar; W [K, N] =
    s q - z in fp64 on the device."""
    kw = ggeo.packed_rows(bits, k)
    qw = rng.integers(0, 1 << 32, (kw, n), dtype=np.uint64).astype(np.uint32).view(np.int32)
    g = _cdiv(k, gs)
    scales = (rng.uniform(0.5, 1.5, (n, g)) * 2.0 ** (1 - bits) / np.sqrt(red)).astype(F32)
    zeros = (scales * rng.integers(2 ** (bits - 1) - 1, 2 ** (bits - 1) + 2, (n, g))).astype(F32)
    w = torch.from_numpy(dequant_weight(qw, scales, zeros, k, gs, bits)).to(dev())
    return [torch.from_numpy(a).to(dev()) for a in (qw, scales, zeros)], w


def _row_factors(wins, tiny, huge):
    """Each window's first row scaled by ``tiny``, its last by ``huge``."""
    fac = {}
    for r0, r1 in wins:
        fac[r0], fac[r1 - 1] = tiny, huge
    return fac


def _pattern(rows, r0, cols, seed, fac, out=None):
    """((r 7 + c 3 + seed) % 17 - 8) / 16 for rows r0 .. r0 + rows, rows in ``fac`` times their factor: a few bits
    each, so that subtracting the pattern in fp64 is exact, and no larger than the O(1) outputs (the fp32 additions into
    out round at the scale of the running value).  Filled in chunks, into ``out`` if given."""
    out = torch.empty(rows, cols, device=dev()) if out is None else out
    c3 = torch.arange(cols, device=dev(), dtype=torch.int32) % 17 * 3
    step = max((1 << 26) // cols, 1)
    for a in range(0, rows, step):
        b = min(a + step, rows)
        r7 = (torch.arange(r0 + a, r0 + b, device=dev(), dtype=torch.int64) % 17 * 7 + seed % 17).to(torch.int32)
        out[a:b] = (r7[:, None] + c3[None, :]).remainder_(17).sub_(8)
        out[a:b] *= 1 / 16
    for r, f in fac.items():
        if r0 <= r < r0 + rows:
            out[r - r0] *= f
    return out


def _normalised_close(got, exp, f, what):
    """got / exp [rows, cols] fp64 with row factors f: rtol = atol = 1e-5 after dividing each row by its factor."""
    fr = torch.tensor(f, dtype=torch.float64)[:, None]
    torch.testing.assert_close(got / fr, exp / fr, rtol=1e-5, atol=1e-5, msg=lambda m: f"{what}: {m}")


def _gptq_forward(case):
    bits, m, k, n, impl = (case.get(x) for x in ("bits", "m", "k", "n", "impl"))
    f16 = case.op == "f16"
    rng = np.random.default_rng(seed_of(case.name))
    seed = seed_of(case.name, "pattern")
    lib = _lib.load()
    (qw, sc, zr), w = _gptq_weights(rng, bits, k, n, GS, k)
    wins = windows(case)
    tiny, huge = (TINY16, HUGE16) if f16 else (TINY, HUGE)
    fac = _row_factors(wins, tiny, huge)
    x = torch.empty(m, k, device=dev()).normal_(generator=_gen(case))
    if f16:
        x = x.half()
    for r, f in fac.items():
        x[r] *= f
    if f16:
        bias = torch.from_numpy(rng.standard_normal(n).astype(F32)).to(dev())
        out = _sentinel((m, n), torch.float16)
        nb = int(lib.sb200_gptq4_linear_f16_workspace_bytes(m, k, n, GS))
        wsp = torch.empty(nb, dtype=torch.uint8, device=dev())
        rc = lib.sb200_gptq4_linear_f16_ex(x.data_ptr(), qw.data_ptr(), out.data_ptr(), bias.data_ptr(), sc.data_ptr(),
                                           zr.data_ptr(), m, k, n, qw.shape[0], GS, None, 0, wsp.data_ptr(), nb, stream())
        assert rc == 0, lib.sb200_last_error()
        del wsp
        _no_sentinel(out)
    else:
        out = _pattern(m, 0, n, seed, fac)

    def call(xs, o):
        if bits == 4:
            return ops.gptq4_matmul(xs, qw, o, sc, zr, GS, impl=impl)
        return ops.gptq_matmul(xs, qw, o, sc, zr, bits, GS)
    if not f16:
        call(x, out)
    torch.cuda.synchronize()
    for r0, r1 in wins:
        f = [fac.get(r, 1.0) for r in range(r0, r1)]
        exp = (x[r0:r1].double() @ w).cpu()
        if f16:
            e = (exp + bias.double().cpu()).numpy()
            y = out[r0:r1].double().cpu().numpy()
            ulp = np.exp2(np.floor(np.log2(np.maximum(np.abs(e), 2.0 ** -14))) - 10)
            assert np.all(np.abs(y - e) <= 0.51 * ulp + 1e-5), f"{case.name} rows [{r0}, {r1})"
        else:
            got = out[r0:r1].double().cpu() - _pattern(r1 - r0, r0, n, seed, fac).double().cpu()
            _normalised_close(got, exp, f, f"{case.name} rows [{r0}, {r1})")

    def run(a, b):
        if f16:
            return ops.gptq4_linear_f16(x[a:b], qw, sc, zr, bias, GS)
        return call(x[a:b], _pattern(b - a, a, n, seed, fac))
    # the SIMT kernel's K slices add into out in whatever order the atomics land: two launches, each within rtol = atol =
    # 1e-5 of the truth, may differ by twice that
    _same_slabs(case, out, run, tol=2e-5 if case.get("bits") != 4 else None, fac=fac)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params([c for c in CASES if c.op in ("gptq", "f16")]))
@_frees_device_memory
def test_gptq_forward_far_end(case):
    with _far_end(case):
        _gptq_forward(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params([c for c in CASES if c.op == "dgrad"]))
@_frees_device_memory
def test_gptq_dgrad_far_end(case):
    """Both kernels are deterministic: the whole grad_in equals the slab launches' bit for bit."""
    m, k, n = case.get("m"), case.get("k"), case.get("n")
    with _far_end(case):
        wins = windows(case)
        fac = _row_factors(wins, TINY, HUGE)
        go = torch.empty(m, n, device=dev()).normal_(generator=_gen(case))
        for r, f in fac.items():
            go[r] *= f
        for bits, impl in case.get("runs"):
            rng = np.random.default_rng(seed_of(case.name, bits))
            seed = seed_of(case.name, bits, "pattern")
            gs = _dg_gs(case, bits)
            (qw, sc, zr), w = _gptq_weights(rng, bits, k, n, gs, n)
            gi = _pattern(m, 0, k, seed, fac)
            ops.gptq_matmul_dgrad(go, qw, gi, sc, zr, bits, gs, impl=impl)
            torch.cuda.synchronize()
            for r0, r1 in wins:
                got = gi[r0:r1].double().cpu() - _pattern(r1 - r0, r0, k, seed, fac).double().cpu()
                exp = (go[r0:r1].double() @ w.T).cpu()
                _normalised_close(got, exp, [fac.get(r, 1.0) for r in range(r0, r1)],
                                  f"{case.name} {bits}-bit rows [{r0}, {r1})")
            if case.get("whole") == "exact":
                _exact_product(case, go, gi, w, sc, zr, seed, fac)
            else:
                _same_slabs(case, gi, lambda a, b: ops.gptq_matmul_dgrad(go[a:b], qw, _pattern(b - a, a, k, seed, fac),
                                                                         sc, zr, bits, gs, impl=impl))
            del gi, qw, sc, zr, w
            gc.collect()


def _exact_product(case, go, gi, w, sc, zr, seed, fac):
    """K = N = 1: the SIMT kernel forms (g s) q and g z with one rounding each, subtracts them, and its reductions add
    only zeros to that, so grad_in = prefill + ((g s) q - g z) in fp32, element for element (values compared, so the
    sign of a zero result is not)."""
    s, z = sc.reshape(()), zr.reshape(())
    q = round((w.reshape(()).item() + float(z)) / float(s))  # the integer weight, from W = s q - z
    step = 1 << 26
    m = case.get("m")
    for a in range(0, m, step):
        b = min(a + step, m)
        g = go[a:b, 0]
        exp = _pattern(b - a, a, 1, seed, fac)[:, 0].add_((g * s).mul_(q).sub_(g * z))
        bad = int((gi[a:b, 0] != exp).sum())
        assert bad == 0, f"{case.name}: {bad} of rows [{a}, {b}) differ from prefill + (g s) q - g z"
