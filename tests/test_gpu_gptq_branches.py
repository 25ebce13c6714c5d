"""Every launch branch of the GPTQ kernels: the dispatch and entry points (csrc/gptq.cu), the SIMT dequant-matmul
(csrc/gptq_simt.cu), the decode kernel (csrc/gptq_decode.cu), the wgmma prefill kernel (csrc/gptq_tc.cu) and the input
gradient (csrc/gptq_dgrad.cu), each reached by a named case and compared with the fp64 truth.

tests/gptq_geometry.py restates the host launch decisions; every case below asserts, with the SM count of the device it
runs on, that it reaches the branches it is listed for, and the CPU test at the bottom checks at 132 SMs (H100 SXM) that
the cases together reach every branch in REQUIRED.  Ids marked (data) depend on the values, not the launch: the case
claims them, its data plants them and the GPU test checks the data really has the property.

Bar: rtol = atol = 1e-5 elementwise against the fp64 truth (the dequantised weights times the operand in float64 on the
device), rows with planted outliers bounded by the row magnitude, fp16 outputs by 0.51 fp16 ulp + 1e-5.  Every output
starts as a finite sentinel: the bias (fp32 forward) or a random prefill (input gradient) for the accumulate contract,
a bit pattern for fp16 outputs and the workspace (where the single-launch fp16 path keeps its partial slots), so an
element a kernel skips fails.  Packed values past K are random, not zero: they meet zero activations only.

  branch                          source                 case (why it gets there)
  dispatch.auto.tc                gptq.cu:96             tc_tail_wrap: M = 300
  dispatch.auto.decode            gptq.cu:100            dec_slab_alias: M = 12
  dispatch.auto.simt              gptq.cu:102            refuse_n4: N = 250 (no decode either)
  dispatch.auto.ws_null           gptq.cu:89-90          ws_null: M = 64 without a workspace -> decode
  dispatch.auto.ws_small          gptq.cu:90             ws_small: one byte short -> decode
  dispatch.refuse.k8              gptq_tc.cu:289         refuse_k8: K = 1004
  dispatch.refuse.n4              gptq_tc.cu:289         refuse_n4: N = 250
  dispatch.refuse.group128        gptq_tc.cu:290         refuse_group128: one group of K = 1000
  dispatch.refuse.x_misaligned    gptq_tc.cu:291         refuse_x_misaligned: x at float offset 1
  dispatch.refuse.qw_misaligned   gptq_tc.cu:291         refuse_qw_misaligned: qweight at word offset 1 -> SIMT
  dispatch.impl1.decode           gptq.cu:100            dec_mpass_slab (forced, M = 70)
  dispatch.impl1.simt_fallback    gptq.cu:100-102        impl1_simt_fallback: N = 250
  dispatch.impl2.tc               gptq.cu:96             tc_odd_wrap2_frac (process-wide impl 2)
  dispatch.impl2.error            gptq.cu:91-95          impl2_error: K = 1004, nothing launched, out untouched
  dispatch.impl4.simt             gptq.cu:102            simt4_* (impl 4)
  dispatch.via.global             gptq.cu:105-112        cases run through sb200_gptq4_matmul + sb200_gptq4_set_impl
  dispatch.via.ex                 gptq.cu:114-128        cases run through sb200_gptq4_matmul_ex while the process-wide
                                                         impl is set to something else (the per-call option wins)
  dispatch.bits2, dispatch.bits3  gptq.cu:218            simt2_*, simt3_* (sb200_gptq_matmul)

SIMT (launch_simt), for b = 2, 3, 4:
  simt<b>.mt1, simt<b>.s_cap      gptq_simt.cu:205-206   simt<b>_cap: M = 1, 11008 x 16384 (S above 1024 / kBlockK)
  simt<b>.short_slice, simt<b>.nb_even   gptq_simt.cu:60, 178   simt<b>_cap; simt<b>_mt4
  simt<b>.mt2, simt<b>.s_free, simt<b>.k_tail, simt<b>.n_tail, simt<b>.rows_past_k, simt<b>.nb_odd
                                  gptq_simt.cu:57-88     simt<b>_mt2: M = 2, K = 1000, N = 300, 3 extra packed rows
  simt<b>.mt4                     gptq_simt.cu:215       simt<b>_mt4: M = 3, 4096 x 11008
  simt<b>.mt8, simt<b>.mpass      gptq_simt.cu:74, 216   simt<b>_mt8_mpass: M = 19
  simt3.straddle                  gptq_unpack.cuh        every 3-bit case (values 10 and 21 of a unit span two words)

Decode (dec_run):
  dec.nbk1, dec.reg, dec.prefetch, dec.wait.strict   gptq_decode.cu:452-455   dec_nbk1_default: M = 1, 4096 x 11008
  dec.nbk2, dec.slab, dec.slab.trow_alias, dec.slab.zero_fill, dec.slab.n_tail, dec.nb1, dec.wait.static
                                  gptq_decode.cu:149-165, 287   dec_slab_alias: M = 12, K = 1000, N = 260, mode 11
  dec.nbk4, dec.mpass, dec.no_pdl gptq_decode.cu:208     dec_mpass_slab: forced impl 1, M = 70, mode 1
  dec.smax, dec.short_slice       gptq_decode.cu:463-465 dec_smax: M = 20, 10880 x 4096 (S 5 > 2, 85 blocks)
  dec.per_sm                      gptq_decode.cu:456     dec_per_sm: mode 0x82
  dec.need_lo, dec.no_lo (data)   gptq_decode.cu:273-276 dec_nbk1_default (fp32); dec_per_sm (fp16-exact activations)
  dec.batch, dec.batch.diff_n, dec.batch.short_k     gptq_decode.cu:104, 116   batch_3: N 512 / 132 / 256, one K 512
  dec.batch (4 problems)          gptq_decode.cu:104     batch_4: M = 32
  dec.f16, dec.f16.unroll4        gptq_decode.cu:379-407 f16_single: M = 1, 4096 x 4096 (16 slices)
  dec.f16.rem                     gptq_decode.cu:401     f16_single_rem_nobias: 9 slices
  dec.f16.counter_reset (data)    gptq_decode.cu:405     f16_single, f16_single_rem_nobias: three calls on one state

wgmma prefill (gptq4_tc):
  tc.f32, tc.k64_tail, tc.ring_wrap, tc.ring_wrap2, tc.m_tail, tc.n_tail, tc.live_a_only, tc.kw_extra
                                  gptq_tc.cu:153-252     tc_tail_wrap: M = 300, K = 1000, N = 264, 3 extra rows
  tc.odd_kb, tc.gq_ne_g           gptq_tc.cu:187, 219    tc_odd_wrap2_frac: K = 704 (11 stages), group 384
  tc.int_zero, tc.two_pass (data) gptq_tc.cu:154-155     tc_tail_wrap
  tc.general.fractional, tc.one_pass (data)   gptq_tc.cu:131   tc_odd_wrap2_frac (fp16-exact activations)
  tc.general.big_zero (data)      gptq_tc.cu:131         tc_big_zero: some |zero| = 1100
  tc.general.scale0 (data)        gptq_tc.cu:131         tc_scale0: one scale 0
  tc.f16_out, tc.f16_out.bias     gptq_tc.cu:232-240     f16_tc: M = 800, N = 260
  tc.f16_out.nobias               gptq_tc.cu:233         f16_tc_nobias: M = 768

fp16 linear (sb200_gptq4_linear_f16_ex):
  f16.tc                          gptq.cu:182            f16_tc, f16_tc_nobias
  f16.single                      gptq.cu:184            f16_single, f16_single_rem_nobias
  f16.staged.no_state             gptq.cu:191-207        f16_staged_no_state: M = 5
  f16.staged.mid                  gptq.cu:191-207        f16_staged_mid: M = 300 (fp32 wgmma inside)
  f16.staged.unsupported          gptq.cu:182, 191       f16_staged_unsupported: M = 800, K = 1004
  f16.null_bias                   gptq.cu:20, 244, 395   f16_tc_nobias, f16_single_rem_nobias

Input gradient (sb200_gptq_matmul_dgrad):
  dg.auto.small_m, dg.simt.slices, dg.simt.k_tail, dg.simt.mt4, dg.simt.m_tiles, dg.simt.b4
                                  gptq.cu:250, gptq_dgrad.cu:135-175   dg_small_m: M = 40, K = 1000, N = 2512
  dg.auto.tc, dg.tc, dg.tc.kw_tail, dg.tc.n_tail, dg.tc.one_group_k128, dg.tc.m_tail, dg.tc.k_tail
                                  gptq_dgrad.cu:183-204  dg_tc_tails: M = 300, K = 516 (one group), N = 264
  dg.auto.unsupported, dg.simt.b3 gptq.cu:243            dg_auto_3bit: 3-bit
  dg.impl1, dg.simt.mt1, dg.simt.one_slice, dg.simt.b2   gptq.cu:253   dg_impl1_mt1: 2-bit, M = 1, N = 61
  dg.simt.mt2                     gptq_dgrad.cu:137      dg_impl1_mt2: M = 2, N = 2516 (5 slices)
  dg.impl2, dg.tc.chunk_restart, dg.tc.ring_wrap, dg.tc.ring_wrap2
                                  gptq_dgrad.cu:287-327  dg_chunk_restart: N = 1032 (17 stages)
  dg.tc.chunk_exact               gptq_dgrad.cu:288      dg_chunk_exact: N = 1024 (16 stages)
  dg.impl2.error                  gptq.cu:245-249        dg_impl2_error: K = 126
  dg.tc.c_clamp (data)            gptq_dgrad.cu:228      dg_c_clamp: group 0 scales ~1e-28 (c = 104 -> 100)
  dg.tc.need_lo, dg.tc.no_lo (data)   gptq_dgrad.cu:259  dg_tc_tails (fp32); dg_chunk_exact (fp16-exact gradients)

Split-kernel data edges (gptq_split_kernel, gptq_tc.cu:37-90), in tiny_fwd_tc, tiny_dgrad_tc and tiny_fwd_decode:
  split.zero_row, split.nonfinite_row, split.tiny_row, split.subnormal_row   (data)
Rows r * 2^-j with max |r| in [1, 2): for j <= 112 the wgmma forward and input gradient and the one-slice decode launch
give exactly y * 2^-j, bit for bit wherever that is a normal number; below (max |x| < 2^-112, subnormal rows) the result
is finite and within 1e-5 sum |x||w| of the fp64 truth, plus 2^-149 for the rounding of a subnormal result stored
plainly.  The decode and SIMT kernels add their K slices into `out` with fp32 atomicAdd, which on sm_90a
(RED.E.ADD.F32.FTZ.RN) flushes a subnormal result to zero: their slack is 2^-126 per atomic addition instead
(test_decode_tiny_rows_lose_only_flushed_subnormals shows that the flush is all the decode kernel loses there).
tiny_fwd_simt runs the same rows through the SIMT kernel, whose staging of x * 16^-(k % 4) underflows below 2^-114 and
adds 15 * 16^3 * 2^-150 per K term; it is exact to y * 2^-j for j <= 100.  A zero row gives exactly the prefill; a row
holding +inf or NaN gives non-finite outputs only in that row.

Each deterministic path runs twice and must repeat bit for bit: the input gradient (both kernels), the wgmma forward and
the single-launch fp16 path.
"""
import ctypes
import re

import numpy as np
import pytest
import torch

import gptq_geometry as geo
from branch_cases import C, assert_table_covers, check_reach, params
from gpu_util import dev, on_device, real_sm, seed, stream
from oracle import gptq as ogptq
from sparsebit_b200 import _lib, ops

F16, F32, F64, U32 = np.float16, np.float32, np.float64, np.uint32
E_UNSUPPORTED = -3
WS_FILL = 0x7B  # workspace / fp16 out sentinel byte: 0x7B7B7B7B = 1.3e36 as fp32, 0x7B7B = 60768 as fp16, both finite
DEFAULT_MODE = geo.DEC_DEFAULT_MODE


# -------------------------------------------------------------------------------------------------- cases
# op: fwd | batch | f16 | dgrad
def _kw(case):
    return geo.packed_rows(case.get("bits", 4), case.get("k")) + case.get("kw_extra", 0)


def _gs(case):
    return case.get("gs") or case.get("k")


def branches(case, sm):
    s = case.spec
    if case.op == "fwd":
        bits, m, k, n = s.get("bits", 4), s["m"], s["k"], s["n"]
        if bits != 4:
            return {f"dispatch.bits{bits}"} | geo.simt_branches(bits, m, k, n, _kw(case), sm)
        kernel, b = geo.dispatch(m, k, n, _gs(case), s["impl"], s.get("x_off", 0), s.get("qw_off", 0), s.get("ws", "ok"))
        b.add("dispatch.via." + s.get("via", "global"))
        if kernel == "tc":
            b |= geo.tc_branches(m, k, n, _kw(case), _gs(case))
        elif kernel == "decode":
            b |= geo.dec_branches([(k, n, _kw(case))], m, s.get("mode", DEFAULT_MODE), sm)
        elif kernel == "simt":
            b |= geo.simt_branches(4, m, k, n, _kw(case), sm)
        return b
    if case.op == "batch":
        probs = [(k, n, geo.packed_rows(4, k)) for k, n in s["problems"]]
        return geo.dec_branches(probs, s["m"], s.get("mode", DEFAULT_MODE), sm)
    if case.op == "f16":
        return geo.f16_branches(s["m"], s["k"], s["n"], _kw(case), _gs(case), s["state"], s["bias"], sm)
    return geo.dgrad_branches(s.get("bits", 4), s["m"], s["k"], s["n"], _kw(case), _gs(case), s["impl"])


SPLIT_DATA = ("split.zero_row", "split.nonfinite_row", "split.tiny_row", "split.subnormal_row")
FWD_CASES = [
    C("tc_tail_wrap", "fwd", ["dispatch.auto.tc", "dispatch.via.global", "tc.f32", "tc.k64_tail", "tc.ring_wrap",
                              "tc.ring_wrap2", "tc.m_tail", "tc.n_tail", "tc.live_a_only", "tc.kw_extra"],
      ["tc.int_zero", "tc.two_pass"], m=300, k=1000, n=264, gs=128, impl=0, kw_extra=3, data="outliers"),
    C("tc_odd_wrap2_frac", "fwd", ["dispatch.impl2.tc", "tc.odd_kb", "tc.gq_ne_g", "tc.ring_wrap2"],
      ["tc.general.fractional", "tc.one_pass"], m=128, k=704, n=512, gs=384, impl=2, zeros="frac", data="f16x"),
    C("tc_big_zero", "fwd", ["dispatch.auto.tc", "dispatch.via.ex"], ["tc.general.big_zero"],
      m=40, k=384, n=132, gs=128, impl=0, via="ex", zeros="big"),
    C("tc_scale0", "fwd", ["dispatch.auto.tc"], ["tc.general.scale0"], m=33, k=256, n=128, gs=128, impl=0, zeros="scale0"),
    C("refuse_k8", "fwd", ["dispatch.refuse.k8", "dispatch.auto.decode", "dec.nbk4", "dec.mpass"],
      m=40, k=1004, n=256, gs=0, impl=0),
    C("refuse_n4", "fwd", ["dispatch.refuse.n4", "dispatch.auto.simt", "simt4.mt8", "simt4.mpass", "simt4.n_tail"],
      m=48, k=512, n=250, gs=128, impl=0),
    C("refuse_group128", "fwd", ["dispatch.refuse.group128", "dispatch.auto.decode"], m=64, k=1000, n=256, gs=0, impl=0),
    C("refuse_x_misaligned", "fwd", ["dispatch.refuse.x_misaligned", "dispatch.auto.decode"],
      m=32, k=512, n=256, gs=128, impl=0, x_off=1),
    C("refuse_qw_misaligned", "fwd", ["dispatch.refuse.qw_misaligned", "dispatch.auto.simt"],
      m=36, k=512, n=256, gs=128, impl=0, qw_off=1),
    C("ws_null", "fwd", ["dispatch.auto.ws_null", "dispatch.auto.decode"], m=64, k=512, n=256, gs=128, impl=0, ws="null"),
    C("ws_small", "fwd", ["dispatch.auto.ws_small", "dispatch.auto.decode"], m=64, k=512, n=256, gs=128, impl=0, ws="small"),
    C("impl1_simt_fallback", "fwd", ["dispatch.impl1.simt_fallback", "dispatch.via.ex"],
      m=3, k=640, n=250, gs=128, impl=1, via="ex"),
    C("impl2_error", "fwd", ["dispatch.impl2.error"], m=40, k=1004, n=256, gs=0, impl=2, via="ex"),
    # decode kernel
    C("dec_nbk1_default", "fwd", ["dec.nbk1", "dec.reg", "dec.prefetch", "dec.wait.strict", "dispatch.auto.decode"],
      ["dec.need_lo"], m=1, k=4096, n=11008, gs=128, impl=0),
    C("dec_slab_alias", "fwd", ["dec.nbk2", "dec.slab", "dec.slab.trow_alias", "dec.slab.zero_fill", "dec.slab.n_tail",
                                "dec.nb1", "dec.wait.static", "dispatch.auto.decode"],
      m=12, k=1000, n=260, gs=0, impl=0, mode=11, kw_extra=2),
    C("dec_mpass_slab", "fwd", ["dispatch.impl1.decode", "dec.nbk4", "dec.mpass", "dec.slab", "dec.no_pdl",
                                "dec.slab.zero_fill", "dec.slab.trow_alias"],
      m=70, k=328, n=64, gs=0, impl=1, via="ex", mode=1),
    C("dec_smax", "fwd", ["dec.smax", "dec.short_slice", "dec.nbk4"], m=20, k=10880, n=4096, gs=128, impl=1, mode=14),
    C("dec_per_sm", "fwd", ["dec.per_sm", "dec.nbk2"], ["dec.no_lo"], m=9, k=2048, n=1028, gs=256, impl=1, mode=0x82,
      data="f16x", zeros="frac"),
]
for _b in (4, 3, 2):
    _simt = dict(bits=_b, impl=4) if _b == 4 else dict(bits=_b, impl=0)
    _via = ["dispatch.impl4.simt"] if _b == 4 else [f"dispatch.bits{_b}"]
    _p = f"simt{_b}."
    _st = [_p + "straddle"] if _b == 3 else []
    FWD_CASES += [
        C(f"simt{_b}_cap", "fwd", [_p + "mt1", _p + "s_cap", _p + "short_slice", _p + "nb_even", *_via, *_st],
          m=1, k=11008, n=16384, gs=128, **_simt),
        C(f"simt{_b}_mt2", "fwd", [_p + "mt2", _p + "s_free", _p + "k_tail", _p + "n_tail", _p + "rows_past_k", _p + "nb_odd",
                                   *_st], m=2, k=1000, n=300, gs=0, kw_extra=3, **_simt),
        C(f"simt{_b}_mt4", "fwd", [_p + "mt4", _p + "short_slice", _p + "nb_odd", _p + "nb_even", *_st],
          m=3, k=4096, n=11008, gs=128, **_simt),
        C(f"simt{_b}_mt8_mpass", "fwd", [_p + "mt8", _p + "mpass", *_st], m=19, k=640, n=128, gs=128, **_simt),
    ]
TINY_CASES = [
    C("tiny_fwd_tc", "fwd", ["dispatch.impl2.tc", "dispatch.via.ex", "tc.f32"], SPLIT_DATA,
      m=12, k=1024, n=512, gs=128, impl=2, via="ex", data="tiny"),
    C("tiny_fwd_decode", "fwd", ["dispatch.impl1.decode", "dec.nbk2"], SPLIT_DATA,
      m=12, k=128, n=512, gs=128, impl=1, via="ex", data="tiny"),
    C("tiny_fwd_simt", "fwd", ["dispatch.impl4.simt", "simt4.mt8", "simt4.mpass"],
      m=12, k=128, n=512, gs=128, impl=4, via="ex", data="tiny"),
    C("tiny_dgrad_tc", "dgrad", ["dg.impl2", "dg.tc"], SPLIT_DATA, m=12, k=512, n=1024, gs=128, impl=2, data="tiny"),
]
BATCH_CASES = [
    C("batch_3", "batch", ["dec.batch", "dec.batch.diff_n", "dec.batch.short_k", "dec.nbk2"],
      m=9, problems=((1024, 512), (1024, 132), (512, 256))),
    C("batch_4", "batch", ["dec.batch", "dec.nbk4"], m=32, problems=((2048, 512), (2048, 512), (1024, 1024), (2048, 256))),
]
F16_CASES = [
    C("f16_tc", "f16", ["f16.tc", "tc.f16_out", "tc.f16_out.bias", "tc.live_a_only"], m=800, k=1024, n=260, gs=128,
      state=True, bias=True),
    C("f16_tc_nobias", "f16", ["f16.tc", "tc.f16_out.nobias", "f16.null_bias"], m=768, k=512, n=512, gs=128, state=True,
      bias=False),
    C("f16_single", "f16", ["f16.single", "dec.f16", "dec.f16.unroll4"], ["dec.f16.counter_reset"],
      m=1, k=4096, n=4096, gs=128, state=True, bias=True),
    C("f16_single_rem_nobias", "f16", ["f16.single", "dec.f16.rem", "dec.f16.unroll4", "f16.null_bias"],
      ["dec.f16.counter_reset"], m=17, k=1152, n=132, gs=128, state=True, bias=False),
    C("f16_staged_no_state", "f16", ["f16.staged.no_state", "dispatch.auto.decode"], m=5, k=1024, n=512, gs=128,
      state=False, bias=True),
    C("f16_staged_mid", "f16", ["f16.staged.mid", "dispatch.auto.tc"], m=300, k=1024, n=520, gs=128, state=True, bias=True),
    C("f16_staged_unsupported", "f16", ["f16.staged.unsupported", "dispatch.refuse.k8"], m=800, k=1004, n=256, gs=0,
      state=True, bias=True),
]
DGRAD_CASES = [
    C("dg_small_m", "dgrad", ["dg.auto.small_m", "dg.simt.slices", "dg.simt.k_tail", "dg.simt.mt4", "dg.simt.m_tiles",
                              "dg.simt.b4"], m=40, k=1000, n=2512, gs=128, impl=0),
    C("dg_tc_tails", "dgrad", ["dg.auto.tc", "dg.tc", "dg.tc.kw_tail", "dg.tc.n_tail", "dg.tc.one_group_k128",
                               "dg.tc.m_tail", "dg.tc.k_tail"], ["dg.tc.need_lo"], m=300, k=516, n=264, gs=0, impl=0),
    C("dg_auto_3bit", "dgrad", ["dg.auto.unsupported", "dg.simt.b3"], bits=3, m=64, k=768, n=136, gs=128, impl=0),
    C("dg_impl1_mt1", "dgrad", ["dg.impl1", "dg.simt.mt1", "dg.simt.one_slice", "dg.simt.b2", "dg.simt.k_tail"],
      bits=2, m=1, k=6661, n=61, gs=0, impl=1),
    C("dg_impl1_mt2", "dgrad", ["dg.impl1", "dg.simt.mt2", "dg.simt.slices"], m=2, k=256, n=2516, gs=128, impl=1),
    C("dg_chunk_restart", "dgrad", ["dg.impl2", "dg.tc.chunk_restart", "dg.tc.ring_wrap", "dg.tc.ring_wrap2"],
      m=64, k=512, n=1032, gs=128, impl=2),
    C("dg_chunk_exact", "dgrad", ["dg.auto.tc", "dg.tc.chunk_exact"], ["dg.tc.no_lo"], m=128, k=256, n=1024, gs=128,
      impl=0, data="f16x"),
    C("dg_impl2_error", "dgrad", ["dg.impl2.error"], m=64, k=126, n=64, gs=0, impl=2),
    C("dg_c_clamp", "dgrad", ["dg.impl2", "dg.tc"], ["dg.tc.c_clamp"], m=64, k=256, n=128, gs=128, impl=2, zeros="tiny_g0"),
]
ALL_CASES = FWD_CASES + TINY_CASES + BATCH_CASES + F16_CASES + DGRAD_CASES

REQUIRED = {
    "dispatch.auto.tc", "dispatch.auto.decode", "dispatch.auto.simt", "dispatch.auto.ws_null", "dispatch.auto.ws_small",
    "dispatch.refuse.k8", "dispatch.refuse.n4", "dispatch.refuse.group128", "dispatch.refuse.x_misaligned",
    "dispatch.refuse.qw_misaligned", "dispatch.impl1.decode", "dispatch.impl1.simt_fallback", "dispatch.impl2.tc",
    "dispatch.impl2.error", "dispatch.impl4.simt", "dispatch.via.global", "dispatch.via.ex", "dispatch.bits2",
    "dispatch.bits3",
    *[f"simt{b}.{x}" for b in (2, 3, 4) for x in ("mt1", "mt2", "mt4", "mt8", "mpass", "s_cap", "s_free", "short_slice",
                                                  "nb_odd", "nb_even", "k_tail", "n_tail", "rows_past_k")],
    "simt3.straddle",
    "dec.nbk1", "dec.nbk2", "dec.nbk4", "dec.mpass", "dec.smax", "dec.short_slice", "dec.nb1", "dec.per_sm", "dec.reg",
    "dec.slab", "dec.slab.trow_alias", "dec.slab.zero_fill", "dec.slab.n_tail", "dec.wait.strict", "dec.wait.static",
    "dec.no_pdl", "dec.prefetch", "dec.need_lo", "dec.no_lo", "dec.batch", "dec.batch.diff_n", "dec.batch.short_k",
    "dec.f16", "dec.f16.unroll4", "dec.f16.rem", "dec.f16.counter_reset",
    "tc.f32", "tc.f16_out", "tc.f16_out.bias", "tc.f16_out.nobias", "tc.int_zero", "tc.general.fractional",
    "tc.general.big_zero", "tc.general.scale0", "tc.one_pass", "tc.two_pass", "tc.k64_tail", "tc.odd_kb", "tc.ring_wrap",
    "tc.ring_wrap2", "tc.m_tail", "tc.n_tail", "tc.live_a_only", "tc.gq_ne_g", "tc.kw_extra",
    "f16.tc", "f16.single", "f16.staged.no_state", "f16.staged.mid", "f16.staged.unsupported", "f16.null_bias",
    "dg.auto.small_m", "dg.auto.tc", "dg.auto.unsupported", "dg.impl1", "dg.impl2", "dg.impl2.error", "dg.tc",
    "dg.simt.mt1", "dg.simt.mt2", "dg.simt.mt4", "dg.simt.one_slice", "dg.simt.slices", "dg.simt.k_tail",
    "dg.simt.m_tiles", "dg.simt.b2", "dg.simt.b3", "dg.simt.b4", "dg.tc.kw_tail", "dg.tc.n_tail", "dg.tc.chunk_restart",
    "dg.tc.chunk_exact", "dg.tc.one_group_k128", "dg.tc.m_tail", "dg.tc.k_tail", "dg.tc.ring_wrap", "dg.tc.ring_wrap2",
    "dg.tc.c_clamp", "dg.tc.need_lo", "dg.tc.no_lo", *SPLIT_DATA,
}


def doc_alias(x):
    """The docstring names the SIMT cases and ids of the three bit widths through simt<b>."""
    return x if x == "simt3.straddle" else re.sub(r"^simt[234]([._])", r"simt<b>\1", x)


# -------------------------------------------------------------------------------------------------- CPU tests
def test_case_table_covers_every_branch():
    assert_table_covers(ALL_CASES, REQUIRED, lambda c: check_reach(c, branches(c, geo.SM_COUNT_H100)), __doc__,
                        doc_alias=doc_alias, reject_unknown=True)


def test_geometry_matches_documented_launches():
    """Spot values of the restated formulas, worked by hand from the .cu files at 132 SMs."""
    sm = geo.SM_COUNT_H100
    # SIMT, 4096 x 11008 at M = 1: 86 column blocks, ceil(1056 / 86) = 13 slices wanted, S = ceil(32 / 13) = 3, 11 slices,
    # the last one 2 blocks long
    p = geo.simt_plan(4, 1, 4096, 11008, sm)
    assert (p["colblocks"], p["S"], p["slices"], p["capped"], p["mt"], p["nbs"][-1]) == (86, 3, 11, False, 1, 2)
    # ... 11008 x 16384: 128 column blocks, 9 wanted, S = ceil(86 / 9) = 10 capped at 1024 / 128 = 8, 11 slices; 2-bit:
    # 172 blocks of 64, S = 20 capped at 16
    p = geo.simt_plan(4, 1, 11008, 16384, sm)
    assert (p["S"], p["capped"], p["slices"], p["nbs"][-1]) == (8, True, 11, 6)
    p = geo.simt_plan(2, 1, 11008, 16384, sm)
    assert (p["nblk"], p["S"], p["capped"], p["slices"]) == (172, 16, True, 11)
    assert geo.simt_plan(4, 19, 640, 128, sm)["passes"] == 3 and geo.simt_plan(3, 5, 640, 128, sm)["mt"] == 8
    # decode, 4096 x 11008 at M = 1: ceil(5 x 132 / 86) = 8 slices wanted, S = 4 (<= smax 8), 8 slices
    p = geo.dec_plan([(4096, 11008, 512)], 1, DEFAULT_MODE, sm)
    assert (p["nbk"], p["S"], p["slices"], p["capped"]) == (1, 4, 8, False)
    # ... 11008 x 4096 at M = 20: nbk 4, 21 wanted, S = ceil(86 / 21) = 5 clamped to smax 2, 43 slices
    p = geo.dec_plan([(11008, 4096, 1376)], 20, DEFAULT_MODE, sm)
    assert (p["nbk"], p["S"], p["capped"], p["slices"]) == (4, 2, True, 43)
    # mode 0x82: 8 CTAs per SM
    assert geo.dec_plan([(2048, 1028, 256)], 9, 0x82, sm)["per_sm"] == 8
    # the single-launch fp16 path at 4096 x 4096, M = 1: 32 column blocks, 21 wanted, S = 2, 16 slices
    assert geo.dec_plan([(4096, 4096, 512)], 1, DEFAULT_MODE, sm)["slices"] == 16
    # dgrad SIMT plan, 4096 x 4096 at M = 32: mt 4, 128 units x 8 row tiles = 1024 CTAs already, one slice of all N
    assert geo.dgrad_simt_plan(32, 4096, 4096) == dict(mt=4, slice_n=4096, slices=1, m_tiles=8, grid=(128, 8, 1),
                                                        m_passes=1)
    # ... M = 40, K = 1000, N = 2512: 32 units x 10 tiles = 320, 4 slices of 640 columns
    assert geo.dgrad_simt_plan(40, 1000, 2512) == dict(mt=4, slice_n=640, slices=4, m_tiles=10, grid=(32, 10, 4),
                                                        m_passes=1)
    assert geo.dgrad_simt_plan(1, 6661, 61) == dict(mt=1, slice_n=128, slices=1, m_tiles=1, grid=(209, 1, 1), m_passes=1)
    # ... M = 600001: 150001 row tiles, gridDim.y capped at 65535, so some CTAs walk 3 tiles
    assert geo.dgrad_simt_plan(600001, 64, 256) == dict(mt=4, slice_n=256, slices=1, m_tiles=150001,
                                                        grid=(2, 65535, 1), m_passes=3)
    # wgmma refusals and the tile whose second feature row is past N
    assert geo.tc_refusal(1004, 256, 1004) == "k8" and geo.tc_refusal(1000, 256, 1000) == "group128"
    assert geo.tc_refusal(512, 256, 128, x_off=1) == "x_misaligned" and geo.tc_refusal(512, 256, 128, qw_off=2) == "qw_misaligned"
    assert geo.tc_live_a_only(264) and geo.tc_live_a_only(132) and not geo.tc_live_a_only(144) and not geo.tc_live_a_only(256)
    assert geo.dispatch(31, 512, 256, 128, 0)[0] == "decode" and geo.dispatch(32, 512, 256, 128, 0)[0] == "tc"
    assert geo.dispatch(64, 512, 256, 128, 0, ws="null")[0] == "decode"
    assert geo.dgrad_branches(4, 47, 512, 256, 64, 128, 0) >= {"dg.auto.small_m"}
    assert geo.dgrad_branches(4, 48, 512, 256, 64, 128, 0) >= {"dg.auto.tc"}
    # the probe and the split, on data
    s = np.full((4, 2), 0.01, F32)
    assert geo.zero_probe(s, (s * 3).astype(F32)) == set()
    assert geo.zero_probe(s, (s * 3.5).astype(F32)) == {"tc.general.fractional"}
    assert geo.zero_probe(s, (s * 1100).astype(F32)) == {"tc.general.big_zero"}
    s0 = s.copy()
    s0[1, 1] = 0
    assert geo.zero_probe(s0, (s * 3).astype(F32)) == {"tc.general.scale0"}
    assert not geo.split_need_lo(np.ones((2, 8), F32)) and geo.split_need_lo(np.full((1, 8), 1 + 2.0 ** -20, F32))
    raw, c = geo.dgrad_table_c(np.array([[1e-28, 0.01]], F32).repeat(3, 0), np.zeros((3, 2), F32))
    assert raw[0] > 100 and c[0] == 100 and c[1] == raw[1]


def test_pack_and_truth_match_hand_packed_words():
    """The test's packer and the unpacking inside its fp64 truth both follow oracle.gptq's slot map; here both are held
    to words packed by hand from QuantLinear.pack (utils/quant.py:214-257): 4-bit q = 1..8 -> 0x87654321; 2-bit
    q = 0,1,2,3,... -> 0xE4E4E4E4; 3-bit, one 32-value unit with q0 = 5, q9 = 3, q10 = 7 (bits 1:0 at << 30 of word 0, bit
    2 at bit 0 of word 1), q11 = 3 (<< 1), q21 = 5 (bit 0 at << 31 of word 1, bits 2:1 at bit 0 of word 2), q22 = 1
    (<< 2), q31 = 6 (<< 29)."""
    q3 = np.zeros(32, np.int64)
    q3[[0, 9, 10, 11, 21, 22, 31]] = [5, 3, 7, 3, 5, 1, 6]
    for bits, q, words in ((4, np.arange(1, 9), [0x87654321]), (2, np.arange(16) % 4, [0xE4E4E4E4]),
                           (3, q3, [0xD8000005, 0x80000007, 0xC0000006])):
        k = q.size
        got = pack(q[:, None], bits, len(words))
        assert got.view(U32).reshape(-1).tolist() == words, (bits, [hex(w) for w in got.view(U32).reshape(-1)])
        one = torch.ones(1, 1, dtype=torch.float32)
        # x = e_i, scale 1, zero 0: the truth's row i is q_i
        y, _ = truth(torch.eye(k), torch.from_numpy(np.asarray(words, U32).view(np.int32)[:, None].copy()), one,
                     torch.zeros(1, 1), k, k, bits, torch.zeros(k, 1))
        assert y[:, 0].tolist() == q.tolist(), bits


# -------------------------------------------------------------------------------------------------- helpers
def filled_bytes(nbytes):
    return torch.full((max(int(nbytes), 16),), WS_FILL, dtype=torch.uint8, device=dev())


def _values_held(bits, kw):
    """The K values `kw` packed rows hold."""
    return kw * 32 // bits


def pack(q, bits, kw):
    """q: [values held by kw rows, N] integers in [0, 2^bits) -> qweight [kw, N] int32, QuantLinear.pack's layout."""
    n = q.shape[1]
    q = q.astype(np.uint64)
    if bits in (2, 4):
        per = 32 // bits
        q3 = q.reshape(kw, per, n)
        w = np.zeros((kw, n), np.uint64)
        for j in range(per):
            w |= q3[:, j] << np.uint64(bits * j)
        return w.astype(U32).view(np.int32)
    units = kw // 3
    q3 = q.reshape(units, 32, n)
    w = np.zeros((units, 3, n), np.uint64)
    for j, (row, shift, srow, sshift) in enumerate(ogptq._bit_slots(3, 32)):
        w[:, row] |= (q3[:, j] << np.uint64(shift)) & np.uint64(0xFFFFFFFF)
        if srow is not None:
            w[:, srow] |= q3[:, j] >> np.uint64(sshift)
    return w.reshape(kw, n).astype(U32).view(np.int32)


def make_weights(rng, bits, k, n, gs, kw_extra=0, zeros="int"):
    """Random GPTQ weights: integer q (random past K too), scales ~ 2 / sqrt(K) / maxq, zeros = zero * scale with an
    integer zero point (the checkpoint convention), or the variants the wgmma zero probe refuses."""
    kw0 = geo.packed_rows(bits, k)
    maxq = 2 ** bits - 1
    q = rng.integers(0, maxq + 1, (_values_held(bits, kw0), n))
    qw = pack(q, bits, kw0)
    if kw_extra:
        qw = np.concatenate([qw, rng.integers(0, 2 ** 32, (kw_extra, n), dtype=np.uint64).astype(U32).view(np.int32)])
    g = -(-k // gs)
    scales = (rng.uniform(0.5, 1.5, (n, g)) * 2 / np.sqrt(k) / maxq).astype(F32)
    zint = rng.integers(1, maxq, (n, g)).astype(F32)
    zr = (zint * scales).astype(F32)
    if zeros == "frac":
        zr = ((zint + rng.uniform(-0.45, 0.45, zint.shape).astype(F32)) * scales).astype(F32)
    elif zeros == "big":
        big = rng.random(zint.shape) < 0.02
        big[0, 0] = True
        zr = np.where(big, np.where(rng.random(zint.shape) < 0.5, F32(-1100), F32(1100)) * scales, zr).astype(F32)
    elif zeros == "scale0":
        scales[3, 0] = 0
        zr[3, 0] = F32(-0.03)
    elif zeros == "tiny_g0":
        scales[:, 0] *= F32(1e-26)
        zr[:, 0] *= F32(1e-26)
    return qw, scales, zr


def truth(x, qw_d, sc_d, zr_d, k, gs, bits, prefill):
    """fp64 truth on the device: prefill + x @ W and sum |x| |W|, W [K, N] dequantised in float64, 2048 rows of K at a
    time.  x: [M, K] device float32 (may hold non-finite values)."""
    kw, n = qw_d.shape
    d = qw_d.device
    q64 = qw_d.to(torch.int64) & 0xFFFFFFFF
    xd = x.double()
    y = prefill.double().clone()
    mag = torch.zeros_like(y)
    slots = ogptq._bit_slots(bits, k)
    for k0 in range(0, k, 2048):
        ks = range(k0, min(k, k0 + 2048))
        row = torch.tensor([slots[i][0] for i in ks], device=d)
        sh = torch.tensor([slots[i][1] for i in ks], device=d)[:, None]
        v = q64[row] >> sh
        spill = [i for i in ks if slots[i][2] is not None]
        if spill:
            loc = torch.tensor([i - k0 for i in spill], device=d)
            srow = torch.tensor([slots[i][2] for i in spill], device=d)
            ssh = torch.tensor([slots[i][3] for i in spill], device=d)[:, None]
            v[loc] |= q64[srow] << ssh
        qv = (v & (2 ** bits - 1)).double()
        gi = torch.arange(k0, k0 + len(ks), device=d) // gs
        w = sc_d.double()[:, gi].T * qv - zr_d.double()[:, gi].T
        y += xd[:, k0:k0 + len(ks)] @ w
        mag += xd[:, k0:k0 + len(ks)].abs() @ w.abs()
    return y, mag


def bit_identical(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def assert_close_rows(got, exp, outlier_rows=()):
    """rtol = atol = 1e-5 elementwise; rows with planted outliers: 1e-5 + 1e-5 max |row|."""
    got, exp = got.double(), exp.double()
    plain = [r for r in range(got.shape[0]) if r not in outlier_rows]
    if plain:
        torch.testing.assert_close(got[plain], exp[plain], rtol=1e-5, atol=1e-5)
    for r in outlier_rows:
        bound = 1e-5 + 1e-5 * max(exp[r].abs().max().item(), 1.0)
        assert (got[r] - exp[r]).abs().max().item() <= bound, f"row {r}"


def activations(rng, case, m, length):
    """[m, length] fp32 rows for the case's data variant; returns (x, outlier rows)."""
    data = case.get("data", "plain")
    if data == "tiny":
        return tiny_rows(rng, length), ()
    x = rng.standard_normal((m, length)).astype(F32)
    if data == "f16x":
        return x.astype(F16).astype(F32), ()
    if data == "outliers":
        x[0, :5] = [3e4, -7e4, 1e-6, 0.0, 123.0]  # fp16-overflowing magnitudes are fine after the row scaling
        x[2] *= F32(1e-4)
        return x, (0, 2)
    return x, ()


TINY_EXACT_J = (0, 40, 100, 112)  # rows 0..3: r * 2^-j, max |x| >= 2^-112
TINY_ROWS = 12


def tiny_rows(rng, length):
    """Rows 0..3: r 2^-j for TINY_EXACT_J (|r| in [0.01, 2), max in [1, 2), so every element stays a normal number);
    4: r 2^-113; 5: r 2^-118 and 6: r 2^-125 (max |x| in [2^-126, 2^-113)); 7: zeros and one subnormal; 8: subnormals;
    9: zeros; 10: one +inf; 11: one NaN."""
    r = (rng.uniform(0.01, 1.99, length) * np.where(rng.random(length) < 0.5, -1, 1)).astype(F32)
    r[0] = F32(1.75)
    r[5::97] = 0
    x = np.zeros((TINY_ROWS, length), F32)
    for i, j in enumerate(TINY_EXACT_J + (113, 118, 125)):
        x[i] = np.ldexp(r, -j).astype(F32)
    x[7, length // 3] = np.array([0x00012345], U32).view(F32)[0]
    x[8] = (rng.integers(1, 1 << 23, length, dtype=np.int64).astype(U32)
            | ((rng.random(length) < 0.5).astype(U32) << U32(31))).view(F32)
    x[10] = r
    x[10, 7] = np.inf
    x[11] = r
    x[11, 9] = np.nan
    return x


def check_tiny(got, exp, mag, prefill, atomics=0, exact_rows=len(TINY_EXACT_J), extra=0.0):
    """The tiny-row contract of the module docstring; got / exp / mag / prefill [TINY_ROWS, N] device tensors.

    `atomics`: fp32 atomic additions per output (0: plain stores).  A plain store rounds a subnormal result once (2^-149);
    a float atomicAdd on sm_90a (RED.E.ADD.F32.FTZ.RN) flushes a subnormal result to zero, which loses up to 2^-126 per
    addition.  The first `exact_rows` rows must be y * 2^-j bit for bit wherever that is a normal number and within that
    slack elsewhere; rows 0..8 must be finite and within 1e-5 sum |x||w| + slack + `extra` of the fp64 truth."""
    slack = atomics * 2.0 ** -126 if atomics else 2.0 ** -149
    g, e, a, p = (t.double().cpu().numpy() for t in (got, exp, mag, prefill))
    y0 = g[0]
    for i, j in enumerate(TINY_EXACT_J[:exact_rows]):
        want = np.ldexp(y0, -j).astype(F32).astype(F64)
        normal = np.abs(want) >= 2.0 ** -126
        assert np.array_equal(g[i][normal], want[normal]), f"row {i} (x 2^-{j}) is not y * 2^-{j} bit for bit"
        assert np.all(np.abs(g[i][~normal] - want[~normal]) <= slack), f"row {i}"
    for i in range(0, 9):
        assert np.isfinite(g[i]).all(), f"row {i}: {np.count_nonzero(~np.isfinite(g[i]))} non-finite outputs"
        err = np.abs(g[i] - e[i])
        bound = 1e-5 * a[i] + slack + extra
        assert np.all(err <= bound), f"row {i}: error {err.max():.3g} above {bound[np.argmax(err - bound)]:.3g}"
    assert np.array_equal(g[9], p[9]), "the zero row changed its prefill"
    for i in (10, 11):
        assert np.array_equal(np.isfinite(g[i]), np.isfinite(e[i])) and not np.isfinite(g[i]).any(), f"row {i}"


@pytest.fixture
def gptq_globals():
    """sb200_gptq4_set_impl and sb200_gptq4_set_decode are process-wide: set them per case, restore the defaults (impl 0,
    decode mode 6) afterwards, also when the case fails."""
    lib = _lib.load()

    def set_(impl=0, mode=DEFAULT_MODE):
        _lib.check(lib.sb200_gptq4_set_impl(impl))
        _lib.check(lib.sb200_gptq4_set_decode(mode))

    yield set_
    lib.sb200_gptq4_set_impl(0)
    lib.sb200_gptq4_set_decode(DEFAULT_MODE)


# -------------------------------------------------------------------------------------------------- fp32 forward
def _fwd_call(case, x_d, qw_d, out, sc_d, zr_d, ws, ws_bytes, gptq_globals):
    lib = _lib.load()
    bits, m, k, n = case.get("bits", 4), case.get("m"), case.get("k"), case.get("n")
    gs, impl, kw = case.get("gs"), case.get("impl"), qw_d.shape[0]
    mode = case.get("mode", DEFAULT_MODE)
    args = (x_d.data_ptr(), qw_d.data_ptr(), out.data_ptr(), sc_d.data_ptr(), zr_d.data_ptr(), m, k, n, kw)
    wsp = ws.data_ptr() if ws is not None else None
    if bits != 4:
        gptq_globals(impl=2, mode=mode)  # the 2 / 3-bit entry point ignores the process-wide 4-bit selection
        return lib.sb200_gptq_matmul(*args, bits, gs, wsp, ws_bytes, stream())
    if case.get("via", "global") == "ex":
        gptq_globals(impl=4 if impl != 4 else 1, mode=mode)  # a decoy: the per-call option must win
        opts = ops._Gptq4Options(impl, 0, 0)
        return lib.sb200_gptq4_matmul_ex(*args, gs, ctypes.byref(opts), wsp, ws_bytes, stream())
    gptq_globals(impl=impl, mode=mode)
    return lib.sb200_gptq4_matmul(*args, gs, wsp, ws_bytes, stream())


def _check_data_claims(case, x, scales, zeros):
    probe = geo.zero_probe(scales, zeros)
    for c in case.claims:
        if c == "tc.int_zero":
            assert probe == set(), probe
        elif c.startswith("tc.general."):
            assert probe == {c}, probe  # the probe is refused for this reason alone
        elif c in ("tc.two_pass", "dec.need_lo", "dg.tc.need_lo"):
            assert geo.split_need_lo(x)
        elif c in ("tc.one_pass", "dec.no_lo", "dg.tc.no_lo"):
            assert not geo.split_need_lo(x)
        elif c.startswith("split."):
            assert c in geo.split_row_kinds(x)
        elif c == "dg.tc.c_clamp":
            raw, clamped = geo.dgrad_table_c(scales, zeros)
            assert (raw != clamped).any()


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(FWD_CASES + [c for c in TINY_CASES if c.op == "fwd"]))
def test_forward_branch_vs_fp64(case, gptq_globals):
    check_reach(case, branches(case, real_sm()))
    rng = np.random.default_rng(seed(case.name))
    bits, m, k, n = case.get("bits", 4), case.get("m"), case.get("k"), case.get("n")
    gs = _gs(case)
    qw, scales, zeros = make_weights(rng, bits, k, n, gs, case.get("kw_extra", 0), case.get("zeros", "int"))
    x, outliers = activations(rng, case, m, k)
    _check_data_claims(case, x, scales, zeros)
    bias = np.zeros(n, F32) if case.get("data") == "tiny" else rng.standard_normal(n).astype(F32)
    x_d, qw_d = on_device(x, case.get("x_off", 0)), on_device(qw, case.get("qw_off", 0))
    sc_d, zr_d = on_device(scales), on_device(zeros)
    prefill = torch.from_numpy(np.broadcast_to(bias, (m, n)).copy()).to(dev())
    lib = _lib.load()
    need = int(lib.sb200_gptq4_workspace_bytes(m, k, n, case.get("gs")))
    ws_kind = case.get("ws", "ok")
    ws = None if ws_kind == "null" else filled_bytes(need)
    ws_bytes = {"ok": ws.numel() if ws is not None else 0, "null": 0, "small": max(need - 1, 0)}[ws_kind]
    runs = []
    for _ in range(2):
        out = prefill.clone()
        torch.cuda.synchronize()
        before = _lib.launch_count()
        rc = _fwd_call(case, x_d, qw_d, out, sc_d, zr_d, ws, ws_bytes, gptq_globals)
        torch.cuda.synchronize()
        if case.get("impl") == 2 and "dispatch.impl2.error" in case.targets:
            assert rc == E_UNSUPPORTED and b"unsupported" in lib.sb200_last_error()
            assert _lib.launch_count() == before and torch.equal(out, prefill)
            return
        assert rc == 0, lib.sb200_last_error()
        runs.append(out)
    kernel = geo.dispatch(m, k, n, gs, case.get("impl"), case.get("x_off", 0), case.get("qw_off", 0), ws_kind)[0] if bits == 4 else "simt"
    if kernel == "tc":
        assert bit_identical(runs[0], runs[1])  # one CTA per output tile, fixed fold order
    exp, mag = truth(x_d.reshape(m, k), qw_d, sc_d, zr_d, k, gs, bits, prefill)
    if case.get("data") == "tiny":
        if kernel == "tc":
            check_tiny(runs[0], exp, mag, prefill)
        elif kernel == "decode":
            # one K slice: each output is one atomicAdd of the exactly scaled partial sum onto the zero prefill
            assert geo.dec_plan([(k, n, qw.shape[0])], m, case.get("mode", DEFAULT_MODE), real_sm())["slices"] == 1
            check_tiny(runs[0], exp, mag, prefill, atomics=1)
        else:
            # one K slice as well.  The SIMT kernel stages x * 16^-(k % 4) (gptq_simt.cu:82-89), which is a subnormal
            # for x below 2^-114: each staged value is then exact to 2^-150 only, i.e. to 15 * 16^3 * 2^-150 after
            # the nibble decode, for each of the K terms (times the scale and zero point, both below 1 here).  The
            # same staging leaves the rows from 2^-112 on not exactly scaled, so only rows 0..2 are compared bit for
            # bit.
            assert geo.simt_plan(4, m, k, n, real_sm())["slices"] == 1
            check_tiny(runs[0], exp, mag, prefill, atomics=1, exact_rows=3, extra=k * 15 * 16.0 ** 3 * 2.0 ** -150)
        return
    assert_close_rows(runs[0], exp, outliers)


@pytest.mark.gpu
def test_decode_tiny_rows_lose_only_flushed_subnormals(gptq_globals):
    """One row r 2^-j per launch (M = 1, K = 128: one K slice) through the decode kernel, j past its exponent clamp.
    Each output is one atomicAdd of the kernel's partial sum onto a zero prefill, and the float atomic flushes a
    subnormal result to zero (RED.E.ADD.F32.FTZ.RN on sm_90a).  So every output is within 1e-5 sum |x||w| (+ one
    subnormal rounding) of the fp64 truth, except outputs that are exactly zero where the truth is below 2^-126 (plus
    that bound): nothing but the flush is lost.  The flush does occur at these magnitudes."""
    gptq_globals()
    rng = np.random.default_rng(seed("decode_tiny_rows_lose_only_flushed_subnormals"))
    qw, scales, zeros = make_weights(rng, 4, 128, 512, 128)
    qw_d, sc_d, zr_d = on_device(qw), on_device(scales), on_device(zeros)
    r = tiny_rows(rng, 128)[0]
    flushed = 0
    for j in (113, 116, 118, 120, 125):
        x_d = on_device(np.ldexp(r, -j).astype(F32)[None])
        out = torch.zeros(1, 512, device=dev())
        ops.gptq4_matmul(x_d, qw_d, out, sc_d, zr_d, 128, impl=1)
        exp, mag = truth(x_d, qw_d, sc_d, zr_d, 128, 128, 4, torch.zeros(1, 512, device=dev()))
        g = out.double()
        bound = 1e-5 * mag + 2.0 ** -149
        close = (g - exp).abs() <= bound
        flush = (g == 0) & (exp.abs() < 2.0 ** -126 + bound)
        assert (close | flush).all(), f"x 2^-{j}: {int((~(close | flush)).sum())} outputs off by more than a flush"
        flushed += int((flush & ~close).sum())
    assert flushed > 0


# -------------------------------------------------------------------------------------------------- batch
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(BATCH_CASES))
def test_batch_branch_vs_fp64(case, gptq_globals):
    check_reach(case, branches(case, real_sm()))
    gptq_globals(mode=case.get("mode", DEFAULT_MODE))
    rng = np.random.default_rng(seed(case.name))
    m = case.get("m")
    probs, keep = [], []
    for k, n in case.get("problems"):
        qw, scales, zeros = make_weights(rng, 4, k, n, 128)
        x = rng.standard_normal((m, k)).astype(F32)
        bias = rng.standard_normal(n).astype(F32)
        prefill = torch.from_numpy(np.broadcast_to(bias, (m, n)).copy()).to(dev())
        t = (on_device(x), on_device(qw), prefill.clone(), on_device(scales), on_device(zeros))
        probs.append(ops._Gptq4Problem(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(),
                                       k, n, qw.shape[0], 128))
        keep.append((t, prefill, k))
    arr = (ops._Gptq4Problem * len(probs))(*probs)
    before = _lib.launch_count()
    assert _lib.load().sb200_gptq4_matmul_batch(arr, len(probs), m, stream()) == 0
    assert _lib.launch_count() - before == 1
    for (x_d, qw_d, out, sc_d, zr_d), prefill, k in keep:
        exp, _ = truth(x_d, qw_d, sc_d, zr_d, k, 128, 4, prefill)
        assert_close_rows(out, exp)


# -------------------------------------------------------------------------------------------------- fp16 linear
def _ulp16(v):
    """The fp16 spacing at |v| (normal binades; 2^-24 below 2^-14)."""
    a = np.abs(v)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return np.exp2(e - 10)


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(F16_CASES))
def test_linear_f16_branch_vs_fp64(case, gptq_globals):
    check_reach(case, branches(case, real_sm()))
    gptq_globals()
    rng = np.random.default_rng(seed(case.name))
    m, k, n, gs = case.get("m"), case.get("k"), case.get("n"), _gs(case)
    qw, scales, zeros = make_weights(rng, 4, k, n, gs)
    xh = rng.standard_normal((m, k)).astype(F16)
    bias = rng.standard_normal(n).astype(F32) if case.get("bias") else None
    x_d, qw_d, sc_d, zr_d = on_device(xh), on_device(qw), on_device(scales), on_device(zeros)
    b_d = on_device(bias) if bias is not None else None
    lib = _lib.load()
    need = int(lib.sb200_gptq4_linear_f16_workspace_bytes(m, k, n, case.get("gs")))
    ws = filled_bytes(need)
    state = torch.zeros(int(lib.sb200_gptq4_linear_f16_state_bytes()), dtype=torch.uint8, device=dev()) if case.get("state") else None
    runs = []
    for _ in range(3 if "f16.single" in case.targets else 1):
        out = torch.full((m, n), WS_FILL * 257, dtype=torch.int16, device=dev()).view(torch.float16)  # 0x7B7B = 60768
        before = _lib.launch_count()
        rc = lib.sb200_gptq4_linear_f16_ex(x_d.data_ptr(), qw_d.data_ptr(), out.data_ptr(), b_d.data_ptr() if b_d is not None else None,
                                           sc_d.data_ptr(), zr_d.data_ptr(), m, k, n, qw.shape[0], case.get("gs"),
                                           state.data_ptr() if state is not None else None, 0, ws.data_ptr(), ws.numel(), stream())
        assert rc == 0, lib.sb200_last_error()
        if "f16.single" in case.targets:
            assert _lib.launch_count() - before == 1
            ws.fill_(WS_FILL)  # the next call must rewrite every partial slot it reads
        runs.append(out.cpu().numpy())
    for r in runs[1:]:  # the counters reset themselves; the slots are added in slice order
        assert np.array_equal(r.view(np.uint16), runs[0].view(np.uint16))
    if state is not None:
        assert not state.any()  # every feature block's counter is back at zero
    prefill = torch.from_numpy(np.broadcast_to(bias if bias is not None else np.zeros(n, F32), (m, n)).copy()).to(dev())
    exp, _ = truth(x_d.float(), qw_d, sc_d, zr_d, k, gs, 4, prefill)
    e = exp.cpu().numpy()
    y = runs[0].astype(F64)
    err = np.abs(y - e)
    bound = 0.51 * _ulp16(e) + 1e-5
    assert np.all(err <= bound), f"{np.count_nonzero(err > bound)} fp16 outputs off by more than 0.51 ulp + 1e-5"


# -------------------------------------------------------------------------------------------------- input gradient
@pytest.mark.gpu
@pytest.mark.parametrize("case", params(DGRAD_CASES + [c for c in TINY_CASES if c.op == "dgrad"]))
def test_dgrad_branch_vs_fp64(case):
    check_reach(case, branches(case, real_sm()))
    rng = np.random.default_rng(seed(case.name))
    bits, m, k, n, gs = case.get("bits", 4), case.get("m"), case.get("k"), case.get("n"), _gs(case)
    qw, scales, zeros = make_weights(rng, bits, k, n, gs, 0, case.get("zeros", "int"))
    go, _ = activations(rng, case, m, n)
    _check_data_claims(case, go, scales, zeros)
    tiny = case.get("data") == "tiny"
    pre = np.zeros((m, k), F32) if tiny or "dg.tc.c_clamp" in case.claims else rng.standard_normal((m, k)).astype(F32)
    go_d, qw_d, sc_d, zr_d = on_device(go), on_device(qw), on_device(scales), on_device(zeros)
    prefill = on_device(pre)
    lib = _lib.load()
    need = int(lib.sb200_gptq_dgrad_workspace_bytes(m, k, n, bits, case.get("gs")))
    ws = filled_bytes(need)
    runs = []
    for _ in range(2):
        gi = prefill.clone()
        before = _lib.launch_count()
        rc = lib.sb200_gptq_matmul_dgrad(go_d.data_ptr(), qw_d.data_ptr(), gi.data_ptr(), sc_d.data_ptr(), zr_d.data_ptr(), m, k,
                                         n, qw.shape[0], bits, case.get("gs"), case.get("impl"), ws.data_ptr(), ws.numel(),
                                         stream())
        if "dg.impl2.error" in case.targets:
            assert rc == E_UNSUPPORTED and b"unsupported" in lib.sb200_last_error()
            assert _lib.launch_count() == before and torch.equal(gi, prefill)
            return
        assert rc == 0, lib.sb200_last_error()
        runs.append(gi)
    assert bit_identical(runs[0], runs[1])  # both kernels: fixed reduction orders, no float atomics
    # grad_in = prefill + go @ W^T: the forward's truth with the roles of K and N swapped
    exp, mag = _dgrad_truth(go_d, qw_d, sc_d, zr_d, k, n, gs, bits, prefill)
    if tiny:
        check_tiny(runs[0], exp, mag, prefill)  # plain stores, no atomics
        return
    assert_close_rows(runs[0], exp)
    if "dg.tc.c_clamp" in case.claims:
        # group 0 (k < 128) has weights ~1e-28, far below atol: there the bar is relative to sum |g||w|
        err = (runs[0][:, :128].double() - exp[:, :128]).abs()
        assert (err <= 1e-5 * mag[:, :128]).all()


def _dgrad_truth(go_d, qw_d, sc_d, zr_d, k, n, gs, bits, prefill):
    """prefill + go @ W^T and |go| @ |W|^T with W [K, N] dequantised in float64 on the device."""
    eye_rows = torch.eye(k, dtype=torch.float32, device=dev())
    w, _ = truth(eye_rows, qw_d, sc_d, zr_d, k, gs, bits, torch.zeros(k, n, device=dev()))  # [K, N]: row i = e_i @ W
    g = go_d.double()
    return prefill.double() + g @ w.T, g.abs() @ w.abs().T
