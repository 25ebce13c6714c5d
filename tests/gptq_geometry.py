"""Plain-Python restatement of the host-side launch decisions of the GPTQ kernels: the dispatch and the entry points
(csrc/gptq.cu), the SIMT dequant-matmul (csrc/gptq_simt.cu), the decode kernel (csrc/gptq_decode.cu), the wgmma
prefill kernel (csrc/gptq_tc.cu) and the input gradient (csrc/gptq_dgrad.cu).

Test infrastructure only, in the manner of tests/weight_geometry.py: given a shape, the pointer offsets and the SM count
it names the kernel bodies and loops one call reaches, so that the cases in tests/test_gpu_gptq_branches.py can be tied to
the branch each exists for, and a CPU test can check that together they reach every branch.  It is not a second
dispatcher; when the formulas in the .cu files change, this file has to follow (the GPU cases re-check their branches
with the real SM count, so a stale restatement fails loudly).

Offsets are in elements from a 16-byte aligned allocation (floats for x / grad_out, int32 for qweight).  group_size is
the real group size (0 already replaced by K, as check_gptq_args does, gptq.cu:47).
"""

SM_COUNT_H100 = 132

SIMT_COLS = 128             # gptq_simt.cu:24 kCols
SIMT_CTAS_PER_SM = 8        # gptq_simt.cu:202
SIMT_STAGED_K = 1024        # gptq_simt.cu:205 s_cap = 1024 / kBlockK
DEC_COLS = 128              # gptq_decode.cu:31 kDecCols
DEC_BLOCK_K = 128           # gptq_decode.cu:32 kDecBlockK
DEC_DEFAULT_PER_SM = 5      # gptq_decode.cu:456
DEC_DEFAULT_MODE = 6        # gptq_decode.cu:416 g_dec_mode
DEC_MAX_PROBLEMS = 4        # gptq_launch.cuh:15 kDecMaxProblems
TC_MIN_M = 32               # gptq.cu:96 auto dispatch takes the wgmma kernel from this M on
TC_STAGES = 5               # gptq_tc.cu:30 kTcStages
TC_GROUP_K = 128            # gptq_tc.cu:31 kGroupK
WG_FEAT, WG_TOK, WG_BK = 128, 128, 64  # tc_common.cuh:21-23
F16_TC_MIN_M = 768          # gptq.cu:182
F16_SINGLE_MAX_M = 32       # gptq.cu:151 kF16SingleLaunchMaxM
F16_STATE_BYTES = 65536     # gptq.cu:152 kF16StateBytes
DG_TC_MIN_M = 48            # gptq.cu:225 kDgradTcMinM
DG_COLS = 128               # gptq_dgrad.cu:40 kDgCols
DG_UNIT_K = 32              # gptq_dgrad.cu:41 kDgUnitK
DG_TARGET_CTAS = 1024       # gptq_dgrad.cu:42 kDgTargetCtas
DG_MAX_GRID_Y = 65535       # gptq_dgrad.cu:43 kDgMaxGridY
DG_STAGES = 5               # gptq_dgrad.cu:179 kDgStages
DG_CHUNK = 8                # gptq_dgrad.cu:180 kDgChunk
DG_C_CLAMP = 100            # gptq_dgrad.cu:228


def _cdiv(a, b):
    return (a + b - 1) // b


def _a16(off):
    return off % 4 == 0


def block_k(bits):
    """GptqFmt<BITS>::kBlockK, gptq_unpack.cuh:21-22."""
    return 64 if bits == 2 else 128


def packed_rows(bits, k):
    """gptq_packed_rows, gptq_unpack.cuh:28-30."""
    return _cdiv(k, 8) if bits == 4 else (_cdiv(k, 16) if bits == 2 else _cdiv(k * 3, 96) * 3)


# ----------------------------------------------------------------------------------------------- dispatch (gptq.cu)
def tc_refusal(k, n, gs, x_off=0, qw_off=0):
    """gptq4_tc_supported, gptq_tc.cu:284-294: None, or the first reason it refuses."""
    if k % 8:
        return "k8"
    if n % 4:
        return "n4"
    if gs % TC_GROUP_K:
        return "group128"
    if not _a16(x_off):
        return "x_misaligned"
    if not _a16(qw_off):
        return "qw_misaligned"
    return None


def decode_supported(n, qw_off=0):
    """gptq4_decode_supported, gptq_decode.cu:410."""
    return n % 4 == 0 and _a16(qw_off)


def dispatch(m, k, n, gs, impl, x_off=0, qw_off=0, ws="ok"):
    """gptq4_dispatch, gptq.cu:81-103.  ws: "ok" | "null" | "small".  Returns (kernel, branches), kernel one of
    "tc" | "decode" | "simt" | "error"."""
    b = set()
    refusal = tc_refusal(k, n, gs, x_off, qw_off)
    if impl in (0, 2):
        ok2 = refusal is None and ws == "ok"
        if impl == 2 and not ok2:
            return "error", {"dispatch.impl2.error"}
        if impl == 2:
            return "tc", {"dispatch.impl2.tc"}
        if m >= TC_MIN_M:
            if ok2:
                return "tc", {"dispatch.auto.tc"}
            b.add(f"dispatch.refuse.{refusal}" if refusal else f"dispatch.auto.ws_{ws}")
    if impl != 4 and decode_supported(n, qw_off):
        b.add("dispatch.impl1.decode" if impl == 1 else "dispatch.auto.decode")
        return "decode", b
    b.add({0: "dispatch.auto.simt", 1: "dispatch.impl1.simt_fallback", 4: "dispatch.impl4.simt"}[impl])
    return "simt", b


# ----------------------------------------------------------------------------------------------- SIMT (gptq_simt.cu)
def simt_plan(bits, m, k, n, sm):
    """launch_simt, gptq_simt.cu:194-220."""
    bk = block_k(bits)
    nblk = _cdiv(k, bk)
    colblocks = _cdiv(n, SIMT_COLS)
    want = max(1, min(_cdiv(sm * SIMT_CTAS_PER_SM, colblocks), nblk))
    s = _cdiv(nblk, want)
    s_cap = SIMT_STAGED_K // bk
    capped = s > s_cap
    s = min(s, s_cap)
    mt = 1 if m == 1 else 2 if m == 2 else 4 if m <= 4 else 8
    slices = _cdiv(nblk, s)
    nbs = [min(y * s + s, nblk) - y * s for y in range(slices)]
    return dict(nblk=nblk, colblocks=colblocks, S=s, capped=capped, slices=slices, mt=mt, passes=_cdiv(m, mt), nbs=nbs)


def simt_branches(bits, m, k, n, kw, sm):
    p = simt_plan(bits, m, k, n, sm)
    pre = f"simt{bits}."
    b = {pre + f"mt{p['mt']}", pre + ("s_cap" if p["capped"] else "s_free")}
    if p["passes"] > 1:
        b.add(pre + "mpass")
    if p["nbs"][-1] < p["S"]:
        b.add(pre + "short_slice")  # gptq_simt.cu:60
    if any(nb % 2 for nb in p["nbs"]):
        b.add(pre + "nb_odd")  # gptq_simt.cu:178-185: the last block has no partner
    if any(nb % 2 == 0 for nb in p["nbs"]):
        b.add(pre + "nb_even")
    if k % block_k(bits):
        b.add(pre + "k_tail")  # gptq_simt.cu:88, 104
    if n % SIMT_COLS:
        b.add(pre + "n_tail")  # col_ok, gptq_simt.cu:57
    if kw * 32 // bits > k:
        b.add(pre + "rows_past_k")  # packed values with k >= K that the kernel loads (row < KW), times x = 0
    if bits == 3 and k > 21:
        b.add(pre + "straddle")  # values 10 and 21 of a 32-k unit span two words (oracle/gptq.py _bit_slots)
    return b


# ----------------------------------------------------------------------------------------------- decode (gptq_decode.cu)
def dec_plan(problems, m, mode, sm):
    """dec_run, gptq_decode.cu:440-477.  problems: [(k, n, kw)]."""
    colblocks = sum(_cdiv(n, DEC_COLS) for _, n, _ in problems)
    nblk_max = max(_cdiv(k, DEC_BLOCK_K) for k, _, _ in problems)
    nbk = 1 if m <= 8 else (2 if m <= 16 else 4)
    per_sm = ((mode >> 4) & 15) or DEC_DEFAULT_PER_SM
    want = max(1, min(_cdiv(sm * per_sm, colblocks), nblk_max))
    s = _cdiv(nblk_max, want)
    smax = {1: 8, 2: 4, 4: 2}[nbk]
    capped = s > smax
    s = min(s, smax)
    return dict(colblocks=colblocks, nblk_max=nblk_max, nbk=nbk, mt=8 * nbk, S=s, capped=capped,
                slices=_cdiv(nblk_max, s), per_sm=per_sm)


def dec_branches(problems, m, mode, sm, static_flag=False, f16=False):
    p = dec_plan(problems, m, mode, sm)
    s, mt = p["S"], p["mt"]
    b = {f"dec.nbk{p['nbk']}"}
    if m > mt:
        b.add("dec.mpass")  # gptq_decode.cu:208, reached through forced impl 1 (M > 32)
    if p["capped"]:
        b.add("dec.smax")
    if p["nblk_max"] % s:
        b.add("dec.short_slice")
    if (mode >> 4) & 15:
        b.add("dec.per_sm")
    slab, pdl, prefetch = bool(mode & 1), bool(mode & 2), bool(mode & 4)
    static = bool(mode & 8) or static_flag
    nbs = []
    for k, n, kw in problems:
        nblk = _cdiv(k, DEC_BLOCK_K)
        for y in range(p["slices"]):
            b0 = y * s
            if b0 >= nblk:
                b.add("dec.batch.short_k")  # gptq_decode.cu:116
                continue
            nbs.append(min(b0 + s, nblk) - b0)
        if slab:
            if nblk * (DEC_BLOCK_K // 8) > kw:
                b.add("dec.slab.zero_fill")  # gptq_decode.cu:162-165
            if n % DEC_COLS:
                b.add("dec.slab.n_tail")  # gptq_decode.cu:158
    if 1 in nbs:
        b.add("dec.nb1")
    if slab:
        b.add("dec.slab")
        if m % mt:
            b.add("dec.slab.trow_alias")  # x_rows < MT in some pass, gptq_decode.cu:287
    else:
        b.add("dec.reg")
        if prefetch and any(nb > 2 for nb in nbs):
            b.add("dec.prefetch")  # gptq_decode.cu:170-185
    b.add(("dec.wait.static" if static else "dec.wait.strict") if pdl else "dec.no_pdl")
    if len(problems) > 1:
        b.add("dec.batch")
        if len({n for _, n, _ in problems}) > 1:
            b.add("dec.batch.diff_n")
    if f16:
        b.add("dec.f16")
        if p["slices"] >= 4:
            b.add("dec.f16.unroll4")  # gptq_decode.cu:396
        if p["slices"] % 4:
            b.add("dec.f16.rem")  # gptq_decode.cu:401
    return b


# ----------------------------------------------------------------------------------------------- wgmma prefill (gptq_tc.cu)
def tc_live_a_only(n):
    """Some consumer thread of the last feature tile has na = n0 + f0 < N <= nb = na + 8 (gptq_tc.cu:176-178):
    f0 = 64 a + 16 b + l (l < 8), so with r = N % 128 some f0 in [r - 8, r - 1] has l < 8 iff r % 16 != 0."""
    r = n % WG_FEAT
    return r != 0 and r % 16 != 0


def tc_branches(m, k, n, kw, gs, f16=False, bias=True):
    num_kb = _cdiv(k, WG_BK)
    b = {"tc.f16_out" if f16 else "tc.f32"}
    if f16:
        b.add("tc.f16_out.bias" if bias else "tc.f16_out.nobias")
    if k % WG_BK:
        b.add("tc.k64_tail")  # the TMA zero-fills the last stage
    if num_kb % 2:
        b.add("tc.odd_kb")  # gptq_tc.cu:219: fold on the last stage
    if num_kb > TC_STAGES:
        b.add("tc.ring_wrap")
    if num_kb > 2 * TC_STAGES:
        b.add("tc.ring_wrap2")
    if m % WG_TOK:
        b.add("tc.m_tail")
    if n % WG_FEAT:
        b.add("tc.n_tail")
    if tc_live_a_only(n):
        b.add("tc.live_a_only")
    if gs != TC_GROUP_K:
        b.add("tc.gq_ne_g")  # gptq_tc.cu:187
    if kw > _cdiv(k, 8):
        b.add("tc.kw_extra")
    return b


def zero_probe(scales, zeros):
    """gptq_zero_probe_kernel, gptq_tc.cu:125-134, on numpy fp32 arrays: the set of reasons the integer-zero epilogue is
    refused (empty: integer zero points)."""
    import numpy as np

    s = np.asarray(scales, np.float32).reshape(-1)
    z = np.asarray(zeros, np.float32).reshape(-1)
    with np.errstate(all="ignore"):
        zi = np.rint(z / s).astype(np.float32)
        resid = np.abs(z.astype(np.float64) - zi.astype(np.float64) * s.astype(np.float64))
        tol = np.abs(z.astype(np.float64)) * 2.0 ** -20 + 1e-30
    out = set()
    if (s == 0).any():
        out.add("tc.general.scale0")
    fin = np.isfinite(zi) & (s != 0)
    if (fin & (np.abs(zi) > 1024)).any():
        out.add("tc.general.big_zero")
    if (fin & (np.abs(zi) <= 1024) & (resid > tol)).any():
        out.add("tc.general.fractional")
    return out


def split_need_lo(x):
    """gptq_split_kernel, gptq_tc.cu:56-89, with the exponent clamped at -126: does some row-scaled element keep a non-zero
    fp16 low part?  x: [M, K] fp32."""
    import numpy as np

    x = np.asarray(x, np.float32)
    amax = np.max(np.where(np.isnan(x), 0, np.abs(x)), axis=1)
    e = np.zeros(x.shape[0], np.int64)
    ok = (amax > 0) & np.isfinite(amax)
    e[ok] = np.maximum(np.frexp(amax[ok])[1] - 1 - 14, -126)
    with np.errstate(all="ignore"):
        v = (x * np.exp2(-e.astype(np.float64))[:, None].astype(np.float32)).astype(np.float32)
        lo = (v - v.astype(np.float16).astype(np.float32)).astype(np.float16)
    return bool(np.any((lo != 0) | np.isnan(lo)))


def split_row_kinds(x):
    """The data edges of gptq_split_kernel a row of x reaches (tests mark them (data))."""
    import numpy as np

    kinds = set()
    for r in np.asarray(x, np.float32):
        a = np.abs(r)
        if not np.isfinite(r).all():
            kinds.add("split.nonfinite_row")
            continue
        amax = a.max()
        if amax == 0:
            kinds.add("split.zero_row")
        elif amax < 2.0 ** -126:
            kinds.add("split.subnormal_row")
        elif amax < 2.0 ** -113:
            kinds.add("split.tiny_row")
    return kinds


# ----------------------------------------------------------------------------------------------- fp16 linear (gptq.cu)
def f16_branches(m, k, n, kw, gs, state, bias, sm, mode=DEC_DEFAULT_MODE, static=False):
    """sb200_gptq4_linear_f16_ex, gptq.cu:171-208."""
    b = set() if bias else {"f16.null_bias"}
    if m >= F16_TC_MIN_M and tc_refusal(k, n, gs) is None:
        return b | {"f16.tc"} | tc_branches(m, k, n, kw, gs, f16=True, bias=bias)
    if state and m <= F16_SINGLE_MAX_M and decode_supported(n) and n <= F16_STATE_BYTES // 4 * 128:
        return b | {"f16.single"} | dec_branches([(k, n, kw)], m, mode, sm, static_flag=static, f16=True)
    if m >= F16_TC_MIN_M:
        b.add("f16.staged.unsupported")
    elif m > F16_SINGLE_MAX_M:
        b.add("f16.staged.mid")
    else:
        b.add("f16.staged.no_state" if not state else "f16.staged.decode_unsupported")
    kernel, d = dispatch(m, k, n, gs, 0)
    b |= d
    if kernel == "tc":
        b |= tc_branches(m, k, n, kw, gs)
    elif kernel == "decode":
        b |= dec_branches([(k, n, kw)], m, mode, sm, static_flag=True)
    else:
        b |= simt_branches(4, m, k, n, kw, sm)
    return b


# ----------------------------------------------------------------------------------------------- input gradient
def dgrad_simt_plan(m, k, n):
    """simt_plan, gptq_dgrad.cu:143-156, and the grid of launch_simt, :167-169 (the workspace sizes are not restated).
    grid = (32-k units, M tiles capped at 65535, N slices); m_passes: the M tiles the busiest CTA walks.  The kernel
    forms its own tile count, ceil(M / MT), in 64 bits (gptq_dgrad.cu:71), so this m_tiles, which Python cannot
    overflow, is the kernel's for every M < 2^31."""
    mt = 1 if m == 1 else (2 if m == 2 else 4)
    m_tiles = _cdiv(m, mt)
    base = _cdiv(k, DG_UNIT_K) * m_tiles
    s = _cdiv(DG_TARGET_CTAS, base)
    s_max = _cdiv(n, 4 * DG_COLS)
    s = max(1, min(s, s_max))
    slice_n = _cdiv(_cdiv(n, s), DG_COLS) * DG_COLS
    slices = _cdiv(n, slice_n)
    grid = (_cdiv(k, DG_UNIT_K), min(m_tiles, DG_MAX_GRID_Y), slices)
    return dict(mt=mt, slice_n=slice_n, slices=slices, m_tiles=m_tiles, grid=grid, m_passes=_cdiv(m_tiles, grid[1]))


def dgrad_tc_ok(bits, k, n, gs, go_off=0):
    """gptq.cu:243 and gptq_dgrad_tc_supported / tc_shape_ok, gptq_dgrad.cu:360-378 (workspace given)."""
    return bits == 4 and n % 8 == 0 and k % 4 == 0 and (gs % 128 == 0 or gs == k) and _a16(go_off)


def dgrad_branches(bits, m, k, n, kw, gs, impl, go_off=0):
    """sb200_gptq_matmul_dgrad, gptq.cu:235-255, and the two launchers of gptq_dgrad.cu."""
    ok = dgrad_tc_ok(bits, k, n, gs, go_off)
    if impl == 2 and not ok:
        return {"dg.impl2.error"}
    use_tc = impl == 2 or (impl == 0 and ok and m >= DG_TC_MIN_M)
    if impl == 0:
        b = {"dg.auto.tc"} if use_tc else {"dg.auto.small_m" if ok else "dg.auto.unsupported"}
    else:
        b = {f"dg.impl{impl}"}
    if use_tc:
        b.add("dg.tc")
        num_nb = _cdiv(n, WG_BK)
        if kw % 8:
            b.add("dg.tc.kw_tail")  # dgrad_repack_kernel, gptq_dgrad.cu:191
        if n % 64:
            b.add("dg.tc.n_tail")  # repack and table padding of the last 64-n stage
        if num_nb > DG_STAGES:
            b.add("dg.tc.ring_wrap")  # gptq_dgrad.cu:294, 323: stage reuse with alternating parity
        if num_nb > 2 * DG_STAGES:
            b.add("dg.tc.ring_wrap2")
        if num_nb > DG_CHUNK:
            b.add("dg.tc.chunk_restart")  # gptq_dgrad.cu:287-327
            if num_nb % DG_CHUNK == 0:
                b.add("dg.tc.chunk_exact")
        if gs == k and k % 128:
            b.add("dg.tc.one_group_k128")
        if m % WG_TOK:
            b.add("dg.tc.m_tail")
        if k % WG_FEAT:
            b.add("dg.tc.k_tail")
        return b
    p = dgrad_simt_plan(m, k, n)
    b |= {f"dg.simt.b{bits}", f"dg.simt.mt{p['mt']}", "dg.simt.slices" if p["slices"] > 1 else "dg.simt.one_slice"}
    if k % DG_UNIT_K:
        b.add("dg.simt.k_tail")  # gptq_dgrad.cu:109
    if p["m_tiles"] > 1:
        b.add("dg.simt.m_tiles")
    if p["m_passes"] > 1:
        b.add("dg.simt.m_loop")  # gptq_dgrad.cu:72: gridDim.y is capped, a CTA walks several M tiles
    return b


def dgrad_table_c(scales, zeros):
    """dgrad_table_kernel, gptq_dgrad.cu:214-228: the per-group exponent c, before and after its clamp."""
    import numpy as np

    s = np.asarray(scales, np.float32)
    z = np.asarray(zeros, np.float32)
    fma = (15.0 * s.astype(np.float64) - z.astype(np.float64)).astype(np.float32)  # fmaf(15, s, -z): one rounding
    bnd = np.maximum(np.abs(z), np.abs(fma))
    bnd = np.where(np.isfinite(bnd), bnd, 0)
    wmax = bnd.max(axis=0)
    raw = np.where(wmax > 0, 14 - (np.frexp(wmax)[1] - 1), 0)
    return raw, np.clip(raw, -DG_C_CLAMP, DG_C_CLAMP)
