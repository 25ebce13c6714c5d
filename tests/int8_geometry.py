"""Plain-Python restatement of the host-side launch decisions and the in-kernel branches of the integer-grid kernels
(csrc/int8_linear.cu): the row quantizer, the column quantizer, the conv2d lowering, the linear / conv GEMM and the
batched matmul GEMM.

Test infrastructure only, in the manner of tests/gptq_geometry.py: given an entry point, its shapes and the byte
offsets of its pointers from a 16-byte aligned allocation, ``branches`` names the kernel paths one call reaches, so that
the cases of tests/test_gpu_int8_branches.py can be tied to the branch each exists for and a CPU test can check that
together they reach every branch.  None of these kernels is persistent: the SM count plays no part.  When the .cu file
changes, this file has to follow.  Line numbers are of csrc/int8_linear.cu.
"""

ROWS_PER_CTA = 8        # :89 one warp per row, 8 warps (:590 grid (rows + 7) / 8)
ROWS_LANE_K = 16        # :101 16 elements per lane step
ROWS_WARP_K = 32 * 16   # :101 a warp covers 512 K per trip
COL_N = 64              # :133 kColN
COL_K = 128             # :134 kColK
LOW_PIX = 128           # :238 kLowPix
LOW_K = 128             # :239 kLowK
GEMM_ROWS = 128         # :38 kI8Rows
GEMM_FEAT = 128         # :39 kI8Feat
GEMM_BK = 128           # :40 kI8BK
STAGES = 6              # :41 kI8Stages
WG_ROWS = 64            # :438 rows per consumer warpgroup
MAX_K = 1 << 17         # kI8MaxK (int8_grid.cuh)


def cdiv(a, b):
    return (a + b - 1) // b


def padded_k(k):
    """:73 padded_k."""
    return cdiv(k, 16) * 16


def aligned16(off):
    return off % 16 == 0


def conv_out(h, w, kh, kw, stride=1, pad=0, dilation=1):
    """conv_shape, :655-658 (symmetric padding)."""
    return (h + 2 * pad - dilation * (kh - 1) - 1) // stride + 1, (w + 2 * pad - dilation * (kw - 1) - 1) // stride + 1


# ----------------------------------------------------------------------------------------------- launch plans
def rows_plan(rows, k, x_off=0):
    """launch_rows, :587-595."""
    kp = padded_k(k)
    return dict(grid=cdiv(rows, ROWS_PER_CTA), kp=kp, vec=k % 4 == 0 and aligned16(x_off), trips=cdiv(kp, ROWS_WARP_K))


def cols_plan(batch, k, n, x_off=0):
    """launch_cols, :634-643."""
    kp = padded_k(k)
    tiles_n = cdiv(n, COL_N)
    return dict(grid=batch * tiles_n, tiles_n=tiles_n, kp=kp, vec=n % 4 == 0 and aligned16(x_off), chunks=cdiv(kp, COL_K),
                last_kc=kp - (cdiv(kp, COL_K) - 1) * COL_K)


def low_plan(n, c, h, w, kh, kw, stride=1, pad=0, dilation=1):
    """launch_im2col, :692-698, and the ConvDims of conv_shape, :647-669."""
    oh, ow = conv_out(h, w, kh, kw, stride, pad, dilation)
    k = c * kh * kw
    kp = padded_k(k)
    m = n * oh * ow
    return dict(oh=oh, ow=ow, p=oh * ow, m=m, k=k, kp=kp, grid=cdiv(m, LOW_PIX), chunks=cdiv(kp, LOW_K),
                last_kc=kp - (cdiv(kp, LOW_K) - 1) * LOW_K)


def gemm_plan(m, k, n, batch=1):
    """run_gemm :623-624 / sb200_int8_matmul :847, :890; num_kb :410 / :500."""
    tiles_m, tiles_n = cdiv(m, GEMM_ROWS), cdiv(n, GEMM_FEAT)
    return dict(tiles_m=tiles_m, tiles_n=tiles_n, grid=batch * tiles_m * tiles_n, num_kb=cdiv(k, GEMM_BK))


def vec2(n, out_off=0):
    """:889: 8-byte stores when N is even and out is 8-byte aligned."""
    return n % 2 == 0 and out_off % 8 == 0


# ----------------------------------------------------------------------------------------------- branches
def rows_branches(rows, k, x_off=0, per_row=False, pre="rows."):
    p = rows_plan(rows, k, x_off)
    b = {pre + ("per_row" if per_row else "per_tensor")}  # :93
    if p["vec"]:
        b.add(pre + "vec")
        b.add(pre + ("vec.tail" if k % ROWS_LANE_K else "vec.full"))  # :103 c + 16 > K in the last chunk
    else:
        b.add(pre + "scalar")  # :109-111
        if k % 4 == 0:
            b.add(pre + "scalar.misaligned")  # :589 K % 4 == 0 but x is not 16-byte aligned
    b.add(pre + ("trips" if p["trips"] > 1 else "one_trip"))  # :101 Kp > 512
    if p["kp"] < ROWS_WARP_K:
        b.add(pre + "idle_lanes")  # lanes with 16 l >= Kp skip the loop
    if rows % ROWS_PER_CTA:
        b.add(pre + "last_cta_partial")  # :90
    if p["kp"] > k:
        b.add(pre + "kpad")  # :116
    return b


def cols_branches(batch, k, n, x_off=0):
    p = cols_plan(batch, k, n, x_off)
    b = {"cols." + ("vec" if p["vec"] else "scalar")}  # :176 / :181
    if n % COL_N:
        b.add("cols.n_tile_partial")  # :201, :220
    if n % 4:
        b.add("cols.quad_partial")  # :181, :190 some of a thread's 4 columns are past N
    b.add("cols." + ("chunks" if p["chunks"] > 1 else "one_chunk"))  # :166
    if p["last_kc"] < COL_K:
        b.add("cols.short_chunk")  # :171 k groups with 4 kq >= kc are skipped
    if k % 4:
        b.add("cols.k4_partial")  # :176, :190 kk + i >= K inside a group
    if batch > 1:
        b.add("cols.batch")  # :153
    return b


def _taps_out(size, osize, ksize, stride, pad, dilation):
    """For each output position along one axis, how many of its ksize taps fall into the padding."""
    return [sum(not 0 <= o * stride - pad + t * dilation < size for t in range(ksize)) for o in range(osize)]


def low_branches(n, c, h, w, kh, kw, stride=1, pad=0, dilation=1):
    p = low_plan(n, c, h, w, kh, kw, stride, pad, dilation)
    b = set()
    if p["m"] % LOW_PIX:
        b.add("low.tile_partial")  # :260 live, :314
    if n > 1 and p["p"] % LOW_PIX:
        b.add("low.tile_spans_images")  # :263 an image boundary j P (0 < j < n) inside a tile
    b.add("low." + ("chunks" if p["chunks"] > 1 else "one_chunk"))  # :276
    if p["chunks"] > 1 and p["last_kc"] < LOW_K:
        b.add("low.short_chunk")  # :277, :291, :310
    ph = _taps_out(h, p["oh"], kh, stride, pad, dilation)
    pw = _taps_out(w, p["ow"], kw, stride, pad, dilation)
    if any(ph) or any(pw):
        b.add("low.pad_taps")  # :299-302
    if kh in ph or kw in pw:
        b.add("low.window_all_pad")  # an output pixel none of whose taps is in x
    if stride > 1:
        b.add("low.stride")
    if dilation > 1:
        b.add("low.dilation")
    if p["kp"] > p["k"]:
        b.add("low.kpad")  # :281, :296
    return b


def ring_branch(num_kb, pre):
    """The 6-stage ring of i8_produce / i8_consume, :342-375: stage kb % 6, phase (kb / 6) & 1."""
    if num_kb == 1:
        return pre + "kb1"
    if num_kb < STAGES:
        return pre + "kb_lt6"
    if num_kb == STAGES:
        return pre + "kb6"
    if num_kb <= 2 * STAGES:
        return pre + "kb_wrap1"  # a stage is refilled once: phase 1
    return pre + "kb_wrap2"  # the phase returns to 0


def _m_tail(m, pre):
    r = m % GEMM_ROWS
    if r == 0:
        return set()
    # :438 rows 64 wg + ...: warpgroup 1 has no live row when the tail is at most 64 rows
    return {pre + ("m_partial_wg1_idle" if r <= WG_ROWS else "m_partial_both")}


def gemm_branches(m, k, n, bias=True, pre="gemm."):
    p = gemm_plan(m, k, n)
    b = {ring_branch(p["num_kb"], pre), pre + ("bias" if bias else "no_bias")} | _m_tail(m, pre)  # :433, :470
    if n % GEMM_FEAT:
        b.add(pre + "n_partial")  # :429, :462
    if p["tiles_m"] > 1 and p["tiles_n"] > 1:
        b.add(pre + "tiles")  # :409 both tile indices from blockIdx.x
    return b


def linear_branches(m, k, n, x_off=0, bias=True):
    return gemm_branches(m, k, n, bias) | rows_branches(m, k, x_off)


def conv_branches(n, c, h, w, kh, kw, c_out, stride=1, pad=0, dilation=1, bias=True):
    p = low_plan(n, c, h, w, kh, kw, stride, pad, dilation)
    b = gemm_branches(p["m"], p["k"], c_out, bias) | low_branches(n, c, h, w, kh, kw, stride, pad, dilation)
    if n > 1 and p["p"] % GEMM_ROWS:
        b.add("nchw.image_in_tile")  # :447-449 rows of one tile in two images
    if p["p"] < GEMM_ROWS:
        b.add("nchw.p_lt_128")
    return b


def matmul_branches(batch, m, k, n, b_k_major, a_off=0, b_off=0, out_off=0):
    p = gemm_plan(m, k, n, batch)
    b = {ring_branch(p["num_kb"], "mm."), "mm.b_rows" if b_k_major else "mm.b_cols"} | _m_tail(m, "mm.")  # :881-884
    if vec2(n, out_off):
        b.add("mm.store.vec2")  # :555-556
    elif n % 2:
        b.add("mm.store.scalar_odd")  # :558-559
    else:
        b.add("mm.store.scalar_even_misaligned")  # :889 out 4 bytes past an 8-byte boundary
    if n % GEMM_FEAT:
        b.add("mm.n_partial")
    if batch > 1 and (m % GEMM_ROWS or n % GEMM_FEAT):
        b.add("mm.batch_partial")  # :480 3-D maps: a partial tile never reads the next entry
    b |= rows_branches(batch * m, k, a_off)
    b |= rows_branches(batch * n, k, b_off) if b_k_major else cols_branches(batch, k, n, b_off)
    return b


def branches(op, **s):
    """The branches one call of entry point ``op`` reaches."""
    if op == "rows":
        return rows_branches(s["rows"], s["k"], s.get("x_off", 0), s.get("per_row", False))
    if op == "cols":
        return cols_branches(s["batch"], s["k"], s["n"], s.get("x_off", 0))
    if op == "im2col":
        return low_branches(*(s[key] for key in ("n", "c", "h", "w", "kh", "kw")), s.get("stride", 1), s.get("pad", 0),
                            s.get("dilation", 1))
    if op == "linear":
        return linear_branches(s["m"], s["k"], s["n"], s.get("x_off", 0), s.get("bias", True))
    if op == "conv":
        return conv_branches(*(s[key] for key in ("n", "c", "h", "w", "kh", "kw", "c_out")), s.get("stride", 1),
                             s.get("pad", 0), s.get("dilation", 1), s.get("bias", True))
    if op == "matmul":
        return matmul_branches(s["batch"], s["m"], s["k"], s["n"], s["b_k_major"], s.get("a_off", 0), s.get("b_off", 0),
                               s.get("out_off", 0))
    raise ValueError(op)


RING = ("kb1", "kb_lt6", "kb6", "kb_wrap1", "kb_wrap2")
REQUIRED = {
    *("rows." + x for x in ("vec", "vec.full", "vec.tail", "scalar", "scalar.misaligned", "one_trip", "trips", "idle_lanes",
                            "last_cta_partial", "per_tensor", "per_row", "kpad")),
    *("cols." + x for x in ("vec", "scalar", "n_tile_partial", "quad_partial", "one_chunk", "chunks", "short_chunk",
                            "k4_partial", "batch")),
    *("low." + x for x in ("tile_partial", "tile_spans_images", "one_chunk", "chunks", "short_chunk", "pad_taps",
                           "window_all_pad", "stride", "dilation", "kpad")),
    *("gemm." + x for x in RING + ("m_partial_both", "m_partial_wg1_idle", "n_partial", "tiles", "bias", "no_bias",
                                   "nan_row")),
    "nchw.image_in_tile", "nchw.p_lt_128",
    *("mm." + x for x in RING + ("b_rows", "b_cols", "store.vec2", "store.scalar_odd", "store.scalar_even_misaligned",
                                 "batch_partial", "m_partial_both", "m_partial_wg1_idle", "n_partial")),
}
