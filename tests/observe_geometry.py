"""Plain-Python restatement of the host-side launch geometry of the observer calibration kernels
(sparsebit_b200/csrc/observe.cu, plus the per-tensor MinMax that qdq.cu runs through its streaming kernel).

Test infrastructure only, in the manner of tests/qdq_geometry.py: given an op, a shape, the pointer offset and the SM
count it names the kernel bodies and loops one call reaches, so that the cases in tests/test_gpu_observe_branches.py can
be tied to the branch each exists for, and a CPU test can check that together they reach every branch.  It is not a
second dispatcher; when the formulas in the .cu files change, this file has to follow (the GPU cases re-check their
intended branch with the real SM count, so a stale restatement fails loudly instead of silently testing something else).

Offsets are in floats from a 16-byte aligned allocation.  Branch ids are dotted strings ("mm.rows.warp.vec.tail_rows",
"sel.hist.p1.ntpr2", ...).
"""
import math

import qdq_geometry as qgeo

SM_COUNT_H100 = qgeo.SM_COUNT_H100

K_THREADS = 256            # observe.cu:18
K_ROW_TILE = 8192          # observe.cu:44
COLS_THREADS = 128         # observe.cu:672
K_MSE_TILE = 8192          # observe.cu:227
K_MSE_CAND_CHUNK = 8       # observe.cu:228
K_MSE_MAX_CAND = 128       # observe.cu:229
K_SEL_SEG_MAX = 65536      # observe.cu:329
K_SEL_SEG_MIN = 16384      # observe.cu:329
K_MOM_TILE = 16384         # observe.cu:584
K_MOM_VALS = 5             # observe.cu:585
SELECT_BINS = 2048         # include/sparsebit_b200.h SB200_SELECT_BINS


def _cdiv(a, b):
    return (a + b - 1) // b


def persistent_grid(tiles, ctas_per_sm, sm):
    """observe.cu:565-569."""
    return min(max(tiles, 1), sm * ctas_per_sm)


def sel_seg(rows, row_len, sm):
    """observe.cu:570-575: halve the segment from 64 Ki while the tiles would give fewer than 6 per SM."""
    seg = K_SEL_SEG_MAX
    while seg > K_SEL_SEG_MIN and rows * _cdiv(row_len, seg) < sm * 6:
        seg >>= 1
    return seg


def strided_finish_threads(tpr, nval):
    """common.cuh:312-319."""
    t = max((tpr + 3) // 4, 1) * nval
    if t > 1024:
        t = (1024 // nval) * nval
    t = max(t, nval)
    return min(_cdiv(t, 32) * 32, 1024)


def finish_branches(tpr, nval, prefix):
    """strided_finish_kernel, observe.cu:630-652: S slices per output; the 4-wide loop (:639-642) runs for slice 0 when
    3 S < tpr."""
    s = strided_finish_threads(tpr, nval) // nval
    out = {f"{prefix}.finish.S1" if s == 1 else f"{prefix}.finish.S_gt1"}
    if 3 * s < tpr:
        out.add(f"{prefix}.finish.unroll4")
    return out


def _span(base_off, length, nthr, prefix):
    """span_minmax (observe.cu:26-41) / the select loads (:379-397) over one span starting `base_off` floats from a
    16-byte boundary: head, 4-wide vector loop, 1-wide vector loop, scalar tail."""
    out = set()
    head = min((4 - base_off % 4) % 4, length)
    nv = (length - head) >> 2
    if head:
        out.add(f"{prefix}.head")
    if nv > 3 * nthr:
        out.add(f"{prefix}.loop4")
    if (length - head) % 4:
        out.add(f"{prefix}.tail")
    return out


# ----------------------------------------------------------------------------------------------- MinMax
def minmax_regime(inner):
    """sb200_observe_minmax_perchannel, observe.cu:667-696."""
    if inner == 1:
        return "cols"
    if inner >= 4096:
        return "cta"
    if inner <= 64:
        return "tiny"
    return "warp"


def minmax_cols(outer, channels, vec, sm):
    """observe.cu:668-679."""
    nq = channels // 4 if vec else channels
    gx = _cdiv(nq, COLS_THREADS)
    want = _cdiv(sm * 8 * (128 // COLS_THREADS), gx)
    limited = "outer" if want > outer else "sm"
    want_y = max(min(want, outer, 65535), 1)
    rpb = _cdiv(outer, want_y)
    return dict(gx=gx, want=want, limited=limited, want_y=want_y, rpb=rpb, grid_y=_cdiv(outer, rpb))


def minmax_blocks(outer, channels, vec, sm):
    """Row ranges [r0, r1) of the column kernel's grid.y blocks."""
    g = minmax_cols(outer, channels, vec, sm)
    return [(r0, min(r0 + g["rpb"], outer)) for r0 in range(0, outer, g["rpb"])]


def minmax_branches(outer, channels, inner, sm, x_off=0):
    b = set()
    rows = outer * channels
    reg = minmax_regime(inner)
    if reg == "cols":
        vec = channels % 4 == 0 and x_off % 4 == 0
        g = minmax_cols(outer, channels, vec, sm)
        b.add(f"mm.cols.gy_{g['limited']}")
        if vec:
            b.add("mm.cols.v4")
            sizes = {r1 - r0 for r0, r1 in minmax_blocks(outer, channels, vec, sm)}
            if any(n >= 4 for n in sizes):
                b.add("mm.cols.v4.loop4")  # observe.cu:149-156
            if any(n % 4 for n in sizes):
                b.add("mm.cols.v4.tail")   # observe.cu:157-160
        else:
            b.add("mm.cols.v1")            # observe.cu:162
        return b
    if reg == "cta":
        tpr = _cdiv(inner, K_ROW_TILE)
        tiles = rows * tpr
        grid = persistent_grid(tiles, 8, sm)
        b.add("mm.rows.cta")
        b.add("mm.rows.cta.tpr1" if tpr == 1 else "mm.rows.cta.tpr_gt1")
        if tpr > 1 and inner % K_ROW_TILE:
            b.add("mm.rows.cta.tpr_gt1.partial")
        if tiles > grid:
            b.add("mm.rows.cta.gridstride")
        for r in range(min(rows, 8)):
            for j in range(tpr):
                ln = min(K_ROW_TILE, inner - j * K_ROW_TILE)
                b |= _span(x_off + r * inner + j * K_ROW_TILE, ln, K_THREADS, "mm.rows.cta.span")
        return b
    if reg == "warp":
        ctas = _cdiv(rows, 4 * (K_THREADS // 32))
        grid = persistent_grid(ctas, 8, sm)
        vec = inner % 4 == 0 and x_off % 4 == 0  # observe.cu:71
        b.add("mm.rows.warp")
        if vec:
            if rows >= 4:
                b.add("mm.rows.warp.vec")            # observe.cu:76-83
            if rows % 4:
                b.add("mm.rows.warp.vec.tail_rows")  # observe.cu:84-88 for the last rows % 4 rows
        else:
            b.add("mm.rows.warp.scalar")             # observe.cu:84-88 for every row
        if rows > grid * (K_THREADS // 32) * 4:
            b.add("mm.rows.warp.gridstride")
        return b
    # tiny
    ctas = _cdiv(rows, 32 * (K_THREADS // 32))
    grid = persistent_grid(ctas, 3, sm)
    b.add("mm.rows.tiny")
    for row0 in range(0, rows, 32):
        cnt = min(32, rows - row0) * inner
        v4 = x_off % 4 == 0 and cnt % 4 == 0 and (row0 * inner) % 4 == 0  # observe.cu:111
        b.add("mm.rows.tiny.stage.v4" if v4 else "mm.rows.tiny.stage.scalar")
    b.add("mm.rows.tiny.rot" if inner % 2 == 0 else "mm.rows.tiny.norot")  # observe.cu:123
    if rows % 32:
        b.add("mm.rows.tiny.last_group_lt32")  # observe.cu:108
    if ctas > grid:
        b.add("mm.rows.tiny.gridstride")
    return b


def minmax_tensor_branches(n, sm, x_off=0):
    """sb200_observe_minmax (qdq.cu:651-656): launch_stream<MODE_TENSOR, STATS> (qdq.cu:429-452), restated in
    qdq_geometry.launch_stream."""
    vec = x_off % 4 == 0 and n >= 4  # qdq.cu:433 (no out, no mask)
    b = {"mm.tensor.v4"} if vec else {"mm.tensor.v1", f"mm.tensor.v1.off{x_off % 4}"}
    if vec and n % 4:
        b.add("mm.tensor.v4.scalar_tail")  # qdq.cu:211-228
    if qgeo.launch_stream(n, 1, n, vec, sm, per_channel=False)["iterations"] > 1:
        b.add("mm.tensor.gridstride")      # qdq.cu:108
    return b


# ----------------------------------------------------------------------------------------------- histogram
def hist_geometry(n, sm):
    """sb200_observe_hist, observe.cu:705-707."""
    blocks = _cdiv(n // 4, K_THREADS * 4)
    grid = persistent_grid(blocks, 8, sm)
    return dict(blocks=blocks, grid=grid, T=grid * K_THREADS)


def hist_branches(n, sm, x_off=0):
    g = hist_geometry(n, sm)
    T = g["T"]
    b = set()
    if x_off % 4:
        b.add("hist.scalar")  # observe.cu:214-216
    else:
        nv = n >> 2
        q, r = divmod(nv, T)
        per_thread = ({q + 1} if r else set()) | ({q} if q and r < T else set())  # vectors each thread reads
        if any(c >= 4 for c in per_thread):
            b.add("hist.v4.loop4")  # observe.cu:202-208
        if any(c % 4 for c in per_thread):
            b.add("hist.v4.loop1")  # observe.cu:209-212
        if n % 4:
            b.add("hist.v4.tail")   # observe.cu:213
    if g["blocks"] > g["grid"]:
        b.add("hist.gridstride")
    return b


# ----------------------------------------------------------------------------------------------- MSE sweep
def mse_tpr(row_len):
    return _cdiv(row_len, K_MSE_TILE)


def mse_workspace_bytes(rows, row_len, ncand):
    """sb200_mse_workspace_bytes, observe.cu:713-717."""
    if rows <= 0 or row_len <= 0 or ncand <= 0:
        return 0
    return rows * mse_tpr(row_len) * ncand * 8


def mse_branches(rows, row_len, ncand, sm, x_off=0):
    """sb200_observe_mse_sweep, observe.cu:719-743 -> mse_sweep_kernel (:246-319) + strided_finish_kernel."""
    tpr = mse_tpr(row_len)
    tiles = rows * tpr
    grid = persistent_grid(tiles, 4, sm)
    b = set()
    kinds = set()
    for tile in range(tiles):
        row, j = divmod(tile, tpr)
        ln = min(K_MSE_TILE, row_len - j * K_MSE_TILE)
        kinds.add("bulk" if (x_off + row * row_len + j * K_MSE_TILE) % 4 == 0 and ln % 4 == 0 else "nonbulk")  # :269
    b |= {f"mse.{k}" for k in kinds}
    if len(kinds) == 2:
        b.add("mse.mixed")
    if tpr > 1:
        b.add("mse.tpr_gt1")
    # a CTA's grid-stride loop (tiles blockIdx.x, + gridDim.x, ...) meets a second row: candidate table reload, :278-286
    if any(len({t // tpr for t in range(blk, tiles, grid)}) > 1 for blk in range(grid)):
        b.add("mse.reload")
    if ncand % K_MSE_CAND_CHUNK:
        b.add("mse.cand_pad")  # :300
    if ncand == 1:
        b.add("mse.ncand1")
    if ncand == K_MSE_MAX_CAND:
        b.add("mse.ncand128")
    b |= finish_branches(tpr, ncand, "mse")
    return b


# ----------------------------------------------------------------------------------------------- radix select
def select_geometry(rows, row_len, sm):
    seg = sel_seg(rows, row_len, sm)
    tiles = rows * _cdiv(row_len, seg)
    return dict(seg=seg, tiles=tiles, grid=persistent_grid(tiles, 6, sm))  # observe.cu:768-770


def select_hist_branches(rows, row_len, ntpr, passes, sm, x_off=0, key_mode=0):
    """sb200_select_hist[_counts] -> select_hist_kernel<PASS> (observe.cu:342-433) for each pass in `passes`."""
    g = select_geometry(rows, row_len, sm)
    seg = g["seg"]
    b = {f"sel.hist.p{p}.ntpr{ntpr}" for p in passes}
    b.add(f"sel.hist.seg{seg}")
    if key_mode:
        b.add("sel.hist.key_mode1")
    if g["tiles"] > g["grid"]:
        b.add("sel.hist.gridstride")
    spr = _cdiv(row_len, seg)
    for r in range(min(rows, 8)):
        for j in range(spr):
            ln = min(seg, row_len - j * seg)
            b |= _span(x_off + r * row_len + j * seg, ln, K_THREADS, "sel.hist")
    return b


def count_sign_branches(rows, row_len, sm):
    """sb200_count_sign, observe.cu:806-815 -> count_sign_kernel (:540-563)."""
    seg = sel_seg(rows, row_len, sm)
    tiles = rows * _cdiv(row_len, seg)
    b = {"count_sign"}
    if rows > 1:
        b.add("count_sign.multirow")
    if tiles > persistent_grid(tiles, 8, sm):
        b.add("count_sign.gridstride")
    return b


def percentile_ranks(neg, pos, total, alpha):
    """percentile_ranks_kernel, observe.cu:522-538: 0-based ranks (min side, max side) and the clamps they hit.
    Python's round() on the double product is half-to-even, i.e. rint."""
    hit = set()
    pn, pp = neg * alpha, pos * alpha
    kmin = _rint(pn)
    if kmin < 1:
        kmin = 1
        hit.add("sel.ranks.kmin_clamp_lo")
    kpos = max(_rint(pp), 0)
    kmax = total - kpos
    if kmax < 1:
        kmax = 1
        hit.add("sel.ranks.kmax_clamp")
    if kmin > total:
        kmin = total
        hit.add("sel.ranks.kmin_clamp_total")
    if (pn != math.floor(pn) and pn - math.floor(pn) == 0.5) or (pp != math.floor(pp) and pp - math.floor(pp) == 0.5):
        hit.add("sel.ranks.tie_half_even")
    return kmin - 1, kmax - 1, hit


def _rint(v):
    """rint() of a double: round half to even (Python's round on a float)."""
    return int(round(v))


# ----------------------------------------------------------------------------------------------- moments
def moments_branches(rows, row_len, centre, sm):
    """sb200_observe_moments, observe.cu:831-848 -> moments_tile_kernel (:587-628) + strided_finish_kernel."""
    tpr = _cdiv(row_len, K_MOM_TILE)
    b = {"moments.centre" if centre else "moments.nocentre"}
    if tpr > 1:
        b.add("moments.tpr_gt1")
    return b | finish_branches(tpr, K_MOM_VALS, "moments")


def moments_workspace_bytes(rows, row_len):
    """observe.cu:826-829."""
    return rows * _cdiv(row_len, K_MOM_TILE) * K_MOM_VALS * 8
