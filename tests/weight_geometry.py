"""Plain-Python restatement of the host-side launch geometry of the weight-side kernels: the one-launch multi-tensor
QDQ, structured pruning masks and the MinMax qparams table (csrc/multi.cu), PACT's clamp backward (multi.cu), AdaRound
(csrc/adaround.cu), DoReFa (csrc/dorefa.cu) and the mask helpers of csrc/qdq.cu.

Test infrastructure only, in the manner of tests/qdq_geometry.py and tests/observe_geometry.py: given a shape, the
pointer offsets and the SM count it names the kernel bodies and loops one call reaches, so that the cases in
tests/test_gpu_weight_branches.py can be tied to the branch each exists for, and a CPU test can check that together they
reach every branch.  It is not a second dispatcher; when the formulas in the .cu files change, this file has to follow
(the GPU cases re-check their branches with the real SM count, so a stale restatement fails loudly).

Offsets are in elements from a 16-byte aligned allocation: floats for float buffers, bytes for uint8 masks.
"""
import numpy as np

SM_COUNT_H100 = 132

MULTI_THREADS = 256        # multi.cu:28 kMultiThreads
MULTI_CTAS_PER_SM = 8      # multi.cu:303
MULTI_MAX_TENSORS = 4096   # multi.cu:220
ROWS_CTAS_PER_SM = 8       # multi.cu:293
CLAMP_THREADS = 256        # multi.cu:282
CLAMP_CTAS_PER_SM = 4      # multi.cu:205
CLAMP_FLUSH_ITERS = 64     # multi.cu:180
QPARAMS_THREADS = 128      # multi.cu:135, 266
CHUNK_THREADS = 256        # adaround.cu:19, dorefa.cu:19 kThreads
CHUNK = CHUNK_THREADS * 4  # adaround.cu:93, dorefa.cu:70 kChunk
CHUNK_CTAS_PER_SM = 8      # adaround.cu:143, dorefa.cu:108, 130
QDQ_THREADS = 256          # qdq.cu:27 kThreads
QDQ_UNROLL = 4             # qdq.cu:28 kUnroll
QDQ_CTAS_PER_SM = 4        # qdq.cu:29 kCtasPerSm


def _cdiv(a, b):
    return (a + b - 1) // b


def _a16(off):
    """A float buffer `off` floats into a 16-byte aligned allocation is 16-byte aligned."""
    return off % 4 == 0


# ----------------------------------------------------------------------------------------------- multi-tensor QDQ
def multi_launch(total_rows, sm):
    """sb200_qdq_multi_run, multi.cu:300-309: one warp per row, 8 warps per CTA, at most 8 CTAs per SM."""
    want = _cdiv(total_rows, MULTI_THREADS // 32)
    ctas = min(want, sm * MULTI_CTAS_PER_SM)
    warps = ctas * (MULTI_THREADS // 32)
    return dict(ctas=ctas, capped=want > ctas, warps=warps, rows_per_warp=_cdiv(total_rows, warps))


def multi_row_aligned(inner, x_off, out_off, mask_off):
    """The per-row predicate of qdq_multi_kernel, multi.cu:89-91 (mask_off None: no mask).  inner % 4 == 0 keeps every
    row on the alignment of the tensor's base, so the predicate is the same for all rows of a tensor."""
    return inner % 4 == 0 and _a16(x_off) and _a16(out_off) and (mask_off is None or mask_off % 4 == 0)


def multi_branches(tensors, sm):
    """tensors: [(outer, channels, inner, x_off, out_off, mask_off or None)] in plan order."""
    b = set()
    rows = [o * c for o, c, *_ in tensors]
    begins = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    total = int(begins[-1])
    g = multi_launch(total, sm)
    if g["capped"]:
        b.add("multi.cap")
    for outer, c, inner, x_off, out_off, mask_off in tensors:
        if outer > 1 and c > 1:
            b.add("multi.channels.cycle")  # multi.cu:80 r % channels wraps
        if multi_row_aligned(inner, x_off, out_off, mask_off):
            nv = inner // 4
            b.add("multi.aligned.mask" if mask_off is not None else "multi.aligned.nomask")
            if nv > 32:
                b.add("multi.aligned.two")  # multi.cu:39, 53-56: the second float4 half
            if nv % 64:
                b.add("multi.aligned.half")  # a lane whose i + 32 >= nv stores one float4 only
        else:
            b.add("multi.scalar.mask" if mask_off is not None else "multi.scalar.nomask")
            if inner % 4:
                b.add("multi.scalar.inner_odd")
            elif not _a16(x_off):
                b.add("multi.scalar.x_misaligned")
            elif not _a16(out_off):
                b.add("multi.scalar.out_misaligned")
            else:
                b.add("multi.scalar.mask_misaligned")
    if len(tensors) >= 2048:
        b.add("multi.smem_table_16k")  # (count + 1) * 8 bytes of s_begin, multi.cu:69, 305
    nw = g["warps"]
    if total > nw:
        b.add("multi.stride")  # multi.cu:76: some warp takes a second row
        r = np.arange(total - nw, dtype=np.int64)
        t0 = np.searchsorted(begins, r, side="right") - 1
        t1 = np.searchsorted(begins, r + nw, side="right") - 1
        step = t1 - t0
        if (step >= 1).any():
            b.add("multi.stride.skip1")  # multi.cu:77: the walk resumes from the previous tensor
        if (step >= 2).any():
            b.add("multi.stride.skip2")  # ... and crosses two or more tensors in one stride
    first = np.searchsorted(begins, np.arange(min(nw, total), dtype=np.int64), side="right") - 1
    if (first >= 2).any():
        b.add("multi.walk.entry_skip2")  # a warp's first row lies two or more tensors past tensor 0
    return b


def mask_rows_gt_branches(rows, inner, mask_off, sm):
    """sb200_mask_rows_gt, multi.cu:289-298, and mask_rows_gt_kernel, multi.cu:100-116."""
    b = set()
    want = _cdiv(rows, 8)
    ctas = min(want, sm * ROWS_CTAS_PER_SM)
    if want > ctas:
        b.add("rows.cap")
    if rows > ctas * 8:
        b.add("rows.stride")
    if inner % 4 == 0 and _a16(mask_off):
        b.add("rows.vec")
        if inner // 4 > 32:
            b.add("rows.vec.lane_loop")  # a lane stores more than one float4 per row
    elif inner % 4:
        b.add("rows.scalar.inner_odd")
    else:
        b.add("rows.scalar.misaligned")
    return b


# ----------------------------------------------------------------------------------------------- PACT clamp backward
def clamp_bwd_ctas(n, sm):
    """multi.cu:204-207."""
    c = (n // 4 + 255) // 256
    return max(1, min(c, sm * CLAMP_CTAS_PER_SM))


def clamp_bwd_workspace_bytes(n, sm):
    """sb200_clamp_bwd_workspace_bytes, multi.cu:271: one double2 partial per CTA."""
    return clamp_bwd_ctas(n, sm) * 16 if n > 0 else 0


def clamp_bwd_geometry(n, x_off, gy_off, gx_off, sm):
    ctas = clamp_bwd_ctas(n, sm)
    nt = ctas * CLAMP_THREADS
    vec = _a16(x_off) and _a16(gy_off) and _a16(gx_off)  # multi.cu:173
    nv = n >> 2 if vec else 0
    vec_iters = _cdiv(nv, nt)  # of thread 0, the most any thread runs
    tail = n - 4 * nv
    tail_iters = _cdiv(tail, nt)
    return dict(ctas=ctas, capped=(n // 4 + 255) // 256 > sm * CLAMP_CTAS_PER_SM, nt=nt, vec=vec, nv=nv,
                vec_iters=vec_iters, tail=tail, tail_iters=tail_iters,
                # fp32 additions into a_hi / a_lo that one thread can make before they reach the fp64 d_hi / d_lo
                fp32_terms=4 * min(vec_iters, CLAMP_FLUSH_ITERS) + tail_iters)


def clamp_bwd_branches(n, x_off, gy_off, gx_off, sm, null_hi=False, null_lo=False):
    g = clamp_bwd_geometry(n, x_off, gy_off, gx_off, sm)
    b = set()
    if g["capped"]:
        b.add("clamp.cap")
    if g["vec"]:
        b.add("clamp.vec")
        if g["vec_iters"] > 1:
            b.add("clamp.vec.stride")
        if g["vec_iters"] >= CLAMP_FLUSH_ITERS:
            b.add("clamp.vec.flush")  # multi.cu:180
        if g["vec_iters"] > CLAMP_FLUSH_ITERS:
            b.add("clamp.vec.flush_then_more")
        if g["tail"]:
            b.add("clamp.vec.tail")  # multi.cu:182 after the vector loop
    else:
        b.add("clamp.scalar")
        b.add("clamp.scalar." + ("x" if not _a16(x_off) else "gy" if not _a16(gy_off) else "gx") + "_misaligned")
        if g["tail_iters"] > 1:
            b.add("clamp.scalar.stride")
    if null_hi:
        b.add("clamp.null_hi")
    if null_lo:
        b.add("clamp.null_lo")
    return b


# ----------------------------------------------------------------------------------------------- AdaRound / DoReFa
ADA_OPS = ("hard", "soft", "bwd", "init")  # launch<0..3>, adaround.cu:162-187
DOREFA_OPS = ("norm", "qdq", "bwd")        # launch<0..2>, dorefa.cu:136-153


def chunk_launch(outer, c, inner, sm):
    """launch<OP> of adaround.cu:138-153 and dorefa.cu:103-117: one CTA per chunk of 1024 elements of a row, at most
    8 CTAs per SM."""
    rows = outer * c
    chunks = rows * _cdiv(inner, CHUNK)
    grid = min(chunks, sm * CHUNK_CTAS_PER_SM)
    return dict(rows=rows, chunks=chunks, grid=grid, iters=_cdiv(chunks, grid))


def chunk_vec(family, op, inner, offs):
    """The VEC predicate: adaround.cu:145-146 (x, out, v unless init, gy for bwd), dorefa.cu:110 (x, out, gy for bwd).
    Returns (vec, reason) where reason names the first operand that sends the call to the scalar body."""
    if inner % 4:
        return False, "inner_odd"
    need = ["x", "out"]
    if family == "ada" and op != "init":
        need.append("v")
    if op == "bwd":
        need.append("gy")
    for name in need:
        if not _a16(offs.get(name, 0)):
            return False, name + "_misaligned"
    return True, None


def chunk_branches(family, op, outer, c, inner, offs, sm):
    """family "ada" | "dorefa"; offs: {operand: float offset}."""
    g = chunk_launch(outer, c, inner, sm)
    vec, why = chunk_vec(family, op, inner, offs)
    path = "vec" if vec else "scalar"
    p = f"{family}.{op}.{path}"
    b = {p}
    if not vec:
        b.add(f"{p}.{why}")
    if g["iters"] > 1:
        b.add(f"{p}.stride")  # the chunk loop (adaround.cu:96, dorefa.cu:74) runs more than once in some CTA
    if inner % CHUNK:
        b.add(f"{p}.partial")  # the last chunk of a row has fewer than 1024 elements
        if g["iters"] > 1:
            b.add(f"{p}.stride.partial")
    if outer > 1 and c > 1:
        b.add(f"{family}.{op}.perchannel")  # row % C wraps
    return b


def dorefa_absmax_launch(n, x_off, sm):
    """sb200_dorefa_absmax, dorefa.cu:126-134, and dorefa_absmax_kernel, dorefa.cu:21-48."""
    want = (n // 4 + CHUNK_THREADS - 1) // CHUNK_THREADS + 1
    grid = min(want, sm * CHUNK_CTAS_PER_SM)
    nt = grid * CHUNK_THREADS
    vec = _a16(x_off)
    nv = n >> 2 if vec else 0
    return dict(grid=grid, capped=want > grid, nt=nt, vec=vec, nv=nv, tail=n - 4 * nv)


def dorefa_absmax_branches(n, x_off, sm):
    g = dorefa_absmax_launch(n, x_off, sm)
    b = set()
    if g["capped"]:
        b.add("absmax.cap")
    if g["vec"]:
        b.add("absmax.vec")
        if g["nv"] > g["nt"]:
            b.add("absmax.vec.stride")
        if g["tail"]:
            b.add("absmax.vec.tail")
    else:
        b.add("absmax.scalar")
        if n > g["nt"]:
            b.add("absmax.scalar.stride")
    return b


# ----------------------------------------------------------------------------------------------- qdq.cu mask helpers
def grid_for(nvec, sm):
    """qdq.cu:505-510."""
    want = max(_cdiv(nvec, QDQ_THREADS * QDQ_UNROLL), 1)
    cap = sm * QDQ_CTAS_PER_SM
    return min(want, cap), want > cap


def mask_gt_branches(n, w_off, mask_off, sm):
    """sb200_mask_gt, qdq.cu:707-713 (grid from n >> 2), and mask_gt_kernel, qdq.cu:595-614."""
    grid, capped = grid_for(n >> 2, sm)
    t = grid * QDQ_THREADS
    b = {"gt.cap"} if capped else set()
    if _a16(w_off) and mask_off % 4 == 0:
        b.add("gt.vec")
        if (n >> 2) > t:
            b.add("gt.vec.stride")
        if n % 4:
            b.add("gt.vec.tail")
    else:
        b.add("gt.scalar.w_misaligned" if not _a16(w_off) else "gt.scalar.mask_misaligned")
        if n > t:
            b.add("gt.scalar.stride")
    return b


def mask_apply_f32_branches(n, offs, sm):
    """sb200_mask_apply_f32, qdq.cu:699-705 (grid from n), and mul_f32_kernel, qdq.cu:616-622: scalar only."""
    grid, capped = grid_for(n, sm)
    b = {"mulf.cap"} if capped else set()
    if n > grid * QDQ_THREADS:
        b.add("mulf.stride")
    if any(not _a16(o) for o in offs.values()):
        b.add("mulf.misaligned")
    return b


# ----------------------------------------------------------------------------------------------- MinMax qparams
def qparams_branches(entries):
    """sb200_minmax_qparams_multi, multi.cu:246-269: one 128-thread CTA per entry; entries: [(channels, symmetric)]."""
    b = set()
    for c, sym in entries:
        b.add("qparams.sym" if sym else "qparams.asym")
        b.add("qparams.chan_loop" if _cdiv(c, QPARAMS_THREADS) > 1 else "qparams.one_pass")
    if len(entries) > 1:
        b.add("qparams.multi_entry")
        if len({bool(s) for _, s in entries}) == 2:
            b.add("qparams.mixed_table")
    return b
