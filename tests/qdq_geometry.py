"""Plain-Python restatement of the host-side launch geometry of the fake-quant forward (csrc/qdq.cu) and STE
backward (csrc/bwd.cu) kernels.

Test infrastructure only: given an op, a shape, the channel axis, the pointer offsets and the SM count it names the
kernel bodies and loops one call reaches, so that the cases in tests/test_gpu_qdq_branches.py can be tied to the branch
each exists for, and a CPU test can check that together they reach every branch.  It is not a second dispatcher; when
the formulas in the .cu files change, this file has to follow (the GPU cases re-check their intended branch on the real
device, so a stale restatement fails loudly instead of silently testing something else).

Branch ids are dotted strings ("fwd.cols.v4.loop4", "bwd.finish.rows.tpr_gt1.multichannel", ...); a case with
rounding != 0 also reaches "R-1@<id>" for each of them (the ROUNDING = -1 template instantiations).
"""
import numpy as np

SM_COUNT_H100 = 132

# csrc/qdq.cu
K_THREADS = 256          # qdq.cu:25
K_UNROLL = 4             # qdq.cu:26
K_CTAS_PER_SM = 4        # qdq.cu:27
K_TMA_TILE = 4096        # qdq.cu:246
K_TAB_MAX_CHANNELS = 2048  # qdq.cu:443 (use_tab)
COLS_THREADS = 128       # qdq.cu:480

# csrc/bwd.cu
BWD_THREADS = 256        # bwd.cu:25
BWD_K_TILE = 8192        # bwd.cu:26
BWD_CTA_TILE_MIN_INNER = 1024  # bwd.cu:396
BWD_CTAS_PER_SM = 8      # bwd.cu:398
BWD_DRAIN_ROWS = 256     # bwd.cu:242, 262, 281


def channel_geometry(shape, ch_axis):
    """[outer, C, inner] (ops.channel_geometry)."""
    ch_axis = ch_axis % len(shape)
    outer = int(np.prod(shape[:ch_axis], dtype=np.int64))
    inner = int(np.prod(shape[ch_axis + 1:], dtype=np.int64))
    return outer, int(shape[ch_axis]), inner


def _cdiv(a, b):
    return (a + b - 1) // b


# ----------------------------------------------------------------------------------------------- forward
def grid_for(nvec, sm):
    """qdq.cu:421-426."""
    want = max(_cdiv(nvec, K_THREADS * K_UNROLL), 1)
    return min(want, sm * K_CTAS_PER_SM)


def launch_stream(n, channels, inner, vec, sm, per_channel):
    """launch_stream, qdq.cu:429-444: grid, per-step cursor increments, table choice and the number of iterations of
    the grid-stride loop (qdq.cu:108)."""
    nvec = n >> 2 if vec else n
    grid = grid_for(nvec, sm)
    step = grid * K_THREADS * (4 if vec else 1)
    inner = max(inner, 1)
    channels = max(channels, 1)
    return dict(nvec=nvec, grid=grid, step=step, dpos=step % inner, dc=(step // inner) % channels,
                use_tab=bool(per_channel and channels <= K_TAB_MAX_CHANNELS),
                iterations=_cdiv(nvec, K_UNROLL * grid * K_THREADS))


def launch_cols(outer, channels, vec, sm):
    """launch_cols, qdq.cu:468-478."""
    nq = channels // 4 if vec else channels
    gx = _cdiv(nq, COLS_THREADS)
    want_y = min(_cdiv(sm * 8, gx), outer, 65535)
    want_y = max(want_y, 1)
    rpb = _cdiv(outer, want_y)
    return dict(gx=gx, want_y=want_y, rpb=rpb, grid_y=_cdiv(outer, rpb))


def use_tma(n, x_off, out_off, variant):
    """use_tma, qdq.cu:359-366 (offsets in floats from a 16-byte aligned allocation)."""
    if variant == 1:
        return False
    ok = x_off % 4 == 0 and out_off % 4 == 0 and n >= 4 * K_TMA_TILE
    return ok if variant == 2 else False


def _tab_vec4_subbranches(n, inner):
    """Which of the three table paths (qdq.cu:142, 147, 156) some warp of the VEC = 4 body takes.  A warp holds 32
    consecutive vectors (T is a multiple of 32 and every lane steps by T); lanes past the end do not vote."""
    if inner < 4:
        return {"inner_lt4"}
    if inner % 4 == 0:
        return {"nocross"}
    nvec = n >> 2
    e = np.arange(nvec, dtype=np.int64) * 4
    cross = (e % inner) + 3 >= inner
    nwin = _cdiv(nvec, 32)
    anyc = np.concatenate([cross, np.zeros(nwin * 32 - nvec, bool)]).reshape(nwin, 32).any(axis=1)
    out = set()
    if anyc.any():
        out.add("cross1")
    if not anyc.all():
        out.add("nocross")
    return out


def fwd_branches(op, shape, ch_axis, sm, x_off=0, out_off=0, mask_off=0, variant=0):
    """op: "perchannel" (sb200_qdq_perchannel_fwd), "mask" (sb200_mask_apply_qdq_perchannel), "pertensor" /
    "stats" (sb200_qdq_pertensor_fwd / sb200_qdq_stats_pertensor_fwd).  Offsets: floats for x / out, bytes for the
    mask, from 16-byte aligned allocations."""
    b = set()
    n = int(np.prod(shape, dtype=np.int64))
    if op in ("pertensor", "stats"):
        if use_tma(n, x_off, out_off, variant):  # qdq.cu:566-567
            b.add("fwd.tma")
            if n % 4:
                b.add("fwd.tma.tail")  # qdq.cu:326-330
            return b
        outer, channels, inner, per_channel, mask = 1, 1, n, False, False
    else:
        outer, channels, inner = channel_geometry(shape, ch_axis)
        mask = op == "mask"
        per_channel = channels != 1  # perchannel_fwd, qdq.cu:497-500
        if per_channel and not mask and inner == 1:  # qdq.cu:501-503
            vec = channels % 4 == 0 and x_off % 4 == 0 and out_off % 4 == 0
            g = launch_cols(outer, channels, vec, sm)
            if vec:
                b.add("fwd.cols.v4")
                full, last = g["rpb"], outer - (g["grid_y"] - 1) * g["rpb"]
                if full >= 4 or last >= 4:
                    b.add("fwd.cols.v4.loop4")  # qdq.cu:393-405
                if full % 4 or last % 4:
                    b.add("fwd.cols.v4.tail")   # qdq.cu:406-413
            else:
                b.add("fwd.cols.v1")            # qdq.cu:415-416
            return b
    # launch_stream, qdq.cu:433-434
    vec = x_off % 4 == 0 and out_off % 4 == 0 and n >= 4 and (not mask or mask_off % 4 == 0)
    v = "v4" if vec else "v1"
    kind = "mask" if mask else ("chan" if per_channel else "tensor")
    b.add(f"fwd.{kind}.{v}")
    if vec and n % 4:
        b.add(f"fwd.{kind}.v4.scalar_tail")  # qdq.cu:211-228
    if not per_channel:
        return b
    g = launch_stream(n, channels, inner, vec, sm, per_channel=True)
    tab = "tab" if g["use_tab"] else "notab"
    if mask:
        b.add(f"fwd.mask.{tab}")
        if inner == 1:
            b.add("fwd.mask.inner1")  # the mask path never takes the cols kernel
    b.add(f"fwd.chan.{tab}.{v}")
    if g["iterations"] > 1:
        b.add(f"fwd.chan.{tab}.{v}.carry")  # cursor update qdq.cu:198-206 carried across grid-stride iterations
    if g["use_tab"]:
        if vec:
            for s in _tab_vec4_subbranches(n, inner):
                b.add(f"fwd.chan.tab.v4.{s}")  # qdq.cu:142-169
    elif vec:
        if inner >= 4 and inner % 4 == 0:
            b.add("fwd.chan.notab.v4.fast")   # qdq.cu:170-176 only
        else:
            b.add("fwd.chan.notab.v4.straddle")  # qdq.cu:177-191
            if inner > 4:
                b.add("fwd.chan.notab.v4.fast")
            if inner < 4:
                b.add("fwd.chan.notab.v4.straddle.inner_lt4")  # the while loop crosses a whole row, qdq.cu:182-185
    return b


# ----------------------------------------------------------------------------------------------- backward
def cols_block_threads(channels):
    """bwd.cu:329-333."""
    nq = channels // 4 if channels % 4 == 0 else channels
    w128 = _cdiv(nq, 128) * 128 - nq
    w64 = _cdiv(nq, 64) * 64 - nq
    return 64 if w64 < w128 else 128


def cols_row_blocks(outer, channels, sm):
    """bwd.cu:334-343: the number of row blocks (grid.y); rows per block is ceil(outer / that)."""
    bt = cols_block_threads(channels)
    gx = _cdiv(channels // 4 if channels % 4 == 0 else channels, bt)
    want = min(_cdiv(sm * 8 * (128 // bt), gx), outer, 65535)
    want = max(want, 1)
    rpb = _cdiv(outer, want)
    return _cdiv(outer, rpb)


def bwd_cols_row_loop(rows, vec):
    """Which loops of bwd_cols_kernel (bwd.cu:219-283) a row block of `rows` rows runs, including the fp32 -> fp64
    drain of the partial sums every 256 rows."""
    out = set()
    if not vec:
        if rows >= BWD_DRAIN_ROWS:
            out.add("drain")  # bwd.cu:281
        return out
    k = 0
    r4 = rows // 4
    if r4:
        out.add("loop4")  # bwd.cu:233-247
    for _ in range(r4):
        k += 4
        if k >= BWD_DRAIN_ROWS:
            out.add("drain")  # bwd.cu:242-246
            k = 0
    if rows % 4 >= 2:
        out.add("loop2")  # bwd.cu:248-267
        k += 2
        if k >= BWD_DRAIN_ROWS:
            out.add("loop2.drain")  # bwd.cu:262-266
    if rows % 2:
        out.add("tail")  # bwd.cu:268-276
    return out


def bwd_ws_bytes(outer, channels, inner, sm):
    """bwd_ws_bytes, bwd.cu:345-350."""
    if outer <= 0 or channels <= 0 or inner <= 0:
        return 0
    if inner == 1 and channels > 1:
        return cols_row_blocks(outer, channels, sm) * channels * 16
    return outer * channels * _cdiv(inner, BWD_K_TILE) * 16


def _span_branches(inner, rows, x_off, gy_off, gx_off, nthr):
    """span_bwd, bwd.cu:50-94, over every tile base (row * inner + j * kTile): scalar path, head, 2x-unrolled
    vector loop."""
    out = set()
    if not (x_off % 4 == gy_off % 4 == gx_off % 4):
        out.add("scalar")  # bwd.cu:56-59
        return out
    tiles = [(r * inner + j * BWD_K_TILE, min(BWD_K_TILE, inner - j * BWD_K_TILE))
             for r in range(min(rows, 8)) for j in range(_cdiv(inner, BWD_K_TILE))]
    for off, ln in tiles:
        head = min((4 - (x_off + off) % 4) % 4, ln)
        if head:
            out.add("head")  # bwd.cu:60-62
        if (ln - head) // 4 > nthr:
            out.add("unroll2")  # bwd.cu:68-82
    return out


def bwd_branches(shape, ch_axis, sm, x_off=0, gy_off=0):
    """sb200_qdq_pertensor_bwd (ch_axis None) / sb200_qdq_perchannel_bwd_ex through bwd_dispatch, bwd.cu:352-412.
    gx is a fresh allocation (ops.qdq_backward), i.e. 16-byte aligned."""
    b = set()
    n = int(np.prod(shape, dtype=np.int64))
    outer, channels, inner = (1, 1, n) if ch_axis is None else channel_geometry(shape, ch_axis)
    if inner == 1 and channels > 1:  # bwd.cu:369
        nb = cols_row_blocks(outer, channels, sm)
        rpb = _cdiv(outer, nb)
        vec = channels % 4 == 0 and x_off % 4 == 0 and gy_off % 4 == 0
        v = "v4" if vec else "v1"
        b.add(f"bwd.cols.{v}")
        b.add(f"bwd.cols.bt{cols_block_threads(channels)}")
        b.add("bwd.finish.cols")  # bwd.cu:294-319
        for rows in {rpb, outer - (nb - 1) * rpb}:
            b |= {f"bwd.cols.{v}.{s}" for s in bwd_cols_row_loop(rows, vec)}
        return b
    rows = outer * channels
    tpr = _cdiv(inner, BWD_K_TILE)
    cta = inner >= BWD_CTA_TILE_MIN_INNER
    kind = "cta" if cta else "warp"
    b.add(f"bwd.rows.{kind}")
    tiles = rows * tpr
    grid = min(max(tiles if cta else _cdiv(tiles, 8), 1), sm * BWD_CTAS_PER_SM)
    slots = grid if cta else grid * BWD_THREADS // 32
    if tiles > slots:
        b.add(f"bwd.rows.{kind}.grid_stride")  # bwd.cu:110
    if inner % BWD_K_TILE == 0 and tpr == 1:
        b.add("bwd.rows.inner_eq_ktile")
    if tpr > 1 and inner % BWD_K_TILE:
        b.add("bwd.rows.partial_last_tile")  # bwd.cu:113
    b |= {f"bwd.span.{s}" for s in _span_branches(inner, rows, x_off, gy_off, 0, BWD_THREADS if cta else 32)}
    if tpr == 1:
        b.add("bwd.finish.rows.tpr1")  # bwd.cu:158-163
    else:
        b.add("bwd.finish.rows.tpr_gt1")  # bwd.cu:164-170
        if channels > 1:
            b.add("bwd.finish.rows.tpr_gt1.multichannel")
    return b


def with_rounding(branches, rounding):
    return set(branches) | ({"R-1@" + x for x in branches} if rounding else set())
