"""Plain-Python restatement of the launch decisions of the channels-last integer-grid convs, in the manner of
tests/int8_geometry.py and tests/int8_group_geometry.py: the NHWC lowering (launch_im2col_nhwc / nhwc_chunk and
int8_im2col_quantize_nhwc_kernel in csrc/int8_linear.cu) and the NHWC grouped / depthwise kernel (nh_plan and
int8_group_conv_nhwc_kernel in csrc/int8_group_conv.cu).  ``lower_branches`` / ``group_branches`` name the paths a
call reaches, so that the cases of tests/test_gpu_int8_conv_nhwc_branches.py can be tied to the branch each exists for
and a CPU test can check that together they reach every branch.  When the .cu files change, this file has to follow."""
from int8_conv_ref import _pads, _pair
from int8_geometry import cdiv

NH_PIX = 64           # kNhPix: output pixels per lowering CTA
NH_MAX_KC = 640       # kNhMaxKC: K bytes per chunk at most
NH_ROWS_MIN_K = 256   # kNhRowsMinK: a stride-1 unpadded 1x1 with c >= this runs the row quantizer
GC_THREADS = 256      # kGcThreads
GC_SMEM_MAX = 48 * 1024
GC_MAX_GRID = 1 << 16
NH_MAX_QUADS = 16     # kNhMaxQuads
NH_ROUNDS = 4         # kNhRounds


def out_hw(h, w, kernel, stride, padding, dilation):
    (kh, kw), (sh, sw), (dh, dw) = _pair(kernel), _pair(stride), _pair(dilation)
    pt, pb, pl, pr = _pads(padding)
    return (h + pt + pb - dh * (kh - 1) - 1) // sh + 1, (w + pl + pr - dw * (kw - 1) - 1) // sw + 1


def lower_plan(n, c, h, w, kernel, stride=1, padding=0, dilation=1, x_off=0):
    """launch_im2col_nhwc: the row quantizer for a stride-1, unpadded 1 x 1 conv of c >= 256, else the NHWC lowering
    with its chunk kc (nhwc_chunk)."""
    (kh, kw), (sh, sw) = _pair(kernel), _pair(stride)
    oh, ow = out_hw(h, w, kernel, stride, padding, dilation)
    m, k = n * oh * ow, c * kh * kw
    kp = cdiv(k, 16) * 16
    taps = kh * kw
    if (kh, kw) == (1, 1) and (sh, sw) == (1, 1) and all(p == 0 for p in _pads(padding)) and k >= NH_ROWS_MIN_K:
        return dict(path="rows", m=m, k=k, kp=kp, vec=k % 4 == 0 and x_off % 16 == 0)
    cb = 16 * max(1, 8 // taps)
    kc = min(cb * taps, NH_MAX_KC, kp)
    return dict(path="nhwc", m=m, k=k, kp=kp, kc=kc, cb=cb, chunks=cdiv(kp, kc), ctas=cdiv(m, NH_PIX),
                vec=c % 4 == 0 and x_off % 16 == 0)


def lower_branches(n, c, h, w, kernel, stride=1, padding=0, dilation=1, x_off=0, nan=False):
    p = lower_plan(n, c, h, w, kernel, stride, padding, dilation, x_off)
    b = {"lower." + p["path"], "load." + ("vec" if p["vec"] else "scalar")}
    if nan:
        b.add("nan")  # the window holds a NaN: the row's flag
    if p["k"] % 16:
        b.add("kp_tail")  # bytes past K in the last piece are the K padding
    if p["path"] == "rows":
        return b
    (kh, kw), (sh, sw), (dh, dw) = _pair(kernel), _pair(stride), _pair(dilation)
    pt, pb, pl, pr = _pads(padding)
    oh, ow = out_hw(h, w, kernel, stride, padding, dilation)
    if any(not 0 <= o * sh - pt + t * dh < h for o in range(oh) for t in range(kh)) or \
       any(not 0 <= o * sw - pl + t * dw < w for o in range(ow) for t in range(kw)):
        b.add("pad_taps")
    if p["m"] % NH_PIX:
        b.add("m_tail")  # the last CTA has fewer than 64 pixels
    if p["chunks"] > 1:
        b.add("k_chunks")
        if p["kp"] % p["kc"]:
            b.add("k_chunk_tail")  # the last chunk is shorter than kc
    if p["kc"] % (kh * kw) or (p["chunks"] > 1 and p["kc"] < p["cb"] * kh * kw):
        b.add("k_chunk_split")  # a chunk boundary cuts a channel's taps: items skip the bytes outside the chunk
    return b


LOWER_REQUIRED = {"lower.rows", "lower.nhwc", "load.vec", "load.scalar", "nan", "kp_tail", "pad_taps", "m_tail",
                  "k_chunks", "k_chunk_tail", "k_chunk_split"}


def group_plan(n, c, h, w, c_out, groups, kernel, stride=1, padding=0, dilation=1, x_off=0, out_off=0):
    """nh_plan: path, quads per CTA, pixels per CTA, grid."""
    (kh, kw) = _pair(kernel)
    oh, ow = out_hw(h, w, kernel, stride, padding, dilation)
    cg, mg = c // groups, c_out // groups
    c4 = cdiv(cg, 4)
    taps = kh * kw
    mode = "dw" if cg == 1 and mg == 1 else "quad" if mg % 4 == 0 else "any"
    qb = 1
    while qb < NH_MAX_QUADS and 4 * qb < c_out:
        qb *= 2
    first = qb
    if mode != "any":
        while True:
            smem = 4 * taps * qb if mode == "dw" else 16 * qb * taps * c4
            if smem <= GC_SMEM_MAX:
                break
            if qb == 1:
                mode = "any"
                break
            qb //= 2
    m = n * oh * ow
    pix = GC_THREADS // qb * NH_ROUNDS
    pblocks, nblocks = cdiv(m, pix), cdiv(c_out, 4 * qb)
    vec = (c % 4 == 0 if mode == "dw" else cg % 4 == 0) and x_off % 16 == 0
    return dict(mode=mode, oh=oh, ow=ow, cg=cg, mg=mg, c4=c4, qb=qb, shrunk=qb != first, pix=pix, m=m,
                pblocks=pblocks, nblocks=nblocks, ctas=pblocks * nblocks, vec=vec,
                vec_out=c_out % 4 == 0 and out_off % 16 == 0)


def group_branches(n, c, h, w, c_out, groups, kernel, stride=1, padding=0, dilation=1, x_off=0, out_off=0, bias=True,
                   nan=False):
    p = group_plan(n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off, out_off)
    b = {"path." + p["mode"], "bias" if bias else "no_bias", "store." + ("vec" if p["vec_out"] else "scalar")}
    if p["mode"] != "any":
        b.add("load." + ("vec" if p["vec"] else "scalar"))
    if nan:
        b.add("nan")
    (kh, kw), (sh, sw), (dh, dw) = _pair(kernel), _pair(stride), _pair(dilation)
    pt, pb, pl, pr = _pads(padding)
    if any(not 0 <= o * sh - pt + t * dh < h for o in range(p["oh"]) for t in range(kh)) or \
       any(not 0 <= o * sw - pl + t * dw < w for o in range(p["ow"]) for t in range(kw)):
        b.add("pad_taps")
    if p["m"] % p["pix"]:
        b.add("pix_tail")
    if c_out % (4 * p["qb"]):
        b.add("nblock_partial")  # quads past C_out in the last channel block
    if c_out % 4:
        b.add("quad_partial")
    if p["nblocks"] > 1:
        b.add("nblocks")  # more than one channel block: weights staged per block
    if p["ctas"] > GC_MAX_GRID:
        b.add("grid.loop")
    if p["shrunk"]:
        b.add("quads.shrunk")  # the staged weights did not fit kGcSmemMax at the first block
    if p["mode"] == "quad" and p["cg"] % 4:
        b.add("quad.c4_pad")
    return b


GROUP_REQUIRED = {"path.dw", "path.quad", "path.any", "bias", "no_bias", "store.vec", "store.scalar", "load.vec",
                  "load.scalar", "nan", "pad_taps", "pix_tail", "nblock_partial", "quad_partial", "nblocks",
                  "grid.loop", "quads.shrunk", "quad.c4_pad"}
