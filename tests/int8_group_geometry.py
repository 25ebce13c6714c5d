"""Plain-Python restatement of the host-side launch plan and the in-kernel branches of the grouped / depthwise
integer-grid conv (csrc/int8_group_conv.cu), in the manner of tests/int8_geometry.py: given a call's shapes and the
byte offset of x from a 16-byte aligned allocation, ``branches`` names the kernel paths the call reaches, so that the
cases of tests/test_gpu_int8_group_branches.py can be tied to the branch each exists for and a CPU test can check that
together they reach every branch.  When the .cu file changes, this file has to follow.  Line numbers are of
csrc/int8_group_conv.cu."""
from int8_conv_ref import _pads, _pair
from int8_geometry import cdiv

THREADS = 256           # :33 kGcThreads
SMEM_MAX = 48 * 1024    # :34 kGcSmemMax
TARGET = 2048           # :35 kGcTarget
MAX_TW = 128            # :36 kGcMaxTW
MAX_MB = 64             # :37 kGcMaxMB
MAX_GRID = 1 << 16      # :38 kGcMaxGrid
MAX_KG = 1 << 17        # kI8MaxK (int8_grid.cuh)


def smem_bytes(mode, cb, ob, c4, tih, tiw, kh, kw):
    """gc_smem_bytes, :344-348."""
    if mode == "depthwise":
        return cb * tih * tiw + 16 + ob * kh * kw
    return 4 * c4 * tih * tiw + 4 * cdiv(ob, 4) * 4 * kh * kw * c4


def plan(n, c, h, w, c_out, groups, kernel, stride=1, padding=0, dilation=1, x_off=0):
    """gc_plan, :357-395, with the output shape of the entry point."""
    (kh, kw), (sh, sw), (dh, dw) = _pair(kernel), _pair(stride), _pair(dilation)
    pt, pb, pl, pr = _pads(padding)
    oh = (h + pt + pb - dh * (kh - 1) - 1) // sh + 1
    ow = (w + pl + pr - dw * (kw - 1) - 1) // sw + 1
    cg, mg = c // groups, c_out // groups
    mode = "depthwise" if cg == 1 else "grouped"
    c4 = cdiv(cg, 4)
    tw = min(ow, MAX_TW)
    cb = mb = 1
    if mode == "depthwise":
        th = max(1, min(oh, TARGET // tw))
        cb = max(1, min(c, TARGET // (th * tw * mg)))
    else:
        mb = min(mg, MAX_MB)
        th = max(1, min(oh, 2 * TARGET // (mb * tw)))
    first = (cb, mb, th, tw)
    while True:
        tih, tiw = (th - 1) * sh + (kh - 1) * dh + 1, (tw - 1) * sw + (kw - 1) * dw + 1
        ob = cb * mg if mode == "depthwise" else mb
        if smem_bytes(mode, cb, ob, c4, tih, tiw, kh, kw) <= SMEM_MAX:
            break
        if mode == "depthwise" and cb > 1:
            cb = (cb + 1) // 2
        elif mode == "grouped" and mb > 1:
            mb = (mb + 1) // 2
        elif th > 1:
            th = (th + 1) // 2
        elif tw > 1:
            tw = (tw + 1) // 2
        else:
            total = n * c_out * oh * ow
            return dict(mode="direct", oh=oh, ow=ow, cg=cg, mg=mg, total=total, grid=min(cdiv(total, THREADS), MAX_GRID))
    if mode == "depthwise":
        mblocks, oblocks = 1, cdiv(c, cb)
    else:
        mblocks = cdiv(mg, ob)
        oblocks = groups * mblocks
    ctas = n * oblocks * cdiv(oh, th) * cdiv(ow, tw)
    return dict(mode=mode, oh=oh, ow=ow, cg=cg, mg=mg, c4=c4, cb=cb, ob=ob, th=th, tw=tw, tih=tih, tiw=tiw,
                mblocks=mblocks, oblocks=oblocks, ctas=ctas, grid=min(ctas, MAX_GRID), shrunk=(cb, mb, th, tw) != first,
                vec=w % 4 == 0 and x_off % 16 == 0)


def branches(n, c, h, w, c_out, groups, kernel, stride=1, padding=0, dilation=1, x_off=0, bias=True, nan=False):
    p = plan(n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off)
    (kh, kw), (sh, sw), (dh, dw) = _pair(kernel), _pair(stride), _pair(dilation)
    pt, pb, pl, pr = _pads(padding)
    b = {"path." + p["mode"], "bias" if bias else "no_bias"}  # :64
    if nan:
        b.add("nan.rescan")  # :280 / :324 a CTA whose tile holds a NaN re-reads each window
    # a window reaching into the padding: :109 / :127 (staged), :173 (direct)
    pad_h = any(not 0 <= o * sh - pt + t * dh < h for o in range(p["oh"]) for t in range(kh))
    pad_w = any(not 0 <= o * sw - pl + t * dw < w for o in range(p["ow"]) for t in range(kw))
    if pad_h or pad_w:
        b.add("pad_taps")
    if p["mode"] == "direct":
        if cdiv(p["total"], THREADS) > MAX_GRID:
            b.add("grid.loop")  # :159
        return b
    b.add("load." + ("vec" if p["vec"] else "scalar"))  # :94, :392
    if p["ctas"] > MAX_GRID:
        b.add("grid.loop")  # :187
    if p["oh"] % p["th"]:
        b.add("tile.partial_h")  # :278 / :323
    if p["ow"] % p["tw"]:
        b.add("tile.partial_w")
    if p["shrunk"]:
        b.add("tile.shrunk")  # :376-379 the first tile did not fit kGcSmemMax
    if p["mode"] == "depthwise":
        if c % p["cb"]:
            b.add("dw.cb_partial")  # :102 channels past C stage 0
        if p["mg"] > 1:
            b.add("dw.multiplier")
    else:
        if p["cg"] % 4:
            b.add("grp.c4_pad")  # :102 channels past C_g stage 0
        if p["mg"] % p["ob"]:
            b.add("grp.mb_partial")
        if any(min(p["ob"], p["mg"] - i * p["ob"]) % 4 for i in range(p["mblocks"])):
            b.add("grp.quad_partial")  # :328
    return b


REQUIRED = {
    "path.depthwise", "path.grouped", "path.direct", "bias", "no_bias", "nan.rescan", "pad_taps", "load.vec",
    "load.scalar", "grid.loop", "tile.partial_h", "tile.partial_w", "tile.shrunk", "dw.cb_partial", "dw.multiplier",
    "grp.c4_pad", "grp.mb_partial", "grp.quad_partial",
}
