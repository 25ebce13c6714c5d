"""Plain-Python restatement of the decisions of sb200_int8_sparse24_conv2d (csrc/int8_sparse24.cu): the conv geometry
it lowers, the sparse GEMM's launch decisions (imported from tests/int8_sparse24_geometry.py) and the NCHW epilogue of
int8_sparse24_gemm_kernel<true>.  Test infrastructure only: ``branches`` names the paths one call reaches, so that the
cases of tests/test_gpu_int8_sparse24_conv_branches.py can be tied to the branch each exists for and a CPU test can
check that together they reach every branch.  When the .cu file changes, this file has to follow.

NCHW epilogue: token m = img P + p of out [M / P, N, P] is stored at (img N + n) P + p.  Lane l of a consumer warp
holds tokens 4 l .. 4 l + 3 of the CTA's 128; they leave as one 16-byte store when all four are live, their out
addresses are consecutive (one image, or N = 1) and the first is 16-byte aligned (out itself 16-byte aligned), and as
scalar stores otherwise.  Feature rows past N and tokens past M are not stored."""
from int8_sparse24_geometry import FEAT, TOK, cdiv, gemm_branches, gemm_plan  # noqa: F401


def conv_plan(n, c, h, w, c_out, kh, kw, stride=1, padding=0, dilation=1):
    """M, K, N, P and the (top, bottom, left, right) padding of a conv geometry."""
    sh, sw = (stride, stride) if isinstance(stride, int) else stride
    dh, dw = (dilation, dilation) if isinstance(dilation, int) else dilation
    pad = (padding,) * 4 if isinstance(padding, int) else tuple(padding)
    if len(pad) == 2:
        pad = (pad[0], pad[0], pad[1], pad[1])
    oh = (h + pad[0] + pad[1] - dh * (kh - 1) - 1) // sh + 1
    ow = (w + pad[2] + pad[3] - dw * (kw - 1) - 1) // sw + 1
    return dict(M=n * oh * ow, K=c * kh * kw, N=c_out, P=oh * ow, OH=oh, OW=ow, pad=pad)


def nchw_store_branches(m, n, p, out_off=0):
    """The store decisions of the NCHW epilogue over every tile, lane and feature row."""
    out = set()
    vec4 = out_off % 16 == 0
    for m0 in range(0, m, TOK):
        imgs = {t // p for t in range(m0, min(m, m0 + TOK))}
        out.add("nchw_tile_spans_images" if len(imgs) > 1 else "nchw_tile_in_image")
        for t0 in range(m0, min(m, m0 + TOK), 4):
            live = [t0 + i < m for i in range(4)]
            base = [(t // p) * n * p + t % p for t in range(t0, t0 + 4)]
            run = live[3] and base[3] - base[0] == 3
            for f in range(n):
                vec = vec4 and run and (base[0] + f * p) % 4 == 0
                out.add("nchw_store_vec4" if vec else "nchw_store_scalar")
            if {"nchw_store_vec4", "nchw_store_scalar"} <= out and len(imgs) > 1:
                break
    if p < TOK:
        out.add("nchw_p_below_tile")
    if p == 1:
        out.add("nchw_p_one")
    return out


def branches(geom, out_off=0, bias=True, unsigned_x=False):
    """Every id one sb200_int8_sparse24_conv2d call on ``geom`` (conv_plan's arguments) reaches."""
    g = conv_plan(**geom)
    out = gemm_branches(g["M"], g["K"], g["N"], bias=bias, unsigned_x=unsigned_x)
    out -= {"gemm_store_vec4", "gemm_store_scalar"}  # the row-major epilogue's stores; NCHW has its own
    out |= nchw_store_branches(g["M"], g["N"], g["P"], out_off)
    if any(g["pad"]):
        out.add("conv_pad_taps")
        if unsigned_x:
            out.add("conv_unsigned_pad_taps")  # a padding tap stores rint(zp) - 128
    return out


REQUIRED = {
    "gemm_one_stage", "gemm_multi_stage", "gemm_ring_wraps", "gemm_pad_steps", "gemm_no_second_box",
    "gemm_partial_m", "gemm_partial_n", "gemm_idle_warpgroup", "gemm_bias", "gemm_no_bias", "gemm_x_signed",
    "gemm_x_unsigned",
    "nchw_tile_in_image", "nchw_tile_spans_images", "nchw_p_below_tile", "nchw_p_one", "nchw_store_vec4",
    "nchw_store_scalar",
    "conv_pad_taps", "conv_unsigned_pad_taps", "(data) conv_nan_window",
}
