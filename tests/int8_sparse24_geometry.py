"""Plain-Python restatement of the launch decisions and in-kernel paths of csrc/int8_sparse24.cu: the 2:4 mask kernel,
the pack kernel and the sparse GEMM.  Test infrastructure only, in the manner of tests/int8_geometry.py: ``branches``
names the paths one call reaches, so that the cases of tests/test_gpu_int8_sparse24_branches.py can be tied to the
branch each exists for and a CPU test can check that together they reach every branch.  None of these kernels is
persistent.  When the .cu file changes, this file has to follow."""

THREADS = 256     # mask and pack kernels: 256 threads, one group / one metadata word each
FEAT = 128        # kSpFeat: features per CTA (two consumer warpgroups x 64)
TOK = 128         # kSpTok: tokens per CTA
BK = 256          # kSpBK: K per stage, four k64 steps
STAGES = 4        # kSpStages
MAX_K = 1 << 17


def cdiv(a, b):
    return (a + b - 1) // b


def mask_branches(rows, cols):
    """sparse24_mask_kernel: one thread per aligned group of 4."""
    groups = rows * cdiv(cols, 4)
    out = {"mask_full_group"} if cols >= 4 else set()
    if cols % 4:
        out.add("mask_tail_group")
    if groups % THREADS:
        out.add("mask_grid_tail")
    return out


def pack_branches(n, k):
    """sparse24_pack_kernel: one thread per metadata word of [ceil(N / 128), K64 / 64, 2, 128]."""
    out = {"pack_word"}
    if n % FEAT:
        out.add("pack_pad_feature")  # features n >= N hold the padding word
    if k % 64:
        out.add("pack_k_tail")       # d = 0 past K inside the last k64 step
    return out


def gemm_plan(m, k, n, out_off=0):
    kb64 = cdiv(k, 64)
    num_kb = cdiv(kb64, 4)
    last_steps = kb64 - 4 * (num_kb - 1)
    return dict(tiles=cdiv(m, TOK) * cdiv(n, FEAT), kb64=kb64, num_kb=num_kb, last_steps=last_steps,
                vec4=n % 4 == 0 and out_off % 16 == 0)


def gemm_branches(m, k, n, out_off=0, bias=True, unsigned_x=False):
    p = gemm_plan(m, k, n, out_off)
    out = {"gemm_store_vec4" if p["vec4"] else "gemm_store_scalar", "gemm_bias" if bias else "gemm_no_bias",
           "gemm_x_unsigned" if unsigned_x else "gemm_x_signed"}
    out.add("gemm_one_stage" if p["num_kb"] == 1 else "gemm_multi_stage")
    if p["num_kb"] > STAGES:
        out.add("gemm_ring_wraps")
    if p["last_steps"] < 4:
        out.add("gemm_pad_steps")      # the last stage's steps past K64 multiply zeros under the padding word
    if p["last_steps"] <= 2:
        out.add("gemm_no_second_box")  # the last stage loads one activation box
    if m % TOK:
        out.add("gemm_partial_m")
    if n % FEAT:
        out.add("gemm_partial_n")
        if n % FEAT <= 64:
            out.add("gemm_idle_warpgroup")  # the second warpgroup's features all lie past N
    return out


REQUIRED = {
    "mask_full_group", "mask_tail_group", "mask_grid_tail",
    "pack_word", "pack_pad_feature", "pack_k_tail", "(data) pack_nan_row", "(data) pack_zero_point",
    "gemm_store_vec4", "gemm_store_scalar", "gemm_bias", "gemm_no_bias", "gemm_x_signed", "gemm_x_unsigned",
    "gemm_one_stage", "gemm_multi_stage", "gemm_ring_wraps", "gemm_pad_steps", "gemm_no_second_box",
    "gemm_partial_m", "gemm_partial_n", "gemm_idle_warpgroup", "(data) gemm_nan_row",
}
