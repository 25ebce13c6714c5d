"""ctypes binding of the C-ABI in ``include/sparsebit_b200.h`` (``csrc/libsparsebit_b200.so``).

There is no CPU fallback: if the shared library is missing, importing any op raises
``SparsebitB200Error`` telling the user to build it (``python -c "import __graft_entry__ as g;
g.build()"`` or ``make -C sparsebit_b200/csrc``).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libsparsebit_b200.so")


class SparsebitB200Error(RuntimeError):
    """Raised for every non-zero status of the native library (the reference raises RuntimeError
    from its pybind modules for the same conditions)."""


c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_vp = ctypes.c_void_p
c_sz = ctypes.c_size_t
c_f = ctypes.c_float
c_d = ctypes.c_double


class Conv2dGeom(ctypes.Structure):
    """``sb200_conv2d_geom``: input [n, c, h, w], kernel kh x kw, stride, dilation, paddings top / bottom / left / right."""
    _fields_ = [(name, ctypes.c_int64) for name in ("n", "c", "h", "w", "kh", "kw", "stride_h", "stride_w", "dilation_h",
                                                    "dilation_w", "pad_top", "pad_bottom", "pad_left", "pad_right")]


c_geom = ctypes.POINTER(Conv2dGeom)

# name -> (restype, argtypes); every symbol include/sparsebit_b200.h declares
PROTOTYPES = {
    "sb200_last_error": (ctypes.c_char_p, []),
    "sb200_version": (c_int, []),
    "sb200_sm_count": (c_int, []),
    "sb200_set_variant": (c_int, [c_int]),
    "sb200_launch_count": (c_i64, []),
    "sb200_qdq_pertensor_fwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int, c_int, c_vp]),
    "sb200_qdq_perchannel_fwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_vp]),
    "sb200_qdq_stats_pertensor_fwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int, c_int, c_vp]),
    "sb200_qdq_pertensor_fwd_host": (c_int, [c_vp, c_f, c_f, c_vp, c_vp, c_i64, c_int, c_int, c_int]),
    "sb200_qdq_pertensor_fwd_host_async": (c_int, [c_vp, c_f, c_f, c_vp, c_vp, c_i64, c_int, c_int, c_int]),
    "sb200_host_sync": (c_int, []),
    "sb200_qdq_perchannel_fwd_host": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_int]),
    "sb200_qdq_bwd_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64]),
    "sb200_qdq_pertensor_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int, c_int, c_vp, c_sz, c_vp]),
    "sb200_qdq_perchannel_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_vp, c_sz, c_vp]),
    "sb200_qdq_perchannel_bwd_ex": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_int, c_vp, c_sz, c_vp]),
    "sb200_clamp_bwd_workspace_bytes": (c_sz, [c_i64]),
    "sb200_clamp_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_sz, c_vp]),
    "sb200_minmax_init": (c_int, [c_vp, c_i64, c_vp]),
    "sb200_observe_minmax": (c_int, [c_vp, c_i64, c_vp, c_vp]),
    "sb200_observe_minmax_perchannel": (c_int, [c_vp, c_i64, c_i64, c_i64, c_vp, c_vp]),
    "sb200_minmax_read": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp]),
    "sb200_observe_hist": (c_int, [c_vp, c_i64, c_vp, c_int, c_vp, c_vp]),
    "sb200_mse_workspace_bytes": (c_sz, [c_i64, c_i64, c_int]),
    "sb200_observe_mse_sweep": (c_int, [c_vp, c_i64, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_sz, c_vp]),
    "sb200_select_init": (c_int, [c_vp, c_vp, c_i64, c_vp, c_vp]),
    "sb200_select_hist": (c_int, [c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_int, c_int, c_vp]),
    "sb200_select_hist_counts": (c_int, [c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_int, c_int, c_vp, c_vp]),
    "sb200_select_scan": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_vp]),
    "sb200_select_read": (c_int, [c_vp, c_i64, c_int, c_vp, c_vp]),
    "sb200_count_sign": (c_int, [c_vp, c_i64, c_i64, c_vp, c_vp]),
    "sb200_percentile_ranks": (c_int, [c_vp, c_vp, c_i64, c_d, c_vp, c_vp]),
    "sb200_moments_workspace_bytes": (c_sz, [c_i64, c_i64]),
    "sb200_observe_moments": (c_int, [c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "sb200_mask_gt": (c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "sb200_minmax_qparams_multi": (c_int, [c_vp, c_int, c_vp, c_sz, c_vp]),
    "sb200_gptq4_matmul_batch": (c_int, [c_vp, c_int, c_i64, c_vp]),
    "sb200_gptq4_matmul_batch_ex": (c_int, [c_vp, c_int, c_i64, c_int, c_vp]),
    "sb200_mask_rows_gt": (c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_vp]),
    "sb200_mask_apply": (c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "sb200_mask_apply_f32": (c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "sb200_mask_apply_qdq_perchannel": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_vp]),
    "sb200_qdq_multi_table_bytes": (c_sz, [c_int]),
    "sb200_qdq_multi_plan": (c_int, [c_vp, c_int, c_vp, c_sz, c_vp, c_vp]),
    "sb200_qdq_multi_run": (c_int, [c_vp, c_int, c_i64, c_vp]),
    "sb200_adaround_fwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_vp]),
    "sb200_adaround_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_vp]),
    "sb200_adaround_init": (c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp]),
    "sb200_dorefa_absmax": (c_int, [c_vp, c_i64, c_vp, c_vp]),
    "sb200_dorefa_fwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_vp]),
    "sb200_dorefa_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_int, c_int, c_vp]),
    "sb200_gptq4_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_int]),
    "sb200_gptq4_matmul": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_sz, c_vp]),
    "sb200_gptq4_matmul_ex": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_vp, c_sz, c_vp]),
    "sb200_gptq4_linear_f16_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_int]),
    "sb200_gptq4_linear_f16": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_sz, c_vp]),
    "sb200_gptq4_linear_f16_state_bytes": (c_sz, []),
    "sb200_gptq4_linear_f16_ex": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_vp, c_int, c_vp, c_sz, c_vp]),
    "sb200_gptq_matmul": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_vp, c_sz, c_vp]),
    "sb200_gptq_dgrad_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_int, c_int]),
    "sb200_gptq_matmul_dgrad": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_vp, c_sz, c_vp]),
    "sb200_int8_quantize_rows": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp]),
    "sb200_int8_linear_workspace_bytes": (c_sz, [c_i64, c_i64]),
    "sb200_int8_linear": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp,
                                  c_sz, c_vp]),
    "sb200_sparse24_mask": (c_int, [c_vp, c_vp, c_i64, c_i64, c_vp]),
    "sb200_int8_sparse24_pack": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp]),
    "sb200_int8_sparse24_linear": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64,
                                           c_i64, c_vp, c_sz, c_vp]),
    "sb200_int8_im2col_quantize": (c_int, [c_vp, c_geom, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    "sb200_int8_conv2d_workspace_bytes": (c_sz, [c_geom]),
    "sb200_int8_conv2d": (c_int, [c_vp, c_geom, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_sz,
                                  c_vp]),
    "sb200_int8_sparse24_conv2d": (c_int, [c_vp, c_geom, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64,
                                           c_vp, c_sz, c_vp]),
    "sb200_int8_quantize_cols": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp]),
    "sb200_int8_matmul_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_i64]),
    "sb200_int8_matmul": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_int, c_int, c_vp, c_i64, c_i64,
                                  c_i64, c_i64, c_vp, c_sz, c_vp]),
    "sb200_int8_group_conv2d": (c_int, [c_vp, c_geom, c_i64, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                        c_i64, c_vp]),
    "sb200_int8_im2col_quantize_nhwc": (c_int, [c_vp, c_geom, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    "sb200_int8_conv2d_nhwc": (c_int, [c_vp, c_geom, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp,
                                       c_sz, c_vp]),
    "sb200_int8_sparse24_conv2d_nhwc": (c_int, [c_vp, c_geom, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                c_i64, c_vp, c_sz, c_vp]),
    "sb200_int8_group_conv2d_nhwc": (c_int, [c_vp, c_geom, c_i64, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                             c_vp, c_i64, c_vp]),
    "sb200_int8_linear_dorefa": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64,
                                         c_i64, c_vp, c_sz, c_vp]),
    "sb200_int8_conv2d_dorefa": (c_int, [c_vp, c_geom, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                         c_i64, c_vp, c_sz, c_vp]),
    "sb200_int8_conv2d_nhwc_dorefa": (c_int, [c_vp, c_geom, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                              c_vp, c_i64, c_vp, c_sz, c_vp]),
    "sb200_int8_group_conv2d_dorefa": (c_int, [c_vp, c_geom, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp,
                                               c_vp, c_vp, c_i64, c_vp]),
    "sb200_int8_group_conv2d_nhwc_dorefa": (c_int, [c_vp, c_geom, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp,
                                                    c_vp, c_vp, c_vp, c_i64, c_vp]),
    "sb200_int8_attention_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_i64, c_i64]),
    "sb200_int8_attention": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_int,
                                     c_int, c_vp, c_vp, c_int, c_int, c_int, c_f, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64,
                                     c_i64, c_vp, c_sz, c_vp]),
    "sb200_int8_attention_masked_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_i64, c_i64, c_int]),
    "sb200_int8_attention_masked": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_int, c_int, c_vp,
                                            c_vp, c_int, c_int, c_vp, c_vp, c_int, c_int, c_int, c_f, c_vp, c_i64, c_i64,
                                            c_i64, c_i64, c_int, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp,
                                            c_sz, c_vp]),
    "sb200_int8_kv_append": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp,
                                     c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp]),
    "sb200_int8_attention_cached_workspace_bytes": (c_sz, [c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_int]),
    "sb200_int8_attention_cached": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_int,
                                            c_int, c_vp, c_vp, c_int, c_int, c_int, c_f, c_vp, c_i64, c_i64, c_i64,
                                            c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp,
                                            c_i64, c_i64, c_i64, c_i64, c_vp, c_sz, c_vp]),
    "sb200_gptq4_set_impl": (c_int, [c_int]),
    "sb200_gptq4_set_wait_backoff": (c_int, [c_int]),
    "sb200_gptq4_set_decode": (c_int, [c_int]),
}

SELECT_STATE_WORDS = 4
SELECT_BINS = 2048

_lib = None


def load():
    """Load (once) and return the ctypes handle; raise loudly if the library was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SparsebitB200Error(
            f"native library not found: {LIB_PATH}. sparsebit_b200 has no CPU / eager fallback -- build it "
            "with `make -C sparsebit_b200/csrc` (nvcc, sm_90a) or `python -c 'import __graft_entry__ as g; g.build()'`."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the .so is stale -> also loud
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status, what=""):
    if status != 0:
        msg = load().sb200_last_error().decode("utf-8", "replace")
        raise SparsebitB200Error(f"{what}: {msg} (status {status})" if what else f"{msg} (status {status})")


def launch_count():
    return int(load().sb200_launch_count())
