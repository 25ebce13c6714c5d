"""CPU: the C-ABI library loads, exports every symbol include/sparsebit_b200.h declares, and its
argument validation (which runs before any CUDA call) reports errors the way the reference's
pybind modules do.  No kernels are launched here."""
import ctypes
import os
import re

import pytest

from sparsebit_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    hdr = open(os.path.join(ROOT, "include", "sparsebit_b200.h")).read()
    return sorted(set(re.findall(r"\b(sb200_\w+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = header_symbols()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    assert sorted(_lib.PROTOTYPES) == names


def test_version_and_variant_validation():
    lib = _lib.load()
    assert lib.sb200_version() >= 100
    assert lib.sb200_set_variant(0) == 0
    assert lib.sb200_set_variant(7) != 0
    assert b"variant" in lib.sb200_last_error()
    assert lib.sb200_gptq4_set_impl(5) != 0
    assert lib.sb200_gptq4_set_impl(3) != 0 and b"impl" in lib.sb200_last_error()
    assert lib.sb200_gptq4_set_impl(0) == 0


def test_argument_errors_surface_as_runtime_error():
    lib = _lib.load()
    buf = (ctypes.c_float * 8)()
    p = ctypes.addressof(buf)
    # empty tensor -> the reference raises InvalidValueException("Tensor is empty") (common.cuh:51-54)
    st = lib.sb200_qdq_pertensor_fwd(p, p, p, p, 0, -128, 127, 0, None)
    assert st == -1 and b"empty" in lib.sb200_last_error()
    with pytest.raises(RuntimeError):
        _lib.check(st, "qdq")
    assert lib.sb200_qdq_pertensor_fwd(None, p, p, p, 8, -128, 127, 0, None) == -1
    assert lib.sb200_qdq_pertensor_fwd(p, p, p, p, 8, -128, 127, 9, None) == -1  # bad rounding
    assert lib.sb200_qdq_perchannel_fwd(p, p, p, p, 0, 4, 2, -128, 127, 0, None) == -1
    # GPTQ: group size must be a multiple of 128 (cuda_kernel_4bit.cu:60)
    st = lib.sb200_gptq4_matmul(p, p, p, p, p, 1, 256, 8, 32, 64, None, 0, None)
    assert st == -1 and b"divisible by 128" in lib.sb200_last_error()
    st = lib.sb200_gptq4_matmul(p, p, p, p, p, 1, 256, 8, 3, 128, None, 0, None)  # too few packed rows
    assert st == -1
    # per-call options: impl is 0, 1, 2 or 4, chunk_k is reserved (sb200_gptq4_options = 8 ints)
    for impl, chunk_k, what in ((3, 0, b"impl"), (0, 512, b"chunk_k"), (2, 64, b"chunk_k")):
        opts = (ctypes.c_int * 8)(impl, chunk_k)
        st = lib.sb200_gptq4_matmul_ex(p, p, p, p, p, 1, 256, 8, 32, 128, opts, p, 1 << 20, None)
        assert st == -1 and what in lib.sb200_last_error()
    assert lib.sb200_observe_hist(p, 8, p, 0, p, None) == -1
    assert lib.sb200_select_hist(p, 1, 8, 3, p, p, 0, 0, None) == -1


def test_workspace_queries_are_pure():
    lib = _lib.load()
    assert lib.sb200_qdq_bwd_workspace_bytes(1, 1, 8192 * 3) == 3 * 16
    assert lib.sb200_qdq_bwd_workspace_bytes(0, 1, 5) == 0
    assert lib.sb200_mse_workspace_bytes(2, 8192 * 2 + 1, 80) == 2 * 3 * 80 * 8


def test_missing_library_fails_loudly(monkeypatch):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libsparsebit_b200.so")
    with pytest.raises(_lib.SparsebitB200Error, match="no CPU"):
        _lib.load()


def test_widened_entry_points_validate_before_launching():
    """AdaRound, 3 / 2-bit GPTQ, row moments, tuning knobs: bad arguments are rejected on the host."""
    lib = _lib.load()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    assert lib.sb200_adaround_fwd(p, p, p, p, p, 1, 1, 8, -8, 7, 2, None) == -1 and b"soft" in lib.sb200_last_error()
    assert lib.sb200_adaround_fwd(p, p, p, p, p, 1, 1, 0, -8, 7, 0, None) == -1
    assert lib.sb200_adaround_bwd(p, p, p, p, None, p, 1, 1, 8, -8, 7, None) == -1
    assert lib.sb200_adaround_init(p, None, p, 1, 1, 8, None) == -1
    # bits other than 2 / 3 / 4; group sizes (cuda_kernel_2bit.cu:58, cuda_kernel_3bit.cu:60); packed rows
    assert lib.sb200_gptq_matmul(p, p, p, p, p, 1, 256, 8, 64, 5, 0, None, 0, None) == -1 and b"2/3/4" in lib.sb200_last_error()
    assert lib.sb200_gptq_matmul(p, p, p, p, p, 1, 256, 8, 24, 3, 64, None, 0, None) == -1
    assert b"divisible by 128" in lib.sb200_last_error()
    assert lib.sb200_gptq_matmul(p, p, p, p, p, 1, 256, 8, 16, 2, 96, None, 0, None) == -1
    assert b"divisible by 64" in lib.sb200_last_error()
    assert lib.sb200_gptq_matmul(p, p, p, p, p, 1, 256, 8, 23, 3, 0, None, 0, None) == -1 and b"rows" in lib.sb200_last_error()
    assert lib.sb200_gptq_matmul(p, p, p, p, p, 1, 256, 8, 15, 2, 0, None, 0, None) == -1
    # row moments: workspace sizing is pure, too-small workspaces are refused
    assert lib.sb200_moments_workspace_bytes(3, 16384) == 3 * 5 * 8
    assert lib.sb200_moments_workspace_bytes(3, 16385) == 3 * 2 * 5 * 8
    assert lib.sb200_moments_workspace_bytes(0, 5) == 0
    assert lib.sb200_observe_moments(p, 3, 16385, None, p, p, 8, None) == -1 and b"workspace" in lib.sb200_last_error()
    assert lib.sb200_gptq4_set_wait_backoff(-1) == -1
    assert lib.sb200_gptq4_set_wait_backoff(0) == 0
    assert lib.sb200_gptq4_set_decode(256) == -1 and lib.sb200_gptq4_set_decode(6) == 0
    assert lib.sb200_gptq4_matmul_batch_ex(p, 1, 1, 2, None) == -1 and b"flags" in lib.sb200_last_error()
    assert lib.sb200_gptq4_linear_f16_state_bytes() >= 4 * 16384
    assert lib.sb200_gptq4_linear_f16_ex(p, p, p, None, p, p, 1, 128, 128, 16, 128, p, 4, p, 1 << 20, None) == -1 and b"flags" in lib.sb200_last_error()
    # DoReFa (dorefa.py:15-26): null / empty / bad flags
    assert lib.sb200_dorefa_absmax(p, 0, p, None) == -1 and b"empty" in lib.sb200_last_error()
    assert lib.sb200_dorefa_absmax(None, 8, p, None) == -1
    assert lib.sb200_dorefa_fwd(p, p, p, p, p, 1, 1, 8, -8, 7, 2, None) == -1 and b"quantize" in lib.sb200_last_error()
    assert lib.sb200_dorefa_fwd(p, p, None, p, p, 1, 1, 8, -8, 7, 1, None) == -1 and b"qparams" in lib.sb200_last_error()
    assert lib.sb200_dorefa_fwd(p, p, p, p, p, 1, 1, 8, 7, -8, 1, None) == -1
    assert lib.sb200_dorefa_bwd(p, p, p, p, None, p, 1, 1, 8, -8, 7, None) == -1
    assert lib.sb200_dorefa_bwd(p, p, p, p, p, p, 1, 0, 8, -8, 7, None) == -1
