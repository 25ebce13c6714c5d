"""CPU: the fp64 truth of the GPTQ input gradient and the host side of sb200_gptq_matmul_dgrad.

* The truth is the adjoint of the forward oracle:  <g, dequant_matmul(x) - bias> == <dgrad(g), x>  for every bit width
  and group size.
* On the 19 reference-produced cases of tests/golden (gptq.npz, gptq_lowbit.npz) it equals g @ wdq, the dense weights
  the unmodified reference dequantised.
* Every bad argument is rejected on the host with SB200_E_INVALID before any CUDA call (no device here), with the
  forward's messages, and the workspace query is a pure function of its arguments."""
import ctypes

import numpy as np
import pytest

from gptq_dgrad_ref import dequant_matmul_dgrad
from oracle import gptq as ogptq
from sparsebit_b200 import _lib


def _case(rng, bit, k, n, gs, fractional_zero=False):
    w = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
    scale, zero = ogptq.find_params(w, bit, gs)
    qw, scales, zeros = ogptq.pack_bits(ogptq.quantize_weight(w, scale, zero, gs, bit), scale, zero, bit)
    if fractional_zero:
        zeros = (zeros + scales * rng.uniform(-0.5, 0.5, zeros.shape)).astype(np.float32)
    return qw, scales, zeros


GROUPS = {2: [-1, 64, 192], 3: [-1, 128, 384], 4: [-1, 128, 384]}


@pytest.mark.parametrize("bit,gs", [(b, g) for b, gl in GROUPS.items() for g in gl])
@pytest.mark.parametrize("fractional_zero", [False, True])
def test_adjoint_of_the_forward_oracle(bit, gs, fractional_zero):
    rng = np.random.default_rng(100 * bit + gs + fractional_zero)
    k, n, m = 768, 72, 5
    qw, scales, zeros = _case(rng, bit, k, n, gs, fractional_zero)
    x = rng.standard_normal((m, k))
    g = rng.standard_normal((m, n))
    bias = rng.standard_normal(n)
    gs0 = 0 if gs == -1 else gs
    y = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (m, n)), scales, zeros, gs0, bit=bit)
    lhs = np.sum(g * (y - bias))
    rhs = np.sum(dequant_matmul_dgrad(g, qw, scales, zeros, k, gs0, bit) * x)
    assert abs(lhs - rhs) <= 1e-12 * (np.abs(g).sum() * np.abs(x).sum())


def _golden_cases(golden):
    for fixture in ("gptq", "gptq_lowbit"):
        g = golden(fixture)
        for name in g["cases"]:
            bit, gs = (4, int(g[name + "_gs"])) if fixture == "gptq" else (int(v) for v in g[name + "_meta"])
            yield name, bit, gs, g


def test_reference_dense_weights_anchor_the_truth(golden):
    cases = list(_golden_cases(golden))
    assert len(cases) == 19
    for name, bit, gs, g in cases:
        wdq = g[name + "_wdq"].astype(np.float64)  # [N, K] from the reference
        n, k = wdq.shape
        rng = np.random.default_rng(len(name))
        lead = g[name + "_x"].shape[:-1]
        go = rng.standard_normal(lead + (n,))
        got = dequant_matmul_dgrad(go, g[name + "_qweight"], g[name + "_scales"], g[name + "_zeros"], k, 0 if gs == -1 else gs, bit)
        exp = go.reshape(-1, n) @ wdq
        # the reference's fp32 dequantisation is within 4e-7 of s q - z (test_oracle_golden.py)
        bound = 4e-7 * (np.abs(go.reshape(-1, n)).sum(axis=1, keepdims=True)) + 1e-12
        assert np.all(np.abs(got.reshape(-1, k) - exp) <= bound), name


def _ptr():
    buf = (ctypes.c_float * 64)()
    return buf, ctypes.addressof(buf)


def test_bad_arguments_are_rejected_on_the_host():
    lib = _lib.load()
    _keep, p = _ptr()
    call = lib.sb200_gptq_matmul_dgrad
    # (grad_out, qweight, grad_in, scales, zeros, m, k, n, rows, bits, gs, impl, ws, ws_bytes, stream)
    ok = [p, p, p, p, p, 4, 256, 8, 32, 4, 128, 0, p, 1 << 20, None]

    def rejected(i, v, text=None):
        args = list(ok)
        args[i] = v
        assert call(*args) == -1, (i, v)
        if text:
            assert text in lib.sb200_last_error(), (i, v, lib.sb200_last_error())

    for bits in (0, 1, 5, 8):
        rejected(9, bits, b"only support 2/3/4 bit")
    for i in range(5):
        rejected(i, None, b"null pointer")
    for i in (5, 6, 7):
        rejected(i, 0, b"empty operand")
        rejected(i, -3, b"empty operand")
        rejected(i, 1 << 31, b"dimension too large")
    for impl in (-1, 3, 4):
        rejected(11, impl, b"impl")
    # packed rows: ceil(K/8) for 4-bit, ceil(K/16) for 2-bit, ceil(3K/96) * 3 for 3-bit (utils/quant.py:172-184)
    for bits, need in ((4, 32), (2, 16), (3, 24)):
        args = list(ok)
        args[9], args[8], args[10] = bits, need - 1, 0
        assert call(*args) == -1 and b"rows" in lib.sb200_last_error()
        args[8] = need
        fwd = lib.sb200_gptq_matmul(p, p, p, p, p, 4, 256, 8, need - 1, bits, 0, None, 0, None)
        assert fwd == -1
    # group sizes: the forward's rule and its message, word for word
    for bits, gs in ((4, 64), (4, 96), (3, 64), (2, 32), (2, 96), (4, -128), (2, -64)):
        args = list(ok)
        args[9], args[10], args[8] = bits, gs, 32
        assert call(*args) == -1
        msg = lib.sb200_last_error()
        assert lib.sb200_gptq_matmul(p, p, p, p, p, 4, 256, 8, 32, bits, gs, None, 0, None) == -1
        assert lib.sb200_last_error() == msg
        assert b"divisible by" in msg


def test_workspace_query_is_pure():
    lib = _lib.load()
    q = lib.sb200_gptq_dgrad_workspace_bytes
    assert q(0, 256, 8, 4, 128) == 0 and q(4, 0, 8, 4, 128) == 0 and q(4, 256, 0, 4, 0) == 0
    for args in [(2048, 4096, 11008, 4, 128), (1, 6661, 2516, 3, 0), (33, 1024, 260, 2, 64), (7, 127, 61, 4, 0)]:
        first = q(*args)
        assert first > 0 and all(q(*args) == first for _ in range(3))
    # the 4-bit tensor-core path needs the repacked weights and the split gradient on top of the SIMT tables
    m, k, n = 2048, 4096, 11008
    assert q(m, k, n, 4, 128) >= n // 8 * k * 4 + 2 * m * n * 2
    assert q(m, k, n, 3, 128) < n // 8 * k * 4
    assert q(m, k, n, 4, 0) == q(m, k, n, 4, k)  # group_size 0 is one group
