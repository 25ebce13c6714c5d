"""fp64 truth of the GPTQ input gradient (sb200_gptq_matmul_dgrad), built on the oracle's unpackers:
    grad_in[m, k] = sum_n grad_out[m, n] * (scales[n, k//gs] * q[k, n] - zeros[n, k//gs])
It is the adjoint of ``oracle.gptq.dequant_matmul`` (tests/test_gptq_dgrad_host.py checks that identity and the
reference-produced dense weights of tests/golden)."""
import numpy as np

from oracle import gptq as ogptq


def dequant_weight(qweight, scales, zeros, k, group_size=0, bit=4, dtype=np.float64):
    """Dense W [K, N] = scales * q - zeros, in ``dtype``."""
    q = (ogptq.unpack_int4(qweight, k) if bit == 4 else ogptq.unpack_bits(qweight, k, bit)).astype(dtype)
    n = q.shape[1]
    gs = k if group_size in (0, -1) else group_size
    ng = (k + gs - 1) // gs
    s = np.asarray(scales, dtype=np.float32).reshape(n, ng).astype(dtype)
    z = np.asarray(zeros, dtype=np.float32).reshape(n, ng).astype(dtype)
    gi = np.arange(k) // gs
    return s.T[gi] * q - z.T[gi]


def dequant_matmul_dgrad(grad_out, qweight, scales, zeros, k, group_size=0, bit=4, dtype=np.float64):
    g = np.asarray(grad_out)
    n = g.shape[-1]
    w = dequant_weight(qweight, scales, zeros, k, group_size, bit, dtype)
    return (g.reshape(-1, n).astype(dtype) @ w.T).reshape(g.shape[:-1] + (k,))
