"""fp64 truth of the integer-grid matmul (sb200_int8_matmul / QMatMulInt8): the batched matmul of the two fake-quant
operands that ``oracle.qdq.qdq`` produces (pinned bit-exact to the reference's QDQ), in fp64,
    T[b, m, n] = sum_k fa[b, m, k] * fb[b, k, n],   fa = qdq(a, s_a, z_a),  fb = qdq(b, s_b, z_b)  (fp32 tensors)
and the accuracy bound the integer path is held to,
    |y - T| <= 2^-21 * (|fa| @ |fb|)
(the epilogue rounds s_a s_b I once to fp32; each fp32 element fa, fb of the truth is itself within 2^-24 of v * s).
Operands are (x, scale, zero_point, qmin, qmax) tuples; ``a`` is [..., M, K], ``b`` is [..., K, N]."""
import numpy as np

from int8_linear_ref import BOUND, grid_offset
from oracle import qdq as oqdq

F32 = np.float32


def stored_grid(x, s, z, qmin, qmax):
    """The s8 grid as the quantize kernels store it (g - offset; NaN stored as 0) and the NaN mask of ``x``."""
    x = np.asarray(x, F32)
    g = oqdq.quantize_int(x, F32(s), F32(z), qmin, qmax)
    nan = np.isnan(g)
    return (np.where(nan, F32(grid_offset(qmin)), g) - grid_offset(qmin)).astype(np.int64), nan


def quantize_cols(x, s, z, qmin, qmax):
    """What sb200_int8_quantize_cols writes for x [..., K, N]: (q int8 [..., N, Kp], col_sum int32, nan bool)."""
    g, nan = stored_grid(x, s, z, qmin, qmax)
    k = g.shape[-2]
    gt = np.swapaxes(g, -1, -2)
    q = np.zeros(gt.shape[:-1] + ((k + 15) // 16 * 16,), np.int8)
    q[..., :k] = gt
    return q, gt.sum(-1).astype(np.int32), nan.any(-2)


def truth(a, b):
    """(T, bound) as fp64 arrays [..., M, N] (leading dimensions broadcast)."""
    fa, fb = oqdq.qdq(*a).astype(np.float64), oqdq.qdq(*b).astype(np.float64)
    with np.errstate(all="ignore"):
        return np.matmul(fa, fb), BOUND * np.matmul(np.abs(fa), np.abs(fb))


def integer_form(a, b):
    """The value the kernel computes before its one rounding to fp32: the stored zero points, the int64 sum
    I = sum qa qb - Z_b sum_k qa - Z_a sum_k qb + K Z_a Z_b, and fp64(I) * (fp64(s_a) * fp64(s_b)); NaN rows of ``a``
    and NaN columns of ``b`` give NaN rows / columns."""
    (xa, sa, za, amin, amax), (xb, sb, zb, bmin, bmax) = a, b
    qa, nan_a = stored_grid(xa, sa, za, amin, amax)
    qb, nan_b = stored_grid(xb, sb, zb, bmin, bmax)
    k = qa.shape[-1]
    z_a = int(np.rint(F32(za))) - grid_offset(amin)
    z_b = int(np.rint(F32(zb))) - grid_offset(bmin)
    i = np.matmul(qa, qb) - z_b * qa.sum(-1)[..., :, None] - z_a * qb.sum(-2)[..., None, :] + k * z_a * z_b
    y = i.astype(np.float64) * (np.float64(F32(sa)) * np.float64(F32(sb)))
    bad = nan_a.any(-1)[..., :, None] | nan_b.any(-2)[..., None, :]
    return qa, qb, z_a, z_b, i, np.where(bad, np.nan, y)
