"""fp64 truth of the integer-grid linear (sb200_int8_linear / QLinearInt8): the matmul of the fake-quant tensors that
``oracle.qdq.qdq`` produces (pinned bit-exact to the reference's QDQ), in fp64, plus the bias:
    T[m, n] = sum_k fx[m, k] * fw[n, k] + bias[n],   fx = qdq(x, s_x, z_x),  fw = qdq(w, s_w[n], z_w[n])  (fp32 tensors)
and the accuracy bound the integer path is held to,
    |y - T| <= 2^-21 * (sum_k |fx fw| + |bias|)
(the epilogue rounds s_x s_w I once to fp32 and once more after the bias; each fp32 element fx, fw of the truth is
itself within 2^-24 of v * s)."""
import numpy as np

from oracle import qdq as oqdq

BOUND = 2.0 ** -21


def grid_offset(qmin):
    return 128 if qmin >= 0 else 0


def fake_quant_operands(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax):
    x = np.asarray(x, np.float32)
    w = np.asarray(w, np.float32)
    fx = oqdq.qdq(x.reshape(-1, x.shape[-1]), np.float32(np.asarray(xs).reshape(-1)[0]), np.float32(np.asarray(xz).reshape(-1)[0]), xqmin, xqmax)
    fw = oqdq.qdq(w, np.asarray(ws, np.float32).reshape(-1), np.asarray(wz, np.float32).reshape(-1), wqmin, wqmax, ch_axis=0)
    return fx, fw


def truth(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, bias=None):
    """(T, bound) as [M, N] fp64 arrays, M = prod(x.shape[:-1])."""
    fx, fw = fake_quant_operands(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax)
    b = np.zeros(fw.shape[0]) if bias is None else np.asarray(bias, np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        t = fx.astype(np.float64) @ fw.astype(np.float64).T + b
        mag = np.abs(fx).astype(np.float64) @ np.abs(fw).astype(np.float64).T + np.abs(b)
    return t, BOUND * mag


def integer_terms(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax):
    """The integer form the kernel computes: stored grids a, b (offset for unsigned ranges), stored zero points and
    I = sum a b - Z_w sum a - Z_x sum b + K Z_x Z_w in int64."""
    x = np.asarray(x, np.float32).reshape(-1, np.asarray(x).shape[-1])
    k = x.shape[1]
    ox, ow = grid_offset(xqmin), grid_offset(wqmin)
    ga = oqdq.quantize_int(x, np.float32(np.asarray(xs).reshape(-1)[0]), np.float32(np.asarray(xz).reshape(-1)[0]), xqmin, xqmax)
    gb = oqdq.quantize_int(w, np.asarray(ws, np.float32).reshape(-1), np.asarray(wz, np.float32).reshape(-1), wqmin, wqmax, ch_axis=0)
    a = (ga - ox).astype(np.int64)
    b = (gb - ow).astype(np.int64)
    zx = int(np.rint(np.float32(np.asarray(xz).reshape(-1)[0]))) - ox
    zw = (np.rint(np.broadcast_to(np.asarray(wz, np.float32).reshape(-1), (b.shape[0],))) - ow).astype(np.int64)
    i = a @ b.T - zw[None, :] * a.sum(1)[:, None] - zx * b.sum(1)[None, :] + k * zx * zw[None, :]
    return a, b, zx, zw, i
