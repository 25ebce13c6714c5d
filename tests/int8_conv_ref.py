"""fp64 truth of the integer-grid conv2d (sb200_int8_conv2d / QConv2dInt8): the conv2d of the fake-quant tensors that
``oracle.qdq.qdq`` produces, in fp64, zero-padded after the fake-quant (as QConv2d pads), plus the bias:
    T = conv2d(pad(fx, 0.0), fw) + bias,   fx = qdq(x, s_x, z_x),  fw = qdq(w, s_w[n], z_w[n])  (fp32 tensors)
and the bound the integer path is held to, elementwise,
    |y - T| <= 2^-21 * (conv2d(|fx|, |fw|) + |bias|)
(the same two fp32 roundings as the integer linear, tests/int8_linear_ref.py).

The lowering reference: F.unfold of the oracle's integer grid on the stored grid (g - off, NaN stored as 0), with the
padding taps set to rint(zp) - off -- the grid point of the zero padding -- and the K padding up to Kp zero."""
import numpy as np
import torch
import torch.nn.functional as F

from int8_linear_ref import BOUND, grid_offset
from oracle import qdq as oqdq

__all__ = ["BOUND", "grid_offset", "out_hw", "truth", "lowered", "integer_terms"]


def _pads(padding):
    p = (padding, padding) if isinstance(padding, int) else tuple(padding)
    return (p[0], p[0], p[1], p[1]) if len(p) == 2 else tuple(p)  # (top, bottom, left, right)


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def out_hw(h, w, kh, kw, stride=1, padding=0, dilation=1):
    pt, pb, pl, pr = _pads(padding)
    (sh, sw), (dh, dw) = _pair(stride), _pair(dilation)
    return (h + pt + pb - dh * (kh - 1) - 1) // sh + 1, (w + pl + pr - dw * (kw - 1) - 1) // sw + 1


def _conv64(x, w, stride, padding, dilation):
    pt, pb, pl, pr = _pads(padding)
    xp = F.pad(torch.from_numpy(np.ascontiguousarray(x, np.float64)), (pl, pr, pt, pb), value=0.0)
    return F.conv2d(xp, torch.from_numpy(np.ascontiguousarray(w, np.float64)), stride=_pair(stride),
                    dilation=_pair(dilation)).numpy()


def fake_quant_operands(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax):
    fx = oqdq.qdq(np.asarray(x, np.float32), np.float32(np.asarray(xs).reshape(-1)[0]),
                  np.float32(np.asarray(xz).reshape(-1)[0]), xqmin, xqmax)
    fw = oqdq.qdq(np.asarray(w, np.float32), np.asarray(ws, np.float32).reshape(-1), np.asarray(wz, np.float32).reshape(-1),
                  wqmin, wqmax, ch_axis=0)
    return fx, fw


def truth(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, bias=None, stride=1, padding=0, dilation=1):
    """(T, bound) as [N, C_out, OH, OW] fp64 arrays."""
    fx, fw = fake_quant_operands(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax)
    b = np.zeros(fw.shape[0]) if bias is None else np.asarray(bias, np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        t = _conv64(fx, fw, stride, padding, dilation) + b[None, :, None, None]
        mag = _conv64(np.abs(fx), np.abs(fw), stride, padding, dilation) + np.abs(b)[None, :, None, None]
    return t, BOUND * mag


def lowered(x, kernel_size, xs, xz, qmin, qmax, stride=1, padding=0, dilation=1):
    """What sb200_int8_im2col_quantize writes: (q int64 [M, Kp], row_sum int64 [M], nan bool [M])."""
    x = np.asarray(x, np.float32)
    n, c = x.shape[:2]
    kh, kw = _pair(kernel_size)
    off = grid_offset(qmin)
    zp = float(np.rint(np.float32(np.asarray(xz).reshape(-1)[0])))
    g = oqdq.quantize_int(x, np.float32(np.asarray(xs).reshape(-1)[0]), np.float32(np.asarray(xz).reshape(-1)[0]), qmin, qmax)
    nan = np.isnan(g)
    stored = np.where(nan, 0.0, np.nan_to_num(g) - off)
    pt, pb, pl, pr = _pads(padding)

    def unfold(v, pad_value):
        vp = F.pad(torch.from_numpy(np.ascontiguousarray(v, np.float64)), (pl, pr, pt, pb), value=pad_value)
        cols = F.unfold(vp, (kh, kw), dilation=_pair(dilation), stride=_pair(stride))  # [N, K, L], K in (c, kh, kw)
        return cols.transpose(1, 2).reshape(-1, c * kh * kw).numpy()

    q = unfold(stored, zp - off).astype(np.int64)
    win_nan = unfold(nan.astype(np.float64), 0.0).any(axis=1)
    k = q.shape[1]
    kp = (k + 15) // 16 * 16
    q = np.concatenate([q, np.zeros((q.shape[0], kp - k), np.int64)], axis=1)
    return q, q.sum(axis=1), win_nan


def integer_terms(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, stride=1, padding=0, dilation=1):
    """The integer form the kernels compute, on the lowered rows: I [M, C_out] = sum a b - Z_w sum a - Z_x sum b
    + K Z_x Z_w with the real K = C KH KW, plus the stored zero points."""
    w = np.asarray(w, np.float32)
    c_out, _, kh, kw = w.shape
    k = w[0].size
    a, _, _ = lowered(x, (kh, kw), xs, xz, xqmin, xqmax, stride, padding, dilation)
    a = a[:, :k]
    ox, ow = grid_offset(xqmin), grid_offset(wqmin)
    gb = oqdq.quantize_int(w.reshape(c_out, -1), np.asarray(ws, np.float32).reshape(-1), np.asarray(wz, np.float32).reshape(-1),
                           wqmin, wqmax, ch_axis=0)
    b = (gb - ow).astype(np.int64)
    zx = int(np.rint(np.float32(np.asarray(xz).reshape(-1)[0]))) - ox
    zw = (np.rint(np.broadcast_to(np.asarray(wz, np.float32).reshape(-1), (c_out,))) - ow).astype(np.int64)
    i = a @ b.T - zw[None, :] * a.sum(1)[:, None] - zx * b.sum(1)[None, :] + k * zx * zw[None, :]
    return a, b, zx, zw, i


def to_nchw(rows, n, oh, ow):
    """[M, C_out] rows (m = (img OH + oh) OW + ow) -> [N, C_out, OH, OW]."""
    return rows.reshape(n, oh, ow, -1).transpose(0, 3, 1, 2)
