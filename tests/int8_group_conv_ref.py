"""fp64 truth of the integer-grid grouped / depthwise conv2d (sb200_int8_group_conv2d / QConv2dGroupInt8): the grouped
conv2d of the fake-quant tensors that ``oracle.qdq.qdq`` produces, in fp64, zero-padded after the fake-quant, plus the
bias,
    T = conv2d(pad(fx, 0.0), fw, groups) + bias,   |y - T| <= 2^-21 * (conv2d(|fx|, |fw|, groups) + |bias|)
(tests/int8_conv_ref.py for groups = 1), and the per-group integer form: group g is the dense conv of input channels
g C_g .. (g + 1) C_g - 1 with weight rows g M_g .. (g + 1) M_g - 1, whose integer terms int8_conv_ref.integer_terms
gives."""
import numpy as np
import torch
import torch.nn.functional as F

from int8_conv_ref import BOUND, _pads, _pair, fake_quant_operands, integer_terms, out_hw, to_nchw

__all__ = ["BOUND", "out_hw", "truth", "group_integer_form"]


def _conv64(x, w, groups, stride, padding, dilation):
    pt, pb, pl, pr = _pads(padding)
    xp = F.pad(torch.from_numpy(np.ascontiguousarray(x, np.float64)), (pl, pr, pt, pb), value=0.0)
    return F.conv2d(xp, torch.from_numpy(np.ascontiguousarray(w, np.float64)), stride=_pair(stride),
                    dilation=_pair(dilation), groups=groups).numpy()


def truth(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, groups, bias=None, stride=1, padding=0, dilation=1):
    """(T, bound) as [N, C_out, OH, OW] fp64 arrays."""
    fx, fw = fake_quant_operands(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax)
    b = np.zeros(fw.shape[0]) if bias is None else np.asarray(bias, np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        t = _conv64(fx, fw, groups, stride, padding, dilation) + b[None, :, None, None]
        mag = _conv64(np.abs(fx), np.abs(fw), groups, stride, padding, dilation) + np.abs(b)[None, :, None, None]
    return t, BOUND * mag


def group_integer_form(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, groups, stride=1, padding=0, dilation=1):
    """(I, s) with I int64 [N, C_out, OH, OW] the exact integer sum of each output and s = s_x s_w[n] fp64 [C_out]:
    the group's dense integer terms, group by group."""
    x, w = np.asarray(x, np.float32), np.asarray(w, np.float32)
    n, c, h, wd = x.shape
    c_out, c_g, kh, kw = w.shape
    m_g = c_out // groups
    oh, ow = out_hw(h, wd, kh, kw, stride, padding, dilation)
    ws = np.broadcast_to(np.asarray(ws, np.float32).reshape(-1), (c_out,))
    wz = np.broadcast_to(np.asarray(wz, np.float32).reshape(-1), (c_out,))
    parts = []
    for g in range(groups):
        o = slice(g * m_g, (g + 1) * m_g)
        *_, i = integer_terms(x[:, g * c_g:(g + 1) * c_g], xs, xz, xqmin, xqmax, w[o], ws[o], wz[o], wqmin, wqmax,
                              stride, padding, dilation)
        parts.append(to_nchw(i, n, oh, ow))
    s = np.float64(np.float32(np.asarray(xs).reshape(-1)[0])) * ws.astype(np.float64)
    return np.concatenate(parts, axis=1), s
