"""numpy reference of the fused integer-grid attention (sb200_int8_attention / QAttentionInt8).

Operands are (x, scale, zero_point, qmin, qmax) tuples: q [..., Tq, d], k [..., Tk, d], v [..., Tk, dv]; p's qparams
are (scale, zero_point, qmin, qmax).  The kernel computes, per batch entry,
    s   = RN32(fp64(I_qk) * (fp64(s_q) fp64(s_k)))   [then RN32(s * RN32(scale))]   -- exact, reproduced here
    p   = softmax(s) in fp32                                                        -- the only inexact step
    g   = the stored grid of p (QDQ rule)
    out = RN32(fp64(I_pv) * (fp64(s_p) fp64(s_v))),  I_pv = sum_j (g - Z_p)(v_v - Z_v)  -- exact given g
The accuracy contract of p (DESIGN §4): |p - p64| <= EPS p64 + ALPHA, p64 the fp64 softmax of the same fp32 scores.
A grid value is admissible when it is the grid of some fp32 t within those bounds of p64.

The branch suites (test_gpu_int8_attention*_branches.py) share their inputs and output sentinels from here."""
import numpy as np

from int8_matmul_ref import BOUND, grid_offset, stored_grid
from oracle import qdq as oqdq

F32, F64 = np.float32, np.float64
EPS = 13 * 2.0 ** -24
ALPHA = 2.0 ** -125
SENTINEL = 1234.5   # out is pre-filled with this, TAIL elements past its end included
PSENT = 0x5A        # ... and p_q with this byte
TAIL = 64


def case_qkv(name, lead, tq, tk, d, dv):
    """(rng, q, k, v) of a branch case: standard normal q [*lead, Tq, d], k [*lead, Tk, d], v [*lead, Tk, dv], drawn in
    that order from a generator seeded by the case name, which the case goes on drawing from."""
    rng = np.random.default_rng(sum(map(ord, name)))
    q = rng.standard_normal(lead + (tq, d)).astype(F32)
    k = rng.standard_normal(lead + (tk, d)).astype(F32)
    v = rng.standard_normal(lead + (tk, dv)).astype(F32)
    return rng, q, k, v


def case_operands(q, k, v):
    """Operand tuples with scales from the largest magnitude, NaNs aside: q and k signed 8-bit at zero point 0, v
    unsigned 8-bit at zero point 7."""
    return ((q, F32(np.nanmax(np.abs(q)) / 127), F32(0), -128, 127),
            (k, F32(np.nanmax(np.abs(k)) / 127), F32(0), -128, 127),
            (v, F32(np.nanmax(np.abs(v)) / 255), F32(7), 0, 255))


def padded(k):
    return (k + 15) // 16 * 16


def stored_zero(z, qmin):
    return int(np.rint(F32(z))) - grid_offset(qmin)


def scores(q, k, scale=None):
    """The kernel's fp32 scores [..., Tq, Tk] from the int64 sums, and the NaN mask of the output rows (a NaN in row i
    of q, or anywhere in k of the entry)."""
    gq, nq = stored_grid(*q)
    gk, nk = stored_grid(*k)
    zq, zk = stored_zero(q[2], q[3]), stored_zero(k[2], k[3])
    i = np.matmul(gq - zq, np.swapaxes(gk - zk, -1, -2))
    s = (i.astype(F64) * (F64(F32(q[1])) * F64(F32(k[1])))).astype(F32)
    if scale is not None:
        s = (s * F32(scale)).astype(F32)
    bad = nq.any(-1) | nk.any((-1, -2))[..., None]
    return s, bad


def softmax64(s):
    """p64: the fp64 softmax of the fp32 scores along the keys."""
    s = s.astype(F64)
    e = np.exp(s - s.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def p_grid(t, p):
    """Stored grid of fp32 values t with p's qparams (s, z, qmin, qmax)."""
    return stored_grid(np.asarray(t, F32), *p)[0]


def admissible_range(p64, p):
    """(lo, hi): the stored grid values of p that the contract admits, elementwise."""
    lo = np.nextafter((p64 * (1 - EPS) - ALPHA).astype(F32), F32(-np.inf))
    hi = np.nextafter((p64 * (1 + EPS) + ALPHA).astype(F32), F32(np.inf))
    return p_grid(lo, p), p_grid(hi, p)


def stage3(pq, tk, p, v):
    """The integer form of p @ v on a given stored p grid pq [..., Tq, >= Tk] (int8), with v's NaN columns."""
    gv, nv = stored_grid(*v)
    zp, zv = stored_zero(p[1], p[2]), stored_zero(v[2], v[3])
    i = np.matmul(pq[..., :tk].astype(np.int64) - zp, gv - zv)
    y = (i.astype(F64) * (F64(F32(p[0])) * F64(F32(v[1])))).astype(F32)
    return np.where(nv.any(-2)[..., None, :], F32(np.nan), y)


def expected(pq, q, k, v, p, scale=None):
    """What the kernel must write given its own p grid: stage3 with the NaN rows of q / k."""
    _, bad = scores(q, k, scale)
    y = stage3(pq, k[0].shape[-2], p, v)
    return np.where(bad[..., None], F32(np.nan), y)


def truth(q, k, v, p, scale=None):
    """(T, f_p64 grid g64, the matmul bound term 2^-21 |f_p64| @ |f_v|, f_v): T = f_p64 @ f_v in fp64, f_p64 the QDQ of
    p64 with p's qparams."""
    s, _ = scores(q, k, scale)
    p64 = softmax64(s)
    fp = oqdq.qdq(p64.astype(F32), F32(p[0]), F32(p[1]), p[2], p[3]).astype(F64)
    fv = oqdq.qdq(*v).astype(F64)
    with np.errstate(all="ignore"):
        return np.matmul(fp, fv), p_grid(p64.astype(F32), p), BOUND * np.matmul(np.abs(fp), np.abs(fv)), fv


def truth_bound(g, g64, p, v, mm_bound):
    """|y - T| bound given the kernel's grid g: the matmul bound plus s_p s_v sum_j |g - g64| |v_v - Z_v| (with one
    fp32 rounding of slack)."""
    gv, _ = stored_grid(*v)
    zv = stored_zero(v[2], v[3])
    diff = np.matmul(np.abs(g.astype(np.int64) - g64), np.abs(gv - zv)).astype(F64)
    return mm_bound + diff * (F64(F32(p[0])) * F64(F32(v[1]))) * (1 + 2.0 ** -22)
