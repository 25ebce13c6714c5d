"""Chunked torch references for tests/test_gpu_far_end.py: the oracle's per-element terms restated in torch, so that
they run on the device over tensors of more than 2^31 elements, one bounded chunk at a time.

Every function takes a [outer, C, inner] view (per-tensor: [n, 1, 1]) and per-channel parameters of C entries, works on
CPU and CUDA tensors alike, and reduces in fp64.  Divisions are tensor / tensor: torch on CUDA turns a division by a
Python scalar into a multiplication by its reciprocal, which is not the correctly rounded quotient the oracle uses.
tests/test_gpu_far_end.py pins each restatement to its numpy oracle (oracle/qdq.py, oracle/observers.py) on a small
tensor."""
import torch

CHUNK = 1 << 25  # elements per reference chunk: a few hundred MB of fp64 temporaries


def slab_chunks(outer, slab, limit=CHUNK):
    """[o0, o1) ranges of whole slabs (slab = C * inner elements) of at most ``limit`` elements (one slab at least)."""
    per = max(limit // slab, 1)
    return [(o, min(o + per, outer)) for o in range(0, outer, per)]


def _bc(p):
    return p.reshape(1, -1, 1)


def ste_sums(x3, gy3, scale, zero_point, qmin, qmax, gzp_open_top=False):
    """oracle.qdq._ste_terms (round half to even) on one chunk: gx, and per channel the fp64 sums of the scale and
    zero-point terms and of their absolute values: (gx, gs, |gs| sum, gzp, |gzp| sum)."""
    s = _bc(scale)
    zp = torch.round(_bc(zero_point))
    q = x3 / s
    r = torch.round(q)
    vq = r + zp
    below = vq < qmin
    inside = (vq >= qmin) & (vq <= qmax)
    term = torch.where(inside, r - q, torch.where(below, qmin - zp, qmax - zp))
    g = gy3.double()
    gs_e = term.double() * g
    inside_z = inside & (vq < qmax) if gzp_open_top else inside
    gz_e = torch.where(inside_z, torch.zeros_like(g), (-s).double() * g)
    gx = torch.where(inside, gy3, torch.zeros_like(gy3))
    return gx, gs_e.sum((0, 2)), gs_e.abs().sum((0, 2)), gz_e.sum((0, 2)), gz_e.abs().sum((0, 2))


def clamp_sums(x, gy, lo, hi):
    """oracle.qdq.clamp_backward on one chunk: (gx, g_hi, g_lo, |g_hi| sum, |g_lo| sum), sums in fp64."""
    g = gy.double()
    zero = torch.zeros_like(g)
    above, under = x > hi, x < lo
    gx = torch.where((x >= lo) & (x <= hi), gy, torch.zeros_like(gy))
    gh, gl = torch.where(above, g, zero), torch.where(under, g, zero)
    return gx, gh.sum(), gl.sum(), gh.abs().sum(), gl.abs().sum()


def mse_sums(x2, cand_scale, cand_zp, qmin, qmax):
    """Per row and candidate, sum (x - xdq)^2 in fp64 with xdq the oracle's fake-quant value (oracle.qdq.qdq, fp32 op by
    op): the loss sb200_observe_mse_sweep approximates.  x2 [rows, len], candidates [rows, ncand] -> [rows, ncand]."""
    x64 = x2.double()
    out = torch.empty(cand_scale.shape, dtype=torch.float64, device=x2.device)
    for i in range(cand_scale.shape[1]):
        s = cand_scale[:, i:i + 1]
        zp = torch.round(cand_zp[:, i:i + 1])
        v = torch.clamp(torch.round(x2 / s) + zp, qmin, qmax)
        d = x64 - ((v - zp) * s).double()
        out[:, i] = (d * d).sum(1)
    return out


def sel_keys(x, key_mode):
    """sel_key (csrc/observe.cu): the enc_f32 total order (-0 < +0) of x, or of |x| with key_mode 1, as int64 in
    [0, 2^32); NaN is the largest key."""
    v = x.abs() if key_mode else x
    b = v.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    k = torch.where(b >= 0x80000000, 0xFFFFFFFF - b, b | 0x80000000)
    return torch.where(torch.isnan(x), torch.full_like(k, 0xFFFFFFFF), k)
