"""Every branch of the fused integer-grid attention (csrc/int8_attention.cu): one named case per branch of
tests/int8_attention_geometry.py, run through the C-ABI into sentinel-filled outputs (a tail past the end of out and
p_q checks that nothing is written beyond them) and through ops.int8_attention, which must agree.  Each output must
equal the integer form of p @ v on the kernel's own p grid, bit for bit, every p grid value must be admissible, and a
repeat must be bit-identical."""
import numpy as np
import pytest
import torch

import int8_attention_geometry as geo
import int8_attention_ref as ref
from gpu_util import dev, t
from int8_attention_ref import PSENT, SENTINEL, TAIL
from sparsebit_b200 import _lib, ops

F32 = np.float32

# name -> (batch, tq, tk, d, dv, p_q, scale, p_signed, ramp, spread, nan)
CASES = {
    "tiny": (2, 1, 1, 8, 8, True, None, False, False, False, ()),
    "q_tail_key_tail": (2, 70, 100, 40, 40, True, 0.125, False, False, False, ()),
    "full_tiles": (1, 256, 256, 128, 128, True, None, True, False, False, ()),
    "ring_wraps_ramp": (2, 65, 700, 64, 64, True, 0.125, False, True, False, ()),
    "dv_odd_k16_pad": (1, 129, 131, 100, 33, True, None, True, False, False, ()),
    "p_q_off": (3, 197, 197, 64, 64, False, 0.125, False, False, False, ()),
    "spread_underflow": (1, 64, 300, 32, 16, True, 4.0, False, False, True, ()),
    "nan_all": (3, 40, 150, 24, 20, True, None, False, False, False, ("q", "k", "v")),
}


def case_branches(c):
    batch, tq, tk, d, dv, p_q, scale, p_signed, ramp, spread, nan = c
    return geo.branches(batch, tq, tk, d, dv, p_q, scale, p_signed, ramp, spread, nan)


def _inputs(name):
    batch, tq, tk, d, dv, p_q, scale, p_signed, ramp, spread, nan = CASES[name]
    _, q, k, v = ref.case_qkv(name, (batch,), tq, tk, d, dv)
    if ramp:  # later keys score higher: the running max of a row grows block by block
        k = (k * 0.2 + np.linspace(0, 3, tk, dtype=F32)[None, :, None] * np.sign(q.mean(1, keepdims=True))).astype(F32)
    if spread:
        q *= 3
    ops_ = ref.case_operands(q, k, v)
    p = (F32(1 / 127), F32(0), -128, 127) if p_signed else (F32(1 / 255), F32(0), 0, 255)
    for o in nan:
        x = ops_["qkv".index(o)][0]
        x[batch - 1, x.shape[1] // 2, x.shape[2] - 1] = np.nan
    return ops_, p, scale, p_q


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_branch_case(name):
    (q, k, v), p, scale, with_p = _inputs(name)
    batch, tq, d = q[0].shape
    tk, dv = v[0].shape[1:]
    tkp = ref.padded(tk)
    lib = _lib.load()
    dt = lambda x: torch.tensor([x], dtype=torch.float32, device=dev())
    qt, kt, vt = t(q[0]), t(k[0]), t(v[0])
    sc = [dt(o[1]) for o in (q, k)] + [dt(p[0])] + [dt(v[1])]
    zp = [dt(o[2]) for o in (q, k)] + [dt(p[1])] + [dt(v[2])]
    rng_ = [o[3:] for o in (q, k)] + [p[2:]] + [v[3:]]
    out = torch.full((batch * tq * dv + TAIL,), SENTINEL, dtype=torch.float32, device=dev())
    pq = torch.full((batch * tq * tkp + TAIL,), PSENT, dtype=torch.int8, device=dev())
    ws_bytes = int(lib.sb200_int8_attention_workspace_bytes(batch, tq, tk, d, dv))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    args = [qt.data_ptr(), kt.data_ptr(), vt.data_ptr()]
    for i in range(4):
        args += [sc[i].data_ptr(), zp[i].data_ptr(), int(rng_[i][0]), int(rng_[i][1])]
    args += [int(scale is not None), float(scale or 1.0), out.data_ptr(), pq.data_ptr() if with_p else None,
             batch, tq, tk, d, dv, ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream]
    assert lib.sb200_int8_attention(*args) == 0, lib.sb200_last_error()
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.all(o[batch * tq * dv:] == SENTINEL)  # nothing past the output
    y = o[:batch * tq * dv].reshape(batch, tq, dv)
    assert not np.any(y == SENTINEL)  # every element written
    # the ops wrapper computes the same, and so does a repeat
    qp = [(sc[i], zp[i], rng_[i]) for i in range(4)]
    y_ops, pq_ops = ops.int8_attention(qt, kt, vt, *qp, scale=scale, return_p=True)
    assert np.array_equal(y, y_ops.cpu().numpy(), equal_nan=True)
    assert lib.sb200_int8_attention(*args) == 0
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy()[:batch * tq * dv].reshape(batch, tq, dv), y, equal_nan=True)
    g = pq_ops.cpu().numpy()
    if with_p:
        pa = pq.cpu().numpy()
        assert np.all(pa[batch * tq * tkp:] == PSENT)
        assert np.array_equal(pa[:batch * tq * tkp].reshape(batch, tq, tkp), g)
    assert not g[..., tk:].any()
    # exact stage 3 on the kernel's own grid, admissible grid values on the rows without NaN
    assert np.array_equal(y, ref.expected(g, q, k, v, p, scale), equal_nan=True)
    s, bad = ref.scores(q, k, scale)
    lo, hi = ref.admissible_range(ref.softmax64(s), p)
    gg = g[..., :tk].astype(np.int64)
    assert np.all(((gg >= lo) & (gg <= hi))[~bad])
    if "max_rescaled" in case_branches(CASES[name]):  # the ramp really moves the max past the first block
        row_max = s.argmax(-1)
        assert np.any(row_max >= geo.KEYS)
    if "exp_underflow" in case_branches(CASES[name]):
        assert np.any(s.max(-1, keepdims=True) - s > 104)

