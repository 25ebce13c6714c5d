"""Every branch of the masked fused attention (int8_attention_kernel<true>, csrc/int8_attention.cu): one named case
per branch of tests/int8_attention_mask_ref.py, run through the C-ABI into sentinel-filled outputs (a tail past the
end of out and p_q checks that nothing is written beyond them) and through ops.int8_attention, which must agree.
Each output must equal the integer form of p @ v on the kernel's own p grid, bit for bit, every p grid value must be
admissible, the keys whose p is exactly 0 (hidden, or skipped) must hold the grid of 0 in p_q, and a repeat must be
bit-identical."""
import numpy as np
import pytest
import torch

import int8_attention_mask_ref as mref
import int8_attention_ref as ref
from gpu_util import dev, t
from int8_attention_ref import PSENT, SENTINEL, TAIL
from int8_harness import check_p
from sparsebit_b200 import _lib, ops

F32 = np.float32

# name -> (heads, entries per head group, tq, tk, d, dv, mask_kind, causal, p_q, nan); batch = entries * heads
CASES = {
    "padding_two_level": (2, 2, 70, 150, 40, 40, "row_two_level", False, True, ()),
    "full_mask": (1, 3, 65, 200, 64, 33, "full", False, True, ()),
    "causal_square": (1, 2, 300, 300, 64, 64, None, True, True, ()),
    "causal_tq_gt_tk": (1, 2, 300, 100, 32, 16, None, True, True, ()),
    "causal_one_row": (1, 2, 1, 700, 128, 128, None, True, True, ()),
    "causal_padded_nan": (3, 2, 256, 256, 64, 40, "row_two_level", True, True, ("k_hidden", "v_hidden")),
    "causal_p_q_off": (1, 1, 260, 260, 64, 64, "full", True, False, ()),
}


def case_branches(c):
    heads, entries, tq, tk, d, dv, mask_kind, causal, p_q, nan = c
    return mref.branches(heads * entries, tq, tk, mask_kind, causal, p_q, nan)


def _inputs(name):
    heads, entries, tq, tk, d, dv, mask_kind, causal, p_q, nan = CASES[name]
    lead = (entries, heads)
    rng, q, k, v = ref.case_qkv(name, lead, tq, tk, d, dv)
    mask = None
    if mask_kind is not None and mask_kind.startswith("row"):  # key padding per entry, broadcast over heads and rows
        mask = np.zeros((entries, 1, 1, tk), F32)
        for e in range(entries):
            mask[e, ..., tk - (e + 1) * tk // 5:] = -np.inf if e % 2 else -10000.0
    elif mask_kind == "full":
        mask = (rng.standard_normal(lead + (tq, tk)) * 2).astype(F32)
        mask[rng.random(mask.shape) < 0.2] = -np.inf
    if "k_hidden" in nan:  # key 200 of the last entry: hidden by causal from rows < 200
        k[-1, -1, 200, 3] = np.nan
    if "v_hidden" in nan:
        v[-1, -1, 220, 5] = np.nan
    p = (F32(1 / 255), F32(0), 0, 255)
    return lead, ref.case_operands(q, k, v), p, 0.125, mask, causal, p_q


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_branch_case(name):
    lead, (q, k, v), p, scale, mask, causal, with_p = _inputs(name)
    tq, d = q[0].shape[-2:]
    tk, dv = v[0].shape[-2:]
    batch = int(np.prod(lead))
    tkp = ref.padded(tk)
    lib = _lib.load()
    dt = lambda x: torch.tensor([x], dtype=torch.float32, device=dev())
    qt, kt, vt = t(q[0]), t(k[0]), t(v[0])
    mt = t(mask) if mask is not None else None
    sc = [dt(o[1]) for o in (q, k)] + [dt(p[0])] + [dt(v[1])]
    zp = [dt(o[2]) for o in (q, k)] + [dt(p[1])] + [dt(v[2])]
    rng_ = [o[3:] for o in (q, k)] + [p[2:]] + [v[3:]]
    out = torch.full((batch * tq * dv + TAIL,), SENTINEL, dtype=torch.float32, device=dev())
    pq = torch.full((batch * tq * tkp + TAIL,), PSENT, dtype=torch.int8, device=dev())
    ws_bytes = int(lib.sb200_int8_attention_masked_workspace_bytes(batch, tq, tk, d, dv, int(causal)))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    args = [qt.data_ptr(), kt.data_ptr(), vt.data_ptr()]
    for i in range(4):
        args += [sc[i].data_ptr(), zp[i].data_ptr(), int(rng_[i][0]), int(rng_[i][1])]
    if mt is not None:
        so, si, inner, sr = ops.attention_mask_strides(mt.shape, mt.stride(), lead, tq, tk)
        if CASES[name][6].endswith("two_level"):
            assert inner > 1 and so > 0  # the view really uses both levels
        margs = [mt.data_ptr(), so, si, inner, sr]
    else:
        margs = [None, 0, 0, 1, 0]
    args += [1, scale] + margs + [int(causal), out.data_ptr(), pq.data_ptr() if with_p else None,
                                  batch, tq, tk, d, dv, ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream]
    assert lib.sb200_int8_attention_masked(*args) == 0, lib.sb200_last_error()
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.all(o[batch * tq * dv:] == SENTINEL)  # nothing past the output
    y = o[:batch * tq * dv].reshape(lead + (tq, dv))
    assert not np.any(y == SENTINEL)  # every element written
    qp = [(sc[i], zp[i], rng_[i]) for i in range(4)]
    y_ops, pq_ops = ops.int8_attention(qt, kt, vt, *qp, scale=scale, return_p=True, attn_mask=mt, causal=causal)
    assert np.array_equal(y, y_ops.cpu().numpy(), equal_nan=True)
    assert lib.sb200_int8_attention_masked(*args) == 0
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy()[:batch * tq * dv].reshape(y.shape), y, equal_nan=True)
    g = pq_ops.cpu().numpy()
    if with_p:
        pa = pq.cpu().numpy()
        assert np.all(pa[batch * tq * tkp:] == PSENT)
        assert np.array_equal(pa[:batch * tq * tkp].reshape(g.shape), g)
    assert np.array_equal(y, mref.expected(g, q, k, v, p, scale, mask, causal), equal_nan=True)
    s, bad = mref.scores(q, k, scale, mask, causal)
    check_p(g, s, bad, p, tq, tk, causal, name)
    br = case_branches(CASES[name])
    if "rows_without_keys" in br:
        assert np.isnan(y[..., :tq - tk, :]).all() and not np.isnan(y[..., tq - tk:, :]).any()
    if "nan_k_hidden" in br:  # rows 200.. of the last entry see the NaN key; the rows before do not
        assert np.isnan(y[-1, -1, 200:]).all()
        assert not np.isnan(y[-1, -1, :200, np.arange(dv) != 5]).any()
    if "nan_v_hidden" in br:  # column 5 is NaN in every row, also those that do not see key 220
        assert np.isnan(y[-1, -1, :, 5]).all()
