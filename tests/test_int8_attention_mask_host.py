"""CPU: the host side of sb200_int8_attention_masked, the mask addressing of ops.int8_attention
(ops.attention_mask_strides), the masked and causal QAttention composition, hand-checked cases of
tests/int8_attention_mask_ref.py and the coverage of the masked branch cases.

* Every bad argument of the masked entry point is rejected on the host before any CUDA call (there is no device here).
* Its workspace query is a pure function: that of sb200_int8_attention, plus the causal column sums of v; the query of
  sb200_int8_attention keeps its values."""
import numpy as np
import pytest
import torch

import int8_attention_mask_ref as mref
import int8_attention_ref as ref
from int8_harness import E_INVALID, E_UNSUPPORTED, E_WORKSPACE, buf, rejector
from sparsebit_b200 import _lib, ops
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.modules import QAttention
from sparsebit_b200.quantization.tools import trace_quant_model
from test_gpu_int8_attention_mask_branches import CASES, case_branches

F32 = np.float32


# q k v | q: s z lo hi | k: s z lo hi | p: s z lo hi | v: s z lo hi | has_scale scale |
# mask so si inner sr causal | out p_q | b tq tk d dv | ws ws_bytes stream
def _ok_args(p, ws_bytes, causal=1):
    return [p, p, p, p, p, -128, 127, p, p, -128, 127, p, p, 0, 255, p, p, -128, 127, 1, 0.125,
            p, 7, 0, 3, 0, causal, p, p, 6, 5, 7, 64, 32, p, ws_bytes, None]


def test_masked_entry_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    ws_ok = int(lib.sb200_int8_attention_masked_workspace_bytes(6, 5, 7, 64, 32, 1))
    ok = _ok_args(p, ws_ok)
    rejected = rejector(lib.sb200_int8_attention_masked, ok, prefix=b"sb200_int8_attention_masked")
    for i in (0, 1, 2, 3, 4, 7, 8, 11, 12, 15, 16, 27, 34):  # null pointers (the mask, 21, and p_q, 28, may be null)
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    for i in range(29, 34):
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
    rejected(E_UNSUPPORTED, b"d <= 128", a32=129)
    rejected(E_INVALID, b"wider than 8 bits", a13=-128, a14=128)
    rejected(E_INVALID, b"not finite", a20=float("nan"))
    rejected(E_INVALID, b"16-byte aligned", a28=p + 2)
    for bad in (2, -1, 7):  # causal
        rejected(E_INVALID, b"causal must be 0 or 1", a26=bad)
    for i in (22, 23, 25):  # the three strides
        rejected(E_INVALID, b"negative mask stride", **{f"a{i}": -1})
    for inner in (0, -3, 4, 5):  # mask_inner: positive and dividing batch = 6
        rejected(E_INVALID, b"mask_inner", a24=inner)
    for off in (1, 2, 3):
        rejected(E_INVALID, b"4-byte aligned", a21=p + off)
    rejected(E_INVALID, b"2^62", a22=1 << 62)  # (6 / 3 - 1) 2^62 + ... >= 2^62
    rejected(E_WORKSPACE, b"workspace too small", a35=ws_ok - 1)
    # without a mask the four mask arguments are not read; without causal the column sums are not needed
    assert lib.sb200_int8_attention_masked(*(ok[:21] + [None, -1, -1, 0, -1] + ok[26:35] + [0, None])) == E_WORKSPACE
    assert b"workspace too small" in lib.sb200_last_error()
    ws0 = int(lib.sb200_int8_attention_masked_workspace_bytes(6, 5, 7, 64, 32, 0))
    assert lib.sb200_int8_attention_masked(*(ok[:26] + [0] + ok[27:35] + [ws0 - 1, None])) == E_WORKSPACE
    rejected(E_WORKSPACE, b"workspace too small", a26=1, a35=ws0)  # causal needs the column sums on top


def _layout_total(b, tq, tk, d, dv):
    """csrc/int8_attention.cu at_layout: the three stored operands with their sums and NaN flags."""
    up = lambda x, a: (x + a - 1) // a * a
    o = 0
    for rows, width in ((b * tq, ref.padded(d)), (b * tk, ref.padded(d)), (b * dv, ref.padded(tk))):
        o = up(o + rows * width, 256)
        o = up(o + rows * 4, 256)
        o = up(o + rows, 1024)
    return o


SHAPES = [(1, 1, 1, 1, 1), (768, 197, 197, 64, 64), (2, 16384, 16384, 64, 64), (1, 3, (1 << 17) - 1, 128, 128),
          (96, 1024, 1024, 64, 64), (5, 7, 300, 40, 33)]


@pytest.mark.parametrize("shape", SHAPES)
def test_workspace_queries(shape):
    lib = _lib.load()
    b, tq, tk, d, dv = shape
    old = int(lib.sb200_int8_attention_workspace_bytes(*shape))
    assert old == _layout_total(*shape) + 1024  # the unmasked query keeps its values
    assert lib.sb200_int8_attention_masked_workspace_bytes(*shape, 0) == old
    extra = (b * dv * mref.cdiv(tk, 128) * 4 + 1023) // 1024 * 1024
    assert all(lib.sb200_int8_attention_masked_workspace_bytes(*shape, 1) == old + extra for _ in range(3))


def test_masked_workspace_query_rejections():
    q = _lib.load().sb200_int8_attention_masked_workspace_bytes
    for causal in (0, 1):
        assert q(0, 5, 7, 64, 32, causal) == 0 and q(1, 5, 7, 129, 32, causal) == 0
        assert q(1, 5, 1 << 17, 64, 32, causal) == 0 and q(1 << 20, 1 << 11, 7, 64, 32, causal) == 0
    assert q(1, 5, 7, 64, 32, 2) == 0 and q(1, 5, 7, 64, 32, -1) == 0


# ---------------------------------------------------------------------------------------------- mask addressing
def _plan(mask, lead, tq, tk):
    return ops.attention_mask_strides(mask.shape, mask.stride(), lead, tq, tk)


def _addressed(plan, mask_flat, lead, tq, tk):
    """The [*lead, Tq, Tk] values the kernel reads through ``plan`` from the flat storage."""
    so, si, inner, sr = plan
    batch = int(np.prod(lead)) if lead else 1
    b = np.arange(batch)[:, None, None]
    off = (b // inner) * so + (b % inner) * si + np.arange(tq)[None, :, None] * sr + np.arange(tk)[None, None, :]
    return mask_flat[off].reshape(tuple(lead) + (tq, tk))


@pytest.mark.parametrize("shape,lead,view", [
    ((4, 1, 1, 50), (4, 3), (50, 0, 3, 0)),        # BERT key padding over [B, H]
    ((4, 3, 20, 50), (4, 3), (1000, 0, 1, 50)),     # a full mask: the two batch dimensions fold into one
    ((1, 1, 20, 50), (4, 3), (0, 0, 1, 50)),        # one mask for every entry
    ((20, 50), (4, 3), (0, 0, 1, 50)),
    ((4, 1, 20, 50), (4, 3), (1000, 0, 3, 50)),     # per entry, broadcast over heads
    ((1, 3, 1, 50), (4, 3), (0, 50, 3, 0)),         # per head
    ((50,), (2,), (0, 0, 1, 0)),
    ((2, 1, 50), (2,), (50, 0, 1, 0)),
    ((1, 50), (), (0, 0, 1, 0)),
])
def test_mask_strides_are_views(shape, lead, view):
    tq, tk = 20, 50
    mask = torch.randn(shape)
    plan = _plan(mask, lead, tq, tk)
    assert plan == view
    want = mask.expand(tuple(lead) + (tq, tk)).numpy()
    assert np.array_equal(_addressed(plan, mask.reshape(-1).numpy(), lead, tq, tk), want)


def test_mask_strides_that_need_a_copy():
    tq, tk = 20, 50
    assert _plan(torch.randn(4, 3, 50, 20).transpose(-2, -1), (4, 3), tq, tk) is None  # key stride 20
    assert _plan(torch.randn(4, 3, 20, 1), (4, 3), tq, tk) is None  # broadcast along the keys
    assert _plan(torch.randn(4, 1, 2, 20, 50), (4, 3, 2), tq, tk) is None  # three batch levels
    assert _plan(torch.randn(4, 3, 2, 20, 50), (4, 3, 2), tq, tk) == (1000, 0, 1, 50)  # contiguous: they fold
    assert _plan(torch.randn(3, 1, 20, 50).transpose(0, 1), (1, 3), tq, tk) == (1000, 0, 1, 50)
    assert _plan(torch.randn(4, 3, 20, 1), (4, 3), tq, 1) == (20, 0, 1, 1)  # Tk = 1: any key stride
    for bad in ((4, 3, 20, 49), (5, 1, 1, 50), (2, 4, 3, 20, 50)):
        with pytest.raises(ValueError, match="does not broadcast"):
            _plan(torch.randn(bad), (4, 3), tq, tk)


def test_bool_and_non_float_masks_are_rejected():
    with pytest.raises(TypeError, match="additive float mask"):
        ops.attention_mask_check(torch.ones(2, 3, dtype=torch.bool))
    for dt in (torch.int32, torch.float64, torch.uint8):
        with pytest.raises(TypeError, match="float32, float16 or bfloat16"):
            ops.attention_mask_check(torch.zeros(2, 3, dtype=dt))
    with pytest.raises(TypeError, match="tensor"):
        ops.attention_mask_check([0.0, -1e4])
    h = torch.tensor([0.0, -10000.0, float("-inf"), 0.1], dtype=torch.float16)
    assert ops.attention_mask_check(h).dtype == torch.float32 and torch.equal(ops.attention_mask_check(h), h.float())
    m = _plain_qattention(0.5)
    q, k, v = torch.randn(1, 2, 4), torch.randn(1, 3, 4), torch.randn(1, 3, 2)
    with pytest.raises(TypeError, match="bool mask"):
        m(q, k, v, attn_mask=torch.ones(1, 2, 3, dtype=torch.bool))


# ---------------------------------------------------------------------------------------------- the composition
def _plain_qattention(scale):
    m = QAttention(scale=scale)  # quantizers off: plain softmax attention
    for c in (m.qk.left, m.qk.right, m.pv.left, m.pv.right):
        c.build_quantizer(sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature"))
        c.set_quant(a_quant=False)
    return m


def _plain(q, k, v, scale, mask, causal):
    s = (q @ k.transpose(-2, -1)) * scale
    tq, tk = s.shape[-2:]
    if causal:  # bottom-right: the last query row sees every key
        s = torch.where(torch.ones(tq, tk, dtype=torch.bool).tril(tk - tq), s, float("-inf"))
    if mask is not None:
        s = s + mask.float()
    return torch.softmax(s, -1) @ v


@pytest.mark.parametrize("tq,tk", [(6, 6), (3, 9), (9, 3), (1, 7), (1, 1)])
@pytest.mark.parametrize("kind", ["causal", "padding", "causal+padding", "full_fp16"])
def test_qattention_masked_forward_is_the_composition(tq, tk, kind):
    torch.manual_seed(tq * 31 + tk)
    m = _plain_qattention(0.5)
    q, k, v = torch.randn(2, 3, tq, 8), torch.randn(2, 3, tk, 8), torch.randn(2, 3, tk, 5)
    causal = kind.startswith("causal")
    mask = None
    if "padding" in kind:
        keep = torch.ones(2, 1, 1, tk)
        keep[1, ..., tk // 2:] = 0
        mask = (1 - keep) * -10000.0
    if kind == "full_fp16":
        mask = torch.randn(2, 3, tq, tk).half()
    y = m(q, k, v, attn_mask=mask, causal=causal)
    want = _plain(q, k, v, 0.5, mask, causal)
    assert torch.equal(torch.isnan(y), torch.isnan(want))
    assert torch.allclose(y.nan_to_num(), want.nan_to_num(), rtol=1e-6, atol=1e-6)
    if causal and tq > tk:  # the first Tq - Tk rows see no key
        assert torch.isnan(y[..., :tq - tk, :]).all() and not torch.isnan(y[..., tq - tk:, :]).any()
    # the reference restates the same masked scores, bit for bit
    s = (q @ k.transpose(-2, -1) * 0.5).numpy()
    s_t = (q @ k.transpose(-2, -1)) * 0.5
    if causal:
        s_t = s_t.masked_fill(~torch.ones(tq, tk, dtype=torch.bool).tril(tk - tq), float("-inf"))
    if mask is not None:
        s_t = s_t + mask.float()
    assert np.array_equal(mref.masked(s, None if mask is None else mask.float().numpy(), causal), s_t.numpy())
    assert torch.equal(m(q, k, v), _plain(q, k, v, 0.5, None, False))  # the unmasked call is unchanged


def test_qattention_masked_traces_as_one_call():
    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.attn = _plain_qattention(0.25)

        def forward(self, x, mask):
            return self.attn(x, x, x, attn_mask=mask, causal=True)

    blk = Block()
    gm = trace_quant_model(blk)
    calls = [n.target.__name__ for n in gm.graph.nodes if n.op == "call_function"]
    assert "masked_scores" in calls
    leaves = [n.target for n in gm.graph.nodes if n.op == "call_module"]
    assert leaves == ["attn.qk.left", "attn.qk.right", "attn.pv.left", "attn.pv.right"]
    x, mask = torch.randn(2, 5, 4), torch.zeros(2, 1, 5)
    mask[0, 0, 3:] = float("-inf")
    assert torch.equal(gm(x, mask), blk(x, mask))


# ---------------------------------------------------------------------------------------------- the reference by hand
def test_reference_by_hand():
    # one entry, Tq = 2, Tk = 3, scores all 1 on a scale-1 grid (q = k rows = [1, 0])
    q = (np.array([[[1, 0], [1, 0]]], F32), F32(1), F32(0), -128, 127)
    k = (np.array([[[1, 0], [1, 0], [1, 0]]], F32), F32(1), F32(0), -128, 127)
    v = (np.array([[[3], [6], [9]]], F32), F32(1), F32(0), -128, 127)
    # causal, bottom-right: row 0 sees keys 0, 1; row 1 sees all three
    assert np.array_equal(mref.visible(2, 3, True), [[True, True, False], [True, True, True]])
    mask = np.array([[[0, -np.inf, 0]]], F32)  # key padding of key 1
    s, bad = mref.scores(q, k, None, mask, True)
    assert np.array_equal(s, np.array([[[1, -np.inf, -np.inf], [1, -np.inf, 1]]], F32)) and not bad.any()
    p64 = mref.softmax64(s)
    assert np.array_equal(p64, [[[1, 0, 0], [0.5, 0, 0.5]]])
    p = (F32(1 / 200), F32(0), 0, 255)  # p = 1 -> 200, 0.5 -> 100, 0 -> 0 (stored minus 128)
    T, g64, _, _ = mref.truth(q, k, v, p, None, mask, True)
    assert np.array_equal(g64, [[[72, -128, -128], [-28, -128, -28]]]) and mref.p_zero_grid(p) == -128
    assert np.allclose(T[..., 0], [[3, 6]], rtol=1e-6)
    pq = np.zeros((1, 2, 16), np.int8)
    pq[..., :3] = g64
    y = mref.expected(pq, q, k, v, p, None, mask, True)
    assert np.array_equal(y, (np.array([[[600.0], [1200.0]]]) * np.float64(F32(1 / 200))).astype(F32))
    # a NaN at key 2 reaches row 1 only; a NaN v at key 2 still poisons column 0 of both rows
    kn = (k[0].copy(),) + k[1:]
    kn[0][0, 2, 1] = np.nan
    assert np.array_equal(mref.scores(q, kn, None, None, True)[1], [[False, True]])
    vn = (v[0].copy(),) + v[1:]
    vn[0][0, 2, 0] = np.nan
    assert np.isnan(mref.expected(pq, q, k, vn, p, None, mask, True)).all()
    # Tq > Tk: the first rows see no key and are NaN; the fp32 add rounds
    s, bad = mref.scores(q, (k[0][:, :1],) + k[1:], None, None, True)
    assert np.array_equal(bad, [[True, False]])
    assert mref.masked(np.array([[1.0]], F32), np.array([[2.0 ** -30]], F32))[0, 0] == F32(1)


def test_launch_plan_by_hand():
    assert mref.visited_blocks(1024, 1024, True) == [1, 2, 3, 4, 5, 6, 7, 8]  # 36 of 64 pairs: 28 skipped
    assert sum(mref.visited_blocks(1024, 1024, True)) == 36
    assert mref.visited_blocks(1024, 1024, False) == [8] * 8
    assert mref.visited_blocks(300, 100, True) == [0, 1, 1]  # Tq > Tk: the first tile sees no key
    assert mref.visited_blocks(1, 700, True) == [6]  # Tq = 1: the one row sees every key
    assert mref.visited_blocks(200, 1200, True) == [9, 10]
    sk = mref.skipped(256, 256, True)
    assert not sk[128:].any() and sk[:128, 128:].all() and not sk[:128, :128].any()
    assert not (sk & mref.visible(256, 256, True)).any()  # a skipped key is hidden from its row


# ---------------------------------------------------------------------------------------------- branch coverage
def test_branch_cases_reach_every_branch():
    reached = set().union(*(case_branches(c) for c in CASES.values()))
    assert reached == set(mref.ALL), sorted(set(mref.ALL) - reached)
