"""CPU: the host side of sb200_int8_attention, the eligibility rules of QAttentionInt8.from_qattention, what
calibration sees of a QAttention, hand-checked cases of the numpy reference (tests/int8_attention_ref.py) and the
coverage of the branch cases (tests/int8_attention_geometry.py).

* Every bad argument is rejected on the host before any CUDA call (there is no device here), with its code and the
  message of its check (csrc/int8_attention.cu: sb200_int8_attention and check_dims).
* The workspace query is a pure, monotone function of (batch, tq, tk, d, dv), O(batch (tq + tk) d + batch dv tk)."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_attention_geometry as geo
import int8_attention_ref as ref
from int8_harness import E_INVALID, E_UNSUPPORTED, E_WORKSPACE, buf, refusal, rejector
from oracle import qdq as oqdq
from sparsebit_b200 import _lib
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.common import Backend
from sparsebit_b200.quantization.modules import (QAttention, QAttentionInt8, QIdentity, QLinear, QMatMul,
                                                 QMatMulInt8, int8_attention_ineligibility)
from sparsebit_b200.quantization.tools import (CalibrationRunner, to_integer_attentions, to_integer_matmuls,
                                               trace_quant_model)
from sparsebit_b200.quantization.tools.calibration import _is_quant_opr
from test_gpu_int8_attention_branches import CASES, case_branches

F32 = np.float32


def test_attention_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    ws_ok = int(lib.sb200_int8_attention_workspace_bytes(3, 5, 7, 64, 32))
    # q k v | q: s z lo hi | k: s z lo hi | p: s z lo hi | v: s z lo hi | has_scale scale out p_q | b tq tk d dv | ws ws_bytes stream
    ok = [p, p, p, p, p, -128, 127, p, p, -128, 127, p, p, 0, 255, p, p, -128, 127, 1, 0.125, p, p, 3, 5, 7, 64, 32, p,
          ws_ok, None]
    rejected = rejector(lib.sb200_int8_attention, ok)
    for i in (0, 1, 2, 3, 4, 7, 8, 11, 12, 15, 16, 21, 28):  # null pointers (p_q, 22, may be null)
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    for i in range(23, 28):  # check_dims: an empty dimension
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
        rejected(E_INVALID, b"empty operand", **{f"a{i}": -3})
    rejected(E_UNSUPPORTED, b"d <= 128", a26=129)  # check_dims: the limits
    rejected(E_UNSUPPORTED, b"dv <= 128", a27=129)
    rejected(E_UNSUPPORTED, b"Tk < 2^17", a25=1 << 17)
    rejected(E_INVALID, b"too large", a23=1 << 20, a24=1 << 11)  # batch Tq = 2^31
    rejected(E_INVALID, b"too large", a23=1 << 20, a25=1 << 11)  # batch Tk = 2^31
    for lo, hi in ((5, 6), (9, 10), (13, 14), (17, 18)):  # check_range of each of the four operands
        rejected(E_INVALID, b"wider than 8 bits", **{f"a{lo}": -128, f"a{hi}": 128})
        rejected(E_INVALID, b"qmin", **{f"a{lo}": 5, f"a{hi}": 4})
        rejected(E_INVALID, b"neither signed", **{f"a{lo}": -129, f"a{hi}": 0})
    for bad in (float("inf"), float("-inf"), float("nan"), 1e39):  # the scale (1e39 is inf as a float)
        rejected(E_INVALID, b"not finite", a20=bad)
    assert lib.sb200_int8_attention(*(ok[:19] + [0, float("nan")] + ok[21:22] + [None] + ok[23:29] + [0, None])) \
        == E_WORKSPACE  # without has_scale the scale is not read
    rejected(E_INVALID, b"16-byte aligned", a22=p + 2)  # p_q
    rejected(E_WORKSPACE, b"workspace too small", a29=ws_ok - 1)
    rejected(E_WORKSPACE, b"workspace too small", a29=0)


def test_workspace_query_is_pure_and_monotone():
    q = _lib.load().sb200_int8_attention_workspace_bytes
    assert q(0, 5, 7, 64, 32) == 0 and q(1, 0, 7, 64, 32) == 0 and q(1, 5, 0, 64, 32) == 0
    assert q(1, 5, 7, 0, 32) == 0 and q(1, 5, 7, 64, -1) == 0
    assert q(1, 5, 7, 129, 32) == 0 and q(1, 5, 7, 64, 129) == 0 and q(1, 5, 1 << 17, 64, 32) == 0
    assert q(1 << 20, 1 << 11, 7, 64, 32) == 0
    for b, tq, tk, d, dv in [(1, 1, 1, 1, 1), (768, 197, 197, 64, 64), (2, 16384, 16384, 64, 64), (1, 3, (1 << 17) - 1, 128, 128)]:
        first = q(b, tq, tk, d, dv)
        dp, tkp = ref.padded(d), ref.padded(tk)
        assert first >= b * ((tq + tk) * (dp + 5) + dv * (tkp + 5))
        assert first <= b * ((tq + tk) * (dp + 5) + dv * (tkp + 5)) + 4096 * 3 + 1024  # no [Tq, Tk] term
        assert all(q(b, tq, tk, d, dv) == first for _ in range(3))
        assert q(b + 1, tq, tk, d, dv) >= first and q(b, tq + 1, tk, d, dv) >= first
        assert q(b, tq, tk, min(d + 1, 128), dv) >= first and q(b, tq, tk, d, min(dv + 1, 128)) >= first
        if tk + 1 < 1 << 17:
            assert q(b, tq, tk + 1, d, dv) >= first


# ---------------------------------------------------------------------------------------------- the reference by hand
def test_reference_by_hand():
    # q = [[1, 0]], k = [[1, 0], [0, 1]] on a scale-1 grid: scores [1, 0]; p = [e, 1] / (e + 1)
    q = (np.array([[[1, 0]]], F32), F32(1), F32(0), -128, 127)
    k = (np.array([[[1, 0], [0, 1]]], F32), F32(1), F32(0), -128, 127)
    v = (np.array([[[2, 0], [0, 4]]], F32), F32(1), F32(0), -128, 127)
    s, bad = ref.scores(q, k)
    assert np.array_equal(s, np.array([[[1, 0]]], F32)) and not bad.any()
    p64 = ref.softmax64(s)
    assert np.allclose(p64, [[[np.e / (np.e + 1), 1 / (np.e + 1)]]], rtol=0, atol=1e-15)
    # p on an unsigned grid of step 1/100: 0.7311 -> 73, 0.2689 -> 27 (stored minus 128)
    p = (F32(0.01), F32(0), 0, 255)
    T, g64, mm, fv = ref.truth(q, k, v, p)
    assert np.array_equal(g64, np.array([[[73 - 128, 27 - 128]]]))
    pq = np.zeros((1, 1, 16), np.int8)
    pq[..., :2] = g64
    y = ref.expected(pq, q, k, v, p)
    # I = (73 * 2, 27 * 4), times fp64(fp32(0.01)), one fp32 rounding each
    assert np.array_equal(y, (np.array([[[146.0, 108.0]]]) * np.float64(F32(0.01))).astype(F32))
    assert np.allclose(T, [[[1.46, 1.08]]], rtol=1e-6)
    # the admissible range: exactly g64 away from rounding ties, and one more step when p64 sits on a tie
    lo, hi = ref.admissible_range(p64, p)
    assert np.array_equal(lo, g64) and np.array_equal(hi, g64)
    tie = np.array([[[0.255, 0.745]]])
    lo, hi = ref.admissible_range(tie, p)
    assert np.array_equal(hi - lo, [[[1, 1]]])
    # a scale multiplies the fp32 scores in fp32
    s8, _ = ref.scores(q, k, 0.1)
    assert np.array_equal(s8, (s * F32(0.1)).astype(F32))
    # NaN rows: one in q marks its row, one anywhere in k marks the entry
    qn = (np.array([[[1, 0], [np.nan, 0]]], F32),) + q[1:]
    kn = (np.array([[[1, 0], [0, np.nan]]], F32),) + k[1:]
    assert np.array_equal(ref.scores(qn, k)[1], [[False, True]]) and np.array_equal(ref.scores(q, kn)[1], [[True]])


def test_truth_bound_holds_for_the_reference_grid():
    rng = np.random.default_rng(8)
    q, k, v = ((rng.standard_normal((2, 9, 24)).astype(F32), F32(0.02), F32(0), -128, 127) for _ in range(3))
    p = (F32(1 / 200), F32(3), 0, 255)
    T, g64, mm, _ = ref.truth(q, k, v, p, 0.2)
    pq = np.zeros((2, 9, 16), np.int8)
    pq[..., :9] = g64
    y = ref.expected(pq, q, k, v, p, 0.2)
    assert np.all(np.abs(y - T) <= ref.truth_bound(g64, g64, p, v, mm))
    # the fake-quant composition on the same operands agrees with T within the matmul bound plus its own softmax
    s, _ = ref.scores(q, k, 0.2)
    fq = oqdq.qdq(torch.from_numpy(s).softmax(-1).numpy(), p[0], p[1], 0, 255).astype(np.float64) @ oqdq.qdq(*v)
    assert np.abs(fq - T).max() < 1e-3


# ---------------------------------------------------------------------------------------------- eligibility
def _qattn(scheme="per-tensor-symmetric", bit=8, qtype="uniform", backend=Backend.VIRTUAL, scale=0.125, p_cfg=True):
    a = sbcfg.quantizer_config(scheme, bit, "feature", qtype=qtype)
    pc = sbcfg.quantizer_config("per-tensor-affine", 8, "feature") if p_cfg else None
    m = QAttention(scale).build_quantizer(a, pc, backend=backend)
    m.set_quant(a_quant=True)
    return m


def test_eligible_modules():
    assert int8_attention_ineligibility(_qattn()) is None
    assert int8_attention_ineligibility(_qattn(scale=None, p_cfg=False)) is None
    assert int8_attention_ineligibility(_qattn("per-tensor-affine", 4)) is None
    m = _qattn()
    assert m.pv.left.input_quantizer.qdesc.qrange == (0, 255) and m.qk.left.input_quantizer.qdesc.qrange == (-128, 127)


_reason = refusal(int8_attention_ineligibility, QAttentionInt8.from_qattention)


@pytest.mark.parametrize("role,side", [("qk", "left"), ("qk", "right"), ("pv", "left"), ("pv", "right")])
def test_every_ineligible_case_gives_its_reason(role, side):
    def carrier(m):
        return getattr(getattr(m, role), side)

    m = _qattn()
    carrier(m).input_quantizer = None
    assert f"the {role} matmul: the {side} quantizer is missing" in _reason(m)
    m = _qattn()
    carrier(m).set_quant(a_quant=False)
    assert f"the {role} matmul: the {side} quantizer is not enabled" in _reason(m)
    m = _qattn()
    carrier(m).input_quantizer.enable_export_onnx()
    assert f"the {side} quantizer is in export_onnx mode" in _reason(m)
    m = _qattn()
    carrier(m).input_quantizer.scale = torch.ones(3)
    carrier(m).input_quantizer.zero_point = torch.zeros(3)
    assert f"the {side} quantizer holds 3 scales" in _reason(m)
    m = _qattn()
    carrier(m).input_quantizer.zero_point = torch.tensor([300.0])
    assert f"the {side} zero point lies outside" in _reason(m)
    m = _qattn()
    setattr(m, role, QMatMulInt8(torch.device("cpu")))
    assert f"the {role} matmul is already a QMatMulInt8: run to_integer_attentions before to_integer_matmuls" in _reason(m)


def test_module_wide_ineligible_cases():
    assert "the qk matmul: the left quantizer is fake_fused" in _reason(
        QAttention().build_quantizer(sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature", disable=True)))
    assert "DoReFa" in _reason(_qattn(qtype="dorefa", p_cfg=False))
    assert "per-channel" in _reason(_qattn(scheme="per-channel-symmetric", p_cfg=False))
    assert "9 bits" in _reason(_qattn(bit=9, p_cfg=False))
    for bad in (float("inf"), float("nan")):
        assert "is not finite" in _reason(_qattn(scale=bad))
    assert "expected a QAttention" in int8_attention_ineligibility(QMatMul())


class _Block(nn.Module):
    def __init__(self):
        super().__init__()
        a = sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature")
        self.fc = QLinear(nn.Linear(6, 6)).build_quantizer(a, sbcfg.quantizer_config("per-channel-symmetric", 8, "weight"))
        self.attn = _qattn()
        self.bad = _qattn(bit=9)
        self.mm = QMatMul().build_quantizer(a)
        self.mm.set_quant(a_quant=True)

    def forward(self, x):
        y = self.fc(x)
        return self.mm(self.bad(self.attn(y, y, y), y, y), y)


def test_to_integer_attentions_converts_only_eligible_attentions():
    model = _Block()
    assert to_integer_attentions(model) == ["attn"]
    assert isinstance(model.attn, QAttentionInt8) and isinstance(model.bad, QAttention) and isinstance(model.mm, QMatMul)
    assert isinstance(model.fc, QLinear)
    assert model.attn.scale == 0.125 and model.attn.qranges == {"q": (-128, 127), "k": (-128, 127), "p": (0, 255),
                                                                "v": (-128, 127)}
    # in the other order the matmuls are converted one by one and the attention is left alone with a reason
    model = _Block()
    model.bad = _qattn()
    assert to_integer_matmuls(model) == ["attn.qk", "attn.pv", "bad.qk", "bad.pv", "mm"]
    assert to_integer_attentions(model) == []
    assert "run to_integer_attentions before to_integer_matmuls" in int8_attention_ineligibility(model.attn)


def test_qattention_exposes_four_carriers_to_calibration():
    m = _qattn()
    assert not _is_quant_opr(m) and not hasattr(m, "input_quantizer")
    carriers = [m.qk.left, m.qk.right, m.pv.left, m.pv.right]
    assert all(isinstance(c, QIdentity) and _is_quant_opr(c) for c in carriers)
    assert len({id(c.input_quantizer) for c in carriers}) == 4
    model = _Block()
    runner = CalibrationRunner(model, streaming=True, record_inputs=False)
    runner.prepare_calibration()
    hooked = {name for name, mod in model.named_modules() if mod._forward_pre_hooks}
    assert {"attn.qk.left", "attn.qk.right", "attn.pv.left", "attn.pv.right"} <= hooked
    runner._remove_hooks()
    gm = trace_quant_model(_Block())
    leaves = [n.target for n in gm.graph.nodes if n.op == "call_module"]
    assert leaves[:5] == ["fc", "attn.qk.left", "attn.qk.right", "attn.pv.left", "attn.pv.right"]
    assert any(n.op == "call_method" and n.target == "softmax" for n in gm.graph.nodes)


def test_qattention_forward_is_the_composition():
    m = QAttention(scale=0.5)  # quantizers off: plain softmax attention
    for c in (m.qk.left, m.qk.right, m.pv.left, m.pv.right):
        c.build_quantizer(sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature"))
        c.set_quant(a_quant=False)
    q, k, v = torch.randn(2, 4, 8), torch.randn(2, 6, 8), torch.randn(2, 6, 3)
    assert torch.allclose(m(q, k, v), torch.softmax(q @ k.transpose(-2, -1) * 0.5, -1) @ v)


def test_qattention_int8_module_contract():
    mod = QAttentionInt8(torch.device("cpu"), 0.125)
    assert set(dict(mod.named_buffers())) == {f"{r}_{w}" for r in "qkpv" for w in ("scale", "zero_point")}
    with pytest.raises(RuntimeError, match="inference-only"):
        mod(torch.zeros(2, 4, requires_grad=True), torch.zeros(3, 4), torch.zeros(3, 2))


# ---------------------------------------------------------------------------------------------- branch coverage
def test_branch_cases_reach_every_branch():
    reached = set().union(*(case_branches(c) for c in CASES.values()))
    assert reached == set(geo.ALL), sorted(set(geo.ALL) - reached)


def test_plan_by_hand():
    assert geo.plan(2, 197, 197, 64, 64) == dict(ctas=4, nkb=2, nk32=2, dp=64, tkp=208)
    assert geo.plan(1, 1, 1, 8, 8) == dict(ctas=1, nkb=1, nk32=1, dp=16, tkp=16)
    assert geo.plan(1, 300, 1000, 100, 8) == dict(ctas=3, nkb=8, nk32=4, dp=112, tkp=1008)
    assert geo.plan(1, 128, 1 << 17, 8, 8) is None and geo.plan(1, 1, 1, 129, 8) is None
    assert geo.plan(1, 1, 1, 8, 129) is None and geo.plan(0, 1, 1, 8, 8) is None
    assert "ring_wraps" in case_branches(CASES["ring_wraps_ramp"]) and "ring_wraps" not in case_branches(CASES["tiny"])
