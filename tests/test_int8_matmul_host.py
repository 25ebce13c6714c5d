"""CPU: the fp64 truth of the integer-grid matmul, the host side of sb200_int8_quantize_cols / sb200_int8_matmul, the
eligibility rules of QMatMulInt8.from_qmatmul and what calibration sees of a QMatMul.

* The truth (the fp64 matmul of the oracle's fake-quant operands) equals the integer form the kernel computes, s_a s_b I,
  exactly for power-of-two scales and within the stated bound otherwise; the fake-quant torch.matmul agrees with it.
* Every bad argument is rejected on the host, before any CUDA call (there is no device here), with its code and message.
* The workspace query is a pure, monotone function of (batch, m, k, n).
* Every rule of from_qmatmul gives its reason; to_integer_matmuls leaves those modules, QLinear and QConv2d alone.
* QMatMul is not a quant operator for CalibrationRunner; its two carriers are, under hooks and under the fx trace."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from int8_harness import E_INVALID, E_UNSUPPORTED, E_WORKSPACE, buf, refusal, rejector
from int8_matmul_ref import BOUND, integer_form, quantize_cols, truth
from oracle import qdq as oqdq
from sparsebit_b200 import _lib
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.common import Backend
from sparsebit_b200.quantization.modules import (QConv2d, QIdentity, QLinear, QMatMul, QMatMulInt8,
                                                 int8_matmul_ineligibility)
from sparsebit_b200.quantization.tools import (CalibrationRunner, to_integer_convs, to_integer_linears,
                                               to_integer_matmuls, trace_quant_model)
from sparsebit_b200.quantization.tools.calibration import _is_quant_opr

F32 = np.float32
RANGES = [((-128, 127), (-128, 127)), ((0, 255), (-128, 127)), ((0, 255), (0, 255)), ((-8, 7), (0, 15)), ((0, 3), (-2, 1))]


def _operand(rng, shape, qrange, pow2, spread):
    x = (rng.standard_normal(shape) * spread).astype(F32)
    qmin, qmax = qrange
    s = F32(2.0 ** -5) if pow2 else F32(np.abs(x).max() / (0.47 * (qmax - qmin)))
    z = F32(0 if qmin < 0 else rng.integers(qmin, qmax + 1))
    return x, s, z, qmin, qmax


@pytest.mark.parametrize("arange,brange", RANGES)
@pytest.mark.parametrize("pow2", [True, False])
def test_truth_equals_the_integer_form(arange, brange, pow2):
    rng = np.random.default_rng(abs(hash((arange, brange, pow2))) % 2**32)
    a = _operand(rng, (2, 3, 9, 37), arange, pow2, 3.0)
    b = _operand(rng, (3, 37, 13), brange, pow2, 1.5)  # leading dimensions broadcast
    t, bound = truth(a, b)
    qa, qb, za, zb, i, y = integer_form(a, b)
    assert t.shape == (2, 3, 9, 13)
    assert qa.min() >= -128 and qa.max() <= 127 and qb.min() >= -128 and qb.max() <= 127
    assert np.array_equal(i, np.matmul(qa - za, qb - zb))  # the correction terms remove the zero points exactly
    if pow2:
        assert np.array_equal(y, t)
    else:
        assert np.all(np.abs(y - t) <= bound) and np.any(bound > 0)
    # the fake-quant operator (torch.matmul of the QDQ outputs, fp32) computes the same product
    ref = torch.matmul(torch.from_numpy(oqdq.qdq(*a)), torch.from_numpy(oqdq.qdq(*b))).numpy()
    assert np.all(np.abs(ref - t) <= 37 * 2.0 ** -23 * bound / BOUND)


def test_nan_rows_and_columns_of_the_integer_form():
    rng = np.random.default_rng(5)
    a = _operand(rng, (2, 5, 20), (-128, 127), False, 1.0)
    b = _operand(rng, (2, 20, 7), (0, 255), False, 1.0)
    a[0][1, 3, 11] = np.nan
    b[0][0, 4, 2] = np.nan
    y = integer_form(a, b)[-1]
    expect = np.zeros((2, 5, 7), bool)
    expect[1, 3, :] = True
    expect[0, :, 2] = True
    assert np.array_equal(np.isnan(y), expect)
    assert np.array_equal(np.isnan(truth(a, b)[0]), expect)


def test_quantize_cols_reference_layout():
    rng = np.random.default_rng(6)
    x, s, z, qmin, qmax = _operand(rng, (2, 19, 5), (0, 255), False, 1.0)
    q, col_sum, nan = quantize_cols(x, s, z, qmin, qmax)
    assert q.shape == (2, 5, 32) and q.dtype == np.int8 and not q[..., 19:].any() and not nan.any()
    g = oqdq.quantize_int(x, s, z, qmin, qmax) - 128
    assert np.array_equal(q[..., :19], np.swapaxes(g, 1, 2)) and np.array_equal(col_sum, g.sum(1))


def test_matmul_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    ws_ok = int(lib.sb200_int8_matmul_workspace_bytes(3, 4, 64, 8))
    # (a, b, b_k_major, a_scale, a_zp, qmin_a, qmax_a, b_scale, b_zp, qmin_b, qmax_b, out, batch, m, k, n, ws, ws_bytes, stream)
    ok = [p, p, 0, p, p, -128, 127, p, p, 0, 255, p, 3, 4, 64, 8, p, ws_ok, None]
    rejected = rejector(lib.sb200_int8_matmul, ok)
    for i in (0, 1, 3, 4, 7, 8, 11, 16):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    for i in (12, 13, 14, 15):
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
        rejected(E_INVALID, b"empty operand", **{f"a{i}": -5})
    rejected(E_INVALID, b"too large", a13=1 << 31)
    rejected(E_INVALID, b"too large", a15=1 << 31)
    rejected(E_INVALID, b"too large", a12=1 << 20, a13=1 << 11)  # batch M = 2^31
    rejected(E_INVALID, b"too large", a12=1 << 16, a15=1 << 15)  # batch N = 2^31
    rejected(E_INVALID, b"output tiles", a12=1 << 10, a13=(1 << 20) + 1, a15=(1 << 20) + 1)
    for lo, hi in ((5, 6), (9, 10)):  # either operand's range
        rejected(E_INVALID, b"wider than 8 bits", **{f"a{lo}": -128, f"a{hi}": 128})
        rejected(E_INVALID, b"wider than 8 bits", **{f"a{lo}": 0, f"a{hi}": 256})
        rejected(E_INVALID, b"qmin", **{f"a{lo}": 5, f"a{hi}": 4})
        rejected(E_INVALID, b"neither signed", **{f"a{lo}": -129, f"a{hi}": 0})
        rejected(E_INVALID, b"neither signed", **{f"a{lo}": 10, f"a{hi}": 260})
    rejected(E_UNSUPPORTED, b"K < 2^17", a14=1 << 17)
    rejected(E_UNSUPPORTED, b"K < 2^17", a14=(1 << 17) + 5)
    rejected(E_WORKSPACE, b"workspace too small", a17=ws_ok - 1)
    rejected(E_WORKSPACE, b"workspace too small", a17=0)
    rejected(E_WORKSPACE, b"workspace too small", a2=1, a17=ws_ok - 1)


def test_quantize_cols_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    # (x, scale, zp, qmin, qmax, q, col_sum, nan_flag, batch, k, n, stream)
    ok = [p, p, p, -128, 127, p, p, p, 2, 64, 8, None]
    rejected = rejector(lib.sb200_int8_quantize_cols, ok)
    for i in (0, 1, 2, 5, 6, 7):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    for i in (8, 9, 10):
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
    rejected(E_INVALID, b"too many columns", a8=1 << 16, a10=1 << 15)
    rejected(E_INVALID, b"wider than 8 bits", a3=-200, a4=100)
    rejected(E_INVALID, b"neither signed", a3=-1, a4=200)
    rejected(E_INVALID, b"16-byte aligned", a5=p + 8)
    rejected(E_UNSUPPORTED, b"K < 2^17", a9=1 << 17)


def test_workspace_query_is_pure_and_monotone():
    q = _lib.load().sb200_int8_matmul_workspace_bytes
    assert q(0, 4, 64, 8) == 0 and q(2, 0, 64, 8) == 0 and q(2, 4, 0, 8) == 0 and q(2, 4, 64, -1) == 0
    assert q(1 << 20, 1 << 11, 64, 8) == 0 and q(2, 4, 1 << 17, 8) == 0  # what the matmul rejects
    for b, m, k, n in [(1, 1, 1, 1), (12, 197, 64, 197), (768, 197, 197, 64), (3, 7, (1 << 17) - 1, 5)]:
        first = q(b, m, k, n)
        assert first >= b * (m + n) * ((k + 15) // 16 * 16 + 5)
        assert all(q(b, m, k, n) == first for _ in range(3))
        assert q(b + 1, m, k, n) >= first and q(b, m + 1, k, n) >= first and q(b, m, k, n + 1) >= first
        if k + 1 < 1 << 17:
            assert q(b, m, k + 1, n) >= first
    assert q(2, 8, 16, 8) == q(2, 8, 1, 8) and q(2, 8, 17, 8) == q(2, 8, 32, 8)  # rows are padded to 16 bytes


# ---------------------------------------------------------------------------------------------- eligibility
def _qmatmul(scheme="per-tensor-symmetric", bit=8, qtype="uniform", backend=Backend.VIRTUAL, disable=False):
    q = QMatMul().build_quantizer(sbcfg.quantizer_config(scheme, bit, "feature", qtype=qtype, disable=disable), backend=backend)
    q.set_quant(a_quant=True)
    return q


def test_eligible_modules():
    assert int8_matmul_ineligibility(_qmatmul()) is None
    assert int8_matmul_ineligibility(_qmatmul("per-tensor-affine", 4)) is None
    assert int8_matmul_ineligibility(_qmatmul(qtype="lsq")) is None
    assert int8_matmul_ineligibility(_qmatmul(backend=Backend.TENSORRT)) is None
    q = _qmatmul()
    assert q.left.input_quantizer is not q.right.input_quantizer


_reason = refusal(int8_matmul_ineligibility, QMatMulInt8.from_qmatmul)


@pytest.mark.parametrize("side", ["left", "right"])
def test_every_ineligible_case_gives_its_reason(side):
    def case(**kw):
        q = _qmatmul(**kw)
        return q, getattr(q, side)

    q, carrier = case()
    carrier.input_quantizer = None
    assert f"the {side} quantizer is missing" in _reason(q)
    q, carrier = case()
    carrier.set_quant(a_quant=False)
    assert f"the {side} quantizer is not enabled" in _reason(q)
    assert "the left quantizer is fake_fused" in _reason(_qmatmul(disable=True))
    q, carrier = case()
    carrier.input_quantizer.enable_export_onnx()
    assert f"the {side} quantizer is in export_onnx mode" in _reason(q)
    assert "DoReFa" in _reason(_qmatmul(qtype="dorefa"))
    assert "the left quantizer is per-channel" in _reason(_qmatmul(scheme="per-channel-symmetric"))
    assert "9 bits" in _reason(_qmatmul(bit=9))
    q, carrier = case()
    carrier.input_quantizer.scale = torch.ones(3)
    carrier.input_quantizer.zero_point = torch.zeros(3)
    assert f"the {side} quantizer holds 3 scales" in _reason(q)
    q, carrier = case()
    carrier.input_quantizer.zero_point = torch.tensor([200.0])
    assert f"the {side} zero point lies outside [-128, 127]" in _reason(q)
    q, carrier = case(backend=Backend.TENSORRT)
    carrier.input_quantizer.zero_point = torch.tensor([3.0])
    assert f"the {side} quantizer: " in _reason(q) and "tensorrt only support symmetric" in _reason(q)
    assert "expected a QMatMul" in int8_matmul_ineligibility(nn.Linear(3, 4))


class _Block(nn.Module):
    def __init__(self):
        super().__init__()
        a, w = sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature"), sbcfg.quantizer_config("per-channel-symmetric", 8, "weight")
        self.fc = QLinear(nn.Linear(6, 6)).build_quantizer(a, w)
        self.conv = QConv2d(nn.Conv2d(1, 1, 1)).build_quantizer(a, w)
        self.bad = _qmatmul(bit=9)
        self.off = _qmatmul()
        self.off.set_quant(a_quant=False)

    def forward(self, x):
        y = self.fc(x)
        return self.off(self.bad(y, y.transpose(-2, -1)), y)


def test_to_integer_matmuls_skips_ineligible_modules_and_other_operators():
    model = _Block()
    model.fc.set_quant(True, True), model.conv.set_quant(True, True)
    assert to_integer_matmuls(model) == []
    assert isinstance(model.bad, QMatMul) and isinstance(model.off, QMatMul)
    assert isinstance(model.fc, QLinear) and isinstance(model.conv, QConv2d)
    # and the siblings leave a QMatMul alone
    model.bad = _qmatmul()
    assert to_integer_linears(nn.Sequential()) == [] and to_integer_convs(nn.Sequential()) == []
    assert isinstance(model.bad, QMatMul)


def test_qmatmul_is_not_a_quant_operator_but_its_carriers_are():
    q = _qmatmul()
    assert not _is_quant_opr(q) and not hasattr(q, "input_quantizer") and not hasattr(q, "weight_quantizer")
    assert isinstance(q.left, QIdentity) and _is_quant_opr(q.left) and _is_quant_opr(q.right)
    model = _Block()
    runner = CalibrationRunner(model, streaming=True, record_inputs=False)
    runner.prepare_calibration()
    hooked = {name for name, m in model.named_modules() if m._forward_pre_hooks}
    assert hooked == {"fc", "conv", "bad.left", "bad.right", "off.left", "off.right"}
    runner._remove_hooks()
    # the fx trace looks through QMatMul: its carriers are the leaves, torch.matmul is a function node between them
    gm = trace_quant_model(_Block())
    modules = [n.target for n in gm.graph.nodes if n.op == "call_module"]
    assert modules == ["fc", "bad.left", "bad.right", "off.left", "off.right"]
    assert [n.target for n in gm.graph.nodes if n.op == "call_function"].count(torch.matmul) == 2


def test_qmatmul_int8_module_contract():
    mod = QMatMulInt8(torch.device("cpu"))
    assert set(dict(mod.named_buffers())) == {"left_scale", "left_zero_point", "right_scale", "right_zero_point"}
    with pytest.raises(ValueError, match="1-D operands are not supported"):
        mod(torch.zeros(4), torch.zeros(4, 3))
    with pytest.raises(ValueError, match="1-D operands are not supported"):
        mod(torch.zeros(2, 4), torch.zeros(4))
    with pytest.raises(RuntimeError, match="inference-only"):
        mod(torch.zeros(2, 4, requires_grad=True), torch.zeros(4, 3))
