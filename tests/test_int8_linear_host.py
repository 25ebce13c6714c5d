"""CPU: the fp64 truth of the integer-grid linear, the host side of sb200_int8_quantize_rows / sb200_int8_linear and the
eligibility rules of QLinearInt8.from_qlinear.

* The truth (the fp64 matmul of the oracle's fake-quant tensors) equals the integer form the kernel computes,
  s_x s_w I + bias, exactly for power-of-two scales and within the stated bound otherwise.
* Every bad argument is rejected on the host, before any CUDA call (there is no device here), with its code and message.
* The workspace query is a pure function of (m, k).
* Every rule of from_qlinear gives its reason, and to_integer_linears leaves those layers alone."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from int8_harness import E_INVALID, E_UNSUPPORTED, E_WORKSPACE, buf, refusal, rejector
from int8_linear_ref import BOUND, integer_terms, truth
from sparsebit_b200 import _lib
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.common import Backend
from sparsebit_b200.quantization.modules import (QConv2dSparse24Int8, QLinear, QLinearInt8, QLinearSparse24Int8,
                                                 int8_ineligibility)
from sparsebit_b200.quantization.tools import to_integer_linears

def _operands(rng, m, k, n, xrange, wrange, pow2):
    x = (rng.standard_normal((m, k)) * 3).astype(np.float32)
    w = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
    if pow2:
        xs = np.float32(2.0 ** -5)
        ws = (2.0 ** -rng.integers(6, 10, n)).astype(np.float32)
    else:
        xs = np.float32(np.abs(x).max() / 127.3)
        ws = (np.abs(w).max(axis=1) / 119.7).astype(np.float32)
    (xqmin, xqmax), (wqmin, wqmax) = xrange, wrange
    xz = np.float32(0 if xqmin < 0 else rng.integers(xqmin, xqmax + 1))
    wz = (np.zeros(n) if wqmin < 0 else rng.integers(wqmin, wqmax + 1, n)).astype(np.float32)
    return x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax


RANGES = [((-128, 127), (-128, 127)), ((0, 255), (-128, 127)), ((0, 255), (0, 255)), ((-8, 7), (0, 15)), ((0, 3), (-2, 1))]


@pytest.mark.parametrize("xrange,wrange", RANGES)
@pytest.mark.parametrize("pow2", [True, False])
def test_truth_equals_the_integer_form(xrange, wrange, pow2):
    rng = np.random.default_rng(hash((xrange, wrange, pow2)) % 2**32)
    m, k, n = 9, 200, 13
    ops_ = _operands(rng, m, k, n, xrange, wrange, pow2)
    bias = None if pow2 else rng.standard_normal(n).astype(np.float32)
    t, bound = truth(*ops_, bias=bias)
    a, b, zx, zw, i = integer_terms(*ops_)
    assert a.min() >= -128 and a.max() <= 127 and b.min() >= -128 and b.max() <= 127
    # the correction terms remove the zero points exactly
    assert np.array_equal(i, (a - zx) @ (b - zw[:, None]).T)
    x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax = ops_
    y = float(xs) * ws.astype(np.float64)[None, :] * i.astype(np.float64) + (0 if bias is None else bias.astype(np.float64))
    if pow2:
        assert np.array_equal(y, t)
    else:
        assert np.all(np.abs(y - t) <= bound)
        assert np.all(bound > 0)


def test_bound_is_the_stated_one():
    assert BOUND == 2.0 ** -21


def test_linear_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    ws_ok = int(lib.sb200_int8_linear_workspace_bytes(4, 64))
    # (x, xs, xz, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, bias, out, m, k, n, ws, ws_bytes, stream)
    ok = [p, p, p, -128, 127, p, p, p, p, None, p, 4, 64, 8, p, ws_ok, None]
    rejected = rejector(lib.sb200_int8_linear, ok)
    for i in (0, 1, 2, 5, 6, 7, 8, 10, 14):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    for i in (11, 12, 13):
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
        rejected(E_INVALID, b"empty operand", **{f"a{i}": -5})
    rejected(E_INVALID, b"too large", a11=1 << 31)
    rejected(E_INVALID, b"too large", a13=1 << 31)
    rejected(E_INVALID, b"wider than 8 bits", a3=-128, a4=128)
    rejected(E_INVALID, b"wider than 8 bits", a3=0, a4=256)
    rejected(E_INVALID, b"qmin", a3=5, a4=4)
    rejected(E_INVALID, b"neither signed", a3=-129, a4=0)
    rejected(E_INVALID, b"neither signed", a3=10, a4=260)
    rejected(E_INVALID, b"16-byte aligned", a5=p + 1)
    rejected(E_UNSUPPORTED, b"K < 2^17", a12=1 << 17)
    rejected(E_UNSUPPORTED, b"K < 2^17", a12=(1 << 17) + 5)
    rejected(E_WORKSPACE, b"workspace too small", a15=ws_ok - 1)
    rejected(E_WORKSPACE, b"workspace too small", a15=0)


def test_quantize_rows_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    # (x, scale, zp, per_row, qmin, qmax, q, row_sum, nan_flag, rows, k, stream)
    ok = [p, p, p, 0, -128, 127, p, p, p, 4, 64, None]
    rejected = rejector(lib.sb200_int8_quantize_rows, ok)
    for i in (0, 1, 2, 6, 7, 8):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    for i in (9, 10):
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
    rejected(E_INVALID, b"wider than 8 bits", a4=-200, a5=100)
    rejected(E_INVALID, b"neither signed", a4=-1, a5=200)
    rejected(E_INVALID, b"16-byte aligned", a6=p + 8)
    rejected(E_UNSUPPORTED, b"K < 2^17", a10=1 << 17)


def test_workspace_query_is_pure():
    q = _lib.load().sb200_int8_linear_workspace_bytes
    assert q(0, 64) == 0 and q(4, 0) == 0 and q(-1, 64) == 0
    for m, k in [(1, 1), (7, 33), (197 * 64, 768), (2048, 11008), (3, (1 << 17) - 1)]:
        first = q(m, k)
        assert first >= m * ((k + 15) // 16 * 16) + 5 * m
        assert all(q(m, k) == first for _ in range(3))
    assert q(8, 16) == q(8, 1) and q(8, 17) == q(8, 32)  # rows are padded to 16 bytes


# ---------------------------------------------------------------------------------------------- eligibility
def _qlinear(a_scheme="per-tensor-symmetric", a_bit=8, w_scheme="per-channel-symmetric", w_bit=8, w_type="uniform",
             a_type="uniform", backend=Backend.VIRTUAL, a_disable=False):
    lin = nn.Linear(24, 10)
    q = QLinear(lin).build_quantizer(sbcfg.quantizer_config(a_scheme, a_bit, "feature", qtype=a_type, disable=a_disable),
                                     sbcfg.quantizer_config(w_scheme, w_bit, "weight", qtype=w_type), backend=backend)
    q.set_quant(w_quant=True, a_quant=True)
    return q


def test_eligible_layers():
    assert int8_ineligibility(_qlinear()) is None
    assert int8_ineligibility(_qlinear("per-tensor-affine", 8, "per-tensor-symmetric", 4)) is None
    assert int8_ineligibility(_qlinear(w_type="lsq", a_type="lsq")) is None
    assert int8_ineligibility(_qlinear(backend=Backend.TENSORRT)) is None


_reason = refusal(int8_ineligibility, QLinearInt8.from_qlinear)


def test_every_ineligible_case_gives_its_reason():
    q = _qlinear()
    q.set_quant(w_quant=True, a_quant=False)
    assert "input quantizer is not enabled" in _reason(q)
    q = _qlinear()
    q.set_quant(w_quant=False, a_quant=True)
    assert "weight quantizer is not enabled" in _reason(q)
    assert "input quantizer is fake_fused" in _reason(_qlinear(a_disable=True))
    q = _qlinear()
    q.weight_quantizer.enable_export_onnx()
    assert "export_onnx" in _reason(q)
    assert "DoReFa" in _reason(_qlinear(w_type="dorefa"))
    assert "adaround" in _reason(_qlinear(w_type="adaround"))
    assert "input quantizer is per-channel" in _reason(_qlinear(a_scheme="per-channel-symmetric"))
    assert "9 bits" in _reason(_qlinear(a_bit=9))
    assert "16 bits" in _reason(_qlinear(w_bit=16))
    q = _qlinear()
    q.weight_quantizer.qdesc._ch_axis = 1
    assert "axis 1" in _reason(q)
    q = _qlinear()
    q.input_quantizer.zero_point = torch.tensor([200.0])
    assert "input zero point lies outside [-128, 127]" in _reason(q)
    q = _qlinear(w_scheme="per-channel-affine")
    q.weight_quantizer.scale = torch.ones(10, 1)
    q.weight_quantizer.zero_point = torch.tensor([[3.0]] * 9 + [[255.6]])
    assert "weight zero point lies outside [0, 255]" in _reason(q)
    q = _qlinear(w_scheme="per-channel-affine")
    q.weight_quantizer.scale = torch.ones(3, 1)
    q.weight_quantizer.zero_point = torch.zeros(3, 1)
    assert "holds 3 scales" in _reason(q)
    q = _qlinear(backend=Backend.TENSORRT)
    q.input_quantizer.zero_point = torch.tensor([3.0])
    assert "tensorrt only support symmetric" in _reason(q)
    assert "expected a QLinear" in int8_ineligibility(nn.Linear(3, 4))


@pytest.mark.parametrize("alpha,narrowed", [(1.5, False), (3.0, False), (1.0, True)])
def test_signed_pact_inputs_whose_clamp_narrows_the_grid_are_ineligible(alpha, narrowed):
    """alpha / scale = 127.5 in exact arithmetic; where fp32 rounds it to 127, -alpha lands on qmin + 1 and the clamp in
    front of the fake-quant op narrows the grid (SURVEY Q19), which the integer path does not restate."""
    q = _qlinear(a_type="pact")
    q.input_quantizer.dims = 2
    q.input_quantizer.alpha = nn.Parameter(torch.tensor([alpha]))
    s = np.float32(alpha) * np.float32(2) / np.float32(255)
    assert (np.rint(np.float32(alpha) / s) == 127) == narrowed
    if narrowed:
        assert "PACT with alpha on the grid, whose clamp narrows it to [-127, 127]" in _reason(q)
    else:
        assert int8_ineligibility(q) is None


def test_to_integer_linears_skips_ineligible_layers():
    model = nn.Sequential(_qlinear(w_type="dorefa"), nn.ReLU(), _qlinear(a_bit=9))
    assert to_integer_linears(model) == []
    assert all(isinstance(model[i], QLinear) for i in (0, 2))


def test_qlinear_int8_module_contract():
    mod = QLinearInt8(20, 6, torch.device("cpu"))
    buffers = {name: (b.dtype, tuple(b.shape)) for name, b in mod.named_buffers()}
    assert buffers == {"w_q": (torch.int8, (6, 32)), "w_rowsum": (torch.int32, (6,)), "w_scale": (torch.float32, (6,)),
                       "w_zero": (torch.int32, (6,)), "scale": (torch.float32, (1,)), "zero_point": (torch.float32, (1,))}
    assert set(mod.state_dict()) == set(buffers) and "bias" in mod._buffers and mod.bias is None
    assert (mod.in_features, mod.out_features, mod.qmin, mod.qmax) == (20, 6, -128, 127)
    assert repr(mod) == "QLinearInt8(in_features=20, out_features=6, qrange=[-128, 127])"
    with pytest.raises(RuntimeError, match=r"^QLinearInt8 is inference-only and has no backward; .* keep QLinear for"):
        mod(torch.zeros(2, 20, requires_grad=True))


def test_sparse24_int8_module_contract():
    """Both 2:4 modules store the same compressed operand, registered before the activation qparams."""
    lin = QLinearSparse24Int8(20, 6, torch.device("cpu"))
    conv = QConv2dSparse24Int8(3, 5, (3, 2), (1, 2), (1, 0, 1, 1), (2, 1), torch.device("cpu"))
    for mod, n in ((lin, 6), (conv, 5)):  # K = 20 and K = 3 * 3 * 2 = 18: K64 = 64
        buffers = [(name, b.dtype, tuple(b.shape)) for name, b in mod.named_buffers()]
        assert buffers == [("vals", torch.int8, (n, 32)), ("meta", torch.int32, (1, 1, 2, 128)), ("dsum", torch.int32, (n,)),
                           ("w_scale", torch.float32, (n,)), ("scale", torch.float32, (1,)),
                           ("zero_point", torch.float32, (1,))]
        assert list(mod.state_dict()) == [name for name, _, _ in buffers]
        assert "bias" in mod._buffers and mod.bias is None and (mod.qmin, mod.qmax) == (-128, 127)
    assert (lin.in_features, lin.out_features) == (20, 6)
    assert repr(lin) == "QLinearSparse24Int8(in_features=20, out_features=6, qrange=[-128, 127], 2:4 sparse)"
    assert (conv.in_channels, conv.out_channels) == (3, 5)
    assert (conv.kernel_size, conv.stride, conv.padding, conv.dilation) == ((3, 2), (1, 2), (1, 0, 1, 1), (2, 1))
    assert repr(conv) == ("QConv2dSparse24Int8(3, 5, kernel_size=(3, 2), stride=(1, 2), padding=(1, 0, 1, 1), "
                          "dilation=(2, 1), qrange=[-128, 127], 2:4 sparse)")
    with pytest.raises(RuntimeError, match=r"^QLinearSparse24Int8 is inference-only and has no backward; .* keep QLinear for"):
        lin(torch.zeros(2, 20, requires_grad=True))
    for x in (torch.zeros(1, 3, 6, 6, requires_grad=True), torch.zeros(3, 6, 6, requires_grad=True)):
        with pytest.raises(RuntimeError, match=r"^QConv2dSparse24Int8 is inference-only and has no backward; .* keep QConv2d for"):
            conv(x)
