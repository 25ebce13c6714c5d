"""DoReFa and AdaRound integer-grid layers on the host: the conversion rules and the converters' disjointness, host-side
rejection by the five ``_dorefa`` entry points (the plain counterpart's checks, order and codes, then a null
x_absmax), the AdaRound round trip the weight rule relies on, and the DoReFa GPU suite running every branch case of the
plain suites."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_geometry
import int8_group_geometry
import int8_nhwc_geometry
import test_gpu_int8_branches as lin_suite
import test_gpu_int8_conv_nhwc_branches as nhwc_suite
import test_gpu_int8_dorefa as dorefa_suite
import test_gpu_int8_group_branches as grp_suite
from branch_cases import assert_table_covers, check_reach
from int8_harness import E_INVALID, buf, conv_geom, rejector
from sparsebit_b200 import _lib, config as sbcfg
from sparsebit_b200.quantization.modules import (ADAROUND_SCALE_RANGE, QConv2d, QLinear, dorefa_adaround_ineligibility,
                                                 int8_conv_ineligibility, int8_group_conv_ineligibility,
                                                 int8_ineligibility)

F32 = np.float32


def _mod(kind, a_type, w_type, groups=1, a_scheme="per-tensor-affine", w_scheme="per-channel-symmetric", bit=4):
    if kind == "linear":
        m = QLinear(nn.Linear(8, 4))
    else:
        m = QConv2d(nn.Conv2d(8, 8, 3, padding=1, groups=groups))
    m.build_quantizer(sbcfg.quantizer_config(a_scheme, bit, "feature", qtype=a_type),
                      sbcfg.quantizer_config(w_scheme, bit, "weight", qtype=w_type))
    if w_type == "adaround":
        m.weight_quantizer.v = nn.Parameter(torch.zeros_like(m.weight))
        m.weight_quantizer.eval()
    m.set_quant(w_quant=True, a_quant=True)
    return m


@pytest.mark.parametrize("kind,groups", [("linear", 1), ("conv", 1), ("conv", 2), ("conv", 8)])
@pytest.mark.parametrize("a_type,w_type", [("dorefa", "dorefa"), ("lsq+", "dorefa"), ("uniform", "adaround"),
                                           ("dorefa", "uniform"), ("lsq", "dorefa")])
def test_dorefa_adaround_layers_are_eligible_and_disjoint(kind, groups, a_type, w_type):
    m = _mod(kind, a_type, w_type, groups)
    assert dorefa_adaround_ineligibility(m) is None
    plain = int8_ineligibility if kind == "linear" else (int8_conv_ineligibility if groups == 1 else
                                                          int8_group_conv_ineligibility)
    assert plain(m) is not None


@pytest.mark.parametrize("kind,groups", [("linear", 1), ("conv", 1), ("conv", 4)])
def test_plain_layers_belong_to_the_plain_converters(kind, groups):
    m = _mod(kind, "uniform", "uniform", groups)
    assert "use to_integer_linears / to_integer_convs / to_integer_group_convs" in dorefa_adaround_ineligibility(m)


def test_reasons():
    assert "expected a QLinear or a QConv2d" in dorefa_adaround_ineligibility(nn.Linear(2, 2))
    m = _mod("linear", "dorefa", "dorefa")
    m.input_quantizer = None
    assert "input quantizer is missing" in dorefa_adaround_ineligibility(m)
    assert "per-channel" in dorefa_adaround_ineligibility(_mod("conv", "dorefa", "dorefa", a_scheme="per-channel-affine"))
    assert "9 bits" in dorefa_adaround_ineligibility(_mod("linear", "dorefa", "dorefa", bit=9)) or \
        "bits" in dorefa_adaround_ineligibility(_mod("linear", "dorefa", "dorefa", bit=9))
    m = _mod("linear", "dorefa", "dorefa")
    m.input_quantizer.disable_quant()
    assert "not enabled" in dorefa_adaround_ineligibility(m)
    m = _mod("conv", "dorefa", "dorefa")
    m.fwd_kwargs["padding"] = "bogus"
    assert "padding" in dorefa_adaround_ineligibility(m)
    m = _mod("linear", "uniform", "adaround")
    m.weight_quantizer.train()
    assert "training mode" in dorefa_adaround_ineligibility(m)
    m = _mod("linear", "uniform", "adaround")
    del m.weight_quantizer.v
    assert "without its rounding variables" in dorefa_adaround_ineligibility(m)
    m = _mod("linear", "uniform", "adaround", w_scheme="per-tensor-affine")
    m.weight_quantizer.zero_point = torch.tensor([[3.5]])
    assert "non-integral zero point" in dorefa_adaround_ineligibility(m)
    m = _mod("linear", "uniform", "adaround", w_scheme="per-tensor-symmetric")
    m.weight_quantizer.scale = torch.tensor([[2.0 ** 120]])
    assert "scale outside" in dorefa_adaround_ineligibility(m)


def _div_exact(x, s):
    """The kernels' quotient RN32(RN64(x * RN64(1 / s))) (div_exact of common.cuh)."""
    return (x.astype(np.float64) * (1.0 / s.astype(np.float64))).astype(F32)


def test_adaround_output_requantizes_to_its_grid():
    """RN32((q - zp) s) / s rounds back to q - zp for every |q - zp| <= 255 and 2^-126 <= |s| <= 2^119."""
    rng = np.random.default_rng(5)
    d = np.arange(-255, 256).astype(F32)
    lo, hi = ADAROUND_SCALE_RANGE
    mant = np.concatenate([[1.0, np.nextafter(F32(2), F32(0))], rng.uniform(1, 2, 2000)]).astype(F32)
    for e in (-126, -125, -60, -1, 0, 1, 60, 118, 119):
        for sign in (1, -1):
            s = (sign * mant * F32(2.0 ** e)).astype(F32)
            s = s[(np.abs(s) >= lo) & (np.abs(s) <= hi)]
            out = (d[None, :] * s[:, None]).astype(F32)  # RN32((q - zp) s), as sb200_adaround_fwd computes it
            back = np.rint(_div_exact(out, s[:, None]))
            assert np.array_equal(back, np.broadcast_to(d, back.shape)), e


def _nulled(rejected, at):
    rejected(E_INVALID, b"null x_absmax", **{f"a{at}": None})


def test_dorefa_entry_points_reject_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    g = conv_geom()
    # each: the counterpart's null-pointer check first (x), a bad range, then a null x_absmax with all else valid
    lin = [p, p, p, p, -128, 127, p, p, p, p, None, p, 4, 16, 8, p, 1 << 20, None]
    rejected = rejector(lib.sb200_int8_linear_dorefa, lin)
    rejected(E_INVALID, b"null pointer", a0=None)
    rejected(E_INVALID, b"empty operand", a12=0)
    rejected(E_INVALID, b"qmin", a4=5, a5=1)
    rejected(-4, b"workspace too small", a16=16)
    _nulled(rejected, 3)
    for fn in (lib.sb200_int8_conv2d_dorefa, lib.sb200_int8_conv2d_nhwc_dorefa):
        conv = [p, ctypes.byref(g), p, p, p, -128, 127, p, p, p, p, None, p, 8, p, 1 << 20, None]
        rejected = rejector(fn, conv)
        rejected(E_INVALID, b"null pointer", a1=None)
        rejected(E_INVALID, b"empty operand", a13=0)
        rejected(E_INVALID, b"non-positive geometry", a1=ctypes.byref(conv_geom(n=0)))
        rejected(E_INVALID, b"qmin", a5=5, a6=1)
        rejected(-4, b"workspace too small", a15=16)
        _nulled(rejected, 4)
    for fn, dense in ((lib.sb200_int8_group_conv2d_dorefa, b"sb200_int8_conv2d"),
                      (lib.sb200_int8_group_conv2d_nhwc_dorefa, b"sb200_int8_conv2d_nhwc")):
        grp = [p, ctypes.byref(g), 2, p, p, p, -128, 127, p, p, p, p, None, p, 8, None]
        rejected = rejector(fn, grp)
        rejected(E_INVALID, b"null pointer", a0=None)
        rejected(E_INVALID, dense, a2=1)
        rejected(E_INVALID, b"does not divide", a2=3)
        rejected(E_INVALID, b"qmin", a6=5, a7=1)
        _nulled(rejected, 5)


def test_dorefa_cases_reach_every_branch_of_their_kernels():
    """The cases the DoReFa GPU suite runs, through the geometry mirrors of the plain suites, reach every branch of the
    kernels that have a DoReFa instantiation: the row quantizer, the lowering, the GEMM and its NCHW epilogue
    (int8_geometry.REQUIRED without the matmul, the column quantizer and per-row qparams, which a per-tensor DoReFa
    input never takes), the grouped kernel (int8_group_geometry.REQUIRED) and the NHWC lowering and grouped kernel."""
    lin_required = {b for b in int8_geometry.REQUIRED if b.split(".")[0] in ("rows", "low", "gemm", "nchw")}
    lin_required.discard("rows.per_row")
    assert {c.op for c in dorefa_suite.LIN_CASES} == {"linear", "conv"}
    assert_table_covers(dorefa_suite.LIN_CASES, lin_required, lin_suite._covers, lin_suite.__doc__, doc_branches=False)

    def group_covers(item):
        name, case = item
        return int8_group_geometry.branches(*case)

    reached = set()
    for item in dorefa_suite.GROUP_CASES.items():
        reached |= group_covers(item)
    assert reached == int8_group_geometry.REQUIRED, (int8_group_geometry.REQUIRED - reached, reached - int8_group_geometry.REQUIRED)
    assert set(grp_suite.CASES) <= set(dorefa_suite.GROUP_CASES)
    assert dorefa_suite.nhwc_suite.CASES is nhwc_suite.CASES
    assert_table_covers(nhwc_suite.LOWER, int8_nhwc_geometry.LOWER_REQUIRED,
                        lambda c: check_reach(c, nhwc_suite.reached(c)) or nhwc_suite.reached(c), nhwc_suite.__doc__)
    assert_table_covers(nhwc_suite.GROUP, int8_nhwc_geometry.GROUP_REQUIRED,
                        lambda c: check_reach(c, nhwc_suite.reached(c)) or nhwc_suite.reached(c), nhwc_suite.__doc__)


def test_x_absmax_argument_rules(monkeypatch):
    """ops._x_absmax_args: no x_absmax keeps the plain entry point; otherwise one fp32 element on x's device selects the
    _dorefa entry point, anything else is refused before any call."""
    from sparsebit_b200 import SparsebitB200Error, ops
    x = torch.zeros(4, 8)
    assert ops._x_absmax_args("int8_linear", x, None) == ("", [])
    with pytest.raises(SparsebitB200Error, match="CUDA tensor"):
        ops._x_absmax_args("int8_linear", x, torch.zeros(1))  # the tensor rules of every operand come first
    monkeypatch.setattr(ops, "_req", lambda t, name, *a, **k: t)  # the remaining rules, on host tensors
    m = torch.zeros(1)
    assert ops._x_absmax_args("int8_linear", x, m) == ("_dorefa", [m.data_ptr()])
    with pytest.raises(SparsebitB200Error, match="int8_conv2d: x_absmax must be one fp32 element on x's device"):
        ops._x_absmax_args("int8_conv2d", x, torch.zeros(2))
    with pytest.raises(SparsebitB200Error, match="on x's device"):
        ops._x_absmax_args("int8_conv2d", x, torch.zeros(1, device="meta"))
