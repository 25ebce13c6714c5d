"""GPU: 2:4 sparsity on the integer grid (sb200_sparse24_mask, sb200_int8_sparse24_pack, sb200_int8_sparse24_linear,
QLinearSparse24Int8, to_sparse24_integer_linears).

* The mask equals the numpy rule (tests/int8_sparse24_ref.py) bit for bit, directly and through the l1norm sparser.
* pack equals the numpy restatement bit for bit: vals, the metadata words, dsum, bad.
* Bit-identity: the sparse linear equals sb200_int8_linear on the same stored weight bit for bit, NaNs included, over
  signed and unsigned activations, zero points away from 0, per-tensor and per-channel weights, 4-bit weights, with and
  without bias, K in {16, 33, 768, 1001, 11008}, partial M and N tiles, and the DeiT-base and LLaMA-7B shapes.
* Truth: the output meets int8_linear's bound against the fp64 fake-quant truth.
* Determinism and a captured CUDA graph that replays after a larger eager call.
* End to end: nn.Linear -> SLinear with the 2:4 sparser -> mask folded -> calibrated QLinear ->
  to_sparse24_integer_linears converts exactly the 2:4 layers and leaves a dense one with its reason."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_sparse24_ref as ref
from gpu_util import dev, t
from int8_harness import calibrated, cfg, stored_rows
from int8_linear_ref import truth
from oracle import observers as oobs
from sparsebit_b200 import SparsebitB200Error, ops
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.modules import (QLinear, QLinearSparse24Int8, int8_ineligibility,
                                                 int8_sparse24_ineligibility)
from sparsebit_b200.quantization.tools import to_integer_linears, to_sparse24_integer_linears
from sparsebit_b200.sparse.modules import SLinear

pytestmark = pytest.mark.gpu

F32 = np.float32


def _bits(y):
    return np.asarray(y, F32).view(np.uint32)


def _specials(rng, w):
    w = w.copy()
    n, k = w.shape
    w[rng.random((n, k)) < 0.05] = 0.0
    w[rng.random((n, k)) < 0.05] = -0.0
    flat = w.reshape(-1)
    idx = rng.choice(flat.size, size=min(flat.size, 12), replace=False)
    flat[idx] = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, np.nan, 3.0, -3.0, 3.0, np.inf, -np.inf], F32)[: len(idx)]
    if k >= 4:  # exact ties inside a group
        w[0, :4] = [2.0, -2.0, 2.0, 1.0]
    return w


# ---------------------------------------------------------------------------------------------- sparser
@pytest.mark.parametrize("shape", [(37, 33), (16, 3, 3, 3), (5, 1), (64, 768), (9, 6)])
def test_mask_is_the_rule(shape):
    rng = np.random.default_rng(sum(shape))
    w = rng.standard_normal(shape).astype(F32)
    w = _specials(rng, w.reshape(shape[0], -1)).reshape(shape)
    m = ops.sparse24_mask(t(w))
    assert m.dtype == torch.bool and m.shape == w.shape
    assert np.array_equal(m.cpu().numpy(), ref.mask24(w))


def test_sparser_type_and_ratio():
    from sparsebit_b200.sparse.sparsers import build_sparser

    w = torch.randn(24, 40, device=dev())
    lin = SLinear(nn.Linear(40, 24)).to(dev())
    sp = build_sparser(sbcfg.sparser_config(0.5, stype="2:4"), lin)
    m = sp.calc_mask(w)
    assert m.dtype == ops.mask_gt(w, torch.zeros(1, device=dev())).dtype  # the unstructured mask's dtype
    assert np.array_equal(m.cpu().numpy(), ref.mask24(w.cpu().numpy()))
    assert torch.equal(build_sparser(sbcfg.sparser_config(0.0, stype="2:4"), lin).calc_mask(w), torch.ones_like(w))
    with pytest.raises(ValueError, match="2:4"):
        build_sparser(sbcfg.sparser_config(0.3, stype="2:4"), lin).calc_mask(w)


# ---------------------------------------------------------------------------------------------- pack
def _sparse_weights(rng, n, k, wr, ws, wz, scale=0.45):
    """Weights 2:4 sparse in value (so on the grid), spread over +-scale of the range around 0."""
    wqmin, wqmax = wr
    w = (rng.uniform(-scale, scale, (n, k)) * (wqmax - wqmin) * np.asarray(ws, F32).reshape(-1, 1)).astype(F32)
    return np.where(ref.mask24(rng.standard_normal((n, k)).astype(F32)), w, F32(0))


@pytest.mark.parametrize("n, k, wr, zero", [(37, 33, (-128, 127), 0), (130, 1001, (0, 255), 128), (8, 16, (-8, 7), 0),
                                            (300, 768, (0, 15), 7), (64, 11008, (-128, 127), 0)])
def test_pack_is_the_restatement(n, k, wr, zero):
    rng = np.random.default_rng(n + k)
    ws = (2.0 ** -rng.integers(3, 8, n)).astype(F32)
    wz = np.full(n, zero, F32)
    w = _sparse_weights(rng, n, k, wr, ws, wz)
    w[1, 5] = np.nan  # a NaN row: packed as zeros
    if n > 3:
        w[3, :4] = (np.array([1, 1, 1, 0], F32) * ws[3] * 3)  # three nonzeros: bad
    w_q, _, w_scale, w_zero = stored_rows(w, ws, wz, *wr)
    vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero, w_scale, k)
    ev, em, ed, eb = ref.pack(w_q.cpu().numpy(), w_zero.cpu().numpy(), w_scale.cpu().numpy(), k)
    assert np.array_equal(vals.cpu().numpy(), ev)
    assert np.array_equal(meta.cpu().numpy().view(np.uint32), em)
    assert np.array_equal(dsum.cpu().numpy(), ed) and np.array_equal(bad.cpu().numpy(), eb)
    assert eb[1] == 0 and (n <= 3 or eb[3] == 1)


# ---------------------------------------------------------------------------------------------- bit-identity
def _both(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, bias=None):
    """(sparse y, dense y) as fp32 [M, N] arrays from the same stored weight."""
    k = w.shape[1]
    w_q, w_sum, w_scale, w_zero = stored_rows(w, ws, wz, wqmin, wqmax)
    vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero, w_scale, k)
    assert not bad.any()
    xt, xst, xzt = t(x), t(np.array([xs], F32)), t(np.array([xz], F32))
    bt = None if bias is None else t(bias)
    ys = ops.int8_sparse24_linear(xt, xst, xzt, xqmin, xqmax, vals, meta, dsum, w_scale, bt)
    yd = ops.int8_linear(xt, xst, xzt, xqmin, xqmax, w_q, w_sum, w_scale, w_zero, bt)
    return ys.cpu().numpy().reshape(-1, w.shape[0]), yd.cpu().numpy().reshape(-1, w.shape[0])


def _case(rng, m, k, n, xr, wr, zx, zw, per_channel):
    (xqmin, xqmax), (wqmin, wqmax) = xr, wr
    xs = F32(2.0 ** -4) * F32(1.37)
    ws = (rng.uniform(0.5, 2.0, n if per_channel else 1) * 2.0 ** -6).astype(F32)
    wz = np.full(n if per_channel else 1, zw, F32) + (rng.integers(-3, 4, n if per_channel else 1) if zw else 0)
    span = (xqmax - xqmin) * float(xs)
    x = (rng.uniform(-0.7 * span, 0.7 * span, (m, k)) + (0.4 * span if xqmin >= 0 else 0)).astype(F32)
    w = _sparse_weights(rng, n, k, wr, ws, wz)
    return x, xs, F32(zx), xqmin, xqmax, w, ws, wz, wqmin, wqmax


SIGNED, UNSIGNED = (-128, 127), (0, 255)
CASES = [
    # (m, k, n, x range, w range, zx, zw, per-channel w, bias)
    (1, 16, 8, SIGNED, SIGNED, 0, 0, True, True),
    (7, 33, 100, UNSIGNED, SIGNED, 131, 0, True, False),
    (129, 768, 200, SIGNED, SIGNED, 5, 0, False, True),
    (300, 1001, 129, UNSIGNED, UNSIGNED, 255, 128, True, True),
    (77, 11008, 64, SIGNED, SIGNED, -9, 0, True, False),
    (255, 768, 300, UNSIGNED, (-8, 7), 0, 0, True, True),
    (17, 1001, 257, SIGNED, (0, 15), 0, 8, False, False),
    (130, 33, 1, UNSIGNED, (-8, 7), 77, 2, True, True),
]


@pytest.mark.parametrize("m,k,n,xr,wr,zx,zw,per_channel,with_bias", CASES)
def test_bit_identical_to_the_dense_layer(m, k, n, xr, wr, zx, zw, per_channel, with_bias):
    rng = np.random.default_rng(m * 7 + k + n)
    args = _case(rng, m, k, n, xr, wr, zx, zw, per_channel)
    bias = rng.standard_normal(n).astype(F32) if with_bias else None
    ys, yd = _both(*args, bias=bias)
    assert np.array_equal(_bits(ys), _bits(yd))


def test_nan_rows_nan_columns_and_inf_inputs_are_bit_identical():
    rng = np.random.default_rng(3)
    x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax = _case(rng, 40, 200, 72, SIGNED, SIGNED, 0, 0, True)
    x[3, 17] = np.nan
    x[5, 0], x[6, 199], x[7, 100] = np.inf, -np.inf, np.inf
    w[9, 2] = np.nan  # the NaN weight row marks its column through w_scale
    bias = rng.standard_normal(72).astype(F32)
    ys, yd = _both(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, bias)
    assert np.isnan(ys[3]).all() and np.isnan(ys[:, 9]).all() and np.isnan(ys).sum() == 72 + 40 - 1
    assert np.array_equal(_bits(ys), _bits(yd))


@pytest.mark.parametrize("m, k, n", [(197 * 64, 768, 2304), (197 * 64, 768, 3072), (197 * 64, 3072, 768),
                                     (16, 4096, 4096), (16, 4096, 11008), (16, 11008, 4096),
                                     (2048, 4096, 4096), (2048, 4096, 11008), (2048, 11008, 4096)])
def test_model_shapes_are_bit_identical(m, k, n):
    rng = np.random.default_rng(m + k + n)
    x = rng.standard_normal((m, k)).astype(F32)
    ws = (rng.uniform(0.5, 2.0, n) / 128 / np.sqrt(k) * 4).astype(F32)
    w = np.where(ref.mask24(rng.standard_normal((n, k)).astype(F32)), rng.standard_normal((n, k)) / np.sqrt(k), 0).astype(F32)
    ys, yd = _both(x, F32(0.03), F32(0), -128, 127, w, ws, np.zeros(n, F32), -128, 127, rng.standard_normal(n).astype(F32))
    assert np.array_equal(_bits(ys), _bits(yd))


def test_meets_the_truth_bound():
    rng = np.random.default_rng(21)
    m, k, n = 300, 1001, 264
    x = (rng.standard_normal((m, k)) * 2 + 0.8).astype(F32)
    w = np.where(ref.mask24(rng.standard_normal((n, k)).astype(F32)), rng.standard_normal((n, k)) / np.sqrt(k), 0).astype(F32)
    xs, xz = oobs.calc_qparams_with_minmax(*oobs.minmax([x]), 0, 255, False)
    ws, wz = oobs.calc_qparams_with_minmax(*oobs.minmax([w], per_channel=True), -128, 127, True)
    bias = rng.standard_normal(n).astype(F32)
    args = (x, F32(xs), F32(xz), 0, 255, w, ws, wz, -128, 127)
    ys, _ = _both(*args, bias=bias)
    t_, bound = truth(*args, bias=bias)
    assert np.all(np.abs(ys - t_) <= bound)


def test_deterministic_and_graph_replay_after_a_larger_call():
    rng = np.random.default_rng(12)
    x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax = _case(rng, 33, 768, 300, UNSIGNED, SIGNED, 100, 0, True)
    w_q, _, w_scale, w_zero = stored_rows(w, ws, wz, wqmin, wqmax)
    vals, meta, dsum, _ = ops.int8_sparse24_pack(w_q, w_zero, w_scale, 768)
    xt, xst, xzt = t(x), t(np.array([xs], F32)), t(np.array([xz], F32))
    big = t(rng.standard_normal((4000, 768)).astype(F32))

    def call(inp):
        return ops.int8_sparse24_linear(inp, xst, xzt, xqmin, xqmax, vals, meta, dsum, w_scale)

    y1, y2 = call(xt), call(xt)
    assert torch.equal(y1, y2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call(xt)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            yg = call(xt)
        yb = call(big)  # outgrows the captured workspace
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, y1)
    assert torch.equal(yb, call(big))


def test_k_limit_is_unsupported():
    k = 1 << 17
    x = torch.zeros(2, k, device=dev())
    one = torch.ones(1, device=dev())
    vshape, mshape = ops.int8_sparse24_shapes(8, k)
    vals = torch.zeros(vshape, dtype=torch.int8, device=dev())
    meta = torch.zeros(mshape, dtype=torch.int32, device=dev())
    with pytest.raises(SparsebitB200Error, match=r"K < 2\^17.*status -3"):
        ops.int8_sparse24_linear(x, one, one * 0, -128, 127, vals, meta, torch.zeros(8, dtype=torch.int32, device=dev()),
                                 torch.ones(8, device=dev()))


# ---------------------------------------------------------------------------------------------- modules
class Mlp(nn.Module):
    """Two 2:4-pruned layers (fc1 4-bit per-channel weights, fc2 affine activations) and a dense one."""

    def __init__(self):
        super().__init__()
        self.fc1 = SLinear(nn.Linear(768, 1001))
        self.fc2 = SLinear(nn.Linear(1001, 96))
        self.head = nn.Linear(96, 40)
        for m in (self.fc1, self.fc2):
            m.build_sparser(sbcfg.sparser_config(0.5, stype="2:4"))

    def forward(self, x):
        return self.head(torch.relu(self.fc2(torch.relu(self.fc1(x)))))


class QMlp(nn.Module):
    """``Mlp`` with each mask folded into its weight and every layer a QLinear."""

    def __init__(self, mlp):
        super().__init__()
        for name, bits, scheme, ascheme in (("fc1", 4, "per-channel-symmetric", "per-tensor-symmetric"),
                                            ("fc2", 8, "per-channel-symmetric", "per-tensor-affine"),
                                            ("head", 8, "per-tensor-symmetric", "per-tensor-symmetric")):
            src = getattr(mlp, name)
            lin = nn.Linear(src.weight.shape[1], src.weight.shape[0]).to(dev())
            with torch.no_grad():
                lin.weight.copy_(src.weight * src.w_mask if isinstance(src, SLinear) else src.weight)
                lin.bias.copy_(src.bias)
            setattr(self, name, QLinear(lin).build_quantizer(cfg(ascheme, "feature", layout="NLC"),
                                                             cfg(scheme, "weight", bit=bits)))

    def forward(self, x):
        return self.head(torch.relu(self.fc2(torch.relu(self.fc1(x)))))


def test_pruned_model_converts_exactly_its_sparse_layers():
    torch.manual_seed(0)
    mlp = Mlp().to(dev())
    for m in (mlp.fc1, mlp.fc2):
        m.calc_mask()
        assert np.array_equal(m.w_mask.cpu().numpy(), ref.mask24(m.weight.detach().cpu().numpy()))
    model = QMlp(mlp)
    batches = [torch.randn(4, 50, 768, device=dev()) for _ in range(2)]
    calibrated(model, batches, streaming=True, record_inputs=None)
    assert "not 2:4 sparse" in int8_sparse24_ineligibility(model.head)
    assert "row 0, group" in int8_sparse24_ineligibility(model.head)
    dense = copy.deepcopy(model)
    assert to_sparse24_integer_linears(model) == ["fc1", "fc2"]
    assert isinstance(model.fc1, QLinearSparse24Int8) and isinstance(model.head, QLinear)
    assert not any(name.startswith("w_q") for name, _ in model.fc1.named_buffers())
    assert to_integer_linears(model) == ["head"]
    assert to_integer_linears(dense) == ["fc1", "fc2", "head"]
    x = torch.randn(3, 50, 768, device=dev())
    with torch.no_grad():
        for name in ("fc1", "fc2"):
            xin = torch.relu(dense.fc1(x)) if name == "fc2" else x
            assert torch.equal(getattr(model, name)(xin).view(torch.int32), getattr(dense, name)(xin).view(torch.int32))
            assert torch.equal(getattr(model, name)(xin.half()), getattr(dense, name)(xin.half()))
        assert torch.equal(model(x), dense(x))


def test_ineligibility_names_the_row_and_group():
    torch.manual_seed(1)
    lin = nn.Linear(64, 16).to(dev())
    with torch.no_grad():
        lin.weight.mul_(torch.from_numpy(ref.mask24(lin.weight.cpu().numpy())).to(dev()))
        lin.weight[5, 9] = 0.3  # group 2 of row 5 now has three nonzeros
    q = QLinear(lin).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"), cfg("per-channel-symmetric", "weight"))
    q.input_quantizer.update_observer(torch.randn(2, 8, 64, device=dev()))
    q.input_quantizer.calc_qparams()
    q.weight_quantizer.update_observer(q.weight)
    q.weight_quantizer.calc_qparams()
    q.set_quant(True, True)
    assert int8_ineligibility(q) is None
    assert int8_sparse24_ineligibility(q) == ("the weight is not 2:4 sparse on the grid: row 5, group 2 (k = 8 .. 11) has "
                                              "more than two nonzeros")
    with pytest.raises(ValueError, match="QLinearSparse24Int8.from_qlinear: .*row 5, group 2"):
        QLinearSparse24Int8.from_qlinear(q)
    # an affine 8-bit weight whose centred grid leaves s8
    with torch.no_grad():
        lin.weight[5, 9] = 0.0
        lin.weight.abs_()
    qa = QLinear(lin).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"), cfg("per-tensor-affine", "weight"))
    qa.input_quantizer.update_observer(torch.randn(2, 8, 64, device=dev()))
    qa.input_quantizer.calc_qparams()
    qa.weight_quantizer.update_observer(qa.weight)
    qa.weight_quantizer.calc_qparams()
    qa.set_quant(True, True)
    if int8_ineligibility(qa) is None:
        assert "leaves s8" in int8_sparse24_ineligibility(qa)
