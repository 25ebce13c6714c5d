"""GPU: the 2:4-sparse integer-grid conv2d (sb200_int8_sparse24_conv2d / ops.int8_sparse24_conv2d) and
QConv2dSparse24Int8.

* Bit-identity with ops.int8_conv2d on the same stored weight over strides, paddings (asymmetric included), dilations,
  output sizes down to 1x1, C_out from 1 to 2048, signed and unsigned activations with non-zero zero points, 4-bit and
  affine 8-bit weights, per-tensor and per-channel, with and without bias.
* NaN windows, +-inf inputs and NaN weight rows, bit-identical to the dense path.
* Every distinct ResNet-50 conv at batch 4, bit-identical.
* Determinism, CUDA graph replay after a larger eager call, K = 2^17 unsupported.
* A pruned CNN: to_sparse24_integer_convs converts exactly its 2:4-pruned dense convs, and the converted model equals
  the all-dense conversion bit for bit."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_sparse24_ref as ref
from gpu_util import dev, t
from int8_harness import calibrated, cfg, stored_rows
from sparsebit_b200 import SparsebitB200Error, ops
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.modules import (QConv2d, QConv2dGroupInt8, QConv2dInt8, QConv2dSparse24Int8,
                                                 int8_conv_ineligibility, int8_sparse24_conv_ineligibility)
from sparsebit_b200.quantization.tools import to_integer_convs, to_integer_group_convs, to_sparse24_integer_convs
from sparsebit_b200.sparse.modules import SConv2d

pytestmark = pytest.mark.gpu

F32 = np.float32
SIGNED, UNSIGNED = (-128, 127), (0, 255)


def _bits(y):
    return np.asarray(y, F32).view(np.uint32)


def _both(x, xs, xz, xr, w, ws, wz, wr, bias=None, stride=1, padding=0, dilation=1):
    """(sparse y, dense y) as fp32 NCHW arrays from the same stored weight."""
    kernel = w.shape[2:]
    w_q, w_sum, w_scale, w_zero = stored_rows(w, ws, wz, *wr)
    vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero, w_scale, w[0].size)
    assert not bad.any()
    xt, xst, xzt = t(x), t(np.array([xs], F32)), t(np.array([xz], F32))
    bt = None if bias is None else t(bias)
    ys = ops.int8_sparse24_conv2d(xt, xst, xzt, *xr, vals, meta, dsum, w_scale, kernel, bt, stride, padding, dilation)
    yd = ops.int8_conv2d(xt, xst, xzt, *xr, w_q, w_sum, w_scale, w_zero, kernel, bt, stride, padding, dilation)
    return ys.cpu().numpy(), yd.cpu().numpy()


def _pruned(rng, shape, wr, ws, scale=0.45):
    """A conv weight 2:4 sparse in value along the rows of weight.reshape(C_out, -1), spread over +-scale of the range."""
    wqmin, wqmax = wr
    s = np.asarray(ws, F32).reshape(-1, 1, 1, 1)
    w = (rng.uniform(-scale, scale, shape) * (wqmax - wqmin) * s).astype(F32)
    return np.where(ref.mask24(rng.standard_normal(shape).astype(F32)), w, F32(0))


def _case(rng, n, c, h, w_, c_out, kh, kw, xr, wr, zx, zw, per_channel):
    (xqmin, xqmax), (wqmin, wqmax) = xr, wr
    xs = F32(2.0 ** -4) * F32(1.37)
    nw = c_out if per_channel else 1
    ws = (rng.uniform(0.5, 2.0, nw) * 2.0 ** -6).astype(F32)
    wz = np.full(nw, zw, F32) + (rng.integers(-3, 4, nw) if zw else 0)
    span = (xqmax - xqmin) * float(xs)
    x = (rng.uniform(-0.7 * span, 0.7 * span, (n, c, h, w_)) + (0.4 * span if xqmin >= 0 else 0)).astype(F32)
    w = _pruned(rng, (c_out, c, kh, kw), wr, ws)
    return x, xs, F32(zx), xr, w, ws, wz, wr


GEOMS = [
    # (n, c, h, w, c_out, kh, kw, stride, padding, dilation, x range, w range, zx, zw, per-channel w, bias)
    (2, 3, 32, 32, 64, 7, 7, 2, 3, 1, SIGNED, SIGNED, 0, 0, True, True),             # the stem, K = 147
    (3, 16, 14, 14, 200, 3, 3, 1, 1, 1, UNSIGNED, SIGNED, 131, 0, True, False),      # 3x3 p1
    (2, 64, 15, 15, 2048, 1, 1, 2, 0, 1, SIGNED, SIGNED, -7, 0, False, True),        # 1x1 s2
    (2, 8, 17, 17, 64, 3, 3, 1, 2, 2, UNSIGNED, (-8, 7), 60, 0, True, True),         # dilation 2, 4-bit weights
    (1, 12, 11, 10, 1, 3, 3, 2, (1, 0, 2, 1), 1, SIGNED, SIGNED, 3, 0, True, False),  # asymmetric padding, C_out = 1
    (4, 32, 14, 14, 64, 3, 3, 2, 1, 1, UNSIGNED, UNSIGNED, 255, 128, True, True),     # 7x7 output, affine 8-bit weights
    (5, 64, 3, 3, 200, 3, 3, 1, 0, 1, UNSIGNED, (0, 15), 77, 8, False, False),        # 1x1 output, 4-bit affine
    (2, 48, 9, 9, 64, 3, 3, 1, 1, 1, SIGNED, UNSIGNED, 0, 128, False, True),          # affine 8-bit, per-tensor
]


@pytest.mark.parametrize("n,c,h,w,c_out,kh,kw,stride,padding,dilation,xr,wr,zx,zw,per_channel,with_bias", GEOMS)
def test_bit_identical_to_the_dense_conv(n, c, h, w, c_out, kh, kw, stride, padding, dilation, xr, wr, zx, zw,
                                         per_channel, with_bias):
    rng = np.random.default_rng(n * 1000 + c * 7 + c_out + kh)
    x, xs, xz, xr, wt, ws, wz, wr = _case(rng, n, c, h, w, c_out, kh, kw, xr, wr, zx, zw, per_channel)
    bias = rng.standard_normal(c_out).astype(F32) if with_bias else None
    ys, yd = _both(x, xs, xz, xr, wt, ws, wz, wr, bias, stride, padding, dilation)
    assert ys.shape == yd.shape and np.array_equal(_bits(ys), _bits(yd))


def test_nan_windows_inf_inputs_and_nan_weight_rows_are_bit_identical():
    rng = np.random.default_rng(3)
    x, xs, xz, xr, w, ws, wz, wr = _case(rng, 2, 8, 12, 12, 72, 3, 3, SIGNED, SIGNED, 0, 0, True)
    x[1, 3, 5, 7] = np.nan
    x[0, 0, 0, 0], x[0, 5, 11, 11], x[1, 7, 2, 3] = np.inf, -np.inf, np.inf
    w[9, 2, 1, 1] = np.nan  # the NaN weight row marks its channel through w_scale
    bias = rng.standard_normal(72).astype(F32)
    ys, yd = _both(x, xs, xz, xr, w, ws, wz, wr, bias, 1, 1)
    assert np.array_equal(_bits(ys), _bits(yd))
    # the NaN pixel NaNs exactly the outputs whose 3x3 windows hold it, in every channel of image 1
    win = np.zeros((2, 12, 12), bool)
    win[1, 4:7, 6:9] = True
    nan = np.isnan(ys)
    expect = np.broadcast_to(win[:, None], ys.shape).copy()
    expect[:, 9] = True
    assert np.array_equal(nan, expect)


def _r50_convs():
    """(c_in, hw, c_out, kernel, stride, padding) of the distinct convs of ResNet-50."""
    convs = [(3, 224, 64, 7, 2, 3)]
    inplanes, hw = 64, 56
    for planes, blocks, stride in [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)]:
        for b in range(blocks):
            s = stride if b == 0 else 1
            convs += [(inplanes, hw, planes, 1, 1, 0), (planes, hw, planes, 3, s, 1), (planes, hw // s, planes * 4, 1, 1, 0)]
            if b == 0:
                convs.append((inplanes, hw, planes * 4, 1, s, 0))
            inplanes, hw = planes * 4, hw // s
    return sorted(set(convs))


@pytest.mark.parametrize("c, hw, c_out, k, stride, padding", _r50_convs())
def test_resnet50_shapes_are_bit_identical(c, hw, c_out, k, stride, padding):
    rng = np.random.default_rng(c * 3 + hw + c_out * 5 + k + stride)
    x = rng.standard_normal((4, c, hw, hw)).astype(F32)
    w = _pruned(rng, (c_out, c, k, k), SIGNED, np.full(c_out, 1.0 / 127 / np.sqrt(c * k * k), F32), scale=0.4)
    ws = np.abs(w).reshape(c_out, -1).max(1).astype(F32) / 127 + F32(1e-8)
    ys, yd = _both(x, F32(0.03), F32(0), SIGNED, w, ws, np.zeros(c_out, F32), SIGNED,
                   rng.standard_normal(c_out).astype(F32), stride, padding)
    assert np.array_equal(_bits(ys), _bits(yd))


def test_deterministic_and_graph_replay_after_a_larger_call():
    rng = np.random.default_rng(12)
    x, xs, xz, xr, w, ws, wz, wr = _case(rng, 2, 16, 10, 10, 96, 3, 3, UNSIGNED, SIGNED, 100, 0, True)
    w_q, _, w_scale, w_zero = stored_rows(w, ws, wz, *wr)
    vals, meta, dsum, _ = ops.int8_sparse24_pack(w_q, w_zero, w_scale, w[0].size)
    xt, xst, xzt = t(x), t(np.array([xs], F32)), t(np.array([xz], F32))
    big = t(rng.standard_normal((16, 16, 40, 40)).astype(F32))

    def call(inp):
        return ops.int8_sparse24_conv2d(inp, xst, xzt, *xr, vals, meta, dsum, w_scale, 3, padding=1)

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
    c = (1 << 17) // 9 + 1  # K = 9 c >= 2^17
    x = torch.zeros(1, c, 3, 3, device=dev())
    one = torch.ones(1, device=dev())
    vshape, mshape = ops.int8_sparse24_shapes(8, 9 * c)
    vals = torch.zeros(vshape, dtype=torch.int8, device=dev())
    meta = torch.zeros(mshape, dtype=torch.int32, device=dev())
    with pytest.raises(SparsebitB200Error, match=r"K < 2\^17.*status -3"):
        ops.int8_sparse24_conv2d(x, one, one * 0, -128, 127, vals, meta, torch.zeros(8, dtype=torch.int32, device=dev()),
                                 torch.ones(8, device=dev()), 3)


# ---------------------------------------------------------------------------------------------- modules
class Cnn(nn.Module):
    """An unpruned stem, 2:4-pruned 3x3 and 1x1 convs, a depthwise conv and a dense 1x1."""

    def __init__(self):
        super().__init__()
        self.stem = nn.Conv2d(3, 32, 3, stride=2, padding=1)
        self.c3 = SConv2d(nn.Conv2d(32, 64, 3, padding=1))
        self.c1 = SConv2d(nn.Conv2d(64, 48, 1, stride=2, bias=False))
        self.dw = nn.Conv2d(48, 48, 3, padding=1, groups=48)
        self.head = nn.Conv2d(48, 10, 1)
        for m in (self.c3, self.c1):
            m.build_sparser(sbcfg.sparser_config(0.5, stype="2:4"))

    def forward(self, x):
        return self.head(torch.relu(self.dw(torch.relu(self.c1(torch.relu(self.c3(torch.relu(self.stem(x)))))))))


class QCnn(nn.Module):
    """``Cnn`` with each mask folded into its weight and every conv a QConv2d."""

    def __init__(self, cnn):
        super().__init__()
        for name, bits, scheme, ascheme in (("stem", 8, "per-channel-symmetric", "per-tensor-symmetric"),
                                            ("c3", 4, "per-channel-symmetric", "per-tensor-affine"),
                                            ("c1", 8, "per-tensor-symmetric", "per-tensor-affine"),
                                            ("dw", 8, "per-channel-symmetric", "per-tensor-affine"),
                                            ("head", 8, "per-channel-symmetric", "per-tensor-affine")):
            src = getattr(cnn, name)
            kw = src.fwd_kwargs if isinstance(src, SConv2d) else dict(stride=src.stride, padding=src.padding,
                                                                       dilation=src.dilation, groups=src.groups)
            conv = nn.Conv2d(src.weight.shape[1] * kw["groups"], src.weight.shape[0], tuple(src.weight.shape[2:]),
                             bias=src.bias is not None, **kw).to(dev())
            with torch.no_grad():
                conv.weight.copy_(src.weight * src.w_mask if isinstance(src, SConv2d) else src.weight)
                if src.bias is not None:
                    conv.bias.copy_(src.bias)
            setattr(self, name, QConv2d(conv).build_quantizer(cfg(ascheme, "feature"), cfg(scheme, "weight", bit=bits)))

    def forward(self, x):
        return self.head(torch.relu(self.dw(torch.relu(self.c1(torch.relu(self.c3(torch.relu(self.stem(x)))))))))


def test_pruned_cnn_converts_exactly_its_sparse_convs():
    torch.manual_seed(0)
    cnn = Cnn().to(dev())
    for m in (cnn.c3, cnn.c1):
        m.calc_mask()
        assert np.array_equal(m.w_mask.cpu().numpy(), ref.mask24(m.weight.detach().cpu().numpy()))
    model = QCnn(cnn)
    calibrated(model, (torch.randn(4, 3, 32, 32, device=dev()) for _ in range(2)), streaming=True, record_inputs=None)
    assert "not 2:4 sparse" in int8_sparse24_conv_ineligibility(model.stem)
    assert int8_sparse24_conv_ineligibility(model.dw) == int8_conv_ineligibility(model.dw)
    dense = copy.deepcopy(model)
    assert to_sparse24_integer_convs(model) == ["c3", "c1"]
    assert isinstance(model.c3, QConv2dSparse24Int8) and isinstance(model.c1, QConv2dSparse24Int8)
    for m in (model.c3, model.c1):
        assert not any(name.startswith("w_q") for name, _ in m.named_buffers())
    assert to_integer_convs(model) == ["stem", "head"]
    assert to_integer_group_convs(model) == ["dw"]
    assert to_integer_convs(dense) == ["stem", "c3", "c1", "head"] and to_integer_group_convs(dense) == ["dw"]
    assert isinstance(model.stem, QConv2dInt8) and isinstance(model.dw, QConv2dGroupInt8)
    x = torch.randn(3, 3, 32, 32, device=dev())
    with torch.no_grad():
        y, yd = model(x), dense(x)
        assert torch.equal(y.view(torch.int32), yd.view(torch.int32))
        assert torch.equal(model(x.half()).view(torch.int32), dense(x.half()).view(torch.int32))
        yu = model(x[1])
        assert yu.shape == yd.shape[1:] and torch.equal(yu.view(torch.int32), yd[1].view(torch.int32))
        with pytest.raises(RuntimeError, match="inference-only"):
            with torch.enable_grad():
                model.c3(torch.randn(1, 32, 8, 8, device=dev(), requires_grad=True))


def test_ineligibility_names_the_row_and_group():
    torch.manual_seed(1)
    conv = nn.Conv2d(8, 16, 3, padding=1).to(dev())
    with torch.no_grad():
        conv.weight.mul_(torch.from_numpy(ref.mask24(conv.weight.cpu().numpy())).to(dev()))
        conv.weight[5, 1, 0, 0] = 0.3  # k = 9 of row 5: group 2 (k = 8 .. 11) now has three nonzeros
        conv.weight[5, 1, 0, 1] = 0.2
        conv.weight[5, 1, 0, 2] = -0.25
    q = QConv2d(conv).build_quantizer(cfg("per-tensor-symmetric", "feature"), cfg("per-channel-symmetric", "weight"))
    q.input_quantizer.update_observer(torch.randn(2, 8, 6, 6, device=dev()))
    q.input_quantizer.calc_qparams()
    q.weight_quantizer.update_observer(q.weight)
    q.weight_quantizer.calc_qparams()
    q.set_quant(True, True)
    assert int8_conv_ineligibility(q) is None
    reason = int8_sparse24_conv_ineligibility(q)
    assert reason == "the weight is not 2:4 sparse on the grid: row 5, group 2 (k = 8 .. 11) has more than two nonzeros"
    with pytest.raises(ValueError, match=r"QConv2dSparse24Int8.from_qconv2d: .*row 5, group 2"):
        QConv2dSparse24Int8.from_qconv2d(q)
