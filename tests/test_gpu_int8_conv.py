"""GPU: the integer-grid conv2d (sb200_int8_im2col_quantize, sb200_int8_conv2d, QConv2dInt8, to_integer_convs).

* The lowering equals F.unfold of the oracle's integer grid bit for bit (tests/int8_conv_ref.py): 1x1, 3x3, 7x7
  (ragged K = 147), dilation, 1x3 / 5x1 kernels, asymmetric padding, odd H / W, M not a multiple of 128; signed,
  unsigned (zero point away from 0), 4- and 2-bit ranges; ties, +-inf, +-0, subnormals and NaN -- the NaN flags set
  on exactly the windows that cover a NaN; and sampled rows at the far end of a case with M Kp >= 2^31.
* Exact mode: power-of-two scales and zero bias, every output whose integer sum is exact in fp32 equals the truth.
* General data with MinMax qparams: |y - T| <= 2^-21 (conv(|fx|, |fw|) + |bias|) elementwise; NaN positions as the
  fake-quant QConv2d; a NaN weight row gives a NaN channel.
* Determinism, CUDA graph replay, K = 2^17 unsupported, fp16 / unbatched input, no backward.
* Modules: a calibrated CNN and a seeded torchvision ResNet-18 converted by to_integer_convs meet the bound per layer."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from gpu_util import dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from int8_conv_ref import lowered, truth
from int8_harness import calibrated, cfg, check_converted, layer_qparams, qrange, stored_rows, wrap_quantized
from oracle import observers as oobs
from sparsebit_b200 import SparsebitB200Error, ops
from sparsebit_b200.quantization.modules import QConv2d, QConv2dInt8, QLinear, QReLU
from sparsebit_b200.quantization.tools import to_integer_convs

pytestmark = pytest.mark.gpu

F32 = np.float32


# ---------------------------------------------------------------------------------------------- the lowering
GEOMS = [
    # (n, c, h, w, kernel, stride, padding, dilation)
    (3, 5, 9, 11, 1, 1, 0, 1),
    (2, 8, 10, 10, 1, 2, 0, 1),
    (2, 6, 9, 9, 3, 1, 1, 1),
    (3, 4, 11, 10, 3, 2, 1, 1),
    (2, 3, 23, 21, 7, 2, 3, 1),           # K = 147: ragged, two K chunks
    (1, 16, 17, 15, 3, 1, 2, 2),          # dilation 2
    (2, 7, 8, 13, (1, 3), 1, (0, 1), 1),
    (2, 5, 12, 6, (5, 1), 1, (2, 0), 1),
    (2, 6, 9, 8, 3, 1, (0, 2, 1, 0), 1),  # asymmetric (top, bottom, left, right)
    (5, 3, 13, 7, 3, 1, 1, 1),            # M = 455: not a multiple of 128
    (1, 40, 6, 6, 3, 1, 1, 1),            # K = 360: three K chunks
]
LOW_RANGES = [(-128, 127), (0, 255), (-8, 7), (0, 15), (-2, 1)]


def _specials(rng, x, s):
    """Ties (k + 1/2) s, +-inf, +-0, subnormals; one NaN in image 0."""
    ties = (rng.integers(-140, 140, x.shape).astype(F32) + F32(0.5)) * F32(s)
    x = np.where(rng.random(x.shape) < 0.25, ties.astype(F32), x)
    flat = x.reshape(-1)
    special = np.array([np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39], F32)
    flat[rng.choice(flat.size, size=len(special), replace=False)] = special
    x = flat.reshape(x.shape)
    # at even (h, w): a tap of every geometry below, stride 2 included
    x[0, rng.integers(0, x.shape[1]), 2 * rng.integers(0, (x.shape[2] + 1) // 2), 2 * rng.integers(0, (x.shape[3] + 1) // 2)] = np.nan
    return x


def _check_lowering(x, kernel, s, z, qmin, qmax, stride, padding, dilation):
    q, row_sum, nan = ops.int8_im2col_quantize(t(x), kernel, t(np.array([s], F32)), t(np.array([z], F32)), qmin, qmax,
                                               stride, padding, dilation)
    eq, esum, enan = lowered(x, kernel, s, z, qmin, qmax, stride, padding, dilation)
    assert q.shape == eq.shape and q.dtype == torch.int8
    assert np.array_equal(q.cpu().numpy().astype(np.int64), eq)
    assert np.array_equal(row_sum.cpu().numpy().astype(np.int64), esum)
    assert np.array_equal(nan.cpu().numpy(), enan)
    return enan


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("qrange", LOW_RANGES)
def test_lowering_is_the_unfolded_oracle_grid(geom, qrange):
    n, c, h, w, kernel, stride, padding, dilation = geom
    qmin, qmax = qrange
    rng = np.random.default_rng(abs(hash((geom, qrange))) % 2**32)
    s = F32(0.37)
    z = F32((qmin + qmax) // 2 + 0.5 if qmin < 0 else qmin + (qmax - qmin) // 3 + 0.5)  # a tie of rint, away from 0
    x = _specials(rng, (rng.standard_normal((n, c, h, w)) * 20).astype(F32), s)
    enan = _check_lowering(x, kernel, s, z, qmin, qmax, stride, padding, dilation)
    assert enan.any() and not enan.all()


def test_lowering_far_end_of_a_workspace_past_2_31():
    """M Kp >= 2^31 (C = 1, 7x7, Kp = 64, M = 700 * 224^2): the rows of the first and the last image."""
    n, h = 700, 224
    rng = np.random.default_rng(9)
    x_last = (rng.standard_normal((2, 1, h, h)) * 3).astype(F32)
    x_last[1, 0, 200, 7] = np.nan
    xt = torch.randn(n, 1, h, h, device=dev())
    xt[0] = t(x_last[0])
    xt[-1] = t(x_last[1])
    s, z = F32(0.05), F32(131)
    q, row_sum, nan = ops.int8_im2col_quantize(xt, 7, t(np.array([s], F32)), t(np.array([z], F32)), 0, 255, 1, 3, 1)
    p = h * h
    assert q.shape == (n * p, 64) and q.numel() >= 2**31
    eq, esum, enan = lowered(x_last, 7, s, z, 0, 255, 1, 3, 1)
    for img, sl in ((0, slice(0, p)), (1, slice((n - 1) * p, n * p))):
        assert np.array_equal(q[sl].cpu().numpy().astype(np.int64), eq[img * p:(img + 1) * p])
        assert np.array_equal(row_sum[sl].cpu().numpy().astype(np.int64), esum[img * p:(img + 1) * p])
        assert np.array_equal(nan[sl].cpu().numpy(), enan[img * p:(img + 1) * p])
    assert nan[-p:].any()
    del q, row_sum, nan, xt
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- the conv
def _run(args, bias=None, stride=1, padding=0, dilation=1):
    x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax = args
    w_q, w_sum, w_scale, w_zero = stored_rows(w, ws, wz, wqmin, wqmax)
    y = ops.int8_conv2d(t(x), t(np.array([xs], F32)), t(np.array([xz], F32)), xqmin, xqmax, w_q, w_sum, w_scale, w_zero,
                        w.shape[2:], None if bias is None else t(bias), stride, padding, dilation)
    return y.cpu().numpy()


CONVS = [
    # (n, c, h, w, c_out, kernel, stride, padding, dilation)
    (2, 3, 30, 30, 64, 7, 2, 3, 1),
    (2, 64, 14, 14, 64, 3, 1, 1, 1),
    (3, 64, 15, 15, 128, 3, 2, 1, 1),
    (2, 256, 7, 7, 200, 1, 1, 0, 1),
    (2, 96, 9, 9, 130, 1, 2, 0, 1),
    (1, 32, 12, 11, 40, 3, 1, (0, 2, 1, 0), 2),
    (1, 1024, 5, 5, 36, 3, 1, 1, 1),
]


@pytest.mark.parametrize("conv", CONVS)
@pytest.mark.parametrize("xr,wr", [((-128, 127), (-128, 127)), ((0, 255), (-128, 127)), (qrange(4, True), qrange(4, False)),
                                   (qrange(2, False), qrange(2, True))])
def test_exact_mode(conv, xr, wr):
    n, c, h, w, c_out, kernel, stride, padding, dilation = conv
    kh, kw = (kernel, kernel) if isinstance(kernel, int) else kernel
    rng = np.random.default_rng(abs(hash((conv, xr, wr))) % 2**32)
    (xqmin, xqmax), (wqmin, wqmax) = xr, wr
    xs, ws = F32(2.0 ** -4), (2.0 ** -rng.integers(3, 8, c_out)).astype(F32)
    zx = F32(0 if xqmin < 0 else xqmin + (xqmax - xqmin) * 2 // 3)
    zw = (np.zeros(c_out) if wqmin < 0 else rng.integers(wqmin, wqmax + 1, c_out)).astype(F32)
    span = (xqmax - xqmin) * float(xs)
    x = rng.uniform(-0.7 * span, 0.7 * span, (n, c, h, w)).astype(F32)
    wt = (rng.uniform(-0.7, 0.7, (c_out, c, kh, kw)) * (wqmax - wqmin) * ws[:, None, None, None]).astype(F32)
    args = (x, xs, zx, xqmin, xqmax, wt, ws, zw, wqmin, wqmax)
    y = _run(args, np.zeros(c_out, F32), stride, padding, dilation)
    t_, _ = truth(*args, stride=stride, padding=padding, dilation=dilation)
    assert y.shape == t_.shape
    i = t_ / (float(xs) * ws.astype(np.float64)[None, :, None, None])
    exact = i.astype(F32).astype(np.float64) == i
    assert exact.mean() > 0.5
    assert np.array_equal(y.astype(np.float64)[exact], t_[exact])


def _minmax_case(rng, n, c, h, w, c_out, kh, kw, affine_x, per_channel_w):
    x = (rng.standard_normal((n, c, h, w)) * 2 + (0.8 if affine_x else 0)).astype(F32)
    wt = (rng.standard_normal((c_out, c, kh, kw)) / np.sqrt(c * kh * kw)).astype(F32)
    xqmin, xqmax = (0, 255) if affine_x else (-128, 127)
    xs, xz = oobs.calc_qparams_with_minmax(*oobs.minmax([x]), xqmin, xqmax, not affine_x)
    ws, wz = oobs.calc_qparams_with_minmax(*oobs.minmax([wt.reshape(c_out, -1)], per_channel=per_channel_w), -128, 127, True)
    bias = rng.standard_normal(c_out).astype(F32)
    return (x, F32(np.asarray(xs).reshape(-1)[0]), F32(np.asarray(xz).reshape(-1)[0]), xqmin, xqmax, wt, ws, wz, -128, 127), bias


@pytest.mark.parametrize("conv", CONVS)
@pytest.mark.parametrize("affine_x,per_channel_w,with_bias", [(False, True, True), (True, True, False), (True, False, True)])
def test_general_data_meets_the_bound(conv, affine_x, per_channel_w, with_bias):
    n, c, h, w, c_out, kernel, stride, padding, dilation = conv
    kh, kw = (kernel, kernel) if isinstance(kernel, int) else kernel
    rng = np.random.default_rng(abs(hash((conv, affine_x, per_channel_w, with_bias))) % 2**32)
    args, bias = _minmax_case(rng, n, c, h, w, c_out, kh, kw, affine_x, per_channel_w)
    bias = bias if with_bias else None
    y = _run(args, bias, stride, padding, dilation)
    t_, bound = truth(*args, bias=bias, stride=stride, padding=padding, dilation=dilation)
    err = np.abs(y - t_)
    assert np.all(err <= bound), float((err / bound).max())


def _qconv_from(args, bias, stride, padding):
    """A QConv2d whose quantizers hold the given qparams (per-tensor activations, per-channel weights)."""
    x, xs, xz, xqmin, xqmax, wt, ws, wz, wqmin, wqmax = args
    c_out, c, kh, kw = wt.shape
    conv = nn.Conv2d(c, c_out, (kh, kw), stride=stride, padding=padding, bias=bias is not None)
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(wt))
        if bias is not None:
            conv.bias.copy_(torch.from_numpy(bias))
    q = QConv2d(conv).build_quantizer(cfg("per-tensor-affine" if xqmin >= 0 else "per-tensor-symmetric", "feature"),
                                      cfg("per-channel-symmetric", "weight")).to(dev())
    q.input_quantizer.scale = t(np.array([xs], F32))
    q.input_quantizer.zero_point = t(np.array([xz], F32))
    q.weight_quantizer.scale = t(np.asarray(ws, F32).reshape(-1, 1, 1, 1))
    q.weight_quantizer.zero_point = t(np.asarray(wz, F32).reshape(-1, 1, 1, 1))
    q.set_quant(w_quant=True, a_quant=True)
    return q


def test_nan_positions_match_the_fake_quant_conv():
    rng = np.random.default_rng(21)
    args, bias = _minmax_case(rng, 2, 16, 13, 13, 24, 3, 3, True, True)
    x = args[0].copy()
    x[0, 3, 4, 5] = np.nan
    x[1, 15, 12, 0] = np.nan
    x[1, 2, 0, 9] = np.inf
    args = (x,) + args[1:]
    y = _run(args, bias, 2, 1)
    qconv = _qconv_from(args, bias, 2, 1)
    with torch.no_grad():
        ref = qconv(t(x)).cpu().numpy()
    t_, bound = truth(*args, bias=bias, stride=2, padding=1)
    assert np.isnan(y).any()
    assert np.array_equal(np.isnan(y), np.isnan(ref)) and np.array_equal(np.isnan(y), np.isnan(t_))
    ok = ~np.isnan(t_)
    assert np.all(np.abs(y[ok] - t_[ok]) <= bound[ok])
    conv = QConv2dInt8.from_qconv2d(qconv)
    with torch.no_grad():
        assert np.array_equal(conv(t(x)).cpu().numpy(), y, equal_nan=True)


def test_weight_nan_row_gives_a_nan_channel():
    rng = np.random.default_rng(22)
    args, bias = _minmax_case(rng, 2, 8, 9, 9, 12, 3, 3, False, True)
    qconv = _qconv_from(args, bias, 1, 1)
    with torch.no_grad():
        qconv.weight[5, 2, 1, 1] = float("nan")
    conv = QConv2dInt8.from_qconv2d(qconv)
    with torch.no_grad():
        y = conv(t(args[0])).cpu().numpy()
    assert np.isnan(y[:, 5]).all() and np.isfinite(np.delete(y, 5, axis=1)).all()


def test_deterministic_and_graph_replay():
    rng = np.random.default_rng(23)
    args, bias = _minmax_case(rng, 4, 64, 28, 28, 96, 3, 3, True, True)
    x, xs, xz, xqmin, xqmax, wt, ws, wz, wqmin, wqmax = args
    w_q, w_sum, w_scale, w_zero = stored_rows(wt, ws, wz, wqmin, wqmax)
    xt, xst, xzt, bt = t(x), t(np.array([xs], F32)), t(np.array([xz], F32)), t(bias)

    def call():
        return ops.int8_conv2d(xt, xst, xzt, xqmin, xqmax, w_q, w_sum, w_scale, w_zero, 3, bt, 1, 1)

    y1, y2 = call(), call()
    assert torch.equal(y1, y2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()  # warm the per-stream workspace outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            yg = call()
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        xt.copy_(t(x))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, y1)


def test_k_limit_is_unsupported():
    c = 1 << 17  # K = c for a 1x1 kernel
    x = torch.zeros(1, c, 1, 2, device=dev())
    one = torch.ones(1, device=dev())
    w_q = torch.zeros(8, c, dtype=torch.int8, device=dev())
    i32 = torch.zeros(8, dtype=torch.int32, device=dev())
    with pytest.raises(SparsebitB200Error, match=r"K < 2\^17.*status -3"):
        ops.int8_conv2d(x, one, one * 0, -128, 127, w_q, i32, torch.ones(8, device=dev()), i32, 1)
    with pytest.raises(SparsebitB200Error, match=r"K < 2\^17.*status -3"):
        ops.int8_im2col_quantize(x, 1, one, one * 0, -128, 127)


# ---------------------------------------------------------------------------------------------- modules
class CnnHead(nn.Module):
    """A stem conv (symmetric), an affine-activation padded 3x3 conv, a strided 1x1 conv, a grouped conv (not
    eligible) and a classifier."""

    def __init__(self):
        super().__init__()
        self.conv1 = QConv2d(nn.Conv2d(3, 16, 3, stride=2)).build_quantizer(cfg("per-tensor-symmetric", "feature"),
                                                                            cfg("per-channel-symmetric", "weight"))
        self.relu = QReLU().build_quantizer(cfg("per-tensor-symmetric", "feature", disable=True))
        self.conv2 = QConv2d(nn.Conv2d(16, 32, 3, padding=1)).build_quantizer(cfg("per-tensor-affine", "feature"),
                                                                              cfg("per-channel-symmetric", "weight"))
        self.conv3 = QConv2d(nn.Conv2d(32, 24, 1, stride=2, bias=False)).build_quantizer(
            cfg("per-tensor-affine", "feature"), cfg("per-tensor-symmetric", "weight"))
        self.dw = QConv2d(nn.Conv2d(24, 24, 3, padding=1, groups=24)).build_quantizer(cfg("per-tensor-affine", "feature"),
                                                                                      cfg("per-channel-symmetric", "weight"))
        self.fc = QLinear(nn.Linear(24, 10)).build_quantizer(cfg("per-tensor-symmetric", "feature"),
                                                             cfg("per-tensor-symmetric", "weight"))

    def forward(self, x):
        x = self.relu(self.conv2(self.conv1(x)))  # conv2 sees signed input: affine activations with Z != 0, padded
        x = torch.relu(self.conv3(x))
        return self.fc(self.dw(x).mean(dim=(2, 3)))


def _truth_of(qconv, x):
    return truth(**layer_qparams(qconv, x))


def test_cnn_head_converts_and_meets_the_bound():
    torch.manual_seed(0)
    batches = [torch.randn(8, 3, 33, 33, device=dev()) for _ in range(3)]
    model = calibrated(CnnHead(), batches, streaming=True, record_inputs=False)
    names = ["conv1", "conv2", "conv3"]
    originals = {nm: getattr(model, nm) for nm in names}
    assert to_integer_convs(model) == names
    assert isinstance(model.dw, QConv2d) and isinstance(model.fc, QLinear)  # grouped conv and the linear stay
    assert model.conv2.qmin == 0 and float(model.conv2.zero_point) != 0  # affine activations, padded
    check_converted(model, originals, batches[:2], names, expected_cls=QConv2dInt8, layer_truth=_truth_of,
                    compare_fake_quant=True)


def test_module_input_forms():
    torch.manual_seed(2)
    batches = [torch.randn(4, 3, 33, 33, device=dev())]
    model = calibrated(CnnHead(), batches, streaming=True, record_inputs=False)
    to_integer_convs(model)
    conv = model.conv2
    x = torch.randn(3, 16, 16, 16, device=dev())
    with torch.no_grad():
        y = conv(x)
        assert y.shape == (3, 32, 16, 16) and y.dtype == torch.float32
        assert torch.equal(conv(x[1]), y[1])  # unbatched [C, H, W]
        x16 = x.half()
        assert torch.equal(conv(x16), conv(x16.float()))
        xcl = x.to(memory_format=torch.channels_last)
        assert torch.equal(conv(xcl), y)
    xg = x.clone().requires_grad_()
    with pytest.raises(RuntimeError, match="no backward"):
        conv(xg)
    with torch.no_grad():
        conv(xg)


def test_resnet18_converts_every_conv_and_meets_the_bound():
    import torchvision

    torch.manual_seed(0)
    qnet = wrap_quantized(torchvision.models.resnet18(weights=None).eval(), cfg("per-tensor-affine", "feature"),
                          cfg("per-channel-symmetric", "weight"))
    torch.manual_seed(1)
    batches = [torch.randn(4, 3, 112, 112, device=dev()) for _ in range(2)]
    qnet = calibrated(qnet, batches, streaming=True, record_inputs=False)
    originals = {nm: m for nm, m in qnet.named_modules() if isinstance(m, QConv2d)}
    names = to_integer_convs(qnet)
    assert len(names) == 20 and names == list(originals)
    assert isinstance(qnet.fc, QLinear)
    check_converted(qnet, originals, [batches[0][:2]], names, expected_cls=QConv2dInt8, layer_truth=_truth_of,
                    compare_fake_quant=False)
