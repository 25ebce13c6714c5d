"""The grouped / depthwise conv on the integer grid (sb200_int8_group_conv2d / QConv2dGroupInt8) against the fp64 truth
of the fake-quant conv (tests/int8_group_conv_ref.py) and, group by group, against the dense integer conv
(ops.int8_conv2d) on the group's channel slice."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from gpu_util import dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from int8_group_conv_ref import truth
from int8_harness import calibrated, cfg, check_converted, layer_qparams, stored_rows, wrap_quantized
from oracle import observers as oobs
from sparsebit_b200 import SparsebitB200Error, ops
from sparsebit_b200.quantization.modules import QConv2d, QConv2dGroupInt8, QConv2dInt8
from sparsebit_b200.quantization.tools import to_integer_convs, to_integer_group_convs

pytestmark = pytest.mark.gpu

F32 = np.float32

# (n, c, h, w, c_out, groups, kernel, stride, padding, dilation)
GEOMS = [
    (2, 16, 14, 14, 16, 16, 3, 1, 1, 1),            # depthwise 3x3
    (2, 24, 15, 13, 24, 24, 5, 2, 2, 1),            # depthwise 5x5, stride 2, odd W
    (1, 8, 16, 16, 8, 8, 7, 1, 3, 1),               # depthwise 7x7
    (2, 12, 17, 17, 12, 12, 3, 1, 2, 2),            # dilation 2
    (2, 10, 9, 12, 10, 10, 4, 1, (1, 2, 1, 2), 1),  # 'same' with an even kernel: asymmetric padding
    (2, 8, 11, 11, 16, 8, 3, 1, 1, 1),              # channel multiplier 2
    (2, 8, 10, 10, 8, 4, 3, 1, 1, 1),               # C_g = 2
    (2, 9, 10, 9, 6, 3, 3, 2, 1, 1),                # C_g = 3, M_g = 2
    (2, 16, 12, 12, 16, 4, 3, 1, 1, 1),             # C_g = 4
    (2, 32, 9, 9, 32, 4, 3, 2, 1, 1),               # C_g = 8
    (2, 64, 8, 8, 64, 4, 3, 1, 1, 1),               # C_g = 16
    (1, 48, 7, 7, 72, 2, 3, 1, 1, 1),               # C_g = 24, M_g = 36
    (2, 64, 7, 7, 64, 2, 3, 1, 1, 1),               # C_g = 32
    (3, 6, 1, 19, 6, 6, 3, 1, 1, 1),                # H = 1
    (2, 8, 13, 1, 16, 4, 3, 1, 1, 1),               # W = 1
    (2, 8, 3, 3, 8, 8, 3, 1, 0, 1),                 # a 1x1 output
]
RANGES = [((-128, 127), (-128, 127)), ((0, 255), (-128, 127)), ((0, 15), (-8, 7))]


def _run(args, groups, bias=None, stride=1, padding=0, dilation=1):
    x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax = args
    wts = stored_rows(w, ws, wz, wqmin, wqmax)
    return ops.int8_group_conv2d(t(x), t(np.array([xs], F32)), t(np.array([xz], F32)), xqmin, xqmax, *wts, w.shape[2:],
                                 groups, None if bias is None else t(bias), stride, padding, dilation).cpu().numpy()


def _per_group_dense(args, groups, bias=None, stride=1, padding=0, dilation=1):
    """ops.int8_conv2d on each group's channel slice and weight rows, concatenated along the channels."""
    x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax = args
    c_g, m_g = x.shape[1] // groups, w.shape[0] // groups
    ws = np.broadcast_to(np.asarray(ws, F32).reshape(-1), (w.shape[0],))
    wz = np.broadcast_to(np.asarray(wz, F32).reshape(-1), (w.shape[0],))
    outs = []
    for g in range(groups):
        o = slice(g * m_g, (g + 1) * m_g)
        wts = stored_rows(np.ascontiguousarray(w[o]), ws[o], wz[o], wqmin, wqmax)
        outs.append(ops.int8_conv2d(t(np.ascontiguousarray(x[:, g * c_g:(g + 1) * c_g])), t(np.array([xs], F32)),
                                    t(np.array([xz], F32)), xqmin, xqmax, *wts, w.shape[2:],
                                    None if bias is None else t(np.ascontiguousarray(bias[o])), stride, padding,
                                    dilation).cpu().numpy())
    return np.concatenate(outs, axis=1)


def _exact_case(rng, geom, xr, wr):
    n, c, h, w, c_out, groups, kernel = geom[:7]
    kh, kw = (kernel, kernel) if isinstance(kernel, int) else kernel
    (xqmin, xqmax), (wqmin, wqmax) = xr, wr
    xs, ws = F32(2.0 ** -4), (2.0 ** -rng.integers(3, 8, c_out)).astype(F32)
    zx = F32(0 if xqmin < 0 else xqmin + (xqmax - xqmin) * 2 // 3)
    zw = (np.zeros(c_out) if wqmin < 0 else rng.integers(wqmin, wqmax + 1, c_out)).astype(F32)
    span = (xqmax - xqmin) * float(xs)
    x = rng.uniform(-0.7 * span, 0.7 * span, (n, c, h, w)).astype(F32)
    wt = (rng.uniform(-0.7, 0.7, (c_out, c // groups, kh, kw)) * (wqmax - wqmin) * ws[:, None, None, None]).astype(F32)
    return (x, xs, zx, xqmin, xqmax, wt, ws, zw, wqmin, wqmax)


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("xr,wr", RANGES)
def test_exact_mode_and_per_group_identity(geom, xr, wr):
    stride, padding, dilation = geom[7:]
    groups = geom[5]
    rng = np.random.default_rng(abs(hash((geom, xr, wr))) % 2**32)
    args = _exact_case(rng, geom, xr, wr)
    bias = np.zeros(geom[4], F32)
    y = _run(args, groups, bias, stride, padding, dilation)
    t_, _ = truth(*args, groups, bias=bias, stride=stride, padding=padding, dilation=dilation)
    assert y.shape == t_.shape
    i = t_ / (float(args[1]) * args[6].astype(np.float64)[None, :, None, None])
    exact = i.astype(F32).astype(np.float64) == i
    assert exact.mean() > 0.5
    assert np.array_equal(y.astype(np.float64)[exact], t_[exact])
    dense = _per_group_dense(args, groups, bias, stride, padding, dilation)
    assert np.array_equal(y, dense)


def _minmax_case(rng, n, c, h, w, c_out, groups, kh, kw, affine_x, per_channel_w):
    x = (rng.standard_normal((n, c, h, w)) * 2 + (0.8 if affine_x else 0)).astype(F32)
    wt = (rng.standard_normal((c_out, c // groups, kh, kw)) / np.sqrt(c // groups * kh * kw)).astype(F32)
    xqmin, xqmax = (0, 255) if affine_x else (-128, 127)
    xs, xz = oobs.calc_qparams_with_minmax(*oobs.minmax([x]), xqmin, xqmax, not affine_x)
    ws, wz = oobs.calc_qparams_with_minmax(*oobs.minmax([wt.reshape(c_out, -1)], per_channel=per_channel_w), -128, 127, True)
    bias = rng.standard_normal(c_out).astype(F32)
    return (x, F32(np.asarray(xs).reshape(-1)[0]), F32(np.asarray(xz).reshape(-1)[0]), xqmin, xqmax, wt, ws, wz, -128, 127), bias


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("affine_x,per_channel_w,with_bias", [(False, True, True), (True, True, False), (True, False, True)])
def test_minmax_data_meets_the_bound(geom, affine_x, per_channel_w, with_bias):
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation = geom
    kh, kw = (kernel, kernel) if isinstance(kernel, int) else kernel
    rng = np.random.default_rng(abs(hash((geom, affine_x, per_channel_w, with_bias))) % 2**32)
    args, bias = _minmax_case(rng, n, c, h, w, c_out, groups, kh, kw, affine_x, per_channel_w)
    bias = bias if with_bias else None
    y = _run(args, groups, bias, stride, padding, dilation)
    t_, bound = truth(*args, groups, bias=bias, stride=stride, padding=padding, dilation=dilation)
    err = np.abs(y - t_)
    assert np.all(err <= bound), float((err / bound).max())
    assert np.array_equal(y, _per_group_dense(args, groups, bias, stride, padding, dilation), equal_nan=True)


@pytest.mark.parametrize("geom", [GEOMS[0], GEOMS[5], GEOMS[10], GEOMS[11]])
def test_nan_and_inf_stay_in_their_group(geom):
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation = geom
    rng = np.random.default_rng(7)
    args, bias = _minmax_case(rng, n, c, h, w, c_out, groups, kernel, kernel, True, True)
    x = args[0].copy()
    c_g = c // groups
    g = groups // 2
    x[0, g * c_g, h // 2, w // 2] = np.nan
    x[n - 1, g * c_g + c_g - 1, 0, w - 1] = np.inf
    x[0, g * c_g, h - 1, 0] = -np.inf
    args = (x,) + args[1:]
    y = _run(args, groups, bias, stride, padding, dilation)
    dense = _per_group_dense(args, groups, bias, stride, padding, dilation)
    assert np.array_equal(y, dense, equal_nan=True)
    t_, bound = truth(*args, groups, bias=bias, stride=stride, padding=padding, dilation=dilation)
    assert np.array_equal(np.isnan(y), np.isnan(t_))
    m_g = c_out // groups
    other = np.ones(c_out, bool)
    other[g * m_g:(g + 1) * m_g] = False
    assert not np.isnan(y[:, other]).any() and np.isnan(y[:, ~other]).any()
    ok = ~np.isnan(t_)
    assert np.all(np.abs(y[ok] - t_[ok]) <= bound[ok])


def test_weight_nan_row_gives_a_nan_channel():
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation = GEOMS[5]
    rng = np.random.default_rng(3)
    args, bias = _minmax_case(rng, n, c, h, w, c_out, groups, kernel, kernel, False, True)
    wt = args[5].copy()
    wt[5, 0, 1, 1] = np.nan
    args = args[:5] + (wt,) + args[6:]
    y = _run(args, groups, bias, stride, padding, dilation)
    assert np.isnan(y[:, 5]).all()
    assert not np.isnan(np.delete(y, 5, axis=1)).any()


def test_deterministic_and_graph_replay():
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation = GEOMS[11]
    rng = np.random.default_rng(5)
    args, bias = _minmax_case(rng, 4, c, 14, 14, c_out, groups, kernel, kernel, True, True)
    x, xs, xz, xqmin, xqmax, wt, ws, wz, wqmin, wqmax = args
    wts = stored_rows(wt, ws, wz, wqmin, wqmax)
    xt, s, z, b = t(x), t(np.array([xs], F32)), t(np.array([xz], F32)), t(bias)

    def call():
        return ops.int8_group_conv2d(xt, s, z, xqmin, xqmax, *wts, kernel, groups, b, stride, padding, dilation)

    ys = [call() for _ in range(3)]
    assert all(torch.equal(ys[0], y) for y in ys[1:])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = call()
    yg.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, ys[0])


def test_far_end_past_2_31_elements():
    """x and out of 129 x 4096 x 4096 floats (> 2^31 elements each): the far end of the last channel."""
    n, c, h, w = 1, 129, 4096, 4096
    g = torch.Generator(device=dev()).manual_seed(11)
    x = torch.randn(n, c, h, w, device=dev(), generator=g)
    assert x.numel() > 2**31
    rng = np.random.default_rng(11)
    wt = rng.standard_normal((c, 1, 3, 3)).astype(F32)
    xs, ws = F32(2.0 ** -5), np.full(c, 2.0 ** -7, F32)
    wts = stored_rows(wt, ws, np.zeros(c, F32), -128, 127)
    y = ops.int8_group_conv2d(x, t(np.array([xs], F32)), t(np.zeros(1, F32)), -128, 127, *wts, 3, c, None, 1, 1, 1)
    assert y.numel() > 2**31
    tail = y[0, c - 1, h - 9:, w - 200:].cpu().numpy()[None, None]
    xin = x[:, c - 1:, h - 10:, w - 201:].cpu().numpy()
    del x, y
    torch.cuda.empty_cache()
    t_, bound = truth(xin, xs, 0, -128, 127, wt[c - 1:], ws[c - 1:], np.zeros(1, F32), -128, 127, 1,
                      padding=(0, 1, 0, 1))
    assert np.array_equal(tail.astype(np.float64), t_)  # power-of-two scales: exact


def test_argument_errors():
    x = torch.randn(2, 8, 6, 6, device=dev())
    s, z = t(np.array([0.1], F32)), t(np.zeros(1, F32))
    w_q = torch.zeros(8, 16, dtype=torch.int8, device=dev())
    w_sum, w_zero = (torch.zeros(8, dtype=torch.int32, device=dev()) for _ in range(2))
    w_scale = torch.ones(8, device=dev())
    with pytest.raises(SparsebitB200Error, match="does not divide"):
        ops.int8_group_conv2d(x, s, z, -128, 127, w_q, w_sum, w_scale, w_zero, 3, 3)
    with pytest.raises(SparsebitB200Error, match="the geometry needs"):
        ops.int8_group_conv2d(x, s, z, -128, 127, w_q, w_sum, w_scale, w_zero, 3, 4)
    with pytest.raises(SparsebitB200Error, match="sb200_int8_conv2d"):
        ops.int8_group_conv2d(x, s, z, -128, 127, torch.zeros(8, 80, dtype=torch.int8, device=dev()), w_sum, w_scale,
                              w_zero, 3, 1)
    with pytest.raises(SparsebitB200Error, match="need 8 elements"):
        ops.int8_group_conv2d(x, s, z, -128, 127, w_q, w_sum[:4], w_scale, w_zero, 3, 8)
    with pytest.raises(SparsebitB200Error, match=r"\[N, C, H, W\]"):
        ops.int8_group_conv2d(x[0], s, z, -128, 127, w_q, w_sum, w_scale, w_zero, 3, 8)


# ---------------------------------------------------------------------------------------------- modules and models
def _truth_of(qconv, x):
    return truth(**layer_qparams(qconv, x), groups=qconv.fwd_kwargs["groups"])


def test_mobilenet_v2_converts_all_52_convs_and_meets_the_bound():
    import torchvision

    torch.manual_seed(0)
    qnet = wrap_quantized(torchvision.models.mobilenet_v2(weights=None).eval(), cfg("per-tensor-affine", "feature"),
                          cfg("per-channel-symmetric", "weight"))
    batches = [torch.randn(2, 3, 96, 96, device=dev()) for _ in range(2)]
    qnet = calibrated(qnet, batches, streaming=True, record_inputs=False)
    originals = {nm: m for nm, m in qnet.named_modules() if isinstance(m, QConv2d)}
    dense = to_integer_convs(qnet)
    grouped = to_integer_group_convs(qnet)
    assert len(dense) == 35 and len(grouped) == 17 and sorted(dense + grouped) == sorted(originals)
    assert all(isinstance(qnet.get_submodule(nm), QConv2dGroupInt8) for nm in grouped)
    assert all(type(qnet.get_submodule(nm)) is QConv2dInt8 for nm in dense)
    check_converted(qnet, originals, [batches[0][:1]], dense + grouped, expected_cls=None, layer_truth=_truth_of,
                    compare_fake_quant=False)


def test_regnet_x_400mf_converts_every_grouped_conv_and_meets_the_bound():
    import torchvision

    torch.manual_seed(1)
    qnet = wrap_quantized(torchvision.models.regnet_x_400mf(weights=None).eval(), cfg("per-tensor-affine", "feature"),
                          cfg("per-channel-symmetric", "weight"))
    batches = [torch.randn(2, 3, 96, 96, device=dev()) for _ in range(2)]
    qnet = calibrated(qnet, batches, streaming=True, record_inputs=False)
    originals = {nm: m for nm, m in qnet.named_modules() if isinstance(m, QConv2d) and m.fwd_kwargs["groups"] > 1}
    grouped = to_integer_group_convs(qnet)
    assert len(grouped) == 22 and grouped == list(originals)
    check_converted(qnet, originals, [batches[0][:1]], grouped, expected_cls=QConv2dGroupInt8, layer_truth=_truth_of,
                    compare_fake_quant=False)


def test_module_input_forms():
    torch.manual_seed(2)
    q = QConv2d(nn.Conv2d(16, 32, 3, padding=1, groups=8)).build_quantizer(cfg("per-tensor-affine", "feature"),
                                                                            cfg("per-channel-symmetric", "weight"))
    q = calibrated(q, [torch.randn(4, 16, 12, 12, device=dev())], streaming=True, record_inputs=False)
    conv = QConv2dGroupInt8.from_qconv2d(q)
    assert "groups=8" in repr(conv)
    x = torch.randn(3, 16, 12, 12, device=dev())
    with torch.no_grad():
        y = conv(x)
        assert y.shape == (3, 32, 12, 12) and y.dtype == torch.float32
        assert torch.equal(conv(x[1]), y[1])
        x16 = x.half()
        assert torch.equal(conv(x16), conv(x16.float()))
        assert torch.equal(conv(x.to(memory_format=torch.channels_last)), y)
    xg = x.clone().requires_grad_()
    with pytest.raises(RuntimeError, match="no backward"):
        conv(xg)
    with torch.no_grad():
        conv(xg)
