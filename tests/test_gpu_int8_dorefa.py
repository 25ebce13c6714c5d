"""Integer-grid layers with DoReFa and AdaRound quantizers on the GPU.

Bit identity: every op given ``x_absmax`` equals, bit for bit (NaN positions included), the plain op run on
``ops.dorefa_forward(x, m)`` with the same qparams, over every launch-branch case of the plain suites (the int8
linear / conv cases of test_gpu_int8_branches.py, the grouped cases of test_gpu_int8_group_branches.py, and the NHWC
lowering and grouped cases of test_gpu_int8_conv_nhwc_branches.py).  Then: NaN / all-zero / +-inf inputs against the
fake-quant DoReFa QConv2d, the weight grids of DoReFa and AdaRound weights, converted layers against the fake-quant
layer, the converter on calibrated ResNet-18 and MobileNetV2, determinism and CUDA graph replay."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import test_gpu_int8_branches as lin_suite
import test_gpu_int8_conv_nhwc_branches as nhwc_suite
import test_gpu_int8_group_branches as grp_suite
from gpu_util import bits_equal, dev, seed
from int8_harness import calibrated, cfg, wrap_quantized
from sparsebit_b200 import SparsebitB200Error, ops
from sparsebit_b200.quantization.modules import (QConv2d, QConv2dDoReFaInt8, QConv2dGroupDoReFaInt8, QConv2dGroupInt8,
                                                 QConv2dInt8, QLinear, QLinearDoReFaInt8, QLinearInt8,
                                                 dorefa_adaround_ineligibility, from_dorefa_adaround)
from sparsebit_b200.quantization.tools import (to_integer_convs, to_integer_dorefa_adaround, to_integer_group_convs,
                                               to_integer_linears)

pytestmark = pytest.mark.gpu

RANGES = {"s8": (-128, 127), "u8": (0, 255), "s4": (-8, 7), "u4": (0, 15), "s2": (-2, 1), "u2": (0, 3)}
LIN_CASES = [c for c in lin_suite.CASES if c.op in ("linear", "conv")]
# the grouped suite's cases, plus one whose CTA tiles pass the 65536-CTA grid (grid.loop; the plain suite reaches it
# with a 2^31-element input, this one with 2^28)
GROUP_CASES = dict(grp_suite.CASES, grid_loop=(1, 16384, 129, 128, 16384, 16384, 3, 1, 1, 1, 0, False, False))


def _qparams(xr, zp):
    qmin, qmax = RANGES[xr]
    z = {"min": qmin, "max": qmax, "mid": (qmin + qmax) // 2}[zp]
    return (torch.tensor([2.0 / (qmax - qmin)], device=dev()), torch.tensor([float(z)], device=dev()), qmin, qmax)


def _x(shape, name, x_off=0, nan=False):
    g = torch.Generator(device=dev()).manual_seed(seed(name))
    n = int(np.prod(shape))
    raw = torch.zeros(x_off // 4 + n + 4, device=dev())
    v = raw[x_off // 4:x_off // 4 + n]
    v.copy_((torch.rand(n, generator=g, device=dev()) - 0.5) * 5)
    if nan:
        v[n // 3] = float("nan")
    return v.view(shape)


def _weights(c_out, k, name):
    g = torch.Generator(device=dev()).manual_seed(seed(name) + 7)
    ws = (2.0 ** -torch.randint(3, 8, (c_out,), generator=g, device=dev()).float()).contiguous()
    wt = ((torch.rand(c_out, k, generator=g, device=dev()) - 0.5) * 255 * ws[:, None]).contiguous()
    w_q, w_sum, _ = ops.int8_quantize_rows(wt, ws, torch.zeros_like(ws), -128, 127)
    bias = torch.randn(c_out, generator=g, device=dev())
    return w_q, w_sum, ws, torch.zeros(c_out, dtype=torch.int32, device=dev()), bias


def _same(op, x, args, kwargs, nhwc=False):
    """op with x_absmax on x against op on dorefa_forward(x, m), bit for bit."""
    m = ops.dorefa_absmax(x.permute(0, 2, 3, 1) if nhwc else x)
    xn = ops.dorefa_forward(x.permute(0, 2, 3, 1) if nhwc else x, m)
    xn = xn.permute(0, 3, 1, 2) if nhwc else xn
    y1 = op(x, *args, **kwargs, x_absmax=m)
    y0 = op(xn, *args, **kwargs)
    torch.cuda.synchronize()
    assert bits_equal(y1.cpu().numpy(), y0.cpu().numpy())
    return y1



@pytest.mark.parametrize("case", LIN_CASES, ids=[c.name for c in LIN_CASES])
def test_linear_and_conv_branch_cases(case):
    s, z, qmin, qmax = _qparams(case.get("xr"), case.get("zp"))
    bias_on = case.get("bias", True)
    if case.op == "linear":
        m, k, n = case.get("m"), case.get("k"), case.get("n")
        x = _x((m, k), case.name, case.get("x_off", 0), nan=True)
        w_q, w_sum, ws, wz, bias = _weights(n, k, case.name)
        _same(ops.int8_linear, x, (s, z, qmin, qmax, w_q, w_sum, ws, wz, bias if bias_on else None), {})
        return
    n, c, h, w = case.get("n"), case.get("c"), case.get("h"), case.get("w")
    kh, kw = case.get("kh"), case.get("kw")
    x = _x((n, c, h, w), case.name, nan=True)
    w_q, w_sum, ws, wz, bias = _weights(case.get("c_out"), c * kh * kw, case.name)
    kwargs = dict(stride=case.get("stride", 1), padding=case.get("pad", 0), dilation=case.get("dilation", 1))
    args = (s, z, qmin, qmax, w_q, w_sum, ws, wz, (kh, kw), bias if bias_on else None)
    y = _same(ops.int8_conv2d, x, args, kwargs)
    # the channels-last entry point computes the same values
    xl = x.contiguous(memory_format=torch.channels_last)
    yl = _same(ops.int8_conv2d_nhwc, xl, args, kwargs, nhwc=True)
    assert bits_equal(yl.contiguous().cpu().numpy(), y.cpu().numpy())


@pytest.mark.parametrize("name", sorted(GROUP_CASES))
def test_group_branch_cases(name):
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x_off, with_bias, with_nan = GROUP_CASES[name]
    s, z, qmin, qmax = _qparams("s8", "mid")
    x = _x((n, c, h, w), name, x_off, with_nan)
    w_q, w_sum, ws, wz, bias = _weights(c_out, c // groups * kernel * kernel, name)
    args = (s, z, qmin, qmax, w_q, w_sum, ws, wz, kernel, groups, bias if with_bias else None)
    kwargs = dict(stride=stride, padding=padding, dilation=dilation)
    y = _same(ops.int8_group_conv2d, x, args, kwargs)
    yl = _same(ops.int8_group_conv2d_nhwc, x.contiguous(memory_format=torch.channels_last), args, kwargs, nhwc=True)
    assert bits_equal(yl.contiguous().cpu().numpy(), y.cpu().numpy())


@pytest.mark.parametrize("case", nhwc_suite.CASES, ids=[c.name for c in nhwc_suite.CASES])
def test_nhwc_branch_cases(case):
    n, c, h, w = case.get("shape")
    x = nhwc_suite._x_channels_last(case)
    s, z, qmin, qmax = _qparams("u8", "mid")
    kernel, stride, padding = case.get("kernel"), case.get("stride", 1), case.get("padding", 0)
    kwargs = dict(stride=stride, padding=padding)
    if case.op == "lower":
        w_q, w_sum, ws, wz, bias = _weights(24, c * kernel * kernel, case.name)
        _same(ops.int8_conv2d_nhwc, x, (s, z, qmin, qmax, w_q, w_sum, ws, wz, kernel, bias), kwargs, nhwc=True)
        return
    c_out, groups = case.get("c_out"), case.get("groups")
    w_q, w_sum, ws, wz, bias = _weights(c_out, c // groups * kernel * kernel, case.name)
    args = (s, z, qmin, qmax, w_q, w_sum, ws, wz, kernel, groups, bias if case.get("bias", True) else None)
    _same(ops.int8_group_conv2d_nhwc, x, args, kwargs, nhwc=True)


def test_normalisation_is_the_true_division():
    """ops.dorefa_forward(x, m) (dorefa_norm, which every DoReFa kernel shares) equals tanh(x) / m under ATen's true
    division, bit for bit, for m at powers of two, random mantissas, subnormals, the largest floats, +-0, +-inf, NaN and
    negative values; tanh(x) is the kernel's own (m = 1, where the quotient is exact)."""
    g = torch.Generator(device=dev()).manual_seed(seed("norm"))
    x = torch.cat([(torch.rand(1 << 16, generator=g, device=dev()) - 0.5) * 20,
                   torch.randn(1 << 16, generator=g, device=dev()) * 1e-3,
                   torch.tensor([0.0, -0.0, 1e-40, -1e-45, 30.0, -30.0, float("inf"), float("-inf"), float("nan")],
                                device=dev())])
    ms = [1.0, 0.5, 2.0 ** -20, 0.7615942, 0.3, 1e-38, 1e-45, 3e38, 0.0, -0.0, float("inf"), float("-inf"),
          float("nan"), -0.25]
    ms += torch.rand(16, generator=g, device=dev()).tolist()
    t = ops.dorefa_forward(x, torch.ones(1, device=dev()))
    for mv in ms:
        m = torch.tensor([mv], device=dev())
        got = ops.dorefa_forward(x, m)
        want = t / m
        assert bits_equal(got.cpu().numpy(), want.cpu().numpy()), mv


def test_x_absmax_is_checked():
    x = _x((4, 32), "chk")
    w_q, w_sum, ws, wz, _ = _weights(16, 32, "chk")
    s, z, qmin, qmax = _qparams("s8", "mid")
    for bad in (torch.zeros(2, device=dev()), torch.zeros(1, dtype=torch.float64, device=dev()), torch.zeros(1)):
        with pytest.raises(SparsebitB200Error):
            ops.int8_linear(x, s, z, qmin, qmax, w_q, w_sum, ws, wz, x_absmax=bad)


# ----------------------------------------------------------------------------- layers
def _layer(kind, a_type, w_type, groups=1, bit=4, w_scheme="per-channel-symmetric", a_scheme="per-tensor-affine", seed_=0):
    torch.manual_seed(seed_)
    if kind == "linear":
        mod = QLinear(nn.Linear(40, 24))
    else:
        mod = QConv2d(nn.Conv2d(16, 16 if groups > 1 else 24, 3, padding=1, groups=groups))
    mod.build_quantizer(cfg(a_scheme, "feature", bit, qtype=a_type), cfg(w_scheme, "weight", bit, qtype=w_type))
    mod = mod.to(dev()).eval()
    x = torch.randn(4, 40, device=dev()) if kind == "linear" else torch.randn(2, 16, 10, 10, device=dev())
    for q, v in ((mod.input_quantizer, x), (mod.weight_quantizer, mod.weight)):
        q.update_observer(v.detach())
        q.calc_qparams()
    if w_type == "adaround":
        mod.weight_quantizer.init_variables(mod.weight)
        with torch.no_grad():
            mod.weight_quantizer.v.normal_()
        mod.weight_quantizer.eval()
    mod.set_quant(w_quant=True, a_quant=True)
    return mod, x


def _bound_check(y, mod, x):
    """|y - fp64 layer over the fake-quant operands| <= 2^-21 (|layer|(|fx|, |fw|) + |bias|)."""
    fx = mod.input_quantizer(x).double()
    fw = mod.weight_quantizer(mod.weight).double()
    b = mod.bias.double() if mod.bias is not None else None
    if isinstance(mod, QLinear):
        t = torch.nn.functional.linear(fx, fw, b)
        a = torch.nn.functional.linear(fx.abs(), fw.abs(), b.abs() if b is not None else None)
    else:
        t = torch.nn.functional.conv2d(fx, fw, b, **mod.fwd_kwargs)
        a = torch.nn.functional.conv2d(fx.abs(), fw.abs(), b.abs() if b is not None else None, **mod.fwd_kwargs)
    assert torch.equal(torch.isnan(y), torch.isnan(t))
    ok = ~torch.isnan(t)
    assert bool(((y.double() - t).abs()[ok] <= 2.0 ** -21 * a[ok] + 1e-30).all())


LAYERS = [("linear", "dorefa", "dorefa", 1), ("conv", "dorefa", "dorefa", 1), ("conv", "dorefa", "dorefa", 16),
          ("conv", "dorefa", "dorefa", 4), ("conv", "lsq", "dorefa", 1), ("linear", "uniform", "adaround", 1),
          ("conv", "uniform", "adaround", 1), ("conv", "dorefa", "adaround", 4)]


@pytest.mark.parametrize("kind,a_type,w_type,groups", LAYERS)
def test_converted_layer_meets_the_bound(kind, a_type, w_type, groups):
    mod, x = _layer(kind, a_type, w_type, groups)
    assert dorefa_adaround_ineligibility(mod) is None
    conv = from_dorefa_adaround(mod)
    dorefa_in = a_type == "dorefa"
    expect = {("linear", True): QLinearDoReFaInt8, ("linear", False): QLinearInt8,
              ("conv", True): QConv2dDoReFaInt8 if groups == 1 else QConv2dGroupDoReFaInt8,
              ("conv", False): QConv2dInt8 if groups == 1 else QConv2dGroupInt8}[(kind, dorefa_in)]
    assert type(conv) is expect
    assert ("input=DoReFa" in repr(conv)) == dorefa_in
    with torch.no_grad():
        y = conv(x)
        _bound_check(y, mod, x)
        if kind == "conv":
            yl = conv(x.contiguous(memory_format=torch.channels_last))
            assert yl.is_contiguous(memory_format=torch.channels_last)
            assert bits_equal(yl.contiguous().cpu().numpy(), y.cpu().numpy())
            assert bits_equal(conv(x[0]).cpu().numpy(), conv(x[:1])[0].cpu().numpy())
            assert bits_equal(conv(x.half()).cpu().numpy(), conv(x.half().float()).cpu().numpy())


@pytest.mark.parametrize("bit", [4, 8])
@pytest.mark.parametrize("scheme", ["per-tensor-symmetric", "per-tensor-affine", "per-channel-symmetric",
                                    "per-channel-affine"])
@pytest.mark.parametrize("w_type", ["dorefa", "adaround"])
def test_weight_grid(w_type, scheme, bit):
    mod, _ = _layer("conv", "uniform", w_type, 1, bit=bit, w_scheme=scheme)
    reason = dorefa_adaround_ineligibility(mod)
    if reason is not None:
        pytest.skip(reason)  # an affine zero point outside the signed range of the stored grid, as the plain rule
    conv = from_dorefa_adaround(mod)
    wq = mod.weight_quantizer
    fw = wq(mod.weight.detach()).reshape(mod.weight.shape[0], -1)
    if w_type == "adaround":
        from oracle.qdq import adaround_forward
        ch = 0 if wq.is_perchannel else None
        ref = adaround_forward(mod.weight.detach().cpu().numpy(), wq.v.detach().cpu().numpy(),
                               wq.scale.reshape(-1).cpu().numpy(), wq.zero_point.reshape(-1).cpu().numpy(),
                               *wq.qdesc.qrange, ch_axis=ch, soft=False)
        fw = torch.from_numpy(np.ascontiguousarray(ref)).to(dev()).reshape(fw.shape)
    scale, zp = wq.scale.reshape(-1, 1).float(), torch.round(wq.zero_point.reshape(-1, 1).float())
    k = fw.shape[1]
    g = conv.w_q[:, :k].to(torch.float32) + ops.int8_grid_offset(wq.qdesc.qrange[0]) - zp
    assert torch.equal(g * scale, fw)


def test_special_inputs_match_the_fake_quant_layer():
    mod, x = _layer("conv", "dorefa", "dorefa", 1)
    conv = from_dorefa_adaround(mod)
    with torch.no_grad():
        xn = x.clone()
        xn[1, 3, 4, 5] = float("nan")
        for xi in (xn, torch.zeros_like(x)):
            y, ref = conv(xi), mod(xi)
            assert bool(torch.isnan(y).all()) and bool(torch.isnan(ref).all())
        xi = x.clone()
        xi[0, 2, 3, 3], xi[1, 5, 0, 0] = float("inf"), float("-inf")
        xo = x.clone()
        xo[0, 2, 3, 3], xo[1, 5, 0, 0] = 30.0, -30.0  # tanh = +-1 exactly
        y = conv(xi)
        assert bits_equal(y.cpu().numpy(), conv(xo).cpu().numpy())
        _bound_check(y, mod, xi)


def test_deterministic_and_graph_replay():
    mod, x = _layer("conv", "dorefa", "dorefa", 1)
    conv = from_dorefa_adaround(mod)
    with torch.no_grad():
        y0 = conv(x)
        assert bits_equal(conv(x).cpu().numpy(), y0.cpu().numpy())
        static = x.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            conv(static)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = conv(static)
        x2 = x * 3.0  # a new max |tanh|: the replay must recompute m
        static.copy_(x2)
        graph.replay()
        torch.cuda.synchronize()
        assert bits_equal(out.cpu().numpy(), conv(x2).cpu().numpy())
        assert not bits_equal(out.cpu().numpy(), y0.cpu().numpy())


# ----------------------------------------------------------------------------- models
@pytest.mark.parametrize("arch,convs", [("resnet18", 20), ("mobilenet_v2", 52)])
@pytest.mark.parametrize("recipe", [("dorefa", "dorefa"), ("pact", "dorefa")])
def test_model_converts_every_layer(arch, convs, recipe):
    tv = pytest.importorskip("torchvision")
    torch.manual_seed(0)
    a_type, w_type = recipe
    model = wrap_quantized(getattr(tv.models, arch)(num_classes=10), cfg("per-tensor-affine", "feature", 4, qtype=a_type),
                           cfg("per-channel-symmetric", "weight", 4, qtype=w_type)).to(dev())
    x = torch.randn(2, 3, 64, 64, device=dev())
    calibrated(model, [x], streaming=True, record_inputs=False).eval()
    _check_converted(model, x, convs + 1)


# not int8_harness.check_converted: each layer runs on the input its fake-quant layer saw, captured before conversion
def _check_converted(model, x, layers):
    """to_integer_dorefa_adaround converts `layers` layers and leaves nothing to the plain converters; each converted
    layer meets the bound against its fake-quant layer on the input that layer saw; channels-last equals NCHW."""
    captured = {}
    hooks = [m.register_forward_pre_hook(lambda m, a, name=name: captured.__setitem__(name, a[0].detach().clone()))
             for name, m in model.named_modules() if isinstance(m, (QConv2d, QLinear))]
    with torch.no_grad():
        model(x)
    for h in hooks:
        h.remove()
    fake = {name: m for name, m in model.named_modules() if isinstance(m, (QConv2d, QLinear))}
    names = to_integer_dorefa_adaround(model)
    assert len(names) == layers
    assert to_integer_linears(model) == [] and to_integer_convs(model) == [] and to_integer_group_convs(model) == []
    mods = dict(model.named_modules())
    with torch.no_grad():
        for name in names:
            _bound_check(mods[name](captured[name]), fake[name], captured[name])
        y = model(x)
        yl = model(x.contiguous(memory_format=torch.channels_last))
    assert bits_equal(yl.contiguous().cpu().numpy(), y.cpu().numpy())


def test_adaround_ptq_resnet18_converts_every_layer():
    """ResNet-18 8w8a AdaRound PTQ (a short reconstruction per layer through the runner's adaround_kwargs): every conv
    and the classifier convert, each within the bound on its captured input, channels-last equal to NCHW."""
    tv = pytest.importorskip("torchvision")
    from sparsebit_b200.quantization.tools import CalibrationRunner, trace_quant_model
    torch.manual_seed(0)
    model = trace_quant_model(wrap_quantized(tv.models.resnet18(num_classes=10), cfg("per-tensor-affine", "feature"),
                                             cfg("per-channel-symmetric", "weight", qtype="adaround")).to(dev()))
    x = torch.randn(4, 3, 64, 64, device=dev())
    runner = CalibrationRunner(model)
    runner.adaround_kwargs = dict(max_steps=30, batch_size=2, print_freq=0)
    runner.prepare_calibration()
    with torch.no_grad():
        model(x)
    runner.layerwise_calibration(dev())
    model.eval()
    for m in model.modules():
        if isinstance(m, (QConv2d, QLinear)):
            m.set_quant(w_quant=True, a_quant=True)
            assert m.weight_quantizer.TYPE == "adaround" and not m.weight_quantizer.training
    _check_converted(model, x, 20 + 1)
