"""Channels-last (NHWC) integer-grid convs against the NCHW ones, on every distinct conv geometry of ResNet-50, the
depthwise convs of MobileNetV2 and EfficientNet-B0 and the grouped convs of RegNetX-400MF and ResNeXt-50 32x4d
(torchvision, 224 x 224 input), 8-bit per-tensor affine activations and per-channel symmetric weights (MinMax qparams).

One JSON line per (geometry, batch in 64, 256), times in us as the median and [min, max] of three alternated repeats
(CUDA events over repeated calls after warm-up):
  nchw_us     -- (a) the NCHW op (ops.int8_conv2d / ops.int8_group_conv2d) on an NCHW input;
  nhwc_us     -- (b) the NHWC op (ops.int8_conv2d_nhwc / ops.int8_group_conv2d_nhwc) on a channels-last input;
  copy_nchw_us -- (c) the route a channels-last input took before the NHWC ops: x.contiguous(), then the NCHW op;
  fq_f32_us, fq_tf32_us -- (d) the fake-quant conv (QDQ of x and W, cuDNN conv2d on NCHW) with TF32 off / on;
  nchw_lower_us, nchw_gemm_us, nhwc_lower_us, nhwc_gemm_us -- dense convs: the lowering (or, for a stride-1 unpadded
      1x1 in NHWC, the row quantizer) and the GEMM alone, torch.profiler in a separate pass;
  nchw_kernel_us, nhwc_kernel_us -- grouped convs: the kernel alone, likewise;
  same_values -- (b) equals (a) bit for bit (NaN-free data).
Then one line per (stack, batch): every conv of each of the five models (ResNet-50 53, MobileNetV2 52, EfficientNet-B0
81, RegNetX-400MF 71, ResNeXt-50 53), each conv on an input of its shape, arms (a) - (d).  The card name and power limit are read in the same run.
Usage: python scripts/bench_int8_conv_nhwc.py [--quick]"""
import collections
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch
import torch.nn as nn
import torch.nn.functional as F

from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import fake_quant, ops

CL = torch.channels_last


def model_convs(name):
    """(c_in, h, w, c_out, groups, k, stride, padding, dilation) of every Conv2d of a torchvision model in forward
    order, at a 1 x 3 x 224 x 224 input."""
    import torchvision

    net = getattr(torchvision.models, name)(weights=None).eval()
    convs = []

    def hook(mod, inp, out):
        x = inp[0]
        convs.append((x.shape[1], x.shape[2], x.shape[3], mod.out_channels, mod.groups, mod.kernel_size[0], mod.stride[0],
                      mod.padding[0], mod.dilation[0]))

    hooks = [m.register_forward_hook(hook) for m in net.modules() if isinstance(m, nn.Conv2d)]
    with torch.no_grad():
        net(torch.zeros(1, 3, 224, 224))
    for h in hooks:
        h.remove()
    return convs


class Layer:
    """One conv with MinMax qparams: 8-bit per-tensor affine activations, per-channel symmetric weights."""

    def __init__(self, geom, x):
        c_in, _, _, c_out, groups, k, stride, padding, dilation = geom
        dev = x.device
        self.groups, self.k, self.stride, self.padding, self.dilation = groups, k, stride, padding, dilation
        self.w = torch.randn(c_out, c_in // groups, k, k, device=dev) / (c_in // groups * k * k) ** 0.5
        self.bias = torch.randn(c_out, device=dev) * 0.1
        lo, hi = torch.clamp(x.min(), max=0.0), torch.clamp(x.max(), min=0.0)
        self.xs = ((hi - lo) / 255).clamp_min(1e-6).reshape(1)
        self.xz = torch.round(-lo / self.xs).clamp(0, 255).reshape(1)
        self.ws = (self.w.reshape(c_out, -1).abs().amax(dim=1) * 2 / 255).clamp_min(1e-6).contiguous()
        self.wz = torch.zeros(c_out, device=dev)
        self.w_q, self.w_sum, _ = ops.int8_quantize_rows(self.w.reshape(c_out, -1).contiguous(), self.ws, self.wz, -128, 127)
        self.w_zero = torch.zeros(c_out, dtype=torch.int32, device=dev)

    def fake_quant(self, x):
        fx = fake_quant.quant_pertensor_forward(x, self.xs, self.xz, 0, 255, 0)
        fw = fake_quant.quant_perchannel_forward(self.w, self.ws, self.wz, -128, 127, 0, 0)
        return F.conv2d(fx, fw, self.bias, stride=self.stride, padding=self.padding, dilation=self.dilation,
                        groups=self.groups)

    def int8(self, x, nhwc):
        args = (x, self.xs, self.xz, 0, 255, self.w_q, self.w_sum, self.ws, self.w_zero, self.k)
        tail = (self.bias, self.stride, self.padding, self.dilation)
        if self.groups == 1:
            return (ops.int8_conv2d_nhwc if nhwc else ops.int8_conv2d)(*args, *tail)
        return (ops.int8_group_conv2d_nhwc if nhwc else ops.int8_group_conv2d)(*args, self.groups, *tail)


def _input(n, c, h, w):
    return torch.relu(torch.randn(n, c, h, w, device="cuda")) + 0.05 * torch.randn(n, c, h, w, device="cuda")


def alternated(arms, repeats=3):
    """{name: (median, min, max)} of `repeats` rounds, each timing every arm once in turn (TF32 set per arm)."""
    times = collections.defaultdict(list)
    for _ in range(repeats):
        for name, (tf32, fn) in arms.items():
            set_tf32(tf32)
            times[name].append(timeit(fn, budget_s=0.1))
    set_tf32(False)
    return {k: (statistics.median(v), min(v), max(v)) for k, v in times.items()}


def _put(rec, key, stats):
    rec[key] = round(stats[0], 2)
    rec[key.replace("_us", "_range_us")] = [round(stats[1], 2), round(stats[2], 2)]


def _arms(layer, x, xc):
    return {"nchw_us": (False, lambda: layer.int8(x, False)), "nhwc_us": (False, lambda: layer.int8(xc, True)),
            "copy_nchw_us": (False, lambda: layer.int8(xc.contiguous(), False)),
            "fq_f32_us": (False, lambda: layer.fake_quant(x)), "fq_tf32_us": (True, lambda: layer.fake_quant(x))}


def bench_geometry(geom, where, n, info):
    c_in, h, w, c_out, groups, k, stride, padding, dilation = geom
    torch.manual_seed(c_in + h + c_out + k + stride + n)
    x = _input(n, c_in, h, w)
    xc = x.to(memory_format=CL)
    layer = Layer(geom, x)
    rec = {"geometry": f"{c_in}x{h}x{w} -> {c_out} g{groups} k{k} s{stride} p{padding}", "models": where, "batch": n}
    y0, y1 = layer.int8(x, False), layer.int8(xc, True)
    rec["same_values"] = bool(torch.equal(y0, y1)) and y1.is_contiguous(memory_format=CL)
    del y0, y1
    for key, v in alternated(_arms(layer, x, xc)).items():
        _put(rec, key, v)
    rec["nhwc_vs_nchw"] = round(rec["nchw_us"] / rec["nhwc_us"], 2)
    rec["nhwc_vs_copy_nchw"] = round(rec["copy_nchw_us"] / rec["nhwc_us"], 2)
    rec.update(info)
    return rec, layer, x, xc


def profile_geometry(rec, layer, x, xc):
    if layer.groups == 1:
        names = ["int8_linear_gemm_kernel", "int8_im2col_quantize_kernel", "int8_im2col_quantize_nhwc_kernel",
                 "int8_quantize_rows_kernel"]
        a = kernel_times(lambda: layer.int8(x, False), names)
        b = kernel_times(lambda: layer.int8(xc, True), names)
        rec["nchw_lower_us"] = round(a.get("int8_im2col_quantize_kernel", 0.0), 2)
        rec["nchw_gemm_us"] = round(a.get("int8_linear_gemm_kernel", 0.0), 2)
        rec["nhwc_lower_us"] = round(b.get("int8_im2col_quantize_nhwc_kernel", 0.0) +
                                     b.get("int8_quantize_rows_kernel", 0.0), 2)
        rec["nhwc_gemm_us"] = round(b.get("int8_linear_gemm_kernel", 0.0), 2)
    else:
        a = kernel_times(lambda: layer.int8(x, False), ["int8_group_conv_kernel"])
        b = kernel_times(lambda: layer.int8(xc, True), ["int8_group_conv_nhwc_kernel"])
        rec["nchw_kernel_us"] = round(a.get("int8_group_conv_kernel", 0.0), 2)
        rec["nhwc_kernel_us"] = round(b.get("int8_group_conv_nhwc_kernel", 0.0), 2)


def bench_stack(family, convs, n, info):
    """The given convs, each on an input of its shape (inputs shared between convs of the same input shape)."""
    torch.manual_seed(7)
    inputs = {}
    for c_in, h, w, *_ in convs:
        if (c_in, h, w) not in inputs:
            x = _input(n, c_in, h, w)
            inputs[(c_in, h, w)] = (x, x.to(memory_format=CL))
    layers = [(Layer(g, inputs[g[:3]][0]),) + inputs[g[:3]] for g in convs]

    def run(fn):
        for layer, x, xc in layers:
            fn(layer, x, xc)

    st = alternated({"nchw_us": (False, lambda: run(lambda l, x, xc: l.int8(x, False))),
                     "nhwc_us": (False, lambda: run(lambda l, x, xc: l.int8(xc, True))),
                     "copy_nchw_us": (False, lambda: run(lambda l, x, xc: l.int8(xc.contiguous(), False))),
                     "fq_f32_us": (False, lambda: run(lambda l, x, xc: l.fake_quant(x))),
                     "fq_tf32_us": (True, lambda: run(lambda l, x, xc: l.fake_quant(x)))})
    rec = {"family": family, "batch": n, "convs": len(layers)}
    for key, v in st.items():
        _put(rec, key, v)
    rec["nhwc_vs_nchw"] = round(rec["nchw_us"] / rec["nhwc_us"], 2)
    rec["nhwc_vs_copy_nchw"] = round(rec["copy_nchw_us"] / rec["nhwc_us"], 2)
    rec.update(info)
    print(json.dumps(rec), flush=True)
    del layers, inputs
    torch.cuda.empty_cache()


def main():
    assert torch.cuda.is_available(), "bench_int8_conv_nhwc.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    convs = {m: model_convs(m) for m in ["resnet50", "mobilenet_v2", "efficientnet_b0", "regnet_x_400mf",
                                         "resnext50_32x4d"]}
    where = collections.defaultdict(list)
    for m, cs in convs.items():
        for g in cs:
            if (m == "resnet50" or g[4] > 1) and m not in where[g]:
                where[g].append(m)
    geoms = list(where)[:4] if quick else list(where)
    batches = [8] if quick else [64, 256]
    for n in batches:
        for g in geoms:
            rec, layer, x, xc = bench_geometry(g, where[g], n, info)
            profile_geometry(rec, layer, x, xc)  # a separate pass after the timed one
            print(json.dumps(rec), flush=True)
            del layer, x, xc
            torch.cuda.empty_cache()
    for n in batches:
        for m in convs:
            bench_stack(m, convs[m], n, info)


if __name__ == "__main__":
    main()
