"""Integer-grid grouped / depthwise conv2d (sb200_int8_group_conv2d) against the fake-quant conv as QConv2d runs it, on
every distinct grouped or depthwise conv geometry of MobileNetV2, EfficientNet-B0, RegNetX-400MF and ResNeXt-50 32x4d
(torchvision, 224 x 224 input), 8-bit per-tensor affine activations and per-channel symmetric weights (MinMax qparams).

One JSON line per (geometry, batch), times in us as the median and [min, max] of three alternated repeats (CUDA events
over repeated calls after warm-up):
  fq_f32_us        -- the fake-quant path: QDQ of x, QDQ of W, cuDNN grouped conv2d with TF32 off;
  fq_tf32_us       -- the same with TF32 on;
  int8_us          -- ops.int8_group_conv2d;
  int8_gbs         -- (4 |x| + 4 |y| + |w_q|) / int8_us, with its share of the data-sheet 3.35 TB/s and of the copy
                      rate measured in the same run (y.copy_(x) over 1 GiB, as the copy arm of scripts/hbm_ceiling.py);
  int8_gops        -- 2 N C_out OH OW K_g / int8_us;
  err_fq_f32, err_fq_tf32, err_int8 -- max |y - T| over the first two images against the fp64 conv of the fake-quant
                      operands (+ bias).
Then one line per (model, batch) for the model's grouped-conv stack, and one per batch for the whole 52-conv
MobileNetV2 stack with ops.int8_conv2d + ops.int8_group_conv2d against fake-quant.  The card name and power limit are
read in the same run.  Usage: python scripts/bench_int8_group_conv.py [--quick]"""
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

from bench_util import card, set_tf32, timeit
from sparsebit_b200 import fake_quant, ops

HBM_PEAK = 3.35e12
MODELS = ["mobilenet_v2", "efficientnet_b0", "regnet_x_400mf", "resnext50_32x4d"]


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

    def kwargs(self):
        return dict(stride=self.stride, padding=self.padding, dilation=self.dilation, groups=self.groups)

    def operands(self, x):
        fx = fake_quant.quant_pertensor_forward(x, self.xs, self.xz, 0, 255, 0)
        fw = fake_quant.quant_perchannel_forward(self.w, self.ws, self.wz, -128, 127, 0, 0)
        return fx, fw

    def fake_quant(self, x):
        fx, fw = self.operands(x)
        return F.conv2d(fx, fw, self.bias, **self.kwargs())

    def int8(self, x):
        if self.groups == 1:
            return ops.int8_conv2d(x, self.xs, self.xz, 0, 255, self.w_q, self.w_sum, self.ws, self.w_zero, self.k,
                                   self.bias, self.stride, self.padding, self.dilation)
        return ops.int8_group_conv2d(x, self.xs, self.xz, 0, 255, self.w_q, self.w_sum, self.ws, self.w_zero, self.k,
                                     self.groups, self.bias, self.stride, self.padding, self.dilation)

    def truth(self, x):
        fx, fw = self.operands(x)
        return F.conv2d(fx.double(), fw.double(), self.bias.double(), **self.kwargs())


def _input(n, c, h, w):
    return torch.relu(torch.randn(n, c, h, w, device="cuda")) + 0.05 * torch.randn(n, c, h, w, device="cuda")


def alternated(arms, repeats=3):
    """{name: (median, min, max)} of `repeats` rounds, each timing every arm once in turn (TF32 set per arm)."""
    times = collections.defaultdict(list)
    for _ in range(repeats):
        for name, (tf32, fn) in arms.items():
            set_tf32(tf32)
            times[name].append(timeit(fn, budget_s=0.2))
    set_tf32(False)
    return {k: (statistics.median(v), min(v), max(v)) for k, v in times.items()}


def _put(rec, key, stats):
    rec[key] = round(stats[0], 2)
    rec[key.replace("_us", "_range_us")] = [round(stats[1], 2), round(stats[2], 2)]


def copy_rate():
    """Bytes/s of y.copy_(x) over 1 GiB of fp32 (2 GiB moved per call), CUDA events after warm-up."""
    x = torch.randn(1 << 28, device="cuda")
    y = torch.empty_like(x)
    us = timeit(lambda: y.copy_(x), budget_s=0.5)
    del x, y
    torch.cuda.empty_cache()
    return 2.0 * 4 * (1 << 28) / (us * 1e-6)


def bench_geometry(geom, where, n, info, copy_bps):
    c_in, h, w, c_out, groups, k, stride, padding, dilation = geom
    torch.manual_seed(c_in + h + c_out + k + stride + n)
    x = _input(n, c_in, h, w)
    layer = Layer(geom, x)
    oh = (h + 2 * padding - dilation * (k - 1) - 1) // stride + 1
    ow = (w + 2 * padding - dilation * (k - 1) - 1) // stride + 1
    kg = c_in // groups * k * k
    rec = {"geometry": f"{c_in}x{h}x{w} -> {c_out} g{groups} k{k} s{stride} p{padding}", "C_g": c_in // groups,
           "models": where, "batch": n}
    xs = x[:2]
    t = layer.truth(xs)
    for name, tf32, fn in (("fq_f32", False, layer.fake_quant), ("fq_tf32", True, layer.fake_quant), ("int8", False, layer.int8)):
        set_tf32(tf32)
        rec["err_" + name] = float((fn(xs).double() - t).abs().max())
    set_tf32(False)
    rec["max_abs_T"] = float(t.abs().max())
    del t
    st = alternated({"fq_f32_us": (False, lambda: layer.fake_quant(x)), "fq_tf32_us": (True, lambda: layer.fake_quant(x)),
                     "int8_us": (False, lambda: layer.int8(x))})
    for key, v in st.items():
        _put(rec, key, v)
    us = rec["int8_us"]
    nbytes = 4.0 * x.numel() + 4.0 * n * c_out * oh * ow + layer.w_q.numel()
    rec["int8_gbs"] = round(nbytes / us * 1e-3, 1)
    rec["share_of_3.35TBs"] = round(nbytes / (us * 1e-6) / HBM_PEAK, 3)
    rec["share_of_copy"] = round(nbytes / (us * 1e-6) / copy_bps, 3)
    rec["int8_gops"] = round(2.0 * n * c_out * oh * ow * kg / us * 1e-3, 1)
    rec["speedup_vs_fq_f32"] = round(rec["fq_f32_us"] / us, 2)
    rec["speedup_vs_fq_tf32"] = round(rec["fq_tf32_us"] / us, 2)
    rec.update(info)
    print(json.dumps(rec), flush=True)


def bench_stack(family, convs, n, info):
    """The given convs, each on an input of its shape (inputs shared between convs of the same input shape)."""
    torch.manual_seed(7)
    inputs = {}
    for c_in, h, w, *_ in convs:
        if (c_in, h, w) not in inputs:
            inputs[(c_in, h, w)] = _input(n, c_in, h, w)
    layers = [(Layer(g, inputs[g[:3]]), inputs[g[:3]]) for g in convs]

    def run(fn):
        for layer, x in layers:
            fn(layer, x)

    st = alternated({"fq_f32_us": (False, lambda: run(Layer.fake_quant)), "fq_tf32_us": (True, lambda: run(Layer.fake_quant)),
                     "int8_us": (False, lambda: run(Layer.int8))}, repeats=3)
    rec = {"family": family, "batch": n, "convs": len(layers)}
    for key, v in st.items():
        _put(rec, key, v)
    rec["speedup_vs_fq_f32"] = round(rec["fq_f32_us"] / rec["int8_us"], 2)
    rec["speedup_vs_fq_tf32"] = round(rec["fq_tf32_us"] / rec["int8_us"], 2)
    rec.update(info)
    print(json.dumps(rec), flush=True)
    del layers, inputs
    torch.cuda.empty_cache()


def main():
    assert torch.cuda.is_available(), "bench_int8_group_conv.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    copy_bps = copy_rate()
    info["copy_gbs"] = round(copy_bps * 1e-9, 1)
    convs = {m: model_convs(m) for m in MODELS}
    where = collections.defaultdict(list)
    for m, cs in convs.items():
        for g in cs:
            if g[4] > 1 and m not in where[g]:
                where[g].append(m)
    geoms = list(where)[:3] if quick else list(where)
    batches = [8] if quick else [64, 256]
    for n in batches:
        for g in geoms:
            bench_geometry(g, where[g], n, info, copy_bps)
            torch.cuda.empty_cache()
    for n in batches:
        for m in MODELS[:1] if quick else MODELS:
            bench_stack(f"{m}_grouped_convs", [g for g in convs[m] if g[4] > 1], n, info)
        bench_stack("mobilenet_v2_all_convs", convs["mobilenet_v2"], n, info)


if __name__ == "__main__":
    main()
