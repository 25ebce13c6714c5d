"""Integer-grid conv2d (sb200_int8_conv2d) against the fake-quant conv QConv2d runs, on every distinct ResNet-50 conv
geometry (torchvision v1.5 layout, as bench.r50_activation_sites / r50_weight_sites), 8-bit per-tensor affine
activations and per-channel symmetric weights (MinMax qparams).

One JSON line per (geometry, batch):
  fq_f32_us        -- the fake-quant path as QConv2d runs it: QDQ of x, QDQ of W, cuDNN conv2d with TF32 off;
  fq_tf32_us       -- the same with TF32 on (PyTorch's default for cuDNN convs; inexact);
  int8_us          -- ops.int8_conv2d end to end (lowering + GEMM);
  lower_us, gemm_us -- the lowering kernel and the GEMM alone (torch.profiler, a separate run);
  lower_gbs        -- the lowering's bytes/s, (4 |x| + M Kp) / lower_us;
  gemm_tops        -- 2 M K N / gemm_us, and int8_tops over the whole call;
  err_fq_f32, err_fq_tf32, err_int8 -- max |y - T| over the first two images against the fp64 conv of the fake-quant
                      operands (+ bias).
Then one line per batch for the whole ResNet-50 conv stack (53 convs, each on an input of its shape), all three ways.
Times are CUDA events over repeated calls after warm-up.  The card name and power limit are read in the same run.
Usage: python scripts/bench_int8_conv.py [--quick]"""
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch
import torch.nn.functional as F

from bench_int8_linear import PEAK_INT8
from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import fake_quant, ops


def r50_convs():
    """(c_in, hw, c_out, kernel, stride, padding) of the 53 convs of ResNet-50 in forward order."""
    convs = [(3, 224, 64, 7, 2, 3)]
    inplanes, hw = 64, 56
    for planes, blocks, stride in [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)]:
        for b in range(blocks):
            s = stride if b == 0 else 1
            convs.append((inplanes, hw, planes, 1, 1, 0))       # conv1 1x1
            convs.append((planes, hw, planes, 3, s, 1))         # conv2 3x3 (stride s)
            convs.append((planes, hw // s, planes * 4, 1, 1, 0))  # conv3 1x1
            if b == 0:
                convs.append((inplanes, hw, planes * 4, 1, s, 0))  # downsample 1x1 (stride s)
            inplanes, hw = planes * 4, hw // s
    return convs


class Layer:
    """One conv with MinMax qparams: 8-bit per-tensor affine activations, per-channel symmetric weights."""

    def __init__(self, c_in, c_out, k, stride, padding, x):
        dev = x.device
        self.k, self.stride, self.padding = k, stride, padding
        self.w = torch.randn(c_out, c_in, k, k, device=dev) / (c_in * k * k) ** 0.5
        self.bias = torch.randn(c_out, device=dev) * 0.1
        lo, hi = torch.clamp(x.min(), max=0.0), torch.clamp(x.max(), min=0.0)
        self.xs = ((hi - lo) / 255).clamp_min(1e-6).reshape(1)
        self.xz = torch.round(-lo / self.xs).clamp(0, 255).reshape(1)
        self.ws = (self.w.reshape(c_out, -1).abs().amax(dim=1) * 2 / 255).clamp_min(1e-6).contiguous()
        self.wz = torch.zeros(c_out, device=dev)
        self.w_q, self.w_sum, _ = ops.int8_quantize_rows(self.w.reshape(c_out, -1).contiguous(), self.ws, self.wz, -128, 127)
        self.w_zero = torch.zeros(c_out, dtype=torch.int32, device=dev)

    def operands(self, x):
        fx = fake_quant.quant_pertensor_forward(x, self.xs, self.xz, 0, 255, 0)
        fw = fake_quant.quant_perchannel_forward(self.w, self.ws, self.wz, -128, 127, 0, 0)
        return fx, fw

    def fake_quant(self, x):
        fx, fw = self.operands(x)
        return F.conv2d(fx, fw, self.bias, stride=self.stride, padding=self.padding)

    def int8(self, x):
        return ops.int8_conv2d(x, self.xs, self.xz, 0, 255, self.w_q, self.w_sum, self.ws, self.w_zero, self.k, self.bias,
                               self.stride, self.padding)

    def truth(self, x):
        fx, fw = self.operands(x)
        return F.conv2d(fx.double(), fw.double(), self.bias.double(), stride=self.stride, padding=self.padding)


def _input(n, c, hw):
    return torch.relu(torch.randn(n, c, hw, hw, device="cuda")) + 0.05 * torch.randn(n, c, hw, hw, device="cuda")


def bench_geometry(geom, count, n, info):
    c_in, hw, c_out, k, stride, padding = geom
    torch.manual_seed(c_in + hw + c_out + k + stride + n)
    x = _input(n, c_in, hw) if c_in != 3 else torch.randn(n, c_in, hw, hw, device="cuda")
    layer = Layer(c_in, c_out, k, stride, padding, x)
    oh = (hw + 2 * padding - k) // stride + 1
    m, kk = n * oh * oh, c_in * k * k
    kp = (kk + 15) // 16 * 16
    rec = {"geometry": f"{c_in}x{hw}x{hw} -> {c_out} k{k} s{stride} p{padding}", "count_in_r50": count, "batch": n, "M": m,
           "K": kk, "N": c_out}
    xs = x[:2]
    t = layer.truth(xs)
    set_tf32(False)
    rec["err_fq_f32"] = float((layer.fake_quant(xs).double() - t).abs().max())
    rec["fq_f32_us"] = timeit(lambda: layer.fake_quant(x))
    set_tf32(True)
    rec["err_fq_tf32"] = float((layer.fake_quant(xs).double() - t).abs().max())
    rec["fq_tf32_us"] = timeit(lambda: layer.fake_quant(x))
    set_tf32(False)
    rec["err_int8"] = float((layer.int8(x)[:2].double() - t).abs().max())
    rec["max_abs_T"] = float(t.abs().max())
    del t
    rec["int8_us"] = timeit(lambda: layer.int8(x))
    kt = kernel_times(lambda: layer.int8(x), ["int8_linear_gemm_kernel", "int8_im2col_quantize_kernel"])
    rec["gemm_us"] = kt.get("int8_linear_gemm_kernel")
    rec["lower_us"] = kt.get("int8_im2col_quantize_kernel")
    ops_ = 2.0 * m * kk * c_out
    rec["int8_tops"] = ops_ / rec["int8_us"] * 1e-6
    if rec["gemm_us"]:
        rec["gemm_tops"] = ops_ / rec["gemm_us"] * 1e-6
        rec["gemm_share_of_1979"] = rec["gemm_tops"] * 1e12 / PEAK_INT8
    if rec["lower_us"]:
        rec["lower_gbs"] = (4.0 * x.numel() + m * kp) / rec["lower_us"] * 1e-3
    rec["speedup_vs_fq_f32"] = rec["fq_f32_us"] / rec["int8_us"]
    rec["speedup_vs_fq_tf32"] = rec["fq_tf32_us"] / rec["int8_us"]
    rec.update(info)
    print(json.dumps(rec), flush=True)


def bench_stack(n, info):
    """The 53 ResNet-50 convs, each on an input of its shape (inputs shared between convs of the same input shape)."""
    torch.manual_seed(7)
    convs = r50_convs()
    inputs = {}
    for c_in, hw, *_ in convs:
        if (c_in, hw) not in inputs:
            inputs[(c_in, hw)] = _input(n, c_in, hw) if c_in != 3 else torch.randn(n, c_in, hw, hw, device="cuda")
    layers = [(Layer(c_in, c_out, k, s, p, inputs[(c_in, hw)]), inputs[(c_in, hw)]) for c_in, hw, c_out, k, s, p in convs]

    def run(fn):
        for layer, x in layers:
            fn(layer, x)

    set_tf32(False)
    fq = timeit(lambda: run(Layer.fake_quant), budget_s=1.0)
    set_tf32(True)
    fq_tf32 = timeit(lambda: run(Layer.fake_quant), budget_s=1.0)
    set_tf32(False)
    i8 = timeit(lambda: run(Layer.int8), budget_s=1.0)
    rec = {"family": "resnet50_conv_stack", "batch": n, "convs": len(layers), "fq_f32_us": fq, "fq_tf32_us": fq_tf32,
           "int8_us": i8, "speedup_vs_fq_f32": fq / i8, "speedup_vs_fq_tf32": fq_tf32 / i8}
    rec.update(info)
    print(json.dumps(rec), flush=True)
    del layers, inputs
    torch.cuda.empty_cache()


def main():
    assert torch.cuda.is_available(), "bench_int8_conv.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    counts = collections.Counter(r50_convs())
    geoms = list(counts)[:3] if quick else list(counts)
    for n in ([8] if quick else [64, 256]):
        for g in geoms:
            bench_geometry(g, counts[g], n, info)
            torch.cuda.empty_cache()
    for n in ([8] if quick else [64, 256]):
        bench_stack(n, info)


if __name__ == "__main__":
    main()
