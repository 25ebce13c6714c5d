"""Integer-grid linear (sb200_int8_linear) against the fake-quant linear QLinear runs, on the DeiT-base and LLaMA-7B
linear shapes, 8-bit per-tensor symmetric activations and per-channel symmetric weights (MinMax qparams).

One JSON line per (shape, M):
  fq_f32_us       -- the fake-quant path as QLinear runs it: QDQ of x, QDQ of W, F.linear with TF32 off;
  fq_tf32_us      -- the same with TF32 on (inexact: TF32 rounds the fake-quant operands to 10-bit mantissas);
  int8_us         -- ops.int8_linear end to end (row quantizer + GEMM);
  gemm_us, rows_us -- the GEMM kernel and the row quantizer alone (torch.profiler, a separate run);
  int8_tops       -- useful TOPS 2 M K N / int8_us, and gemm_tops over the GEMM alone, with their share of the
                     1,979 TOPS data-sheet dense INT8 rate of the H100 SXM;
  rows_gbs        -- the row quantizer's bytes/s at 5 B per activation element (fp32 read, s8 write);
  err_fq_f32, err_fq_tf32, err_int8 -- max |y - T| against the fp64 matmul of the fake-quant operands (+ bias).
Then one line for the DeiT-base linear stack (12 blocks x 4 linears) at M = 197 * 64, both ways.  Times are CUDA
events over repeated calls after warm-up.  The card name and power limit are read in the same run.
Usage: python scripts/bench_int8_linear.py [--quick]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F

from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import fake_quant, ops

DEIT = [("qkv", 768, 2304), ("proj", 768, 768), ("fc1", 768, 3072), ("fc2", 3072, 768)]  # (name, K, N)
LLAMA = [("q", 4096, 4096), ("k", 4096, 4096), ("v", 4096, 4096), ("o", 4096, 4096), ("gate", 4096, 11008),
         ("up", 4096, 11008), ("down", 11008, 4096)]
PEAK_INT8 = 1979e12


class Layer:
    """One linear with MinMax qparams: 8-bit per-tensor symmetric activations, per-channel symmetric weights."""

    def __init__(self, k, n, x):
        dev = x.device
        self.w = torch.randn(n, k, device=dev) / k ** 0.5
        self.bias = torch.randn(n, device=dev) * 0.1
        self.xs = (torch.maximum(x.abs().max(), torch.tensor(0.0, device=dev)) * 2 / 255).clamp_min(1e-6).reshape(1)
        self.xz = torch.zeros(1, device=dev)
        self.ws = (self.w.abs().amax(dim=1) * 2 / 255).clamp_min(1e-6).contiguous()
        self.wz = torch.zeros(n, device=dev)
        w_q, self.w_sum, w_nan = ops.int8_quantize_rows(self.w, self.ws, self.wz, -128, 127)
        self.w_q = w_q
        self.w_zero = torch.zeros(n, dtype=torch.int32, device=dev)

    def fake_quant(self, x):
        fx = fake_quant.quant_pertensor_forward(x, self.xs, self.xz, -128, 127, 0)
        fw = fake_quant.quant_perchannel_forward(self.w, self.ws, self.wz, -128, 127, 0, 0)
        return F.linear(fx, fw, self.bias)

    def int8(self, x):
        return ops.int8_linear(x, self.xs, self.xz, -128, 127, self.w_q, self.w_sum, self.ws, self.w_zero, self.bias)

    def truth(self, x):
        fx = fake_quant.quant_pertensor_forward(x, self.xs, self.xz, -128, 127, 0).double()
        fw = fake_quant.quant_perchannel_forward(self.w, self.ws, self.wz, -128, 127, 0, 0).double()
        return fx @ fw.t() + self.bias.double()


def bench_shape(family, name, k, n, m, info):
    torch.manual_seed(k + n + m)
    x = torch.randn(m, k, device="cuda")
    layer = Layer(k, n, x)
    t = layer.truth(x)
    rec = {"family": family, "shape": name, "M": m, "K": k, "N": n}
    set_tf32(False)
    rec["err_fq_f32"] = float((layer.fake_quant(x).double() - t).abs().max())
    rec["fq_f32_us"] = timeit(lambda: layer.fake_quant(x))
    set_tf32(True)
    rec["err_fq_tf32"] = float((layer.fake_quant(x).double() - t).abs().max())
    rec["fq_tf32_us"] = timeit(lambda: layer.fake_quant(x))
    set_tf32(False)
    rec["err_int8"] = float((layer.int8(x).double() - t).abs().max())
    rec["max_abs_T"] = float(t.abs().max())
    del t
    rec["int8_us"] = timeit(lambda: layer.int8(x))
    kt = kernel_times(lambda: layer.int8(x), ["int8_linear_gemm_kernel", "int8_quantize_rows_kernel"])
    rec["gemm_us"] = kt.get("int8_linear_gemm_kernel")
    rec["rows_us"] = kt.get("int8_quantize_rows_kernel")
    ops_ = 2.0 * m * k * n
    rec["int8_tops"] = ops_ / rec["int8_us"] * 1e-6
    rec["int8_share_of_1979"] = rec["int8_tops"] * 1e12 / PEAK_INT8
    if rec["gemm_us"]:
        rec["gemm_tops"] = ops_ / rec["gemm_us"] * 1e-6
        rec["gemm_share_of_1979"] = rec["gemm_tops"] * 1e12 / PEAK_INT8
    if rec["rows_us"]:
        rec["rows_gbs"] = 5.0 * m * k / rec["rows_us"] * 1e-3
    rec["speedup_vs_fq_f32"] = rec["fq_f32_us"] / rec["int8_us"]
    rec.update(info)
    print(json.dumps(rec), flush=True)
    return rec


def bench_stack(m, info):
    """12 DeiT-base blocks x (qkv, proj, fc1, fc2), each layer on its own input of the right width."""
    torch.manual_seed(7)
    xs = {k: torch.randn(m, k, device="cuda") for k in (768, 3072)}
    layers = [Layer(k, n, xs[k]) for _ in range(12) for (_, k, n) in DEIT]
    set_tf32(False)

    def run(fn):
        for layer in layers:
            fn(layer, xs[layer.w.shape[1]])

    fq = timeit(lambda: run(Layer.fake_quant), budget_s=1.0)
    i8 = timeit(lambda: run(Layer.int8), budget_s=1.0)
    rec = {"family": "deit_base_stack", "M": m, "layers": len(layers), "fq_f32_us": fq, "int8_us": i8, "speedup": fq / i8}
    rec.update(info)
    print(json.dumps(rec), flush=True)


def main():
    assert torch.cuda.is_available(), "bench_int8_linear.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    ms = [197 * 16] if quick else [197 * 16, 197 * 64, 197 * 256]
    for m in ms:
        for name, k, n in DEIT:
            bench_shape("deit_base", name, k, n, m, info)
    for name, k, n in (LLAMA[:1] if quick else LLAMA):
        bench_shape("llama_7b", name, k, n, 2048, info)
    bench_stack(197 * 64, info)


if __name__ == "__main__":
    main()
