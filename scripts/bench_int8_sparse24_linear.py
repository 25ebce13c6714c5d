"""2:4-sparse integer-grid linear (sb200_int8_sparse24_linear) against the dense one (sb200_int8_linear) and the
fake-quant linear, on the DeiT-base shapes at M = 197 * 64 and 197 * 256 and the LLaMA-7B shapes at M = 16 (decode)
and 2048 (prefill): 8-bit per-tensor symmetric activations, per-channel symmetric weights (MinMax qparams) pruned 2:4
by the 2:4 sparser's rule.

One JSON line per (shape, M):
  fq_f32_us                  -- QDQ of x, QDQ of W, F.linear with TF32 off (the fake-quant path QLinear runs);
  dense_us, sparse_us        -- ops.int8_linear / ops.int8_sparse24_linear end to end (row quantizer + GEMM), as
                                QLinearInt8 / QLinearSparse24Int8 call them;
  dense_gemm_us, sparse_gemm_us, rows_us -- the two GEMM kernels and the row quantizer alone (torch.profiler, a
                                separate run);
  *_tops                     -- useful TOPS 2 M K N over each time (the pruned zeros counted as work, as for dense);
  dense_weight_bytes, sparse_weight_bytes -- weight bytes a GEMM reads: 1 B per weight dense; 0.5 B per weight plus
                                4 bits of metadata per kept pair (0.125 B per weight) sparse, with K padded to 64;
  sparse_vs_dense            -- dense_us / sparse_us (> 1: the sparse layer wins), and the same for the GEMMs alone;
  bit_identical              -- the sparse output equals the dense output bit for bit;
  err_fq_f32, err_int8       -- max |y - T| against the fp64 matmul of the fake-quant operands (+ bias).
Times are CUDA events over repeated calls after warm-up.  The card name and power limit are read in the same run.
Usage: python scripts/bench_int8_sparse24_linear.py [--quick]"""
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
LLAMA = [("qkvo", 4096, 4096), ("gate_up", 4096, 11008), ("down", 11008, 4096)]


class Layer:
    """One 2:4-pruned linear with MinMax qparams, stored both ways."""

    def __init__(self, k, n, x):
        dev = x.device
        w = torch.randn(n, k, device=dev) / k ** 0.5
        self.w = w * ops.sparse24_mask(w)
        self.bias = torch.randn(n, device=dev) * 0.1
        self.xs = (x.abs().max() * 2 / 255).clamp_min(1e-6).reshape(1)
        self.xz = torch.zeros(1, device=dev)
        self.ws = (self.w.abs().amax(dim=1) * 2 / 255).clamp_min(1e-6).contiguous()
        self.wz = torch.zeros(n, device=dev)
        self.w_q, self.w_sum, _ = ops.int8_quantize_rows(self.w, self.ws, self.wz, -128, 127)
        self.w_zero = torch.zeros(n, dtype=torch.int32, device=dev)
        self.vals, self.meta, self.dsum, bad = ops.int8_sparse24_pack(self.w_q, self.w_zero, self.ws, k)
        assert not bool(bad.any())

    def fake_quant(self, x):
        fx = fake_quant.quant_pertensor_forward(x, self.xs, self.xz, -128, 127, 0)
        fw = fake_quant.quant_perchannel_forward(self.w, self.ws, self.wz, -128, 127, 0, 0)
        return F.linear(fx, fw, self.bias)

    def dense(self, x):
        return ops.int8_linear(x, self.xs, self.xz, -128, 127, self.w_q, self.w_sum, self.ws, self.w_zero, self.bias)

    def sparse(self, x):
        return ops.int8_sparse24_linear(x, self.xs, self.xz, -128, 127, self.vals, self.meta, self.dsum, self.ws, self.bias)

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
    ys, yd = layer.sparse(x), layer.dense(x)
    rec["err_int8"] = float((ys.double() - t).abs().max())
    rec["bit_identical"] = bool(torch.equal(ys.view(torch.int32), yd.view(torch.int32)))
    del t, ys, yd
    rec["fq_f32_us"] = timeit(lambda: layer.fake_quant(x))
    rec["dense_us"] = timeit(lambda: layer.dense(x))
    rec["sparse_us"] = timeit(lambda: layer.sparse(x))
    kd = kernel_times(lambda: layer.dense(x), ["int8_linear_gemm_kernel", "int8_quantize_rows_kernel"])
    ks = kernel_times(lambda: layer.sparse(x), ["int8_sparse24_gemm_kernel"])
    rec["dense_gemm_us"] = kd.get("int8_linear_gemm_kernel")
    rec["sparse_gemm_us"] = ks.get("int8_sparse24_gemm_kernel")
    rec["rows_us"] = kd.get("int8_quantize_rows_kernel")
    ops_ = 2.0 * m * k * n
    for key in ("fq_f32", "dense", "sparse", "dense_gemm", "sparse_gemm"):
        if rec.get(key + "_us"):
            rec[key + "_tops"] = ops_ / rec[key + "_us"] * 1e-6
    k64 = (k + 63) // 64 * 64
    rec["dense_weight_bytes"] = n * ((k + 15) // 16 * 16)
    rec["sparse_weight_bytes"] = n * k64 // 2 + layer.meta.numel() * 4
    rec["sparse_vs_dense"] = rec["dense_us"] / rec["sparse_us"]
    if rec["dense_gemm_us"] and rec["sparse_gemm_us"]:
        rec["sparse_vs_dense_gemm"] = rec["dense_gemm_us"] / rec["sparse_gemm_us"]
    rec.update(info)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    assert torch.cuda.is_available(), "bench_int8_sparse24_linear.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    for m in ([197 * 64] if quick else [197 * 64, 197 * 256]):
        for name, k, n in DEIT:
            bench_shape("deit_base", name, k, n, m, info)
    for m in (16, 2048):
        for name, k, n in (LLAMA[:1] if quick else LLAMA):
            bench_shape("llama_7b", name, k, n, m, info)


if __name__ == "__main__":
    main()
