"""2:4-sparse integer-grid conv2d (sb200_int8_sparse24_conv2d) against the dense one (sb200_int8_conv2d) and the
fake-quant conv, on every distinct ResNet-50 conv geometry at batch 256 (r50_convs of bench_int8_conv.py): 8-bit
per-tensor affine activations and per-channel symmetric weights (MinMax qparams), the weights pruned 2:4 by
ops.sparse24_mask along the rows of weight.reshape(C_out, -1).

One JSON line per geometry:
  fq_f32_us                  -- QDQ of x, QDQ of W, cuDNN conv2d with TF32 off (the fake-quant path QConv2d runs);
  dense_us, sparse_us        -- ops.int8_conv2d / ops.int8_sparse24_conv2d end to end (lowering + GEMM), as
                                QConv2dInt8 / QConv2dSparse24Int8 call them;
  lower_us, dense_gemm_us, sparse_gemm_us -- the lowering kernel and the two GEMM kernels alone (torch.profiler, a
                                separate run);
  sparse_vs_dense            -- dense_us / sparse_us (> 1: the sparse conv wins), and sparse_vs_dense_gemm for the
                                GEMMs alone;
  dense_weight_bytes, sparse_weight_bytes -- weight bytes a GEMM reads: 1 B per weight (K padded to 16) dense; vals
                                (0.5 B per weight, K padded to 64) plus the metadata words sparse;
  bit_identical              -- the sparse output equals the dense output bit for bit (the whole batch);
  err_fq_f32, err_sparse     -- max |y - T| over the first two images against the fp64 conv of the fake-quant
                                operands (+ bias).
Then one line per batch (256 and 64) for the whole ResNet-50 conv stack (53 convs, each on an input of its shape),
dense against sparse.  Times are CUDA events over repeated calls after warm-up.  The card name and power limit are
read in the same run.
Usage: python scripts/bench_int8_sparse24_conv.py [--quick]"""
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch

from bench_int8_conv import Layer, _input, r50_convs
from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import ops


class SparseLayer(Layer):
    """``Layer`` with its weight pruned 2:4, stored both ways.  Pruning keeps the largest |w| of every row, so the
    per-channel MinMax scales do not change."""

    def __init__(self, c_in, c_out, k, stride, padding, x):
        super().__init__(c_in, c_out, k, stride, padding, x)
        self.w = self.w * ops.sparse24_mask(self.w)
        rows = self.w.reshape(c_out, -1).contiguous()
        self.w_q, self.w_sum, _ = ops.int8_quantize_rows(rows, self.ws, self.wz, -128, 127)
        self.vals, self.meta, self.dsum, bad = ops.int8_sparse24_pack(self.w_q, self.w_zero, self.ws, rows.shape[1])
        assert not bool(bad.any())

    def sparse(self, x):
        return ops.int8_sparse24_conv2d(x, self.xs, self.xz, 0, 255, self.vals, self.meta, self.dsum, self.ws, self.k,
                                        self.bias, self.stride, self.padding)


def bench_geometry(geom, count, n, info):
    c_in, hw, c_out, k, stride, padding = geom
    torch.manual_seed(c_in + hw + c_out + k + stride + n)
    x = _input(n, c_in, hw) if c_in != 3 else torch.randn(n, c_in, hw, hw, device="cuda")
    layer = SparseLayer(c_in, c_out, k, stride, padding, x)
    oh = (hw + 2 * padding - k) // stride + 1
    m, kk = n * oh * oh, c_in * k * k
    rec = {"geometry": f"{c_in}x{hw}x{hw} -> {c_out} k{k} s{stride} p{padding}", "count_in_r50": count, "batch": n, "M": m,
           "K": kk, "N": c_out}
    set_tf32(False)
    t = layer.truth(x[:2])
    rec["err_fq_f32"] = float((layer.fake_quant(x[:2]).double() - t).abs().max())
    ys, yd = layer.sparse(x), layer.int8(x)
    rec["err_sparse"] = float((ys[:2].double() - t).abs().max())
    rec["bit_identical"] = bool(torch.equal(ys.view(torch.int32), yd.view(torch.int32)))
    del t, ys, yd
    rec["fq_f32_us"] = timeit(lambda: layer.fake_quant(x))
    rec["dense_us"] = timeit(lambda: layer.int8(x))
    rec["sparse_us"] = timeit(lambda: layer.sparse(x))
    kd = kernel_times(lambda: layer.int8(x), ["int8_linear_gemm_kernel", "int8_im2col_quantize_kernel"])
    ks = kernel_times(lambda: layer.sparse(x), ["int8_sparse24_gemm_kernel"])
    rec["lower_us"] = kd.get("int8_im2col_quantize_kernel")
    rec["dense_gemm_us"] = kd.get("int8_linear_gemm_kernel")
    rec["sparse_gemm_us"] = ks.get("int8_sparse24_gemm_kernel")
    rec["sparse_vs_dense"] = rec["dense_us"] / rec["sparse_us"]
    if rec["dense_gemm_us"] and rec["sparse_gemm_us"]:
        rec["sparse_vs_dense_gemm"] = rec["dense_gemm_us"] / rec["sparse_gemm_us"]
    rec["dense_weight_bytes"] = c_out * ((kk + 15) // 16 * 16)
    rec["sparse_weight_bytes"] = layer.vals.numel() + layer.meta.numel() * 4
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
    layers = [(SparseLayer(c_in, c_out, k, s, p, inputs[(c_in, hw)]), inputs[(c_in, hw)])
              for c_in, hw, c_out, k, s, p in convs]

    def run(fn):
        for layer, x in layers:
            fn(layer, x)

    set_tf32(False)
    dense = timeit(lambda: run(SparseLayer.int8), budget_s=1.0)
    sparse = timeit(lambda: run(SparseLayer.sparse), budget_s=1.0)
    rec = {"family": "resnet50_conv_stack", "batch": n, "convs": len(layers), "dense_us": dense, "sparse_us": sparse,
           "sparse_vs_dense": dense / sparse}
    rec.update(info)
    print(json.dumps(rec), flush=True)
    del layers, inputs
    torch.cuda.empty_cache()


def main():
    assert torch.cuda.is_available(), "bench_int8_sparse24_conv.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    counts = collections.Counter(r50_convs())
    geoms = list(counts)[:3] if quick else list(counts)
    n = 8 if quick else 256
    for g in geoms:
        bench_geometry(g, counts[g], n, info)
        torch.cuda.empty_cache()
    for n in ([8] if quick else [256, 64]):
        bench_stack(n, info)


if __name__ == "__main__":
    main()
