"""Integer-grid matmul (sb200_int8_matmul) against the fake-quant matmul QMatMul runs, on the two products of DeiT-tiny /
-small / -base attention (197 tokens, head dim 64; 3 / 6 / 12 heads) at batch 64 and 256 and on one long-sequence
shape ([8, 32, 2048, 128]); 8-bit per-tensor operands, symmetric except the unsigned softmax output.
  qk: q [B, H, T, D] @ k^T, k^T the transposed view of a contiguous k (K-major in memory: the row quantizer twice);
  pv: p [B, H, T, T] @ v, v contiguous [B, H, T, D] (N-major: the row quantizer and the transposing column quantizer).

One JSON line per shape; every time is the median of three repeats with [min, max], the three paths alternated:
  fq_f32_us       -- the fake-quant path as QMatMul runs it: QDQ of both operands (of a contiguous copy of k^T, as the
                     quantizer makes one), torch.matmul with TF32 off;
  fq_tf32_us      -- the same with TF32 on (inexact: TF32 rounds the fake-quant operands to 10-bit mantissas);
  int8_us         -- ops.int8_matmul end to end (two quantize passes + GEMM);
  gemm_us, rows_us, cols_us -- the kernels alone, per call (torch.profiler, a separate run);
  int8_tops, gemm_tops      -- useful TOPS 2 B M K N over int8_us / gemm_us, gemm_share_of_1979 against the data-sheet
                               dense INT8 rate of the H100 SXM;
  quant_gbs       -- the quantize passes' bytes/s at 5 B per operand element (fp32 read, s8 write);
  gemm_gbs        -- the GEMM's bytes/s: the s8 operands read once, the fp32 result written;
  err_fq_f32, err_fq_tf32, err_int8 -- max |y - T| against the fp64 matmul of the fake-quant operands, first two
                                       batch entries.
Times are CUDA events over repeated calls after a warm-up per shape.  The card name, power limit and maximum SM clock
are read in the same run.  Usage: python scripts/bench_int8_matmul.py [--quick]"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import fake_quant, ops

PEAK_INT8 = 1979e12
MODELS = [("deit_tiny", 3), ("deit_small", 6), ("deit_base", 12)]
SIGNED, UNSIGNED = (-128, 127), (0, 255)


class Operand:
    """A tensor with MinMax per-tensor qparams on ``qrange``."""

    def __init__(self, x, qrange):
        self.x, self.qrange = x, qrange
        lo, hi = float(x.min()), float(x.max())
        if qrange[0] < 0:
            s, z = max(abs(lo), abs(hi)) * 2 / 255, 0.0
        else:
            s = (max(hi, 0.0) - min(lo, 0.0)) / 255
            z = round(-min(lo, 0.0) / s)
        self.s = torch.tensor([max(s, 1e-6)], device=x.device)
        self.z = torch.tensor([float(z)], device=x.device)

    def fq(self, x=None):
        # the quantizer makes its input contiguous first: for k^T that is a transposing copy
        return fake_quant.quant_pertensor_forward((self.x if x is None else x).contiguous(), self.s, self.z, *self.qrange, 0)


def bench_shape(family, product, a, b, info):
    """``a``: Operand [..., M, K]; ``b``: Operand whose x is [..., K, N], possibly a transposed view."""
    m, k = a.x.shape[-2:]
    n = b.x.shape[-1]
    batch = a.x.numel() // (m * k)
    rec = {"family": family, "product": product, "batch": batch, "M": m, "K": k, "N": n,
           "b_layout": "K-major" if ops._is_k_major(b.x) else "N-major"}

    def fq():
        return torch.matmul(a.fq(), b.fq())

    def int8():
        return ops.int8_matmul(a.x, a.s, a.z, a.qrange, b.x, b.s, b.z, b.qrange)

    sl = (slice(0, 1),) * (a.x.dim() - 3) + (slice(0, 2),)  # two batch entries
    t = torch.matmul(a.fq(a.x[sl].contiguous()).double(), b.fq(b.x[sl]).double())
    for name, fn, tf32 in (("err_fq_f32", fq, False), ("err_fq_tf32", fq, True), ("err_int8", int8, False)):
        set_tf32(tf32)
        rec[name] = float((fn()[sl].double() - t).abs().max())
    rec["max_abs_T"] = float(t.abs().max())
    del t
    runs = {"fq_f32_us": [], "fq_tf32_us": [], "int8_us": []}
    for _ in range(3):  # the three paths alternated
        for name, fn, tf32 in (("fq_f32_us", fq, False), ("fq_tf32_us", fq, True), ("int8_us", int8, False)):
            set_tf32(tf32)
            runs[name].append(timeit(fn, warmup=2, budget_s=0.2))
    set_tf32(False)
    for name, v in runs.items():
        rec[name] = statistics.median(v)
        rec[name + "_range"] = [min(v), max(v)]
    kt = kernel_times(int8, ["int8_matmul_gemm_kernel", "int8_quantize_rows_kernel", "int8_quantize_cols_kernel"], reps=5)
    rec["gemm_us"] = kt.get("int8_matmul_gemm_kernel")
    rec["rows_us"] = kt.get("int8_quantize_rows_kernel")
    rec["cols_us"] = kt.get("int8_quantize_cols_kernel")
    ops_ = 2.0 * batch * m * k * n
    kp = ops.int8_padded_k(k)
    rec["int8_tops"] = ops_ / rec["int8_us"] * 1e-6
    if rec["gemm_us"]:
        rec["gemm_tops"] = ops_ / rec["gemm_us"] * 1e-6
        rec["gemm_share_of_1979"] = rec["gemm_tops"] * 1e12 / PEAK_INT8
        rec["gemm_gbs"] = batch * ((m + n) * kp + 4.0 * m * n) / rec["gemm_us"] * 1e-3
    quant_us = (rec["rows_us"] or 0.0) + (rec["cols_us"] or 0.0)
    if quant_us:
        rec["quant_gbs"] = 5.0 * batch * (m + n) * k / quant_us * 1e-3
    rec["speedup_vs_fq_f32"] = rec["fq_f32_us"] / rec["int8_us"]
    rec["speedup_vs_fq_tf32"] = rec["fq_tf32_us"] / rec["int8_us"]
    rec.update(info)
    print(json.dumps(rec), flush=True)


def attention_shapes(family, bsz, heads, tokens, dim, info):
    torch.manual_seed(bsz + heads + tokens)
    q = torch.randn(bsz, heads, tokens, dim, device="cuda")
    k = torch.randn(bsz, heads, tokens, dim, device="cuda")
    bench_shape(family, "qk", Operand(q * dim ** -0.5, SIGNED), Operand(k.transpose(-2, -1), SIGNED), info)
    del q, k
    p = torch.rand(bsz, heads, tokens, tokens, device="cuda")
    p /= p.sum(dim=-1, keepdim=True)  # rows sum to 1, as softmax output
    v = torch.randn(bsz, heads, tokens, dim, device="cuda")
    bench_shape(family, "pv", Operand(p, UNSIGNED), Operand(v, SIGNED), info)


def main():
    assert torch.cuda.is_available(), "bench_int8_matmul.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    for bsz in ([64] if quick else [64, 256]):
        for family, heads in (MODELS[:1] if quick else MODELS):
            attention_shapes(family, bsz, heads, 197, 64, info)
    if not quick:
        attention_shapes("long_sequence", 8, 32, 2048, 128, info)


if __name__ == "__main__":
    main()
