"""Fused integer-grid attention (ops.int8_attention) against the unfused paths, on the attention of DeiT-tiny / -small /
-base (197 tokens, head dim 64; 3 / 6 / 12 heads) at batch 64 and 256, on [8, 32, 2048, 128] and on [2, 32, 16384, 64],
where one fp32 score tensor alone is 68 GB; 8-bit per-tensor q, k, v (symmetric) and p (unsigned), scale d^-1/2.

One JSON line per shape; every time is the median of three repeats with [min, max], the paths alternated:
  fq_f32_us     -- QAttention as it runs in fake-quant: QDQ of q and of a contiguous k^T, torch.matmul (TF32 off),
                   * scale, softmax, QDQ of p and v, torch.matmul;
  fq_tf32_us    -- the same with TF32 on;
  unfused_us    -- QMatMulInt8 -> * scale -> softmax -> QMatMulInt8 (ops.int8_matmul twice, ATen softmax between);
  fused_us      -- ops.int8_attention end to end (three quantize passes + the fused kernel);
  rows_us, cols_us, fused_kernel_us -- the kernels of the fused path alone, per call (torch.profiler, a separate run);
  fused_gbs     -- algorithmic bytes over fused_us: 4 (|q| + |k| + |v|) read, the int8 copies written and read back
                   once, 4 |y| written;
  fused_tops    -- useful TOPS 2 B Tq Tk (d + dv) over fused_us (the kernel also recomputes q k^T in its second pass:
                   executed_tops counts 2 B Tq Tk (2 d + dv));
  err_*         -- max |y - T| on the first two heads, T the fp64 attention of the fake-quant operands (p from the fp64
                   softmax of the scores of fp64 fake-quant q, k).
A path that cannot allocate its tensors reports "does not fit".  Times are CUDA events over repeated calls after a
warm-up per shape.  The card name, power limit and maximum SM clock are read in the same run.
Usage: python scripts/bench_int8_attention.py [--quick]"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch

from bench_int8_matmul import MODELS, SIGNED, UNSIGNED, Operand
from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import ops

FIT = "does not fit"


def p_operand(device):
    """p's qparams: unsigned 8-bit over [0, 1], zero point 0."""
    p = Operand(torch.tensor([0.0, 1.0], device=device), UNSIGNED)
    return p


def bench(family, bsz, heads, tokens, dim, info):
    torch.manual_seed(bsz + heads + tokens)
    shape = (bsz, heads, tokens, dim)
    q, k, v = (torch.randn(shape, device="cuda") for _ in range(3))
    scale = dim ** -0.5
    oq, ok, ov, op = Operand(q, SIGNED), Operand(k.transpose(-2, -1), SIGNED), Operand(v, SIGNED), p_operand(q.device)
    rec = {"family": family, "batch": bsz, "heads": heads, "Tq": tokens, "Tk": tokens, "d": dim, "dv": dim}

    def fq():
        s = torch.matmul(oq.fq(), ok.fq()) * scale
        return torch.matmul(op.fq(s.softmax(-1)), ov.fq())

    def unfused():
        s = ops.int8_matmul(q, oq.s, oq.z, SIGNED, k.transpose(-2, -1), ok.s, ok.z, SIGNED) * scale
        return ops.int8_matmul(s.softmax(-1), op.s, op.z, UNSIGNED, v, ov.s, ov.z, SIGNED)

    def fused():
        return ops.int8_attention(q, k, v, (oq.s, oq.z, SIGNED), (ok.s, ok.z, SIGNED), (op.s, op.z, UNSIGNED),
                                  (ov.s, ov.z, SIGNED), scale=scale)

    sl = (slice(0, 1), slice(0, 2))
    fqd = lambda o, x: o.fq(x).double()
    s64 = (torch.matmul(fqd(oq, q[sl]), fqd(ok, k[sl].transpose(-2, -1))) * scale)
    t = torch.matmul(op.fq(s64.softmax(-1).float()).double(), fqd(ov, v[sl]))
    del s64
    paths = (("fq_f32", fq, False), ("fq_tf32", fq, True), ("unfused", unfused, False), ("fused", fused, False))
    live = []
    for name, fn, tf32 in paths:
        set_tf32(tf32)
        try:
            rec["err_" + name] = float((fn()[sl].double() - t).abs().max())
            live.append((name, fn, tf32))
        except torch.cuda.OutOfMemoryError:
            rec["err_" + name] = rec[name + "_us"] = FIT
        torch.cuda.empty_cache()
    rec["max_abs_T"] = float(t.abs().max())
    del t
    runs = {name: [] for name, _, _ in live}
    for _ in range(3):
        for name, fn, tf32 in live:
            set_tf32(tf32)
            runs[name].append(timeit(fn, warmup=2, budget_s=0.2))
    set_tf32(False)
    for name, v_ in runs.items():
        rec[name + "_us"] = statistics.median(v_)
        rec[name + "_us_range"] = [min(v_), max(v_)]
    kt = kernel_times(fused, ["int8_attention_kernel", "int8_quantize_rows_kernel", "int8_quantize_cols_kernel"], reps=5)
    rec["fused_kernel_us"] = kt.get("int8_attention_kernel")
    rec["rows_us"] = kt.get("int8_quantize_rows_kernel")
    rec["cols_us"] = kt.get("int8_quantize_cols_kernel")
    b = bsz * heads
    n_in = 3 * b * tokens * dim
    rec["fused_gbs"] = (4.0 * n_in + 2.0 * n_in + 4.0 * b * tokens * dim) / rec["fused_us"] * 1e-3
    rec["fused_tops"] = 2.0 * b * tokens * tokens * (dim + dim) / rec["fused_us"] * 1e-6
    rec["executed_tops"] = 2.0 * b * tokens * tokens * (2 * dim + dim) / rec["fused_us"] * 1e-6
    if rec["fused_kernel_us"]:
        rec["kernel_tops"] = 2.0 * b * tokens * tokens * (dim + dim) / rec["fused_kernel_us"] * 1e-6
    for name in ("fq_f32", "fq_tf32", "unfused"):
        if isinstance(rec.get(name + "_us"), float):
            rec["speedup_vs_" + name] = rec[name + "_us"] / rec["fused_us"]
    rec.update(info)
    print(json.dumps(rec), flush=True)


def main():
    assert torch.cuda.is_available(), "bench_int8_attention.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    for bsz in ([64] if quick else [64, 256]):
        for family, heads in (MODELS[:1] if quick else MODELS):
            bench(family, bsz, heads, 197, 64, info)
    if not quick:
        bench("long_sequence", 8, 32, 2048, 128, info)
        bench("long_sequence", 2, 32, 16384, 64, info)


if __name__ == "__main__":
    main()
