"""Masked and causal fused integer-grid attention (ops.int8_attention with attn_mask / causal) against the unfused
paths, at the attention shapes of the reference's two masked PTQ examples: BERT-base on GLUE ([32, 12, 128, 64] and
[8, 12, 512, 64], a [B, 1, 1, T] key-padding mask (1 - m) * -10000, a quarter of the entries padded to half length)
and GPT-2 on wikitext ([8, 12, 1024, 64], causal, block_size 1024); 8-bit per-tensor q, k, v (symmetric) and p
(unsigned), scale d^-1/2.  At the GPT-2 shape the unmasked fused call is timed too, to show what the causal block
skip saves.

One JSON line per shape; every time is the median of three repeats with [min, max], the paths alternated:
  fq_f32_us        -- QAttention as it runs in fake-quant: QDQ of q and k^T, torch.matmul (TF32 off), * scale, the
                      causal where and / or the mask add, softmax, QDQ of p and v, torch.matmul;
  unfused_us       -- QMatMulInt8 -> * scale -> where / + mask -> softmax -> QMatMulInt8 (ops.int8_matmul twice);
  fused_us         -- ops.int8_attention with the mask / causal, end to end (quantize passes, the causal column sums
                      of v, the fused kernel);
  fused_unmasked_us -- (GPT-2 shape) ops.int8_attention without a mask on the same operands;
  fused_kernel_us, fused_unmasked_kernel_us -- the fused kernel alone, per call (torch.profiler, a separate run);
  err_*            -- max |y - T| on the first two heads, T the fp64 attention of the fake-quant operands.
The card name, power limit and maximum SM clock are read in the same run.
Usage: python scripts/bench_int8_attention_mask.py"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch

from bench_int8_attention import p_operand
from bench_int8_matmul import SIGNED, UNSIGNED, Operand
from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import ops


def bench(family, bsz, heads, tokens, dim, causal, padded, info):
    torch.manual_seed(bsz + heads + tokens)
    shape = (bsz, heads, tokens, dim)
    q, k, v = (torch.randn(shape, device="cuda") for _ in range(3))
    scale = dim ** -0.5
    mask = None
    if padded:
        keep = torch.ones(bsz, tokens, device="cuda")
        keep[: bsz // 4, tokens // 2:] = 0
        mask = (1.0 - keep[:, None, None, :]) * -10000.0
    oq, ok, ov, op = Operand(q, SIGNED), Operand(k.transpose(-2, -1), SIGNED), Operand(v, SIGNED), p_operand(q.device)
    rec = {"family": family, "batch": bsz, "heads": heads, "Tq": tokens, "Tk": tokens, "d": dim, "dv": dim,
           "causal": causal, "key_padding": padded}
    hidden = torch.ones(tokens, tokens, dtype=torch.bool, device="cuda").tril().logical_not()

    def masked(s):
        if causal:
            s = s.masked_fill(hidden, float("-inf"))
        return s + mask if mask is not None else s

    def fq():
        s = masked(torch.matmul(oq.fq(), ok.fq()) * scale)
        return torch.matmul(op.fq(s.softmax(-1)), ov.fq())

    def unfused():
        s = masked(ops.int8_matmul(q, oq.s, oq.z, SIGNED, k.transpose(-2, -1), ok.s, ok.z, SIGNED) * scale)
        return ops.int8_matmul(s.softmax(-1), op.s, op.z, UNSIGNED, v, ov.s, ov.z, SIGNED)

    def fused(m=mask, c=causal):
        return ops.int8_attention(q, k, v, (oq.s, oq.z, SIGNED), (ok.s, ok.z, SIGNED), (op.s, op.z, UNSIGNED),
                                  (ov.s, ov.z, SIGNED), scale=scale, attn_mask=m, causal=c)

    sl = (slice(0, 1), slice(0, 2))
    fqd = lambda o, x: o.fq(x).double()
    s64 = torch.matmul(fqd(oq, q[sl]), fqd(ok, k[sl].transpose(-2, -1))) * scale
    if causal:
        s64 = s64.masked_fill(hidden, float("-inf"))
    if mask is not None:
        s64 = s64 + mask[sl[0]].double()
    t = torch.matmul(op.fq(s64.softmax(-1).float()).double(), fqd(ov, v[sl]))
    paths = [("fq_f32", fq), ("unfused", unfused), ("fused", fused)]
    if causal:
        paths.append(("fused_unmasked", lambda: fused(None, False)))
    set_tf32(False)
    for name, fn in paths[:3]:
        rec["err_" + name] = float((fn()[sl].double() - t).abs().max())
    runs = {name: [] for name, _ in paths}
    for _ in range(3):
        for name, fn in paths:
            runs[name].append(timeit(fn, warmup=2, budget_s=0.2))
    for name, v_ in runs.items():
        rec[name + "_us"] = statistics.median(v_)
        rec[name + "_us_range"] = [min(v_), max(v_)]
    rec["fused_kernel_us"] = kernel_times(fused, ["int8_attention_kernel<true>"], reps=5).get("int8_attention_kernel<true>")
    if causal:
        kt = kernel_times(lambda: fused(None, False), ["int8_attention_kernel<false>"], reps=5)
        rec["fused_unmasked_kernel_us"] = kt.get("int8_attention_kernel<false>")
        rec["causal_vs_unmasked"] = rec["fused_us"] / rec["fused_unmasked_us"]
    for name in ("fq_f32", "unfused"):
        rec["speedup_vs_" + name] = rec[name + "_us"] / rec["fused_us"]
    rec.update(info)
    print(json.dumps(rec), flush=True)


def main():
    assert torch.cuda.is_available(), "bench_int8_attention_mask.py measures on a GPU"
    info = card()
    bench("bert_base", 32, 12, 128, 64, False, True, info)
    bench("bert_base", 8, 12, 512, 64, False, True, info)
    bench("gpt2", 8, 12, 1024, 64, True, False, info)


if __name__ == "__main__":
    main()
