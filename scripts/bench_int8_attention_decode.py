"""Generation on the integer grid: one attention step of a causal decoder with an int8 key/value cache
(QAttentionInt8.forward(..., cache=)) against the routes without one, on GPT-2 small heads [8, 12, L, 64] for
L in {512, 1024} and LLaMA-7B heads [1 and 8, 32, L, 128] for L in {2048, 4096}; Tq in {1, 4, 16} new tokens (the
split-key decode kernels), Tq = 17 and a 64-token prefill chunk (the fused kernel over the cache).  8-bit per-tensor
q, k, v (symmetric) and p (unsigned), scale d^-1/2, causal.

Paths, each timed per step with L keys already in the past (median of three repeats, with [min, max], the paths
alternated; CUDA events over repeated steps after a warm-up):
  cached_us  -- append of the Tq new keys / values plus the cached attention: ops.int8_kv_append and
                ops.int8_attention_cached, the two calls QAttentionInt8.forward(..., cache=) makes.  The cache length
                is rewound to L before every step, so that every step appends at position L and attends to L + Tq
                keys; the column sums of v then drift, which changes no work;
  concat_us  -- today's route without a cache: torch.cat of the fp32 past and the new keys / values, then
                QAttentionInt8 (ops.int8_attention, which re-quantizes all L + Tq keys and values);
  fq_us      -- the fake-quant QAttention on the concatenated fp32 past (QDQ, torch.matmul with TF32 off, softmax);
  sdpa16_us  -- torch.cat of an fp16 past and scaled_dot_product_attention in fp16: a speed reference only, it does not
                compute the same numbers.
The routing threshold: decode_kernels_us is the device time of the three decode kernels (scores, p @ v, combine) in a
cached step, fused_kernel_us that of int8_attention_kernel over the same L + Tq keys in the concat route
(torch.profiler, a separate run after the timings).  At Tq <= 16 they compare the two ways of computing one step's
attention; at Tq = 17 the fused kernel runs in both routes (cached_fused_kernel_us).
Bytes model of the cached step: the cache it reads, E (L + Tq) (dp + dv) bytes, the fp32 scores written and read back
(decode: 8 E Tq (L + Tq)), the fp32 q, new k / v and out; cached_gbs is that over cached_us and copy_gbs the copy rate
of scripts/hbm_ceiling.py (its copy arm at the largest size), run as a subprocess first.  concat_bytes is the fp32
past that the route without a cache reads at least (4 E L (d + dv)).  The card name, power limit and maximum SM
clock are read in the same run.
Usage: python scripts/bench_int8_attention_decode.py [--quick]"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch
import torch.nn.functional as F

from bench_int8_matmul import SIGNED, UNSIGNED, Operand
from bench_util import card, kernel_times, set_tf32, timeit
from sparsebit_b200 import ops

SHAPES = [("gpt2_small", 8, 12, 512, 64), ("gpt2_small", 8, 12, 1024, 64),
          ("llama7b", 1, 32, 2048, 128), ("llama7b", 1, 32, 4096, 128),
          ("llama7b", 8, 32, 2048, 128), ("llama7b", 8, 32, 4096, 128)]
TQS = (1, 4, 16, 17, 64)


def copy_gbs():
    """The copy arm of scripts/hbm_ceiling.py at its largest size (GB/s)."""
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "hbm_ceiling.py"), "--rounds", "3"],
                         capture_output=True, text=True, check=True).stdout
    copy = [r for r in (json.loads(line) for line in out.splitlines() if line.startswith("{")) if r.get("arm") == "copy"]
    return max(copy, key=lambda r: r["elems"])["GB/s"]


def bench(family, bsz, heads, past, dim, tq, info, ceiling):
    torch.manual_seed(bsz + heads + past + tq)
    lead = (bsz, heads)
    kp, vp = (torch.randn(lead + (past, dim), device="cuda") for _ in range(2))
    q, kn, vn = (torch.randn(lead + (tq, dim), device="cuda") for _ in range(3))
    scale = dim ** -0.5
    oq, ok, ov = Operand(q, SIGNED), Operand(kp, SIGNED), Operand(vp, SIGNED)
    op = Operand(torch.tensor([0.0, 1.0], device="cuda"), UNSIGNED)
    qp = [(oq.s, oq.z, SIGNED), (ok.s, ok.z, SIGNED), (op.s, op.z, UNSIGNED), (ov.s, ov.z, SIGNED)]
    cache = ops.Int8KVCache(None, lead, past + tq, dim, dim, q.device)
    ops.int8_kv_append(cache, kp, vp, qp[1], qp[3])
    kp16, vp16, q16, kn16, vn16 = (x.half() for x in (kp, vp, q, kn, vn))

    def cached():
        cache.length = past
        ops.int8_kv_append(cache, kn, vn, qp[1], qp[3])
        return ops.int8_attention_cached(q, cache, *qp, scale=scale, causal=True)

    def concat():
        k, v = torch.cat((kp, kn), -2), torch.cat((vp, vn), -2)
        return ops.int8_attention(q, k, v, *qp, scale=scale, causal=True)

    def fq():
        k, v = torch.cat((kp, kn), -2), torch.cat((vp, vn), -2)
        s = torch.matmul(oq.fq(q), ok.fq(k).transpose(-2, -1)) * scale
        s = s.masked_fill(torch.ones(tq, past + tq, dtype=torch.bool, device="cuda").triu(past + 1), float("-inf"))
        return torch.matmul(op.fq(s.softmax(-1)), ov.fq(v))

    def sdpa16():
        k, v = torch.cat((kp16, kn16), -2), torch.cat((vp16, vn16), -2)
        keep = torch.ones(tq, past + tq, dtype=torch.bool, device="cuda").tril(past)
        return F.scaled_dot_product_attention(q16, k, v, attn_mask=keep)

    y_cached, y_concat = cached(), concat()
    rec = {"family": family, "batch": bsz, "heads": heads, "L": past, "Tq": tq, "d": dim, "dv": dim,
           "route": "decode" if tq <= 16 else "fused",
           "max_abs_cached_vs_concat": float((y_cached - y_concat).abs().max()),
           "bitwise_cached_vs_concat": bool(torch.equal(y_cached, y_concat))}
    paths = (("cached", cached), ("concat", concat), ("fq", fq), ("sdpa16", sdpa16))
    set_tf32(False)
    runs = {name: [] for name, _ in paths}
    for _ in range(3):
        for name, fn in paths:
            runs[name].append(timeit(fn, warmup=3, budget_s=0.2))
    for name, v_ in runs.items():
        rec[name + "_us"] = statistics.median(v_)
        rec[name + "_us_range"] = [min(v_), max(v_)]
    kt = kernel_times(cached, ["int8_attention_decode", "int8_attention_kernel"], reps=5)
    rec["decode_kernels_us"] = kt.get("int8_attention_decode")
    rec["cached_fused_kernel_us"] = kt.get("int8_attention_kernel")
    rec["fused_kernel_us"] = kernel_times(concat, ["int8_attention_kernel"], reps=5).get("int8_attention_kernel")
    e, tk, dp = bsz * heads, past + tq, (dim + 15) // 16 * 16
    cache_bytes = e * tk * (dp + dim)
    scores = 8 * e * tq * tk if tq <= 16 else 0
    rec["cached_bytes"] = cache_bytes + scores + 4 * e * tq * (3 * dim) + 4 * e * tq * dim
    rec["concat_bytes"] = 4 * e * past * 2 * dim
    rec["cached_gbs"] = rec["cached_bytes"] / rec["cached_us"] * 1e-3
    rec["copy_gbs"] = ceiling
    rec["cached_share_of_copy"] = rec["cached_gbs"] / ceiling
    for name in ("concat", "fq", "sdpa16"):
        rec["speedup_vs_" + name] = rec[name + "_us"] / rec["cached_us"]
    rec.update(info)
    print(json.dumps(rec), flush=True)


def main():
    assert torch.cuda.is_available(), "bench_int8_attention_decode.py measures on a GPU"
    quick = "--quick" in sys.argv
    info = card()
    ceiling = copy_gbs()
    print(json.dumps({"copy_gbs": ceiling, **info}), flush=True)
    for family, bsz, heads, past, dim in (SHAPES[:1] if quick else SHAPES):
        for tq in TQS:
            bench(family, bsz, heads, past, dim, tq, info, ceiling)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
