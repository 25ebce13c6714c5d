"""Input gradient of the GPTQ 4-bit g128 linear (sb200_gptq_matmul_dgrad) on the LLaMA-7B linear shapes.

One JSON line per (shape, M, path):
  auto / simt / tc      -- this library's dispatch and each kernel forced;
  deq_f32_matmul        -- dequantise to fp32 + torch.matmul with TF32 off: the same accuracy class, the simple
                           alternative the kernels have to beat (the dequantisation is part of every call: keeping a
                           dense copy of the weights would defeat 4-bit fine-tuning);
  deq_f16_hgemm         -- dequantise to fp16 + cuBLAS HGEMM, for context, with its max error against the fp64 truth.
Times are CUDA events over repeated calls after warm-up; useful TFLOP/s = 2 M K N / time, and its share of the 989
TFLOP/s data-sheet dense FP16 rate of the H100 SXM.  The card name and power limit are read in the same run.
Usage: python scripts/bench_gptq_dgrad.py [M ...]   (default 32 256 2048 4096)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from bench_util import card, timeit
from sparsebit_b200 import ops

SHAPES = [("qkvo", 4096, 4096), ("gate_up", 4096, 11008), ("down", 11008, 4096)]  # (name, K = in, N = out)
GS = 128
PEAK_F16 = 989e12


def dequant(qw, sc, zr, k, dtype):
    """[K, N] dense weights s * q - z (fp64 arithmetic for the fp64 truth, else fp32 and a cast)."""
    ct = torch.float64 if dtype == torch.float64 else torch.float32
    shifts = torch.arange(0, 32, 4, device=qw.device, dtype=torch.int32).view(1, 8, 1)
    q = ((qw.unsqueeze(1) >> shifts) & 15).reshape(-1, qw.shape[1])[:k].to(ct)
    gi = torch.arange(k, device=qw.device) // GS
    return (q * sc.t().to(ct)[gi] - zr.t().to(ct)[gi]).to(dtype)


def main():
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    ms = [int(a) for a in sys.argv[1:]] or [32, 256, 2048, 4096]
    info = card()
    print(json.dumps(info))
    for name, k, n in SHAPES:
        g = torch.Generator(device=dev).manual_seed(k + n)
        qw = torch.randint(-2**31, 2**31 - 1, (k // 8, n), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
        sc = (torch.rand(n, k // GS, device=dev, generator=g) * 0.01 + 0.002).contiguous()
        zr = (sc * torch.randint(0, 16, (n, k // GS), device=dev, generator=g).float()).contiguous()
        w64 = dequant(qw, sc, zr, k, torch.float64)
        for m in ms:
            go = torch.randn(m, n, device=dev, generator=g)
            gi = torch.zeros(m, k, device=dev)
            exp = go[:256].double() @ w64.t()
            paths = {
                "auto": lambda: ops.gptq_matmul_dgrad(go, qw, gi, sc, zr, 4, GS),
                "simt": lambda: ops.gptq_matmul_dgrad(go, qw, gi, sc, zr, 4, GS, impl=1),
                "tc": lambda: ops.gptq_matmul_dgrad(go, qw, gi, sc, zr, 4, GS, impl=2),
                "deq_f32_matmul": lambda: gi.addmm_(go, dequant(qw, sc, zr, k, torch.float32).t()),
                "deq_f16_hgemm": lambda: gi.add_(torch.matmul(go.half(), dequant(qw, sc, zr, k, torch.float16).t()).float()),
            }
            for label, fn in paths.items():
                t = timeit(fn, max_iters=100) * 1e-6  # seconds
                gi.zero_()
                fn()
                err = (gi[:256].double() - exp).abs().max().item()
                print(json.dumps({"shape": name, "K": k, "N": n, "M": m, "path": label, "us": round(t * 1e6, 2),
                                  "tflops": round(2 * m * k * n / t / 1e12, 2),
                                  "frac_of_989": round(2 * m * k * n / t / PEAK_F16, 4),
                                  "max_abs_err_vs_fp64": err, **info}), flush=True)
            del go, gi, exp
        del w64


if __name__ == "__main__":
    main()
