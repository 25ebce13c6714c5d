"""GPTQ 4 / 3 / 2-bit g128 decode (M = 1, 16) on the LLaMA-7B linear shapes: this repo's SIMT kernel (gptq_simt.cu;
4-bit forced through impl 4) vs the reference's own CUDA kernels (oracle/_ref/gptq_ref.so).  One JSON line per
(bits, shape, M, impl) and a per-token summary.  Same timing method as bench_gptq.py (CUDA graphs over rotating weight
copies > L2)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch

from bench_gptq import LAYERS, SHAPES, dev, load_ref, timeit
from sparsebit_b200 import ops
from sparsebit_b200.gptq.quant_linear import pack_rows


def main():
    ref = load_ref()
    ms = [int(a) for a in sys.argv[1:]] or [1, 16]
    totals = {}
    for bits in (4, 3, 2):
        for m in ms:
            for name, k, n, cnt in SHAPES:
                rows = pack_rows(k, bits)
                wbytes = rows * n * 4
                copies = max(2, min(24, (256 << 20) // wbytes + 1))
                g = torch.Generator(device=dev).manual_seed(k + n + bits)
                ws = []
                for _ in range(copies):
                    qw = torch.randint(-2**31, 2**31 - 1, (rows, n), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
                    sc = torch.rand(n, k // 128, device=dev, generator=g) * 0.01 + 0.002
                    zr = sc * torch.randint(0, 2**bits, (n, k // 128), device=dev, generator=g).float()
                    ws.append((qw, sc.contiguous(), zr.contiguous()))
                x = torch.randn(m, k, device=dev).half().float()
                y = torch.zeros(m, n, device=dev)
                if bits == 4:
                    impls = [("ours", lambda i: ops.gptq4_matmul(x, ws[i % copies][0], y, ws[i % copies][1], ws[i % copies][2], 128, impl=4))]
                else:
                    impls = [("ours", lambda i: ops.gptq_matmul(x, ws[i % copies][0], y, ws[i % copies][1], ws[i % copies][2], bits, 128))]
                if ref is not None:
                    fn = {4: ref.vecgroupquant4matmul, 3: ref.vecgroupquant3matmul, 2: ref.vecgroupquant2matmul}[bits]
                    impls.append(("reference_cuda", lambda i, fn=fn: fn(x, ws[i % copies][0], y, ws[i % copies][1], ws[i % copies][2], 128)))
                for label, call in impls:
                    t = timeit(call, 200, copies)
                    print(json.dumps({"bits": bits, "shape": name, "K": k, "N": n, "M": m, "impl": label, "us": t * 1e6,
                                      "weight_GBps": (wbytes + 2 * n * (k // 128) * 4) / t / 1e9}))
                    totals[(bits, m, label)] = totals.get((bits, m, label), 0.0) + t * cnt * LAYERS
                del ws
    for (bits, m, label), t in sorted(totals.items()):
        print(json.dumps({"summary": "llama7b_all_linears", "bits": bits, "M": m, "impl": label, "ms_per_forward": t * 1e3,
                          "tok_per_s": m / t}))


if __name__ == "__main__":
    main()
