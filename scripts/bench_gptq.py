"""GPTQ int4 g128 on the LLaMA-7B linear shapes: this repo (SIMT decode path, wgmma prefill path)
vs the REFERENCE's own CUDA kernel, built from the reference checkout into oracle/_ref/gptq_ref.so
(oracle/build_ref.py) when that is present.  Benchmark infrastructure; prints one JSON line per (shape, M, impl).

Timing: CUDA events, >= 3 warm-ups, rotating over enough distinct weight copies that the packed
weights of consecutive launches exceed L2 (50 MB on an H100) at decode sizes.
"""
import importlib.util
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from sparsebit_b200 import _lib, ops

dev = torch.device("cuda:0")
SHAPES = [("qkvo", 4096, 4096, 4), ("gate_up", 4096, 11008, 2), ("down", 11008, 4096, 1)]  # name, K, N, count per layer
LAYERS = 32
TS_CHUNKS = [int(c) for c in os.environ.get("SB200_TS_CHUNKS", "512").split(",")]
# the packed weights / scales / zeros of a loaded model are constants: the decode kernel may request them while the
# previous linear is still draining (SB200_GPTQ4_STATIC_WEIGHTS, include/sparsebit_b200.h)
STATIC = os.environ.get("SB200_STATIC_WEIGHTS", "1") == "1"


def load_ref():
    path = os.path.join(ROOT, "oracle", "_ref", "gptq_ref.so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location("gptq_ref", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make(k, n, copies, gs=128):
    g = torch.Generator(device=dev).manual_seed(k + n)
    out = []
    for _ in range(copies):
        qw = torch.randint(-2**31, 2**31 - 1, (k // 8, n), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
        scales = torch.rand(n, k // gs, device=dev, generator=g) * 0.01 + 0.002
        zeros = scales * torch.randint(0, 16, (n, k // gs), device=dev, generator=g).float()
        out.append((qw, scales.contiguous(), zeros.contiguous()))
    return out


def timeit(fn, reps, copies=1):
    """GPU time per launch: `copies` launches (one per rotating weight copy) are captured into a CUDA
    graph and the graph is replayed -- decode-sized kernels are shorter than a Python launch."""
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        for i in range(min(copies, 3)):
            fn(i)
        side.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            for i in range(copies):
                fn(i)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    nrep = max(1, reps // copies)
    e0.record()
    for _ in range(nrep):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / (nrep * copies)


def run(ms, with_reference=True, quiet=False):
    """Time all LLaMA-7B linear shapes at every M in `ms`; returns {(M, impl): seconds per forward over all
    32 x 7 linears} and prints one JSON line per measurement unless quiet."""
    ref = load_ref() if with_reference else None
    lib = _lib.load()
    totals = {}

    def emit(rec):
        if not quiet:
            print(json.dumps(rec))

    fp16_acts = os.environ.get("SB200_FP16_ACTS", "1") == "1"
    for m in ms:
        for name, k, n, cnt in SHAPES:
            wbytes = k * n // 2
            copies = max(2, min(24, (256 << 20) // wbytes + 1)) if m <= 64 else 2
            ws = make(k, n, copies)
            x = torch.randn(m, k, device=dev)
            if fp16_acts:
                # the reference's model path: fp16 activations cast to fp32 (utils/quant.py:262-277, SURVEY 8d)
                x = x.half().float()
            y = torch.zeros(m, n, device=dev)
            impls = [("ours_auto", 0, 0)] + ([("ours_simt", 1, 0)] if m <= 64 else []) + [("ours_wgmma_group", 2, 0)]
            if m >= 32:  # the weight-plane kernel, accumulator restarted every chunk_k K
                impls += [(f"ours_wgmma_ts_c{c}", 3, c) for c in TS_CHUNKS]
            for label, impl, chunk in impls:
                try:
                    t = timeit(lambda i: ops.gptq4_matmul(x, *ws[i % copies][:1], y, *ws[i % copies][1:], 128, impl=impl, chunk_k=chunk, static_weights=STATIC),
                               20 if m > 64 else 200, copies)
                except RuntimeError as e:
                    emit({"shape": name, "M": m, "impl": label, "error": str(e)[:100]})
                    continue
                emit({"shape": name, "K": k, "N": n, "M": m, "impl": label, "acts": "fp16->fp32" if fp16_acts else "fp32",
                      "us": t * 1e6, "TFLOPs": 2.0 * m * k * n / t / 1e12, "weight_GBps": (wbytes + 2 * n * (k // 128) * 4) / t / 1e9})
                totals[(m, label)] = totals.get((m, label), 0.0) + t * cnt * LAYERS
            if ref is not None:
                reps = 4 if m > 64 else 200
                t = timeit(lambda i: ref.vecgroupquant4matmul(x, ws[i % copies][0], y, ws[i % copies][1], ws[i % copies][2], 128), reps, copies)
                emit({"shape": name, "K": k, "N": n, "M": m, "impl": "reference_cuda", "us": t * 1e6,
                      "TFLOPs": 2.0 * m * k * n / t / 1e12, "weight_GBps": (wbytes + 2 * n * (k // 128) * 4) / t / 1e9})
                totals[(m, "reference_cuda")] = totals.get((m, "reference_cuda"), 0.0) + t * cnt * LAYERS
            del ws
    # decode with the same-input linears of a layer fused into one launch each: [q, k, v], o, [gate, up], down
    for m in ms:
        if m > 32:
            continue
        try:
            sets = {name: make(k, n, max(2, min(8, (256 << 20) // (k * n // 2 * cnt) + 1)) * cnt) for name, k, n, cnt in SHAPES}
            xq = torch.randn(m, 4096, device=dev).half().float()
            xd = torch.randn(m, 11008, device=dev).half().float()
            ys = {"qkvo": [torch.zeros(m, 4096, device=dev) for _ in range(4)], "gate_up": [torch.zeros(m, 11008, device=dev) for _ in range(2)],
                  "down": [torch.zeros(m, 4096, device=dev)]}
            rounds = min(len(sets["qkvo"]) // 4, len(sets["gate_up"]) // 2, len(sets["down"]))

            def layer(i):
                q4, gu, dn = sets["qkvo"][4 * i:4 * i + 4], sets["gate_up"][2 * i:2 * i + 2], sets["down"][i]
                ops.gptq4_matmul_batch([(xq, w[0], y, w[1], w[2]) for w, y in zip(q4[:3], ys["qkvo"][:3])], 128, static_weights=STATIC)
                ops.gptq4_matmul(xq, q4[3][0], ys["qkvo"][3], q4[3][1], q4[3][2], 128, static_weights=STATIC)
                ops.gptq4_matmul_batch([(xq, w[0], y, w[1], w[2]) for w, y in zip(gu, ys["gate_up"])], 128, static_weights=STATIC)
                ops.gptq4_matmul(xd, dn[0], ys["down"][0], dn[1], dn[2], 128, static_weights=STATIC)

            t = timeit(lambda i: layer(i % rounds), 60, rounds)
            emit({"shape": "layer(qkv|o|gate_up|down)", "M": m, "impl": "ours_fused_launches", "us": t * 1e6,
                  "weight_GBps": (6_476_005_376 / 32 / 2 + 2 * 4 * 6_476_005_376 / 32 / 128) / t / 1e9})
            totals[(m, "ours_fused_launches")] = t * LAYERS
            del sets
        except Exception as e:  # keep the per-linear numbers
            emit({"M": m, "impl": "ours_fused_launches", "error": repr(e)[:160]})
    return totals


def run_f16_linear(m=1, quiet=True):
    """The model path (QuantLinear.forward, fp16 activations): all LLaMA-7B linears through sb200_gptq4_linear_f16_ex, one
    launch per linear vs the staged path (cast, bias, kernel, cast).  Returns seconds per forward for both."""
    out = {}
    for single in (True, False):
        total = 0.0
        for name, k, n, cnt in SHAPES:
            wbytes = k * n // 2
            copies = max(2, min(24, (256 << 20) // wbytes + 1))
            ws = make(k, n, copies)
            x = torch.randn(m, k, device=dev).half()
            bias = torch.zeros(n, device=dev)
            t = timeit(lambda i: ops.gptq4_linear_f16(x, ws[i % copies][0], ws[i % copies][1], ws[i % copies][2], bias, 128,
                                                      static_weights=STATIC, single_launch=single), 200, copies)
            if not quiet:
                print(json.dumps({"shape": name, "M": m, "impl": "f16_linear_one_launch" if single else "f16_linear_staged", "us": t * 1e6}))
            total += t * cnt * LAYERS
            del ws
        out["one_launch" if single else "staged"] = total
    return out


def main():
    ms = [int(a) for a in sys.argv[1:]] or [1, 16, 2048]
    totals = run(ms, with_reference=os.environ.get("SB200_NO_REF", "0") != "1")
    for (m, label), t in sorted(totals.items()):
        print(json.dumps({"summary": "llama7b_all_linears", "M": m, "impl": label, "ms_per_forward": t * 1e3, "tok_per_s": m / t}))
    if 1 in ms:
        for label, t in run_f16_linear(1, quiet=False).items():
            print(json.dumps({"summary": "llama7b_all_linears", "M": 1, "impl": "f16_linear_" + label, "ms_per_forward": t * 1e3, "tok_per_s": 1 / t}))


if __name__ == "__main__":
    main()
