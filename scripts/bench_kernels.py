"""Per-kernel roofline measurements at BASELINE shapes (SURVEY.md 8d): every C-ABI entry point of the
hot path, CUDA events, >= 5 warm-ups, working sets larger than L2 (or rotated buffers).  Prints one
JSON line per kernel: achieved algorithmic GB/s and fraction of the measured HBM peak."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from sparsebit_b200 import _lib, ops

dev = torch.device("cuda:0")
PEAK, PEAK_SRC = 3350.0, "H100 SXM data sheet (HBM3), not measured"
p = os.path.join(ROOT, "MEASURED_PEAKS.json")
if os.path.exists(p):
    PEAK, PEAK_SRC = float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"


def timeit(fn, reps=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / reps


def report(name, shape, alg_bytes, t, note=""):
    gbs = alg_bytes / t / 1e9
    print(json.dumps({"kernel": name, "shape": list(shape), "us": round(t * 1e6, 2), "alg_GBps": round(gbs, 1),
                      "frac_of_hbm_peak": round(gbs / PEAK, 3), "peak_source": PEAK_SRC, "note": note}), flush=True)


def main():
    g = torch.Generator(device=dev).manual_seed(0)
    s1, z1 = torch.tensor([0.02], device=dev), torch.tensor([3.0], device=dev)

    # ---- per-tensor QDQ, fused stats, minmax on the headline tensor and the largest R50 site
    for shape in [(256, 3, 224, 224), (256, 256, 56, 56)]:
        x = torch.randn(shape, device=dev, generator=g)
        y = torch.empty_like(x)
        n = x.numel()
        st = ops.minmax_new(1, dev)
        report("qdq_pertensor_fwd", shape, 8 * n, timeit(lambda: ops.qdq_pertensor(x, s1, z1, 0, 255, out=y)))
        report("qdq_stats_pertensor_fwd", shape, 8 * n, timeit(lambda: ops.qdq_stats_pertensor(x, s1, z1, 0, 255, st, out=y)))
        report("observe_minmax", shape, 4 * n, timeit(lambda: ops.minmax_update(x, st)))
        gy = torch.randn_like(x)
        sg, zg = s1.clone().requires_grad_(True), z1.clone().requires_grad_(True)
        report("qdq_pertensor_bwd(gx,gs,gzp)", shape, 12 * n, timeit(lambda: ops.qdq_backward(x, sg, zg, gy, 0, 255)))
        report("qdq_pertensor_bwd(gx only)", shape, 12 * n, timeit(lambda: ops.qdq_backward(x, s1, z1, gy, 0, 255, need_gs=False, need_gzp=False)))
        del gy, y

    # ---- per-channel QDQ / minmax / backward: NCHW activations (3 regimes), weights, NLC
    for shape, ch in [((256, 64, 112, 112), 1), ((256, 256, 56, 56), 1), ((256, 512, 28, 28), 1), ((256, 2048, 7, 7), 1),
                      ((1024, 197, 768), 2), ((256, 197, 3072), 2), ((2048, 512, 3, 3), 0), ((1000, 2048), 0)]:
        x = torch.randn(shape, device=dev, generator=g)
        c = shape[ch]
        sc = torch.rand(c, device=dev, generator=g) * 0.02 + 0.01
        zc = torch.zeros(c, device=dev)
        y = torch.empty_like(x)
        n = x.numel()
        st = ops.minmax_new(c, dev)
        small = n * 8 < (200 << 20)
        note = "working set < L2 (L2-resident)" if small else ""
        report("qdq_perchannel_fwd", shape, 8 * n, timeit(lambda: ops.qdq_perchannel(x, sc, zc, -128, 127, ch, out=y)), note)
        report("observe_minmax_perchannel", shape, 4 * n, timeit(lambda: ops.minmax_update(x, st, ch)), note)
        if n <= 210_000_000:
            gy = torch.randn_like(x)
            sg, zg = sc.clone().requires_grad_(True), zc.clone().requires_grad_(True)
            report("qdq_perchannel_bwd(gx,gs,gzp)", shape, 12 * n, timeit(lambda: ops.qdq_backward(x, sg, zg, gy, -128, 127, ch)), note)
            del gy
        del x, y

    # ---- observers on a DeiT-base sized shard (128 samples of [197, 768]) and the headline tensor
    for shape in [(128, 197, 768), (256, 3, 224, 224), (128, 197, 3072)]:
        x = torch.randn(shape, device=dev, generator=g)
        n = x.numel()
        rng = torch.tensor([-5.0, 5.0], device=dev)
        counts = torch.zeros(2048, dtype=torch.int64, device=dev)
        report("observe_hist(2048)", shape, 4 * n, timeit(lambda: ops.hist_update(x.reshape(-1), rng, counts)))
        x2 = x.reshape(1, -1)
        cand_s = (torch.linspace(0.2, 1.0, 80, device=dev) * 0.04).reshape(1, 80).contiguous()
        cand_z = torch.zeros(1, 80, device=dev)
        sse = torch.zeros(1, 80, dtype=torch.float64, device=dev)
        t = timeit(lambda: ops.mse_sweep(x2, cand_s, cand_z, -128, 127, sse), reps=5, warm=2)
        report("observe_mse_sweep(80 cand)", shape, 4 * n, t, f"reference = 80 passes; {80 * n / t / 1e12:.2f} Tcand-elem/s")
        sel = ops.RadixSelect(1, 2, dev, 0)
        for pnum in range(3):
            report(f"select_hist(pass {pnum})", shape, 4 * n, timeit(lambda: sel.hist_pass(pnum, x2, with_counts=True), reps=10, warm=2))
            sel.scan(pnum)

        def full_percentile():
            s2 = ops.RadixSelect(1, 2, dev, 0)
            s2.hist_pass(0, x2, with_counts=True)
            s2.percentile_ranks(torch.tensor([n], device=dev), 1e-3)
            s2.scan(0)
            for pp in (1, 2):
                s2.hist_pass(pp, x2)
                s2.scan(pp)
            return s2.values()

        report("percentile(min+max, exact, 3 passes)", shape, 12 * n, timeit(full_percentile, reps=5, warm=2), "torch.kthvalue x2 in the reference")
        del x

    # ---- sparser: threshold select, mask, mask-apply, fused mask + weight QDQ on the largest R50 weight and all-R50-weights-sized
    for shape in [(512, 512, 3, 3), (2048, 1024, 1, 1), (25_502_912,)]:
        w = torch.randn(shape, device=dev, generator=g) * 0.05
        n = w.numel()
        note = "working set < L2" if n * 9 < (200 << 20) else ""
        k = n // 2
        report("l1_threshold(radix select |w|)", shape, 12 * n, timeit(lambda: ops.kth_value(w.reshape(-1), k, 1), reps=5, warm=2), note + " (torch.sort in the reference)")
        thr = ops.kth_value(w.reshape(-1), k, 1)
        mask = ops.mask_gt(w, thr)
        out = torch.empty_like(w)
        report("mask_gt", shape, 5 * n, timeit(lambda: ops.mask_gt(w, thr)), note)
        report("mask_apply", shape, 9 * n, timeit(lambda: ops.mask_apply(w, mask, out=out)), note)
        if len(shape) > 1:
            c = shape[0]
            sc = torch.rand(c, device=dev) * 0.01 + 0.001
            zc = torch.zeros(c, device=dev)
            report("mask_apply_qdq_perchannel(fused)", shape, 9 * n, timeit(lambda: ops.mask_apply_qdq_perchannel(w, mask, sc, zc, -8, 7, 0, out=out)), note)


if __name__ == "__main__":
    main()
