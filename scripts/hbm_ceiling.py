"""HBM ceiling on this card next to the per-tensor fake-quant kernels, at every activation-site size of the bench.

For each distinct element count of the 55 ResNet-50 activation sites at batch 256 (bench.r50_activation_sites), plus
the [256,3,224,224] input, it times five arms on 16-byte aligned fp32 buffers:

    copy        y.copy_(x)                                device-to-device copy, 8 B/elem
    write       y.zero_()                                 4 B/elem
    read        sb200_observe_minmax                      4 B/elem
    qdq_v1      sb200_qdq_stats_pertensor_fwd, variant 1  8 B/elem (fused QDQ + MinMax, the bench's activation kernel)
    qdq_v2      sb200_qdq_stats_pertensor_fwd, variant 2  8 B/elem (TMA ring where it applies)

Every site has its own input and output, as in the bench; below 256 MB the launches rotate over several buffer pairs
so that the working set exceeds the 50 MB L2 and the numbers are HBM numbers.  Each measurement is one CUDA graph
of 30 back-to-back launches timed with CUDA events, after warm-up; the arms are interleaved and every round is
repeated 3 times (the median is reported, with the spread).

Prints one JSON line per (size, arm), then one line with the card, its power limit, clocks.max.sm and the SM
clock sampled during the run.

    python scripts/hbm_ceiling.py [--reps 30] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from bench import ClockSampler, numel, r50_activation_sites  # noqa: E402
from sparsebit_b200 import _lib  # noqa: E402

DATASHEET_GBS = 3350.0  # H100 SXM data sheet, HBM3
ROTATE_BYTES = 256 << 20  # input + output bytes rotated over per size, about 5x the L2
ARMS = ("copy", "write", "read", "qdq_v1", "qdq_v2")
BYTES_PER_ELEM = {"copy": 8, "write": 4, "read": 4, "qdq_v1": 8, "qdq_v2": 8}


def card_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clk = [f.strip() for f in q.stdout.strip().split(",")]
    return {"card": name, "power_limit_w": float(power), "clocks_max_sm_mhz": float(clk)}


def site_sizes():
    sizes = sorted({numel(shape) for shape, _ in r50_activation_sites(256)}, reverse=True)
    assert numel((256, 3, 224, 224)) in sizes
    return sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30, help="launches per timed graph")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hbm_ceiling.py needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    lib = _lib.load()
    side = torch.cuda.Stream(device=dev)
    g = torch.Generator(device=dev).manual_seed(0)

    # graphs[(n, arm)] replays `reps` launches of that arm, rotating over the size's buffer pairs
    graphs = {}
    keep = []
    for n in site_sizes():
        pairs = max(1, -(-ROTATE_BYTES // (8 * n)))
        bufs = []
        for _ in range(pairs):
            x = torch.randn(n, device=dev, generator=g).relu_()
            bufs.append((x, torch.empty_like(x)))
        s = ((x.max() / 255.0).clamp(min=1e-6)).reshape(1)
        z = torch.zeros(1, device=dev)
        mm = torch.empty(2, dtype=torch.int32, device=dev)
        keep += [bufs, s, z, mm]

        def launch(arm, i, st, n=n, bufs=bufs, s=s, z=z, mm=mm):
            x, y = bufs[i % len(bufs)]
            if arm == "copy":
                y.copy_(x)
            elif arm == "write":
                y.zero_()
            elif arm == "read":
                _lib.check(lib.sb200_observe_minmax(x.data_ptr(), n, mm.data_ptr(), st), "observe_minmax")
            else:
                _lib.check(lib.sb200_qdq_stats_pertensor_fwd(x.data_ptr(), s.data_ptr(), z.data_ptr(), y.data_ptr(),
                                                             mm.data_ptr(), n, 0, 255, 0, st), "qdq_stats")

        for arm in ARMS:
            # the variant is read at launch time by the host dispatcher, so it is fixed into the captured graph
            lib.sb200_set_variant({"qdq_v1": 1, "qdq_v2": 2}.get(arm, 0))
            with torch.cuda.stream(side):
                for i in range(len(bufs)):  # eager warm-up of every buffer pair
                    launch(arm, i, side.cuda_stream)
                side.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr, stream=side):
                    for i in range(args.reps):
                        launch(arm, i, torch.cuda.current_stream(dev).cuda_stream)
            graphs[(n, arm)] = gr
        lib.sb200_set_variant(0)
    torch.cuda.synchronize()

    info = card_info()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    times = {k: [] for k in graphs}
    for gr in graphs.values():  # warm-up replay of every graph
        gr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for n in site_sizes():
            for arm in ARMS:  # arms interleaved within each round
                e0.record()
                graphs[(n, arm)].replay()
                e1.record()
                e1.synchronize()
                times[(n, arm)].append(e0.elapsed_time(e1) * 1e3 / args.reps)
    clocks = sampler.stop()

    for n in site_sizes():
        copy_gbs = n * BYTES_PER_ELEM["copy"] / statistics.median(times[(n, "copy")]) / 1e3
        for arm in ARMS:
            t = times[(n, arm)]
            us = statistics.median(t)
            gbs = n * BYTES_PER_ELEM[arm] / us / 1e3
            print(json.dumps({"elems": n, "arm": arm, "us": round(us, 2), "us_min": round(min(t), 2), "us_max": round(max(t), 2),
                              "GB/s": round(gbs, 1), "frac_datasheet": round(gbs / DATASHEET_GBS, 4),
                              "frac_copy": round(gbs / copy_gbs, 4), "bytes_per_elem": BYTES_PER_ELEM[arm]}), flush=True)
    print(json.dumps({**info, "clocks_during_run": clocks, "reps": args.reps, "rounds": args.rounds,
                      "datasheet_GB/s": DATASHEET_GBS}), flush=True)


if __name__ == "__main__":
    main()
