"""Timing and card helpers shared by the benchmark scripts in this directory."""
import subprocess

import torch


def card():
    """The card name, power limit and maximum SM clock, read in the run they describe."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return {"card": name, "power_limit": power, "max_sm_clock": clock}


def set_tf32(on):
    torch.backends.cuda.matmul.allow_tf32 = on
    torch.backends.cudnn.allow_tf32 = on


def timeit(fn, warmup=3, budget_s=0.3, max_iters=200):
    """Mean µs per call of ``fn`` by CUDA events: ``warmup`` calls, one timed call to size the run, then as many calls
    as fit in ``budget_s`` (at least 3, at most ``max_iters``) timed together."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    iters = max(3, min(max_iters, int(budget_s / max(a.elapsed_time(b) * 1e-3, 1e-6))))
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def kernel_times(fn, names, reps=10):
    """Mean device time (µs) per call of ``fn`` spent in each kernel whose name contains one of ``names``
    (torch.profiler)."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for n in names:
            if n in e.key:
                tot = getattr(e, "self_device_time_total", None)
                if tot is None:
                    tot = e.self_cuda_time_total
                out[n] = out.get(n, 0.0) + tot / reps
    return out
