"""Plain-Python restatement of the launch plan of the attention over an int8 key/value cache
(csrc/int8_attention_cache.cu), in the manner of tests/int8_attention_geometry.py: given a call's shapes and options,
``branches`` names the paths the call reaches, so that the cases of tests/test_gpu_int8_attention_cache_branches.py can
be tied to the branch each exists for and a CPU test can check that together they reach every branch.  When the .cu
file changes, this file has to follow."""
from int8_geometry import cdiv

DEC_ROWS = 16         # kDecRows: Tq <= 16 runs the split-key decode kernels, Tq > 16 the fused kernel
KEYS = 128            # kAtKeys: splits are multiples of 128 keys
MAX_SPLIT = 2048      # kDecMaxSplit
WORK = 4 * 132        # kDecWork
MAX_DIM = 128
MAX_C = 1 << 17

ALL = ("route_decode", "route_fused", "one_split", "two_splits", "many_splits", "split_capped", "tail_1", "tail_127",
       "tail_128", "tail_129", "full_cache", "gl_1", "gl_2", "gl_4", "gl_8", "dv_16", "dv_64", "dv_80", "dv_128",
       "p_unsigned", "p_signed", "zero_point_off_range", "causal_band_rows")


def split(batch, length):
    """dec_split: (keys per split, split count)."""
    want = max(1, cdiv(WORK, batch))
    s = cdiv(cdiv(length, want), KEYS) * KEYS
    s = min(max(s, KEYS), MAX_SPLIT)
    return s, cdiv(length, s)


def lanes_per_key(d):
    """gl of int8_attention_decode_scores_kernel: pow2ceil(dp / 16)."""
    dp = cdiv(d, 16) * 16
    return 1 if dp <= 16 else 2 if dp <= 32 else 4 if dp <= 64 else 8


def branches(batch, tq, capacity, length, d, dv, p_signed=False, zp_off=False, causal=False):
    out = set()
    if tq > DEC_ROWS:
        out.add("route_fused")
    else:
        out.add("route_decode")
        s, ns = split(batch, length)
        out.add("one_split" if ns == 1 else "two_splits" if ns == 2 else "many_splits")
        if s == MAX_SPLIT:
            out.add("split_capped")
        tail = length - (ns - 1) * s  # keys of the last split: a partial 128-key block of 1 or 127 keys, whole blocks,
        if tail == 1:                 # or one key past a whole block
            out.add("tail_1")
        elif tail % KEYS == 127:
            out.add("tail_127")
        elif tail % KEYS == 0:
            out.add("tail_128")
        elif tail % KEYS == 1:
            out.add("tail_129")
        out.add(f"gl_{lanes_per_key(d)}")
        if causal and tq > 1:
            out.add("causal_band_rows")
    if length == capacity:
        out.add("full_cache")
    if dv in (16, 64, 80, 128):
        out.add(f"dv_{dv}")
    out.add("p_signed" if p_signed else "p_unsigned")
    if zp_off:
        out.add("zero_point_off_range")
    return out
