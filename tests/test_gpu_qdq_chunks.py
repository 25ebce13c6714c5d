"""The chunked per-tensor QDQ launch (chunk_kernel in csrc/qdq.cu) behind sb200_qdq_pertensor_fwd and
sb200_qdq_stats_pertensor_fwd: every launch branch, compared bit-exact with oracle.qdq.qdq, and the MinMax state
exact against numpy.

The launch runs one CTA per chunk of K_CHUNK_VECS vectors per thread (4096 floats on the 128-bit path, 1024 on the
scalar path) and puts the n % 4 scalar tail of the 128-bit path in the last chunk.  chunk_launch() below restates
that host formula (launch_chunks in qdq.cu); the CPU test checks that the case table reaches every branch and spot
values of the formula, and every GPU case asserts its branches again with the real device's answer to the
alignment question.

  branch            case (why it gets there)
  v4.single         single_partial: n = 1000, one partial chunk; tiny_tail1: n = 5
  v4.multi          exact_3, plus_vec, tail1..3, multi (several chunks)
  v4.exact          exact_1, exact_3: n a multiple of 4096, every chunk full
  v4.partial_last   plus_vec: n = 4096 + 4 (one vector in the last chunk); minus_vec: 4096 - 4
  v4.tail           tiny_tail1, tail1, tail2, tail3, minus_1, multi (n % 4 = 1, 2, 3)
  v1                x_off1, out_off2, v1_plus1, tiny_n3 (misaligned x or out, or n < 4)
  v1.multi          x_off1, out_off2, v1_plus1
  v1.exact          out_off2: n = 5 * 1024
  v1.partial_last   x_off1, v1_plus1: n = 1024 + 1 at x offset 3

Data: x = (k + f) * s with k past [qmin, qmax], a quarter of the elements at (k + 0.5) * s +- 0..3 ulp (ties for all
three rounding modes), the minimum at the first element and the maximum at the last; 'inf' puts -inf first and +inf
last; 'nan_first' / 'nan_last' put a NaN in the first / last chunk (the last element, in the scalar tail when there
is one).
"""
import zlib

import numpy as np
import pytest
import torch

from gpu_util import bits_equal, dev, on_device
from oracle import qdq as oqdq
from sparsebit_b200 import _lib, ops

F32 = np.float32
K_THREADS = 256   # qdq.cu kThreads
K_CHUNK_VECS = 4  # qdq.cu kChunkVecs
K_TMA_TILE = 4096  # qdq.cu kTmaTile (variant 2 takes the TMA kernel when aligned and n >= 4 tiles)


def chunk_launch(n, x_off=0, out_off=0):
    """launch_chunks (qdq.cu): vector width, grid, vectors in the last chunk, scalar tail.  Offsets in floats from a
    16-byte aligned allocation."""
    vec = x_off % 4 == 0 and out_off % 4 == 0 and n >= 4
    nvec = n >> 2 if vec else n
    per = K_CHUNK_VECS * K_THREADS
    grid = -(-nvec // per)
    return dict(vec=vec, nvec=nvec, grid=grid, last=nvec - (grid - 1) * per, tail=(n & 3) if vec else 0)


def takes_chunks(n, x_off, out_off, variant):
    """use_tma (qdq.cu): only variant 2 with aligned pointers and n >= 4 TMA tiles leaves the chunked launch."""
    return not (variant == 2 and x_off % 4 == 0 and out_off % 4 == 0 and n >= 4 * K_TMA_TILE)


def branches(n, x_off=0, out_off=0):
    g = chunk_launch(n, x_off, out_off)
    v = "v4" if g["vec"] else "v1"
    b = {v, f"{v}.single" if g["grid"] == 1 else f"{v}.multi"}
    b.add(f"{v}.exact" if g["last"] == K_CHUNK_VECS * K_THREADS else f"{v}.partial_last")
    if g["tail"]:
        b.add(f"{v}.tail")
    return b


# name, n, x_off, out_off, variant, targets
CASES = [
    ("single_partial", 1000, 0, 0, 0, {"v4.single", "v4.partial_last"}),
    ("tiny_tail1", 5, 0, 0, 1, {"v4.single", "v4.tail"}),
    ("tiny_n3", 3, 0, 0, 0, {"v1", "v1.single"}),
    ("exact_1", 4096, 0, 0, 0, {"v4.single", "v4.exact"}),
    ("exact_3", 3 * 4096, 0, 0, 2, {"v4.multi", "v4.exact"}),
    ("plus_vec", 4096 + 4, 0, 0, 0, {"v4.multi", "v4.partial_last"}),
    ("minus_vec", 4096 - 4, 0, 0, 1, {"v4.single", "v4.partial_last"}),
    ("minus_1", 4096 - 1, 0, 0, 0, {"v4.tail"}),
    ("tail1", 2 * 4096 + 1, 0, 0, 0, {"v4.multi", "v4.exact", "v4.tail"}),
    ("tail2", 2 * 4096 + 2, 0, 0, 2, {"v4.multi", "v4.tail"}),
    ("tail3", 2 * 4096 + 3, 0, 0, 0, {"v4.multi", "v4.tail"}),
    ("x_off1", 3 * 1024 + 5, 1, 0, 0, {"v1", "v1.multi", "v1.partial_last"}),
    ("out_off2", 5 * 1024, 0, 2, 2, {"v1", "v1.multi", "v1.exact"}),
    ("v1_plus1", 1024 + 1, 3, 3, 0, {"v1.multi", "v1.partial_last"}),
    ("multi", 2_000_003, 0, 0, 1, {"v4.multi", "v4.tail"}),
]
DATA = ("ties", "inf", "nan_first", "nan_last")
REQUIRED = {"v4.single", "v4.multi", "v4.exact", "v4.partial_last", "v4.tail", "v1", "v1.single", "v1.multi", "v1.exact",
            "v1.partial_last"}


def make_x(n, s, z, rng, data, qmin, qmax):
    k = rng.integers(qmin - 8, qmax + 8, n, dtype=np.int32).astype(F32) - np.rint(z)
    x = ((k + rng.uniform(-0.5, 0.5, n).astype(F32)) * s).astype(F32)
    sel = rng.random(n) < 0.25
    xt = ((k[sel] + F32(0.5)) * s).astype(F32)
    d = rng.integers(-3, 4, xt.size, dtype=np.int32)
    d[xt == 0] = 0
    x[sel] = (xt.view(np.int32) + d).view(F32)
    if n > 1:  # the extremes sit at the two ends: the first chunk's first element, the last chunk's (or tail's) last
        lo, hi = x.min(), x.max()
        x[0], x[-1] = lo - F32(1), hi + F32(1)
    if data == "inf":
        x[0], x[-1] = -np.inf, np.inf
    elif data == "nan_first":
        x[min(7, n - 1)] = np.nan
    elif data == "nan_last":
        x[-1] = np.nan
    return x


def empty_at(n, offset):
    return torch.empty(n + offset, dtype=torch.float32, device=dev())[offset:]


def expected_minmax(*xs):
    x = np.concatenate(xs)
    return (F32(np.nan), F32(np.nan)) if np.isnan(x).any() else (x.min(), x.max())


# -------------------------------------------------------------------------------------------------- CPU
def test_cases_reach_every_branch():
    reached = set()
    for name, n, xo, oo, variant, targets in CASES:
        assert takes_chunks(n, xo, oo, variant), name
        got = branches(n, xo, oo)
        assert targets <= got, (name, sorted(got))
        reached |= got
    assert REQUIRED <= reached, sorted(REQUIRED - reached)
    for name, *_ in CASES:
        assert name in __doc__, name


def test_launch_formula_spot_values():
    assert chunk_launch(38_535_168) == dict(vec=True, nvec=9_633_792, grid=9408, last=1024, tail=0)
    assert chunk_launch(205_520_896)["grid"] == 50_176
    assert chunk_launch(4096 + 4) == dict(vec=True, nvec=1025, grid=2, last=1, tail=0)
    assert chunk_launch(2 * 4096 + 3) == dict(vec=True, nvec=2048, grid=2, last=1024, tail=3)
    assert chunk_launch(3) == dict(vec=False, nvec=3, grid=1, last=3, tail=0)
    assert chunk_launch(1025, 3, 3) == dict(vec=False, nvec=1025, grid=2, last=1, tail=0)


# -------------------------------------------------------------------------------------------------- GPU
def _params():
    return [pytest.param(c, d, r, id=f"{c[0]}-{d}-r{r}") for c in CASES for d in DATA for r in (0, 1, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,data,rounding", _params())
def test_chunks_vs_oracle(case, data, rounding):
    name, n, x_off, out_off, variant, targets = case
    assert targets <= branches(n, x_off, out_off) and takes_chunks(n, x_off, out_off, variant)
    qmin, qmax = (-128, 127) if rounding != 1 else (0, 255)
    rng = np.random.default_rng(zlib.crc32(repr((name, data, rounding)).encode()))
    s, z = np.float32([0.0173]), np.float32([2.5])
    x = make_x(n, s[0], z[0], rng, data, qmin, qmax)
    xd, sd, zd = on_device(x, x_off), on_device(s), on_device(z)
    lib = _lib.load()
    assert lib.sb200_set_variant(variant) == 0
    try:
        y = ops.qdq_pertensor(xd, sd, zd, qmin, qmax, rounding, out=empty_at(n, out_off))
        st = ops.minmax_new(1, dev())
        y2 = ops.qdq_stats_pertensor(xd, sd, zd, qmin, qmax, st, rounding, out=empty_at(n, out_off))
        mn, mx = ops.minmax_read(st)
    finally:
        lib.sb200_set_variant(0)
    exp = oqdq.qdq(x, s, z, qmin, qmax, 0, rounding)
    got = y.cpu().numpy()
    if not bits_equal(got, exp):
        bad = np.flatnonzero(~((got == exp) | (np.isnan(got) & np.isnan(exp))))
        i = bad[0]
        raise AssertionError(f"{name} {data} r{rounding}: {bad.size} of {n} differ; first at {i}: x={x[i]!r} "
                             f"got={got[i]!r} expected={exp[i]!r}")
    assert bits_equal(y2.cpu().numpy(), got)
    assert bits_equal(np.float32([float(mn), float(mx)]), np.float32(expected_minmax(x)))


@pytest.mark.gpu
@pytest.mark.parametrize("nan", [False, True])
def test_stats_accumulate_across_calls(nan):
    """The state is a running min / max: a second call folds into what the first left."""
    rng = np.random.default_rng(7)
    s, z = np.float32([0.02]), np.float32([0.0])
    a = make_x(3 * 4096 + 1, s[0], z[0], rng, "ties", 0, 255)
    b = make_x(4096 + 4, s[0], z[0], rng, "nan_last" if nan else "ties", 0, 255)
    b[0] = a.min() - F32(3)  # the second call lowers the minimum
    st = ops.minmax_new(1, dev())
    sd, zd = on_device(s), on_device(z)
    for x in (a, b):
        ops.qdq_stats_pertensor(on_device(x), sd, zd, 0, 255, st)
    mn, mx = ops.minmax_read(st)
    assert bits_equal(np.float32([float(mn), float(mx)]), np.float32(expected_minmax(a, b)))


@pytest.mark.gpu
def test_variants_agree_and_graph_replays():
    """Variants 0, 1 (chunks) and 2 (TMA at this size) give the same bits; a captured graph of the chunked launch gives
    them again on every replay, including two replays queued back to back."""
    n = 1_000_003
    rng = np.random.default_rng(11)
    s, z = np.float32([0.013]), np.float32([-3.0])
    x = make_x(n, s[0], z[0], rng, "ties", -128, 127)
    xd, sd, zd = on_device(x), on_device(s), on_device(z)
    lib = _lib.load()
    outs = []
    for variant in (0, 1, 2):
        lib.sb200_set_variant(variant)
        try:
            st = ops.minmax_new(1, dev())
            outs.append((ops.qdq_stats_pertensor(xd, sd, zd, -128, 127, st).cpu().numpy(), ops.minmax_read(st)))
        finally:
            lib.sb200_set_variant(0)
    exp = oqdq.qdq(x, s, z, -128, 127, 0, 0)
    emm = np.float32(expected_minmax(x))
    for y, (mn, mx) in outs:
        assert bits_equal(y, exp)
        assert bits_equal(np.float32([float(mn), float(mx)]), emm)

    y = torch.empty_like(xd)
    st = torch.empty(2, dtype=torch.int32, device=dev())
    side = torch.cuda.Stream(device=dev())
    g = torch.cuda.CUDAGraph()

    def enqueue(stream):
        _lib.check(lib.sb200_minmax_init(st.data_ptr(), 1, stream), "minmax_init")
        _lib.check(lib.sb200_qdq_stats_pertensor_fwd(xd.data_ptr(), sd.data_ptr(), zd.data_ptr(), y.data_ptr(), st.data_ptr(),
                                                     n, -128, 127, 0, stream), "qdq_stats")

    with torch.cuda.stream(side):
        enqueue(side.cuda_stream)
        side.synchronize()
        with torch.cuda.graph(g, stream=side):
            enqueue(torch.cuda.current_stream(dev()).cuda_stream)
    for _ in range(2):
        y.zero_()
        g.replay()
        g.replay()
        torch.cuda.synchronize()
        assert bits_equal(y.cpu().numpy(), exp)
        mn, mx = ops.minmax_read(st)
        assert bits_equal(np.float32([float(mn), float(mx)]), emm)
