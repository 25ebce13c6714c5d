"""GPU parity: GPTQ int4 dequant-matmul through the ``cuda_kernel`` mirror / QuantLinear vs the
reference's known-answer construction (test_cuda_kernel.py: rtol = atol = 1e-5 against
Linear(dequantised W), fp32, TF32 off) and the fp64 oracle."""
import numpy as np
import pytest
import torch

from gpu_util import dev, t
from oracle import gptq as ogptq
from sparsebit_b200 import _lib
from sparsebit_b200.gptq import QuantLinear, cuda_kernel, find_params_int4

pytestmark = pytest.mark.gpu
TOL = dict(rtol=1e-5, atol=1e-5)  # test_cuda_kernel.py:47


def _run(x, qw, bias, scales, zeros, gs):
    y = t(np.broadcast_to(bias, x.shape[:-1] + (qw.shape[1],)).copy())
    if gs == -1:
        cuda_kernel.vecquant4matmul(t(x), t(qw), y, t(scales), t(zeros))
    else:
        cuda_kernel.vecgroupquant4matmul(t(x), t(qw), y, t(scales), t(zeros), gs)
    return y.cpu().numpy()


@pytest.mark.parametrize("impl", [1, 0, 4])  # small-M path (HMMA streaming kernel where N % 4 == 0), auto, scalar kernel
def test_golden_known_answers(golden, impl):
    g = golden("gptq")
    _lib.load().sb200_gptq4_set_impl(impl)
    try:
        for name in g["cases"]:
            gs = int(g[name + "_gs"])
            y = _run(g[name + "_x"], g[name + "_qweight"], g[name + "_bias"], g[name + "_scales"], g[name + "_zeros"], gs)
            np.testing.assert_allclose(y, g[name + "_gt"], err_msg=name, **TOL)
    finally:
        _lib.load().sb200_gptq4_set_impl(0)


def _make_case(rng, bshape, k, n, gs):
    w = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
    scale, zero = ogptq.find_params_int4(w, gs)
    wq = ogptq.quantize_weight(w, scale, zero, gs)
    qw, scales, zeros = ogptq.pack_int4(wq, scale, zero)
    x = rng.standard_normal(bshape + (k,)).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32) * 0.1
    return x, qw, bias, scales, zeros


# shapes of test_cuda_kernel.py:50-126 that fit the time budget (irregular sizes, multi-batch, 3-D
# inputs, GS = 128 / 384), plus the LLaMA-7B linear shapes at decode and prefill-tile M.
CASES = [
    ((1,), 128, 64, -1), ((1,), 127, 61, -1), ((1,), 6661, 2516, -1), ((31,), 6661, 2516, -1),
    ((32, 1), 1024, 1031, -1), ((4, 8), 6661, 512, -1), ((29,), 8192, 1024, 128), ((4,), 6144, 768, 384),
    ((1,), 4096, 4096, 128), ((1,), 4096, 11008, 128), ((1,), 11008, 4096, 128), ((16,), 4096, 4096, 128),
    ((256,), 4096, 4096, 128), ((300,), 1024, 512, 128), ((2, 130), 512, 264, 128),
]


@pytest.mark.parametrize("impl", [0, 4])
@pytest.mark.parametrize("bshape,k,n,gs", CASES)
def test_vs_fp64_oracle(bshape, k, n, gs, impl):
    rng = np.random.default_rng(k + n + len(bshape))
    x, qw, bias, scales, zeros = _make_case(rng, bshape, k, n, gs)
    y = _run_impl(x, qw, bias, scales, zeros, gs, impl=impl)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, x.shape[:-1] + (n,)), scales, zeros, 0 if gs == -1 else gs)
    np.testing.assert_allclose(y, exp, **TOL)


# per-group wgmma path forced (sb200_gptq4_set_impl(2)): ragged M / N tiles, odd number of 64-K stages,
# group sizes 128 / 256 / 384, a single row, outlier activations (per-row power-of-two scaling).
TC_CASES = [
    ((1,), 128, 128, 128), ((128,), 256, 128, 128), ((130,), 512, 264, 128), ((29,), 8192, 1024, 128),
    ((4,), 6144, 768, 384), ((300,), 1024, 512, 256), ((2, 130), 512, 260, 128), ((257,), 192 * 2, 132, 128),
    ((256,), 4096, 4096, 128), ((64,), 11008, 512, 128),
]


@pytest.mark.parametrize("bshape,k,n,gs", TC_CASES)
def test_tcgen05_path_vs_fp64_oracle(bshape, k, n, gs):
    rng = np.random.default_rng(7 * k + n + len(bshape))
    x, qw, bias, scales, zeros = _make_case(rng, bshape, k, n, gs)
    xf = x.reshape(-1, k)
    xf[0, :5] = [3e4, -7e4, 1e-6, 0.0, 123.0]  # fp16-overflowing magnitudes are fine after row scaling
    if xf.shape[0] > 2:
        xf[2] *= 1e-4
    lib = _lib.load()
    assert lib.sb200_gptq4_set_impl(2) == 0
    try:
        y = _run(x, qw, bias, scales, zeros, gs)
    finally:
        lib.sb200_gptq4_set_impl(0)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, x.shape[:-1] + (n,)), scales, zeros, gs)
    yf, ef = y.reshape(-1, n), exp.reshape(-1, n)
    # every ordinary row: the reference's own elementwise form, atol + rtol * |expected| (test_cuda_kernel.py:47)
    plain = [r for r in range(yf.shape[0]) if r not in (0, 2)]
    if plain:
        np.testing.assert_allclose(yf[plain], ef[plain], **TOL)
    # the two rows with injected outliers (|x| up to 7e4 next to 1e-6): an fp32 result cannot meet an elementwise
    # bound against the fp64 oracle where the large terms cancel, so these rows are bounded by the row magnitude
    for r in (0, 2):
        if r < yf.shape[0]:
            mag = max(np.abs(ef[r]).max(), 1.0)
            np.testing.assert_array_less(np.abs(yf[r] - ef[r]), 1e-5 + 1e-5 * mag)


def _run_impl(x, qw, bias, scales, zeros, gs, impl, chunk_k=0):
    from sparsebit_b200 import ops

    y = t(np.broadcast_to(bias, x.shape[:-1] + (qw.shape[1],)).copy())
    ops.gptq4_matmul(t(x), t(qw), y, t(scales), t(zeros), 0 if gs == -1 else gs, impl=impl, chunk_k=chunk_k)
    return y.cpu().numpy()


# warp-level HMMA streaming kernel (impl 1 with N % 4 == 0, gptq_decode.cu): 1 / 8 / 9 / 16 / 17 / 32 / 33 / 70 tokens (the
# three token-block variants and the multi-pass loop), K not a multiple of 128 or 32, ragged feature blocks, fp32 and
# fp16-exact activations, outliers, non-integer zero points
DECODE_CASES = [(1, 4096, 4096, 128), (8, 1024, 512, 128), (9, 1024, 260, 128), (16, 2048, 1028, 256), (17, 512, 132, 128),
                (32, 1536, 384, 384), (33, 1000, 256, -1), (70, 328, 64, -1), (1, 11008, 4096, 128), (5, 6656, 2516, -1)]


@pytest.fixture
def decode_mode():
    """sb200_gptq4_set_decode is process-wide: restore the default (6 = programmatic dependent launch + L2 prefetch) afterwards.
    Bits: 1 bulk-copy weight slab, 2 programmatic launch, 4 L2 prefetch of the later K blocks, 8 every call counts as
    SB200_GPTQ4_STATIC_WEIGHTS (weights requested before griddepcontrol.wait), high nibble CTAs per SM."""
    from sparsebit_b200 import _lib

    lib = _lib.load()
    yield lambda mode: _lib.check(lib.sb200_gptq4_set_decode(mode))
    _lib.check(lib.sb200_gptq4_set_decode(6))


@pytest.mark.parametrize("m,k,n,gs", DECODE_CASES)
@pytest.mark.parametrize("fp16_acts", [False, True])
@pytest.mark.parametrize("mode", [6, 14, 11, 0x82])  # default; + static weights; slab variant; 8 CTAs per SM, no prefetch
def test_decode_hmma_path_vs_fp64_oracle(m, k, n, gs, fp16_acts, mode, decode_mode):
    decode_mode(mode)
    rng = np.random.default_rng(13 * k + n + m)
    x, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, gs)
    if fp16_acts:
        x = x.astype(np.float16).astype(np.float32)
    else:
        x[0, :3] = [2.5e4, -6e4, 1e-7]  # per-token power-of-two scaling
    if m > 1:
        zeros = (zeros + 0.21 * scales).astype(np.float32)  # fractional zero points: the affine part is applied in fp32
    y = _run_impl(x, qw, bias, scales, zeros, gs, impl=1)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (m, n)), scales, zeros, 0 if gs == -1 else gs)
    rows = list(range(1, m)) if not fp16_acts else list(range(m))
    if rows:
        np.testing.assert_allclose(y[rows], exp[rows], **TOL)
    if not fp16_acts:  # the outlier row: bounded by the row magnitude (an fp32 result cannot do better)
        np.testing.assert_array_less(np.abs(y[0] - exp[0]), 1e-5 + 1e-5 * max(1.0, np.abs(exp[0]).max()))


# weight-plane wgmma kernel (impl 3, gptq_ts.cu): ragged token / feature tiles, odd numbers of 64-K stages,
# several chunks, group sizes 128 / 256 / 384, a single row, several 128-token tiles and ragged last tiles
TS_CASES = [
    ((1,), 128, 128, 128), ((128,), 256, 128, 128), ((130,), 512, 264, 128), ((29,), 8192, 1024, 128),
    ((4,), 6144, 768, 384), ((300,), 1024, 512, 256), ((2, 130), 512, 260, 128), ((257,), 192 * 2, 132, 128),
    ((256,), 4096, 4096, 128), ((64,), 11008, 512, 128), ((513,), 384, 392, -1), ((700,), 2048, 136, 128),
]


@pytest.mark.parametrize("bshape,k,n,gs", TS_CASES)
def test_tcgen05_ts_path_vs_fp64_oracle(bshape, k, n, gs):
    rng = np.random.default_rng(11 * k + n + len(bshape))
    x, qw, bias, scales, zeros = _make_case(rng, bshape, k, n, gs)
    y = _run_impl(x, qw, bias, scales, zeros, gs, impl=3)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, x.shape[:-1] + (n,)), scales, zeros, 0 if gs == -1 else gs)
    np.testing.assert_allclose(y, exp, **TOL)  # the reference's elementwise form (test_cuda_kernel.py:47)


def test_tcgen05_ts_outlier_rows_and_fp16_exact_activations():
    rng = np.random.default_rng(3)
    m, k, n = 300, 1024, 520
    x, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, 128)
    x[0, :5] = [3e4, -7e4, 1e-6, 0.0, 123.0]  # fp16-overflowing magnitudes: per-row power-of-two scaling
    x[2] *= 1e-4
    y = _run_impl(x, qw, bias, scales, zeros, 128, impl=3)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (m, n)), scales, zeros, 128)
    plain = [r for r in range(m) if r != 0]
    np.testing.assert_allclose(y[plain], exp[plain], **TOL)
    np.testing.assert_array_less(np.abs(y[0] - exp[0]), 1e-5 + 1e-5 * np.abs(exp[0]).max())
    # fp16 activations cast to fp32 (the model path): the x_lo pass is skipped, rows are bit-identical to the
    # three-pass result on the same data
    xh = x.astype(np.float16).astype(np.float32)
    xh[0, :2] = 1.0
    y1 = _run_impl(xh, qw, bias, scales, zeros, 128, impl=3)
    x2 = xh.copy()
    x2[0, 0] += 1e-5
    y2 = _run_impl(x2, qw, bias, scales, zeros, 128, impl=3)
    np.testing.assert_allclose(y1, ogptq.dequant_matmul(xh, qw, np.broadcast_to(bias, (m, n)), scales, zeros, 128), **TOL)
    np.testing.assert_allclose(y2[1:], y1[1:], rtol=0, atol=0)


def test_tcgen05_ts_general_zero_points_and_chunking():
    rng = np.random.default_rng(5)
    x, qw, bias, scales, zeros = _make_case(rng, (200,), 1024, 384, 128)
    exp_int = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (200, 384)), scales, zeros, 128)
    for chunk in (64, 256, 512, 4096):  # accumulator drained every 1 / 4 / 8 stages, or once
        np.testing.assert_allclose(_run_impl(x, qw, bias, scales, zeros, 128, impl=3, chunk_k=chunk), exp_int, **TOL)
    # zeros that are NOT an integer multiple of scales: the prepare kernel clears the flag, the epilogue subtracts
    # zeros * (row sums of x)
    zeros2 = (zeros + 0.37 * scales * rng.uniform(0.5, 1.5, zeros.shape)).astype(np.float32)
    zeros2[3, 2] = 0.0
    y = _run_impl(x, qw, bias, scales, zeros2, 128, impl=3)
    np.testing.assert_allclose(y, ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (200, 384)), scales, zeros2, 128), **TOL)
    # integer zero points far outside [0, 15] (the contract allows any fp32 zeros)
    zeros3 = (scales * np.rint(rng.uniform(-900, 900, zeros.shape))).astype(np.float32)
    y = _run_impl(x, qw, bias, scales, zeros3, 128, impl=3)
    exp3 = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (200, 384)), scales, zeros3, 128)
    np.testing.assert_allclose(y, exp3, rtol=1e-5, atol=1e-5 * max(1.0, np.abs(exp3).max()))


@pytest.mark.parametrize("m,k,n", [(256, 1024, 512), (77, 512, 132)])
def test_tcgen05_fp16_representable_activations_single_pass(m, k, n):
    """fp16 activations cast to fp32 (the reference's model path): lo == 0 everywhere, the kernel skips the
    second MMA pass -- result must still match the oracle, and equal the 2-pass result on the same data."""
    rng = np.random.default_rng(m + k)
    x, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, 128)
    x = x.astype(np.float16).astype(np.float32)
    lib = _lib.load()
    lib.sb200_gptq4_set_impl(2)
    try:
        y = _run(x, qw, bias, scales, zeros, 128)
        x2 = x.copy()
        x2[0, 0] += 1e-5  # one element with a non-zero low part forces the 2-pass path
        y2 = _run(x2, qw, bias, scales, zeros, 128)
    finally:
        lib.sb200_gptq4_set_impl(0)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (m, n)), scales, zeros, 128)
    np.testing.assert_allclose(y, exp, **TOL)
    np.testing.assert_allclose(y2[1:], y[1:], rtol=0, atol=0)  # rows without the perturbation: bit-identical


def test_tcgen05_general_zero_points_fall_back_to_affine_epilogue():
    """zeros that are NOT an integer multiple of scales (the contract allows any fp32 value): the
    device-side probe must clear the integer-zero flag and the (scale, zeros) epilogue must be used."""
    rng = np.random.default_rng(5)
    x, qw, bias, scales, zeros = _make_case(rng, (200,), 1024, 384, 128)
    zeros = (zeros + 0.37 * scales * rng.uniform(0.5, 1.5, zeros.shape)).astype(np.float32)
    zeros[3, 2] = 0.0
    lib = _lib.load()
    lib.sb200_gptq4_set_impl(2)
    try:
        y = _run(x, qw, bias, scales, zeros, 128)
    finally:
        lib.sb200_gptq4_set_impl(0)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (200, 384)), scales, zeros, 128)
    np.testing.assert_allclose(y, exp, **TOL)


@pytest.mark.parametrize("m,k,n,gs", [(5, 1024, 512, 128), (300, 1024, 520, 128), (1024, 2048, 1028, 256), (777, 512, 260, -1)])
def test_linear_f16_entry_point(m, k, n, gs):
    """sb200_gptq4_linear_f16: fp16 activations in, fp16 ``bias + x @ W`` out without eager casts -- equals the fp32
    entry point's result rounded to fp16 (up to one fp16 ulp where the fp32 results differ in the last bits)."""
    from sparsebit_b200 import ops

    rng = np.random.default_rng(m + k)
    x, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, gs)
    xh = x.astype(np.float16)
    g = 0 if gs == -1 else gs
    y16 = ops.gptq4_linear_f16(t(xh), t(qw), t(scales), t(zeros), t(bias), g).cpu().numpy()
    assert y16.dtype == np.float16 and y16.shape == (m, n)
    exp = ogptq.dequant_matmul(xh.astype(np.float32), qw, np.broadcast_to(bias, (m, n)), scales, zeros, g)
    ulp = np.abs(exp).astype(np.float16).astype(np.float32) * 2.0**-10 + 2.0**-24
    assert np.all(np.abs(y16.astype(np.float64) - exp) <= 0.51 * ulp + 1e-5 * (1 + np.abs(exp)))
    y_nobias = ops.gptq4_linear_f16(t(xh), t(qw), t(scales), t(zeros), None, g).cpu().numpy().astype(np.float32)
    np.testing.assert_allclose(y_nobias, exp - bias, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("m,k,n,gs", [(1, 4096, 4096, 128), (1, 1000, 132, -1), (9, 1024, 520, 128), (17, 2048, 1028, 256), (32, 1536, 384, 384)])
def test_linear_f16_decode_sized_is_one_launch(m, k, n, gs):
    """sb200_gptq4_linear_f16_ex with a counter state: fp16 in -> ONE decode-kernel launch -> fp16 bias + x @ W out (the
    last K-slice CTA of every feature block adds the slices' partial sums in slice order).  Repeated calls on the same
    state (the counters reset themselves), equal to the staged four-launch path up to fp32 summation order, and
    bit-identical run to run."""
    from sparsebit_b200 import launch_count, ops

    rng = np.random.default_rng(3 * m + k + n)
    x, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, gs)
    xh = x.astype(np.float16)
    g = 0 if gs == -1 else gs
    args = (t(xh), t(qw), t(scales), t(zeros), t(bias), g)
    before = launch_count()
    y_a = ops.gptq4_linear_f16(*args)
    assert launch_count() - before == 1
    y_b = ops.gptq4_linear_f16(*args, static_weights=True)  # second call on the same state; weights requested before the wait
    y_c = ops.gptq4_linear_f16(*args)
    before = launch_count()
    y_staged = ops.gptq4_linear_f16(*args, single_launch=False)
    assert launch_count() - before >= 4  # cast, bias, kernel(s), cast (M = 32 runs the per-group wgmma kernel: two more)
    a = y_a.cpu().numpy()
    assert a.dtype == np.float16 and a.shape == (m, n)
    assert np.array_equal(a, y_b.cpu().numpy()) and np.array_equal(a, y_c.cpu().numpy())  # fixed summation order
    exp = ogptq.dequant_matmul(xh.astype(np.float32), qw, np.broadcast_to(bias, (m, n)), scales, zeros, g)
    ulp = np.abs(exp).astype(np.float16).astype(np.float32) * 2.0**-10 + 2.0**-24
    assert np.all(np.abs(a.astype(np.float64) - exp) <= 0.51 * ulp + 1e-5 * (1 + np.abs(exp)))
    assert np.all(np.abs(y_staged.cpu().numpy().astype(np.float64) - exp) <= 0.51 * ulp + 1e-5 * (1 + np.abs(exp)))
    y_nobias = ops.gptq4_linear_f16(t(xh), t(qw), t(scales), t(zeros), None, g).cpu().numpy().astype(np.float32)
    np.testing.assert_allclose(y_nobias, exp - bias, rtol=2e-3, atol=2e-3)


def test_linear_f16_single_launch_inside_a_cuda_graph():
    """Three dependent fp16 linears (each consumes its predecessor's fp16 output) captured into one CUDA graph and
    replayed: the self-resetting counters and the programmatic launches must survive replays."""
    from sparsebit_b200 import ops

    rng = np.random.default_rng(11)
    dims = [(1024, 768), (768, 1536), (1536, 256)]
    m = 2
    layers = []
    for k, n in dims:
        _, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, 128)
        layers.append((t(qw), t(scales), t(zeros), t(bias), qw, scales, zeros, bias))
    x = rng.standard_normal((m, dims[0][0])).astype(np.float16)
    xt = t(x)

    def chain():
        cur = xt
        for qw, sc, zr, bs, *_ in layers:
            cur = ops.gptq4_linear_f16(cur, qw, sc, zr, bs, 128, static_weights=True)
        return cur

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
        s.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            out = chain()
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    exp = x.astype(np.float32)
    for *_, qw, scales, zeros, bias in layers:
        exp = ogptq.dequant_matmul(exp, qw, np.broadcast_to(bias, (m, qw.shape[1])), scales, zeros, 128).astype(np.float16).astype(np.float32)
    np.testing.assert_allclose(out.cpu().numpy().astype(np.float32), exp, rtol=4e-3, atol=4e-3 * np.abs(exp).max())


def test_tcgen05_forced_on_unsupported_shape_is_an_error():
    lib = _lib.load()
    rng = np.random.default_rng(1)
    x, qw, bias, scales, zeros = _make_case(rng, (4,), 127, 61, -1)
    lib.sb200_gptq4_set_impl(2)
    try:
        with pytest.raises(RuntimeError, match="unsupported"):
            _run(x, qw, bias, scales, zeros, -1)
    finally:
        lib.sb200_gptq4_set_impl(0)


def test_quant_linear_module_matches_dense_linear():
    torch.backends.cuda.matmul.allow_tf32 = False
    for (b, k, n, gs) in [(3, 256, 96, -1), (29, 1024, 200, 128)]:
        layer = torch.nn.Linear(k, n)
        scale, zero = find_params_int4(layer.weight.data, gs)
        wq = ogptq.quantize_weight(layer.weight.data.numpy(), scale.reshape(n, -1).numpy(), zero.reshape(n, -1).numpy(), gs)
        layer.weight.data = torch.from_numpy(wq)
        ql = QuantLinear(k, n, 4, gs)
        ql.pack(layer, scale, zero)
        x = torch.randn(b, k)
        gt = layer.to(dev())(x.to(dev()))
        torch.testing.assert_close(ql.to(dev())(x.to(dev())), gt, **TOL)
        with torch.no_grad():
            yh = ql(x.to(dev()).half())  # fp16 model path: sb200_gptq4_linear_f16, no casts
        assert yh.dtype == torch.float16
        torch.testing.assert_close(yh.float(), layer(x.to(dev()).half().float()), rtol=2e-3, atol=2e-3)


def test_linearity_and_accumulate_contract_at_llama_shape():
    """Full L7B down_proj shape, M = 2048: properties instead of a CPU recompute -- the kernel
    ACCUMULATES into out (bias contract), and is linear in x."""
    rng = np.random.default_rng(0)
    k, n, m = 11008, 4096, 2048
    x, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, 128)
    y1 = _run(x, qw, bias, scales, zeros, 128)
    y0 = _run(np.zeros_like(x), qw, bias, scales, zeros, 128)
    np.testing.assert_allclose(y0, np.broadcast_to(bias, (m, n)), rtol=0, atol=1e-6)
    y2 = _run(2 * x, qw, np.zeros(n, np.float32), scales, zeros, 128)
    np.testing.assert_allclose(y2, 2 * (y1 - bias), rtol=2e-5, atol=2e-5)
    rows = [0, 255, 256, 777, 2047]
    exp = ogptq.dequant_matmul(x[rows], qw, np.broadcast_to(bias, (len(rows), n)), scales, zeros, 128)
    np.testing.assert_allclose(y1[rows], exp, **TOL)
    for impl in (2, 3):  # both wgmma kernels at the full shape
        np.testing.assert_allclose(_run_impl(x, qw, bias, scales, zeros, 128, impl=impl)[rows], exp, **TOL)


def test_argument_checks():
    x = torch.randn(4, 256, device=dev())
    qw = torch.zeros(32, 8, dtype=torch.int32, device=dev())
    y = torch.zeros(4, 8, device=dev())
    s = torch.ones(8, 2, device=dev())
    with pytest.raises(RuntimeError, match="divisible by 128"):
        cuda_kernel.vecgroupquant4matmul(x, qw, y, s, s, 64)
    with pytest.raises(RuntimeError, match="dimension >= 2"):
        cuda_kernel.vecquant4matmul(x[0, :], qw, y[0], s, s)
    with pytest.raises(RuntimeError, match="out_channel"):
        cuda_kernel.vecquant4matmul(x, qw, torch.zeros(4, 9, device=dev()), s, s)


def test_layer_streaming_equals_resident_execution():
    """LayerStreamer (the reference's single_device_mode, llama_wrapper.py:848-924): packed weights stream from pinned host
    memory into two device slots, one layer ahead of the compute; outputs equal the fully resident model and only two layers' worth of packed weights are on the device."""
    from sparsebit_b200.gptq import LayerStreamer

    torch.manual_seed(0)

    class Block(torch.nn.Module):
        def __init__(self, k, h):
            super().__init__()
            self.up, self.down = QuantLinear(k, h, 4, 128), QuantLinear(h, k, 4, 128)
            for ql, (i, o) in ((self.up, (k, h)), (self.down, (h, k))):
                lin = torch.nn.Linear(i, o)
                s, z = find_params_int4(lin.weight.data, 128)
                ql.pack(lin, s, z)

        def forward(self, x):
            return x + self.down(torch.relu(self.up(x)))

    blocks = [Block(256, 512) for _ in range(5)]
    x = torch.randn(7, 256, device=dev())
    import copy

    resident = [copy.deepcopy(b).to(dev()) for b in blocks]
    with torch.no_grad():
        ref = x
        for b in resident:
            ref = b(ref)
        streamer = LayerStreamer(blocks, dev())
        out1 = streamer(x)
        out2 = streamer(x)  # slots are reused across forwards
    # (split-K partial sums meet in fp32 atomics: equal up to the summation order)
    torch.testing.assert_close(out1, ref, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(out2, ref, rtol=1e-5, atol=1e-5)
    per_layer = sum(m.qweight.numel() for m in resident[0].modules() if isinstance(m, QuantLinear)) * 4
    assert streamer.resident_bytes() == 2 * per_layer
    assert all(m.qweight.numel() == 0 for b in blocks for m in b.modules() if isinstance(m, QuantLinear))


@pytest.mark.parametrize("mode", [6, 14, 11, 0])
@pytest.mark.parametrize("graph", [False, True])
def test_decode_chain_of_dependent_linears_under_programmatic_launch(mode, graph, decode_mode):
    """y1 = W1 x, y2 = W2 y1, y3 = W3 y2 launched back to back on one stream: with programmatic dependent launch a
    kernel may start (and fetch its weights) before its predecessor has finished, and must still see the predecessor's
    complete output (griddepcontrol.wait in front of the activation staging).  Also as a captured CUDA graph."""
    from sparsebit_b200 import ops

    decode_mode(mode)
    rng = np.random.default_rng(5)
    dims = [(1024, 768), (768, 1536), (1536, 256)]
    m = 3
    layers = []
    for k, n in dims:
        _, qw, _, scales, zeros = _make_case(rng, (m,), k, n, 128)
        layers.append((t(qw), t(scales), t(zeros), qw, scales, zeros))
    x = rng.standard_normal((m, dims[0][0])).astype(np.float32)
    ys = [torch.zeros(m, n, device=dev()) for _, n in dims]

    def chain(xin):
        for y in ys:
            y.zero_()
        cur = xin
        for (qw, sc, zr, *_), y in zip(layers, ys):  # three decode kernels back to back, each reading its predecessor's out
            ops.gptq4_matmul(cur, qw, y, sc, zr, 128, impl=1, static_weights=(mode == 6 and graph))  # also the per-call flag
            cur = y

    xt = t(x)
    if graph:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain(xt)  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            chain(xt)
        for _ in range(3):
            gr.replay()
    else:
        for _ in range(3):
            chain(xt)
    torch.cuda.synchronize()
    exp = x.astype(np.float64)
    for (_, _, _, qw, scales, zeros), (k, n) in zip(layers, dims):
        exp = ogptq.dequant_matmul(exp.astype(np.float32), qw, np.zeros((m, n)), scales, zeros, 128)
    got = ys[-1].cpu().numpy()
    np.testing.assert_allclose(got, exp, rtol=2e-4, atol=2e-4 * np.abs(exp).max())  # three chained fp32 linears vs fp64


@pytest.mark.parametrize("m", [1, 9, 32])
def test_batch_launch_equals_single_launches(m):
    """sb200_gptq4_matmul_batch: q / k / v (same input, three weight matrices of different N, one with a shorter K) in ONE
    launch == three launches == the fp64 oracle; every ``out`` keeps the accumulate-in-place contract."""
    from sparsebit_b200 import launch_count, ops

    rng = np.random.default_rng(m)
    probs, exps = [], []
    for k, n in ((1024, 512), (1024, 132), (512, 256)):
        x, qw, bias, scales, zeros = _make_case(rng, (m,), k, n, 128)
        out = t(np.broadcast_to(bias, (m, n)).copy())
        probs.append((t(x), t(qw), out, t(scales), t(zeros)))
        exps.append(ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, (m, n)), scales, zeros, 128))
    before = launch_count()
    outs = ops.gptq4_matmul_batch(probs, 128)
    assert launch_count() - before == 1
    for o, e in zip(outs, exps):
        np.testing.assert_allclose(o.cpu().numpy(), e, **TOL)
    with pytest.raises(RuntimeError, match="same number of tokens"):
        ops.gptq4_matmul_batch([probs[0], (probs[1][0][:0].reshape(0, 1024).new_zeros(m + 1, 1024),) + probs[1][1:]], 128)
