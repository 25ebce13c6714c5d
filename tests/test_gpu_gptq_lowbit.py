"""GPU parity: GPTQ 3-bit / 2-bit dequant-matmul (SURVEY 8f #3) through the ``cuda_kernel`` mirror /
QuantLinear vs the reference's known-answer construction (test_cuda_kernel.py, bit = 2, 3 cases:
rtol = atol = 1e-5 against Linear(dequantised W), fp32) and the fp64 oracle.  The fp64 oracle cases also run the
4-bit instantiations of the same SIMT kernel (gptq_simt.cu) through ``impl=4``."""
import numpy as np
import pytest
import torch

from gpu_util import dev, t
from oracle import gptq as ogptq
from sparsebit_b200 import ops
from sparsebit_b200.gptq import QuantLinear, cuda_kernel
from sparsebit_b200.gptq.quant_linear import find_params

pytestmark = pytest.mark.gpu
TOL = dict(rtol=1e-5, atol=1e-5)  # test_cuda_kernel.py:47
PLAIN = {2: cuda_kernel.vecquant2matmul, 3: cuda_kernel.vecquant3matmul}
GROUPED = {2: cuda_kernel.vecgroupquant2matmul, 3: cuda_kernel.vecgroupquant3matmul}


def _run(bit, x, qw, bias, scales, zeros, gs):
    y = t(np.broadcast_to(bias, x.shape[:-1] + (qw.shape[1],)).copy())
    if bit == 4:
        ops.gptq4_matmul(t(x), t(qw), y, t(scales), t(zeros), 0 if gs == -1 else gs, impl=4)
    elif gs == -1:
        PLAIN[bit](t(x), t(qw), y, t(scales), t(zeros))
    else:
        GROUPED[bit](t(x), t(qw), y, t(scales), t(zeros), gs)
    return y.cpu().numpy()


def test_golden_known_answers(golden):
    g = golden("gptq_lowbit")
    for name in g["cases"]:
        bit, gs = (int(v) for v in g[name + "_meta"])
        y = _run(bit, g[name + "_x"], g[name + "_qweight"], g[name + "_bias"], g[name + "_scales"], g[name + "_zeros"], gs)
        np.testing.assert_allclose(y, g[name + "_gt"], err_msg=name, **TOL)


# test_cuda_kernel.py:50-126 shapes that fit the time budget: irregular K / N, multi-batch, 3-D inputs,
# minimum and 3x group sizes, plus LLaMA-7B linear shapes at decode M.  For every bit width they run each row tile
# MT in {1, 2, 4, 8} (M = 1, 2, 3..4, >= 5), the multi-pass M loop (M > 8), K % block != 0, N % 128 != 0, and on a
# 132-SM H100 K slices of one block, of an odd and an even number of blocks, and a last slice shorter than the rest
# (e.g. 4096 x 11008: 3 blocks per slice, 2 in the last).
CASES = [
    (2, (1,), 1024, 1024, -1), (3, (1,), 1024, 1024, -1), (2, (1,), 719, 857, -1), (3, (1,), 719, 857, -1),
    (2, (31,), 6661, 1257, -1), (3, (31,), 6661, 1257, -1), (2, (4, 8), 2661, 512, -1), (3, (32, 1), 1024, 1031, -1),
    (2, (29,), 8192, 512, 64), (3, (29,), 8192, 512, 128), (2, (4,), 6144, 768, 192), (3, (4,), 6144, 768, 384),
    (2, (1,), 4096, 11008, 64), (3, (1,), 11008, 4096, 128), (3, (2,), 4096, 4096, 128), (2, (3,), 4096, 4096, 128),
    (2, (2,), 4096, 11008, 64),
    (4, (1,), 4096, 11008, 128), (4, (2,), 719, 857, -1), (4, (3,), 4096, 4096, 128), (4, (31,), 6661, 1257, -1),
    (4, (2,), 11008, 4096, 128), (4, (5, 4), 2048, 11008, 256),
]


@pytest.mark.parametrize("bit,bshape,k,n,gs", CASES)
def test_vs_fp64_oracle(bit, bshape, k, n, gs):
    rng = np.random.default_rng(bit * 1000 + k + n + len(bshape))
    w = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
    scale, zero = ogptq.find_params(w, bit, gs)
    qw, scales, zeros = ogptq.pack_bits(ogptq.quantize_weight(w, scale, zero, gs, bit), scale, zero, bit)
    assert np.asarray(ogptq.unpack_bits(qw, k, bit)).max() <= 2**bit - 1
    x = rng.standard_normal(bshape + (k,)).astype(np.float32)
    bias = (rng.standard_normal(n) * 0.1).astype(np.float32)
    y = _run(bit, x, qw, bias, scales, zeros, gs)
    exp = ogptq.dequant_matmul(x, qw, np.broadcast_to(bias, x.shape[:-1] + (n,)), scales, zeros, 0 if gs == -1 else gs, bit=bit)
    np.testing.assert_allclose(y, exp, **TOL)


@pytest.mark.parametrize("bit,gs", [(2, -1), (2, 64), (3, -1), (3, 128)])
def test_quantlinear_lowbit_roundtrip(bit, gs):
    """run_case of test_cuda_kernel.py:21-47 with our QuantLinear: quantise, pack, compare with the
    dequantised nn.Linear (fp16 activations go through the fp32 path and are cast back)."""
    torch.manual_seed(bit * 10 + (gs > 0))
    k, n = 512, 200
    layer = torch.nn.Linear(k, n)
    scale, zero = find_params(layer.weight.data, bit, gs)
    wv = layer.weight.data.view(n, -1, k if gs == -1 else gs)
    sv, zv = scale.view(n, -1, 1), zero.view(n, -1, 1)
    layer.weight.data = (sv * (torch.clamp(torch.round(wv / sv) + zv, 0, 2**bit - 1) - zv)).view(n, k)
    ql = QuantLinear(k, n, bit=bit, groupsize=gs)
    ql.pack(layer, scale, zero)
    ql, layer = ql.to(dev()), layer.to(dev())
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        x = torch.randn(5, 7, k, device=dev())
        with torch.no_grad():
            torch.testing.assert_close(ql(x), layer(x), rtol=1e-5, atol=1e-5)
            assert ql(x.half()).dtype == torch.float16
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def test_lowbit_argument_errors():
    x, out = torch.zeros(2, 256, device=dev()), torch.zeros(2, 8, device=dev())
    s = torch.ones(8, 4, device=dev())
    qw3 = torch.zeros(ogptq.packed_rows(256, 3), 8, dtype=torch.int32, device=dev())
    qw2 = torch.zeros(ogptq.packed_rows(256, 2), 8, dtype=torch.int32, device=dev())
    with pytest.raises(RuntimeError, match="divisible by 128"):
        cuda_kernel.vecgroupquant3matmul(x, qw3, out, s, s, 64)
    with pytest.raises(RuntimeError, match="divisible by 64"):
        cuda_kernel.vecgroupquant2matmul(x, qw2, out, s, s, 96)
    with pytest.raises(RuntimeError, match="rows"):
        cuda_kernel.vecquant3matmul(x, qw3[:-3].contiguous(), out, s, s)
    with pytest.raises(RuntimeError, match="2/3/4 bit"):
        ops.gptq_matmul(x, qw2, out, s, s, 5)
    with pytest.raises(RuntimeError, match="out_channel"):
        cuda_kernel.vecquant2matmul(x, qw2, torch.zeros(2, 9, device=dev()), s, s)
