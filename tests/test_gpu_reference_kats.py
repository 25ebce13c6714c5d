"""The reference's GPTQ known-answer tests at FULL size (large_language_models/llama/quantization/
test_cuda_kernel.py:21-126, all thirteen 4-bit cases incl. M=6661 / N=25163, 12288 x 49152 and 8192 x 32768):
``QuantLinear(x)`` against a dense ``nn.Linear`` holding the dequantised weights, fp32 with TF32 off, elementwise
``rtol = atol = 1e-5`` (test_cuda_kernel.py:47).  Construction follows run_case line by line, on the GPU
(Quantizer.find_params -> quantize -> QuantLinear.pack -> forward); every case runs the dispatcher's choice
(impl 0), the small-M paths (impl 1: HMMA streaming kernel, impl 4: scalar kernel) and, where the shape is TMA-compatible, both wgmma kernels (impl 2, 3)."""
import pytest
import torch
import torch.nn as nn

from gpu_util import dev
from sparsebit_b200 import _lib
from sparsebit_b200.gptq import QuantLinear, find_params

pytestmark = pytest.mark.gpu

# (B, M=in_features, N=out_features, C, GS) -- test_cuda_kernel.py:50-126, bit = 4 rows
CASES = [
    (1, 12288, 12288 * 4, None, -1),   # test_OPT_175B_FC2_matvec
    (1, 8192, 8192 * 4, None, -1),     # test_regular_FC
    (1, 6661, 25163, None, -1),        # test_irregular_FC
    (1, 128, 64, None, -1),            # test_single_block_regular_FC
    (1, 127, 61, None, -1),            # test_single_block_irregular_FC
    (32, 12288, 12288 * 4, None, -1),  # test_multibatch_OPT_127B_FC2_matvec
    (29, 8192, 8192 * 4, None, -1),    # test_multibatch_regular_FC
    (31, 6661, 25163, None, -1),       # test_multibatch_irregular_FC
    (32, 6661, 25163, 1, -1),          # test_multibatch_1token_FC
    (4, 6661, 25163, 8, -1),           # test_multibatch_8token_FC
    (1, 12288, 12288 * 4, None, 128),  # test_OPT_175B_FC2_matvec_groupsize_min
    (29, 8192, 8192 * 4, None, 128),   # test_multibatch_regular_FC_groupsize_min
    (4, 6144, 6144 * 4, None, 384),    # test_groupsize_3x
]


def _quantize(x, scale, zero, maxq):  # utils/quant.py:8-10
    q = torch.clamp(torch.round(x / scale) + zero, 0, maxq)
    return scale * (q - zero)


@pytest.mark.parametrize("B,M,N,C,GS", CASES)
def test_reference_known_answer_full_size(B, M, N, C, GS):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(B * 7 + M + (C or 0))
    layer = nn.Linear(M, N).to(dev())
    vec = torch.randn((B, M) if C is None else (B, C, M), device=dev())
    with torch.no_grad():
        scale, zero = find_params(layer.weight.data, 4, GS)
        layer.weight.data = _quantize(layer.weight.data.view(-1, M if GS == -1 else GS), scale.view(-1, 1), zero.view(-1, 1),
                                      15).view(N, M)
        ql = QuantLinear(M, N, bit=4, groupsize=GS)
        ql.pack(layer, scale, zero)
        ql = ql.to(dev())
        gt = layer(vec)
        lib = _lib.load()
        tc_ok = (M % 8 == 0) and (N % 4 == 0)
        try:
            for impl in (0, 1, 4, 2, 3):
                if impl >= 2 and not tc_ok:
                    continue
                assert lib.sb200_gptq4_set_impl(impl) == 0
                for _ in range(2):  # twice: the module must not modify its own buffers (bias) between calls
                    out = ql(vec)
                    try:
                        torch.cuda.synchronize()
                    except RuntimeError as e:  # attribute an asynchronous kernel fault to the implementation
                        raise AssertionError(f"impl {impl}: {e}") from e
                    torch.testing.assert_close(out, gt, rtol=1e-5, atol=1e-5, msg=lambda m: f"impl {impl}: {m}")
        finally:
            lib.sb200_gptq4_set_impl(0)
