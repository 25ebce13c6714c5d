"""Drop-in for the reference's JIT-built pybind module ``cuda_kernel``
(large_language_models/llama/quantization/cuda/cuda_kernel.cpp:10-73): same six names, argument order
and in-place-accumulate contract, backed by ``sb200_gptq4_matmul`` (4-bit: wgmma / SIMT) and
``sb200_gptq_matmul`` (3-bit, 2-bit: SIMT)."""
from .. import ops


def vecquant4matmul(inp1, inp2, out, scales, zeros):
    """out += inp1 @ dequant(inp2) with one scale/zero per output column (group_size = K)."""
    ops.gptq4_matmul(inp1, inp2, out, scales, zeros, 0)


def vecgroupquant4matmul(inp1, inp2, out, scales, zeros, group_size):
    """Group-wise variant; group_size must be a multiple of 128 (cuda_kernel_4bit.cu:60)."""
    ops.gptq4_matmul(inp1, inp2, out, scales, zeros, int(group_size))


def vecquant3matmul(inp1, inp2, out, scales, zeros):
    ops.gptq_matmul(inp1, inp2, out, scales, zeros, 3, 0)


def vecgroupquant3matmul(inp1, inp2, out, scales, zeros, group_size):
    """group_size must be a multiple of 128 (cuda_kernel_3bit.cu:60)."""
    ops.gptq_matmul(inp1, inp2, out, scales, zeros, 3, int(group_size))


def vecquant2matmul(inp1, inp2, out, scales, zeros):
    ops.gptq_matmul(inp1, inp2, out, scales, zeros, 2, 0)


def vecgroupquant2matmul(inp1, inp2, out, scales, zeros, group_size):
    """group_size must be a multiple of 64 (cuda_kernel_2bit.cu:58)."""
    ops.gptq_matmul(inp1, inp2, out, scales, zeros, 2, int(group_size))
