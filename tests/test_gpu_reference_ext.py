"""GPU parity against the REFERENCE'S OWN CUDA extensions (torch_extensions/export.cc + fake_quant_tensor.cu: the four
entry points of export.cc:3-8; cuda/cuda_kernel*.cu: vecquant{2,3,4}matmul and the group variants).

Their outputs on the inputs built below are stored in ``tests/golden/ref_ext.npz`` (``tests/golden/make_golden_ref_ext.py``
ran the unmodified extensions once on an H100); every input comes from a seeded CPU generator, so the test needs nothing
outside the repository.  Element-wise outputs are stored as a fixed seeded sample (``sample_index``).

Forward outputs and gx are compared bit for bit, the float reductions gs / gzp at 1e-5 (relative to the L1 norm
of the summed terms: the reference accumulates with fp32 atomics in launch order).  Shapes keep every thread of
the reference kernels inside its data: its backward kernels call __syncthreads() under divergent control flow
(fake_quant_tensor.cu:123,128,260,265), which is only well defined when no thread leaves the loop early."""
import numpy as np
import pytest
import torch

from gpu_util import bits_equal, dev, t
from oracle import qdq as oqdq
from sparsebit_b200 import fake_quant
from sparsebit_b200.gptq import cuda_kernel

pytestmark = pytest.mark.gpu
SAMPLE = 4096  # stored elements per output tensor

PERTENSOR_CASES = [(512 * 40, -128, 127, 0.0), (2560 * 512, 0, 255, 37.0), (2 * 2560 * 512, -8, 7, 0.0)]
PERCHANNEL_CASES = [((8, 16, 32, 32), 1, -128, 127), ((64, 512), 0, -8, 7), ((4, 6, 7, 512), 1, 0, 15), ((16, 3, 1024), 1, 0, 255)]
GPTQ_CASES = [(4, 1, 4096, 4096, 128), (4, 16, 4096, 11008, 128), (4, 5, 1024, 768, -1), (3, 3, 4096, 512, 128), (2, 7, 2048, 256, 64),
              (4, 256, 2048, 1024, 128)]
GATE_CASES = [(False, False), (True, False), (False, True)]


def sample_index(n, key):
    """The fixed positions of a flattened output of n elements that the golden file stores (all of them when n <= SAMPLE)."""
    if n <= SAMPLE:
        return np.arange(n)
    return np.sort(np.random.default_rng(key).choice(n, SAMPLE, replace=False))


def pertensor_inputs(n, qmin, qmax, zp):
    rng = np.random.default_rng(n + qmax)
    x = (rng.standard_normal(n) * 1.5).astype(np.float32)
    gy = rng.standard_normal(n).astype(np.float32)
    s = np.float32([np.abs(x).max() / (qmax - qmin) * 1.2])  # clips ~ 10 % of a symmetric range
    return x, gy, s, np.float32([zp])


def perchannel_inputs(shape, ch_axis, qmin, qmax):
    rng = np.random.default_rng(sum(shape) + qmax)
    x = (rng.standard_normal(shape) * 1.5).astype(np.float32)
    gy = rng.standard_normal(shape).astype(np.float32)
    c = shape[ch_axis]
    s = (rng.uniform(0.6, 1.4, c) * 4.0 / (qmax - qmin)).astype(np.float32)
    z = np.rint(rng.uniform(-2, 2, c) + (0 if qmin < 0 else (qmax + 1) // 2)).astype(np.float32)
    return x, gy, s, z


def gate_inputs():
    g = torch.Generator().manual_seed(17)
    return torch.randn(512 * 8, generator=g), torch.randn(512 * 8, generator=g), torch.tensor([0.05]), torch.tensor([3.0])


def gptq_inputs(bit, m, k, n, gs):
    """Packed checkpoint, activations and bias on the device, plus the entry-point name."""
    from sparsebit_b200.gptq import find_params, pack_intweight

    torch.manual_seed(bit * 1000 + m)
    w = torch.randn(n, k) / k**0.5
    scale, zero = find_params(w, bit, gs)
    g = scale.reshape(n, -1).shape[1]
    q = torch.clamp(torch.round(w.view(n, g, -1) / scale.view(n, g, 1)) + zero.view(n, g, 1), 0, 2**bit - 1)
    qw = pack_intweight(q.view(n, k).to(torch.int64).t().contiguous(), bit).to(dev())
    scales = scale.reshape(n, g).contiguous().to(dev())
    zeros = (zero * scale).reshape(n, g).contiguous().to(dev())
    x = torch.randn(m, k).to(dev())
    bias = (torch.randn(n) * 0.1).to(dev())
    name = f"vec{'group' if gs != -1 else ''}quant{bit}matmul"
    return x, qw, scales, zeros, bias, name


def case_key(*parts):
    return "_".join(str(p) for p in parts).replace("(", "").replace(")", "").replace(", ", "x").replace("-", "m").replace(".", "p")


@pytest.fixture(scope="module")
def ref(golden):
    return golden("ref_ext")


def _close(a, b, l1, tol=1e-5):
    return np.all(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) <= tol * (np.asarray(l1, np.float64) + 1e-30))


@pytest.mark.parametrize("n,qmin,qmax,zp", PERTENSOR_CASES)
def test_pertensor_forward_backward_equal_reference_kernels(ref, n, qmin, qmax, zp):
    key = case_key("pt", n, qmin, qmax, zp)
    x, gy, s, z = pertensor_inputs(n, qmin, qmax, zp)
    idx = sample_index(n, n)
    xt, gt = t(x), t(gy)
    st, zt = t(s).requires_grad_(True), t(z).requires_grad_(True)
    y = fake_quant.quant_pertensor_forward(xt, st, zt, qmin, qmax, 0)
    assert bits_equal(y.cpu().numpy()[idx], ref[key + "_y"])
    gx, gs, gz = fake_quant.quant_pertensor_backward(xt, st, zt, gt, qmin, qmax, 0)
    assert bits_equal(gx.cpu().numpy()[idx], ref[key + "_gx"])
    _, egs, egz = oqdq.ste_backward(x, s, z, gy, qmin, qmax)
    l1g = np.abs(gy).astype(np.float64).sum()
    l1s, l1z = l1g * max(abs(qmin - zp), abs(qmax - zp), 1.0), l1g * s[0]  # L1 norms of the summed terms
    assert _close(gs.cpu().numpy(), egs, l1s, 1e-6) and _close(gz.cpu().numpy(), egz, l1z, 1e-6)  # ours vs fp64
    assert _close(gs.cpu().numpy(), ref[key + "_gs"], l1s) and _close(gz.cpu().numpy(), ref[key + "_gz"], l1z)


@pytest.mark.parametrize("shape,ch_axis,qmin,qmax", PERCHANNEL_CASES)
def test_perchannel_forward_backward_equal_reference_kernels(ref, shape, ch_axis, qmin, qmax):
    key = case_key("pc", shape, ch_axis, qmin, qmax)
    x, gy, s, z = perchannel_inputs(shape, ch_axis, qmin, qmax)
    idx = sample_index(x.size, sum(shape))
    xt, gt = t(x), t(gy)
    st, zt = t(s).requires_grad_(True), t(z).requires_grad_(True)
    y = fake_quant.quant_perchannel_forward(xt, st, zt, qmin, qmax, ch_axis, 0)
    assert bits_equal(y.cpu().numpy().reshape(-1)[idx], ref[key + "_y"])
    gx, gs, gz = fake_quant.quant_perchannel_backward(xt, st, zt, gt, qmin, qmax, ch_axis, 0)
    assert bits_equal(gx.cpu().numpy().reshape(-1)[idx], ref[key + "_gx"])
    gs_r, gz_r = ref[key + "_gs"], ref[key + "_gz"]
    axes = tuple(a for a in range(len(shape)) if a != ch_axis)
    l1g = np.abs(gy).astype(np.float64).sum(axis=axes)
    l1s, l1z = l1g * np.maximum(np.abs(qmin - z), np.abs(qmax - z)), l1g * s
    assert _close(gs.cpu().numpy().reshape(-1), gs_r, l1s)
    # zero-point gradient: the reference kernel's open-top rule (fake_quant_tensor.cu:264) is what ships by default
    assert _close(gz.cpu().numpy().reshape(-1), gz_r, l1z)
    _, _, egz_open = oqdq.ste_backward(x, s, z, gy, qmin, qmax, ch_axis, gzp_open_top=True)
    _, _, egz_closed = oqdq.ste_backward(x, s, z, gy, qmin, qmax, ch_axis)
    assert _close(gz_r, np.reshape(egz_open, -1), l1z) and not _close(gz_r, np.reshape(egz_closed, -1), l1z)


def test_requires_grad_gates_match_reference(ref):
    x, gy, s, z = (v.to(dev()) for v in gate_inputs())
    for i, (rs, rz) in enumerate(GATE_CASES):
        st, zt = s.clone().requires_grad_(rs), z.clone().requires_grad_(rz)
        _, gs, gz = fake_quant.quant_pertensor_backward(x, st, zt, gy, -8, 7, 0)
        gs_zero_r, gz_zero_r = ref["gate_zero"][i]
        assert bool(gs_zero_r) == (float(gs) == 0) and bool(gz_zero_r) == (float(gz) == 0)


@pytest.mark.parametrize("bit,m,k,n,gs", GPTQ_CASES)
def test_gptq_kernels_equal_reference_kernels(ref, bit, m, k, n, gs):
    """Same packed checkpoint, same activations: ours vs the reference's VecQuant{2,3,4}MatMulKernel
    (cuda_kernel_{2,3,4}bit.cu) at the reference's own tolerance rtol = atol = 1e-5 (test_cuda_kernel.py:47)."""
    x, qw, scales, zeros, bias, name = gptq_inputs(bit, m, k, n, gs)
    y = bias.expand(m, n).contiguous()
    if gs == -1:
        getattr(cuda_kernel, name)(x, qw, y, scales, zeros)
    else:
        getattr(cuda_kernel, name)(x, qw, y, scales, zeros, gs)
    key = case_key("gptq", bit, m, k, n, gs)
    got = y.cpu().numpy().reshape(-1)[sample_index(m * n, bit * 1000 + m)]
    torch.testing.assert_close(torch.from_numpy(got), torch.from_numpy(ref[key + "_y"]), rtol=1e-5, atol=1e-5)
