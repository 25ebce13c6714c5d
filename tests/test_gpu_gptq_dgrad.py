"""GPU: the input gradient of the GPTQ dequant-matmul (sb200_gptq_matmul_dgrad) and the backward of QuantLinear.

Bar: rtol = atol = 1e-5 elementwise, the forward's (test_cuda_kernel.py:47), against g @ wdq of the reference-produced
golden cases and against the fp64 truth (tests/gptq_dgrad_ref.py; computed in float64 on the device for the large
shapes).  Gradient rows with injected outliers are bounded by the row magnitude instead, as in the forward's
test_tcgen05_path_vs_fp64_oracle."""
import numpy as np
import pytest
import torch

from gpu_util import dev, no_tf32, t  # noqa: F401 -- no_tf32: a fixture
from gptq_dgrad_ref import dequant_weight
from oracle import gptq as ogptq
from sparsebit_b200 import _lib, ops
from sparsebit_b200.gptq import LayerStreamer, QuantLinear
from sparsebit_b200.gptq.quant_linear import find_params

pytestmark = pytest.mark.gpu
TOL = dict(rtol=1e-5, atol=1e-5)
SIMT, TC = 1, 2


def _dgrad(go, qw, scales, zeros, bit, gs, k, impl, grad_in=None):
    gi = torch.zeros(go.shape[:-1] + (k,), device=dev()) if grad_in is None else grad_in
    ops.gptq_matmul_dgrad(go, qw, gi, scales, zeros, bit, 0 if gs == -1 else gs, impl=impl)
    return gi


def _truth(go, qw, scales, zeros, bit, gs, k):
    """fp64 truth on the device: dense float64 weights times the float64 gradient."""
    w = torch.from_numpy(dequant_weight(qw, scales, zeros, k, 0 if gs == -1 else gs, bit)).to(dev())  # [K, N]
    g = go.reshape(-1, go.shape[-1]).double()
    return (g @ w.T).reshape(go.shape[:-1] + (k,))


def _case(rng, bit, bshape, k, n, gs, fractional_zero=False):
    w = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
    scale, zero = ogptq.find_params(w, bit, gs)
    wq = ogptq.quantize_weight(w, scale, zero, gs, bit)
    qw, scales, zeros = ogptq.pack_int4(wq, scale, zero) if bit == 4 else ogptq.pack_bits(wq, scale, zero, bit)
    if fractional_zero:
        zeros = (zeros + scales * rng.uniform(-0.5, 0.5, zeros.shape)).astype(np.float32)
    go = rng.standard_normal(bshape + (n,)).astype(np.float32)
    return go, qw, scales, zeros


def _check_rows(got, exp, outlier_rows=()):
    k = got.shape[-1]
    gf, ef = got.reshape(-1, k).double(), exp.reshape(-1, k)
    plain = [r for r in range(gf.shape[0]) if r not in outlier_rows]
    torch.testing.assert_close(gf[plain], ef[plain], **TOL)
    for r in outlier_rows:
        if r < gf.shape[0]:
            mag = max(ef[r].abs().max().item(), 1.0)
            assert (gf[r] - ef[r]).abs().max().item() <= 1e-5 + 1e-5 * mag


# ------------------------------------------------------------------------------------------------- golden cases
def _golden(golden):
    for fixture in ("gptq", "gptq_lowbit"):
        g = golden(fixture)
        for name in g["cases"]:
            bit, gs = (4, int(g[name + "_gs"])) if fixture == "gptq" else (int(v) for v in g[name + "_meta"])
            yield name, bit, gs, g


@pytest.mark.parametrize("impl", [0, SIMT, TC])
def test_golden_cases_against_reference_dense_weights(golden, impl):
    ran = 0
    for name, bit, gs, g in _golden(golden):
        wdq = torch.from_numpy(g[name + "_wdq"]).to(dev()).double()  # [N, K]
        n, k = wdq.shape
        if impl == TC and not (bit == 4 and n % 8 == 0 and k % 4 == 0):
            continue
        rng = np.random.default_rng(len(name))
        go = t(rng.standard_normal(g[name + "_x"].shape[:-1] + (n,)).astype(np.float32))
        got = _dgrad(go, t(g[name + "_qweight"]), t(g[name + "_scales"]), t(g[name + "_zeros"]), bit, gs, k, impl)
        exp = (go.double().reshape(-1, n) @ wdq).reshape(got.shape)
        torch.testing.assert_close(got.double(), exp, msg=name, **TOL)
        ran += 1
    assert ran == (5 if impl == TC else 19)


# ------------------------------------------------------------------------------------------------- tensor-core path
TC_CASES = [  # (bshape, k, n, gs, variant)
    ((1,), 256, 128, 128, ""),             # M = 1
    ((130,), 516, 264, -1, ""),            # ragged M, K and 64-n stage tiles, one group
    ((2, 65), 1024, 520, 256, ""),         # 3-D gradient, group 256
    ((4,), 6144, 768, 384, ""),            # group 384
    ((257,), 768, 136, -1, ""),            # one group, ragged M
    ((300,), 1024, 512, 128, "frac"),      # zero points with a fractional part
    ((129,), 1024, 264, 128, "span"),      # scales spanning 2^14 within one group
    ((64,), 512, 1032, 128, "frac+span"),
]


@pytest.mark.parametrize("impl", [TC, 0])
@pytest.mark.parametrize("bshape,k,n,gs,variant", TC_CASES)
def test_tensor_core_path_vs_fp64(bshape, k, n, gs, variant, impl):
    rng = np.random.default_rng(k + 3 * n + len(bshape))
    go, qw, scales, zeros = _case(rng, 4, bshape, k, n, gs, "frac" in variant)
    gf = go.reshape(-1, n)
    if "span" in variant:
        # per-feature factors 2^[-14, 0]: the group's normalisation is set by its largest features, and row 1 of the
        # gradient sees only the features 2^8 .. 2^14 below them, scaled up so that the elementwise bar is meaningful
        f = np.exp2(rng.uniform(-14, 0, (n, 1))).astype(np.float32)
        scales, zeros = (scales * f).astype(np.float32), (zeros * f).astype(np.float32)
        gf[1] = np.where(f[:, 0] < 2.0**-8, gf[1] * 2.0**10, 0.0)
    outliers = ()
    if gf.shape[0] > 2:
        gf[0, :5] = [3e4, -7e4, 1e-6, 0.0, 123.0]  # fp16-overflowing gradients are fine after row scaling
        gf[2] *= 1e-4
        outliers = (0, 2)
    go_t = t(go)
    got = _dgrad(go_t, t(qw), t(scales), t(zeros), 4, gs, k, impl)
    _check_rows(got, _truth(go_t, qw, scales, zeros, 4, gs, k), outliers)


@pytest.mark.parametrize("k,n", [(4096, 4096), (4096, 11008), (11008, 4096)])  # LLaMA-7B qkvo, gate/up, down
def test_tensor_core_path_llama_shapes(k, n):
    rng = np.random.default_rng(k + n)
    go, qw, scales, zeros = _case(rng, 4, (2048,), k, n, 128)
    go_t = t(go)
    exp = _truth(go_t, qw, scales, zeros, 4, 128, k)
    for impl in (TC, 0):
        _check_rows(_dgrad(go_t, t(qw), t(scales), t(zeros), 4, 128, k, impl), exp)


# ------------------------------------------------------------------------------------------------- SIMT path
SIMT_CASES = [  # (bit, bshape, k, n, gs): K = 6661, N not a multiple of 8, 3-bit units ending on a straddler
    (4, (3,), 6661, 2516, -1), (4, (1,), 256, 2516, 128), (4, (2,), 1000, 61, -1), (4, (33,), 127, 61, -1),
    (3, (5,), 6661, 250, -1), (3, (1,), 331, 61, -1), (3, (2,), 342, 200, -1), (3, (40,), 768, 136, 384),
    (2, (7,), 6661, 61, -1), (2, (1,), 320, 2516, 64), (2, (2,), 1152, 130, 192), (2, (33,), 512, 136, 64),
]


@pytest.mark.parametrize("bit,bshape,k,n,gs", SIMT_CASES)
def test_simt_path_vs_fp64(bit, bshape, k, n, gs):
    rng = np.random.default_rng(bit * 1000 + k + n)
    go, qw, scales, zeros = _case(rng, bit, bshape, k, n, gs, fractional_zero=(k % 2 == 0))
    go_t = t(go)
    exp = _truth(go_t, qw, scales, zeros, bit, gs, k)
    for impl in (SIMT, 0):
        _check_rows(_dgrad(go_t, t(qw), t(scales), t(zeros), bit, gs, k, impl), exp)


# ------------------------------------------------------------------------------------------------- contract
@pytest.mark.parametrize("bit,m,k,n,gs,impl", [(4, 300, 1024, 512, 128, TC), (4, 1, 256, 2516, 128, SIMT),
                                               (3, 33, 768, 136, 128, SIMT), (2, 5, 6661, 61, -1, SIMT)])
def test_accumulate_linear_and_deterministic(bit, m, k, n, gs, impl):
    rng = np.random.default_rng(m + k)
    go, qw, scales, zeros = _case(rng, bit, (m,), k, n, gs)
    args = (t(qw), t(scales), t(zeros), bit, gs, k, impl)
    g1, g2 = t(go), t(rng.standard_normal((m, n)).astype(np.float32))
    base = _dgrad(g1, *args)
    again = _dgrad(g1, *args)
    assert torch.equal(base, again)  # run-to-run bit-identical
    prefill = t(rng.standard_normal((m, k)).astype(np.float32))
    acc = _dgrad(g1, *args, grad_in=prefill.clone())
    torch.testing.assert_close(acc, prefill + base, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(_dgrad(2 * g1, *args), 2 * base, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(_dgrad(g1 + g2, *args), base + _dgrad(g2, *args), rtol=2e-5, atol=2e-5)


def test_forcing_the_tensor_core_path_on_unsupported_input_is_an_error():
    rng = np.random.default_rng(5)
    for bit, k, n in ((4, 127, 61), (4, 256, 60), (3, 256, 64), (2, 256, 64)):
        go, qw, scales, zeros = _case(rng, bit, (4,), k, n, -1)
        with pytest.raises(RuntimeError, match="unsupported"):
            _dgrad(t(go), t(qw), t(scales), t(zeros), bit, -1, k, TC)


# ------------------------------------------------------------------------------------------------- autograd
def _quant_linear(k, n, bit, gs, seed):
    torch.manual_seed(seed)
    lin = torch.nn.Linear(k, n)
    scale, zero = find_params(lin.weight.data, bit, gs)
    lin.weight.data = torch.from_numpy(ogptq.quantize_weight(lin.weight.data.numpy(), scale.reshape(n, -1).numpy(),
                                                              zero.reshape(n, -1).numpy(), gs, bit))
    ql = QuantLinear(k, n, bit, gs)
    ql.pack(lin, scale, zero)
    return ql.to(dev()), lin.to(dev())


@pytest.mark.parametrize("bit,gs", [(4, 128), (3, -1), (2, 64)])
@pytest.mark.parametrize("bshape", [(40,), (3, 7)])
def test_quant_linear_input_gradient_matches_dense(bit, gs, bshape, no_tf32):
    k, n = 384, 200
    ql, lin = _quant_linear(k, n, bit, gs, seed=bit)
    x = torch.randn(bshape + (k,), device=dev())
    r = torch.randn(bshape + (n,), device=dev())
    xq, xd = x.clone().requires_grad_(), x.clone().requires_grad_()
    (ql(xq) * r).sum().backward()
    (lin(xd) * r).sum().backward()
    assert xq.grad.shape == x.shape and xq.grad.device == x.device
    torch.testing.assert_close(xq.grad, xd.grad, **TOL)
    assert all(b.grad is None for b in (ql.qweight, ql.scales, ql.zeros, ql.bias))


def test_lora_stack_lower_adapter_gradient_matches_dense(no_tf32):
    k, rank = 256, 8
    layers = [_quant_linear(k, k, 4, 128, seed=s) for s in (1, 2)]
    torch.manual_seed(3)
    adapters = [(torch.nn.Linear(k, rank, bias=False).to(dev()), torch.nn.Linear(rank, k, bias=False).to(dev())) for _ in layers]
    x = torch.randn(48, k, device=dev())

    def run(quantised):
        h = x
        for (ql, lin), (a, b) in zip(layers, adapters):
            h = (ql if quantised else lin)(h) + b(a(h))
        return h.square().sum()

    grads = []
    for quantised in (True, False):
        for a, b in adapters:
            a.zero_grad(), b.zero_grad()
        run(quantised).backward()
        grads.append([p.grad.clone() for a, b in adapters for p in (a.weight, b.weight)])
    for gq, gd in zip(*grads):
        torch.testing.assert_close(gq, gd, rtol=1e-4, atol=1e-4)


def test_forward_is_bit_identical_with_and_without_grad():
    ql, _ = _quant_linear(512, 256, 4, 128, seed=7)
    x = torch.randn(64, 512, device=dev())
    with torch.no_grad():
        y0 = ql(x)
    y1 = ql(x.clone().requires_grad_())
    assert y1.requires_grad and torch.equal(y0, y1.detach())


def test_frozen_input_launches_nothing_in_backward():
    ql, _ = _quant_linear(256, 256, 4, 128, seed=9)
    a = torch.nn.Linear(256, 8, bias=False).to(dev())
    b = torch.nn.Linear(8, 256, bias=False).to(dev())
    x = torch.randn(40, 256, device=dev())
    loss = (ql(x) + b(a(x))).square().sum()
    torch.cuda.synchronize()
    before = _lib.launch_count()
    loss.backward()
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    assert a.weight.grad is not None and b.weight.grad is not None


def test_layer_streamer_backward_fails_loudly():
    """The streamer reuses its device slots, so the packed weights a layer saved for backward are overwritten by a later
    layer's copy: backward must raise instead of computing with another layer's weights."""
    torch.manual_seed(0)
    layers = [torch.nn.Sequential(_quant_linear(256, 256, 4, 128, seed=s)[0]) for s in range(3)]
    for layer in layers:
        layer.cpu()
    streamer = LayerStreamer(layers, dev(), slots=2)
    x = torch.randn(5, 256, device=dev(), requires_grad=True)
    out = streamer(x)
    with pytest.raises(RuntimeError, match="inplace|in-place"):
        out.sum().backward()
