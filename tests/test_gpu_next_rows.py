"""GPU parity for the "next" rows (SURVEY 8f #2): LSQ / LSQ+ / PACT / DoReFa quantizers and the
MovingAverage observer, against golden vectors from the unmodified reference
(tests/golden/make_golden.py::gen_next_rows)."""
import math

import numpy as np
import pytest
import torch

from gpu_util import bits_equal, dev, t
from oracle import qdq as oqdq
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization import build_quantizer
from sparsebit_b200.quantization.common import Backend

pytestmark = pytest.mark.gpu
SCHEMES = {(0, 1): "per-tensor-symmetric", (0, 0): "per-tensor-affine", (1, 1): "per-channel-symmetric", (1, 0): "per-channel-affine"}
QTYPE = {"lsq": "lsq", "lsqp": "lsq+", "pact": "pact", "dorefa": "dorefa", "mavg": "uniform", "aciqg": "uniform", "aciql": "uniform"}
OBSERVER = {"mavg": "moving_average", "aciqg": "aciq", "aciql": "aciq"}
# scheme the reference was CONFIGURED with (LSQ may flip affine -> symmetric when it sees negatives)
CONFIGURED = {"lsq_pt_a4": "per-tensor-affine", "lsq_pt_sym4": "per-tensor-symmetric", "lsq_pc_w4": "per-channel-symmetric",
              "lsqp_pt_a8": "per-tensor-affine", "lsqp_pc_w4": "per-channel-symmetric", "pact_pt_a4": "per-tensor-affine",
              "pact_pt_s8": "per-tensor-symmetric", "dorefa_w4": "per-tensor-symmetric", "mavg_pt": "per-tensor-symmetric",
              "mavg_nlc": "per-tensor-affine", "aciqg_pt_s8": "per-tensor-symmetric", "aciqg_pt_a4": "per-tensor-affine",
              "aciqg_pc_w8": "per-channel-symmetric", "aciql_pt_s8": "per-tensor-symmetric", "aciql_pc_w4": "per-channel-symmetric"}


def _build(g, name):
    qmin, qmax, ch_axis, perch, sym, bit = (int(v) for v in g[name + "_meta"])
    prefix = name.split("_")[0]
    target = "weight" if name.endswith(("w4", "w8")) else "feature"
    layout = "NLC" if ch_axis == 2 else "NCHW"
    cfg = sbcfg.quantizer_config(CONFIGURED[name], bit, target, OBSERVER.get(prefix, "minmax"), layout, qtype=QTYPE[prefix],
                                 pact_alpha=3, ema_ratio=0.9, aciq_distribution="LAPLACE" if prefix == "aciql" else "GAUS")
    q = build_quantizer(cfg).to(dev())
    q.set_backend(Backend.VIRTUAL)
    xs = [g[f"{name}_x{i}"] for i in range(int(g[name + "_nb"]))]
    for x in xs:
        q.update_observer(t(x))
    return q, xs


def test_next_row_quantizers_match_reference(golden):
    g = golden("next_rows")
    for name in g["cases"]:
        prefix = name.split("_")[0]
        q, xs = _build(g, name)
        with torch.no_grad():
            q.calc_qparams()
            q.enable_quant()
            if prefix in ("lsq", "lsqp", "pact"):
                scale, zp = q._qparams_preprocess(t(xs[0]))
            else:
                scale, zp = q.scale, q.zero_point
            # LSQ-type step sizes come from a float mean/std over the data: 2e-6 relative (summation order)
            np.testing.assert_allclose(scale.reshape(-1).cpu().numpy(), g[name + "_scale"], rtol=2e-6, err_msg=name)
            assert bits_equal(zp.reshape(-1).cpu().numpy(), g[name + "_zp"]), name
            if prefix in ("mavg", "aciqg", "pact"):  # min/max-derived qparams: bit-exact
                assert bits_equal(scale.reshape(-1).cpu().numpy(), g[name + "_scale"]), name
            if prefix in ("lsq", "lsqp", "aciql"):  # decouple the forward compare from the float reduction
                q.scale.data.copy_(t(g[name + "_scale"]).reshape(q.scale.shape))
            y = q(t(xs[0])).cpu().numpy()
        if prefix == "dorefa":  # tanh runs in torch (CUDA vs CPU libm may differ by an ulp -> rare grid flips)
            assert np.mean(y != g[name + "_y"]) < 2e-3, name
        else:
            assert bits_equal(y, g[name + "_y"]), name
        assert len(q.observer.data_cache) == 0


def test_lsq_scale_gradient_uses_kernel_gs():
    q = build_quantizer(sbcfg.quantizer_config("per-tensor-symmetric", 4, "feature", qtype="lsq")).to(dev())
    q.set_backend(Backend.VIRTUAL)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(4, 3, 16, 16, generator=g)
    q.update_observer(x.to(dev()))
    q.calc_qparams()
    assert isinstance(q.scale, torch.nn.Parameter)
    q.enable_quant()
    xr = x.to(dev()).requires_grad_(True)
    gy = torch.randn(x.shape, generator=g)
    q(xr).backward(gy.to(dev()))
    s = q.scale.detach().abs().reshape(-1).cpu().numpy()
    egx, egs, _ = oqdq.ste_backward(x.numpy(), s, np.zeros(1, np.float32), gy.numpy(), -8, 7)
    ratio = 1.0 / math.sqrt(x.numel() * 7)
    sign = np.sign(q.scale.detach().reshape(-1).cpu().numpy())  # d|s|/ds
    np.testing.assert_allclose(q.scale.grad.reshape(-1).cpu().numpy(), egs * ratio * sign, rtol=1e-5)
    assert bits_equal(xr.grad.cpu().numpy(), egx)


def _ada_quantizer(g, name):
    qmin, qmax, ch_axis, perch, sym, bit = (int(v) for v in g[name + "_meta"])
    q = build_quantizer(sbcfg.quantizer_config(SCHEMES[(perch, sym)], bit, "weight", qtype="adaround")).to(dev())
    q.set_backend(Backend.VIRTUAL)
    w = t(g[name + "_w"])
    q.update_observer(w)
    q.calc_qparams()
    q.enable_quant()
    return q, w


def test_adaround_matches_reference(golden):
    """AdaRound (adaround.py:26-54) through the plugin class: qparams and the eval branch bit-exact,
    init / soft branch / dL/dv within 1e-5 relative (expf / logf vs the CPU libm)."""
    g = golden("next_rows")
    for name in g["ada_cases"]:
        q, w = _ada_quantizer(g, name)
        assert bits_equal(q.scale.reshape(-1).cpu().numpy(), g[name + "_scale"]), name
        assert bits_equal(q.zero_point.reshape(-1).cpu().numpy(), g[name + "_zp"]), name
        q.init_variables(w)
        assert isinstance(q.v, torch.nn.Parameter) and q.v.shape == w.shape
        np.testing.assert_allclose(q.v.detach().cpu().numpy(), g[name + "_v0"], rtol=1e-5, atol=1e-6, err_msg=name)
        q.v = torch.nn.Parameter(t(g[name + "_v1"]))
        q.eval()
        with torch.no_grad():
            assert bits_equal(q(w).cpu().numpy(), g[name + "_yhard"]), name
        q.train()
        y = q(w)
        np.testing.assert_allclose(y.detach().cpu().numpy(), g[name + "_ysoft"], rtol=1e-5, atol=1e-7, err_msg=name)
        (y * t(g[name + "_gy"])).sum().backward()
        np.testing.assert_allclose(q.v.grad.cpu().numpy(), g[name + "_gv"], rtol=1e-5, atol=1e-8, err_msg=name)
        # the differentiable regulariser input equals the oracle restatement
        np.testing.assert_allclose(q._get_soft_round_values().detach().cpu().numpy(),
                                   oqdq.adaround_soft_values(g[name + "_v1"])[0], rtol=1e-5, atol=1e-7)


def test_adaround_kernels_vs_oracle_ragged():
    """Odd inner sizes (scalar path), large per-tensor tensors (float4 path), NaN / inf inputs."""
    from sparsebit_b200 import ops

    rng = np.random.default_rng(7)
    for shape, ch_axis in [((5, 7, 3), 0), ((3, 4, 1031), 1), ((1 << 18,), None), ((64, 147), 0), ((2, 2048, 9), 1)]:
        x = (rng.standard_normal(shape) * 0.3).astype(np.float32)
        v = (rng.standard_normal(shape) * 3).astype(np.float32)
        c = 1 if ch_axis is None else shape[ch_axis]
        s = (rng.uniform(0.01, 0.05, c)).astype(np.float32)
        zp = np.rint(rng.uniform(-3, 3, c)).astype(np.float32)
        if x.size > 100:
            x.reshape(-1)[3], x.reshape(-1)[17], v.reshape(-1)[29] = np.nan, np.inf, np.nan
        ax = 0 if ch_axis is None else ch_axis
        hard = ops.adaround_forward(t(x), t(v), t(s), t(zp), -8, 7, ch_axis, soft=False).cpu().numpy()
        assert bits_equal(hard, oqdq.adaround_forward(x, v, s, zp, -8, 7, ax, soft=False)), shape
        soft = ops.adaround_forward(t(x), t(v), t(s), t(zp), -8, 7, ch_axis, soft=True).cpu().numpy()
        np.testing.assert_allclose(soft, oqdq.adaround_forward(x, v, s, zp, -8, 7, ax, soft=True), rtol=1e-5, atol=1e-7)
        gy = rng.standard_normal(shape).astype(np.float32)
        ok = np.isfinite(x) & np.isfinite(v)
        gv = ops.adaround_backward(t(x), t(v), t(s), t(zp), t(gy), -8, 7, ch_axis).cpu().numpy()
        np.testing.assert_allclose(gv[ok], oqdq.adaround_grad_v(x, v, s, zp, gy, -8, 7, ax)[ok], rtol=1e-5, atol=1e-8)
        v0 = ops.adaround_init(t(x), t(s), ch_axis).cpu().numpy()
        np.testing.assert_allclose(v0[ok], oqdq.adaround_init(x, s, ax)[ok], rtol=1e-5, atol=1e-6)


def test_adaround_reconstruct_qlayer_reduces_error():
    """reconstruct_qlayer (adaround.py:57-110) on a tiny linear layer: the learned rounding must not be
    worse than round-to-nearest on the layer's outputs, and every v must have left the soft zone."""
    from sparsebit_b200.quantization.quantizers.adaround import reconstruct_qlayer

    class QLinear(torch.nn.Module):  # the slice of QuantOpr the routine uses (modules/base.py:48-66)
        def __init__(self, lin, wq):
            super().__init__()
            self.weight, self.bias, self.weight_quantizer = lin.weight, lin.bias, wq

        def set_quant(self, w_quant=False, a_quant=False):
            self.weight_quantizer.enable_quant() if w_quant else self.weight_quantizer.disable_quant()

        def forward(self, x):
            return torch.nn.functional.linear(x, self.weight_quantizer(self.weight), self.bias)

    torch.manual_seed(0)
    lin = torch.nn.Linear(32, 16).to(dev())
    wq = build_quantizer(sbcfg.quantizer_config("per-channel-symmetric", 3, "weight", qtype="adaround")).to(dev())
    wq.set_backend(Backend.VIRTUAL)
    wq.update_observer(lin.weight)
    wq.calc_qparams()
    layer = QLinear(lin, wq)
    x = torch.randn(256, 32, device=dev())
    with torch.no_grad():
        ref = lin(x)
        nearest = torch.nn.functional.linear(x, torch.round(lin.weight / wq.scale).clamp(-4, 3) * wq.scale, lin.bias)
        err_nearest = (nearest - ref).pow(2).mean().item()
    reconstruct_qlayer(layer, x, ref, batch_size=64, max_steps=600, print_freq=0)
    assert not wq.training
    with torch.no_grad():
        err_ada = (layer(x) - ref).pow(2).mean().item()
    assert err_ada <= err_nearest * 1.02, (err_ada, err_nearest)


def test_row_moments_vs_fp64_numpy():
    """sb200_observe_moments (LSQ / LSQ+ / ACIQ-laplace initialisation statistics): fp64 sums in a fixed order,
    accumulated across batches, bit-identical run to run."""
    from sparsebit_b200 import ops

    rng = np.random.default_rng(11)
    for rows, row_len in [(1, 100_003), (7, 33), (64, 20_000), (3, 1)]:
        batches = [(rng.standard_normal((rows, row_len)) * 3 + 0.5).astype(np.float32) for _ in range(2)]
        centre = rng.standard_normal(rows)
        acc = ops.moments_new(rows, dev())
        for b in batches:
            ops.moments_update(t(b), acc, centre=torch.from_numpy(centre).to(dev()))
        x = np.concatenate(batches, axis=1).astype(np.float64)
        d = x - centre[:, None]
        exp = np.stack([x.sum(1), (x * x).sum(1), np.abs(x).sum(1), np.abs(d).sum(1), (d * d).sum(1)], axis=1)
        got = acc.cpu().numpy()
        np.testing.assert_allclose(got, exp, rtol=1e-12, atol=1e-9)
        again = ops.moments_new(rows, dev())
        for b in batches:
            ops.moments_update(t(b), again, centre=torch.from_numpy(centre).to(dev()))
        assert np.array_equal(again.cpu().numpy(), got)  # deterministic
        plain = ops.moments_update(t(batches[0]), ops.moments_new(rows, dev())).cpu().numpy()
        np.testing.assert_allclose(plain[:, 3], plain[:, 2], rtol=1e-15)  # centre = 0: |x - 0| == |x|
    with pytest.raises(RuntimeError):
        ops.moments_update(t(batches[0]), torch.zeros(2, 5, device=dev()))  # wrong dtype / shape


def _dorefa_eager(x, scale, zp, qdesc_q):
    """The reference op chain on the GPU (dorefa.py:15-20): ATen tanh / abs / max / div, then STE (native QDQ)."""
    from sparsebit_b200.quantization.quantizers.quant_tensor import STE

    t_ = x.tanh()
    xn = t_ / t_.detach().abs().max()
    return xn, STE.apply(xn, scale, zp, qdesc_q.qdesc, qdesc_q.backend)


@pytest.mark.parametrize("scheme,shape", [("per-tensor-symmetric", (64, 3, 7, 7)), ("per-tensor-affine", (33, 5, 3)),
                                          ("per-channel-symmetric", (48, 16, 3, 3)), ("per-channel-affine", (10, 1031))])
def test_dorefa_fused_kernels_match_the_eager_chain(scheme, shape):
    """sb200_dorefa_absmax / _fwd / _bwd against tanh -> / max|.| -> STE run as separate ATen ops + autograd: the
    normalised tensor to 1 ulp, fake-quantised values and gradients equal except where that ulp moves a rounding."""
    from sparsebit_b200 import ops

    g = torch.Generator().manual_seed(hash(shape) % 1000)
    x = (torch.randn(shape, generator=g) * 1.3).to(dev())
    q = build_quantizer(sbcfg.quantizer_config(scheme, 4, "weight", qtype="dorefa")).to(dev())
    q.set_backend(Backend.VIRTUAL)
    q.update_observer(x)
    q.calc_qparams()
    q.enable_quant()
    assert len(q.observer.data_cache) == 0
    # what the observer saw: tanh(x) / max|tanh(x)|, so min / max lie in [-1, 1] and one of them is +-1
    m = ops.dorefa_absmax(x)
    assert abs(float(m) - float(x.tanh().abs().max())) <= 1.2e-7  # libdevice tanhf on both sides (1 ulp of slack below 1.0)
    xn_fused = ops.dorefa_forward(x, m)
    xr = x.clone().requires_grad_(True)
    xn, y_eager = _dorefa_eager(xr, q.scale, q.zero_point, q)
    np.testing.assert_allclose(xn_fused.cpu().numpy(), xn.detach().cpu().numpy(), rtol=5e-7, atol=0)
    assert float(xn_fused.abs().max()) == 1.0
    gy = torch.randn(shape, generator=g).to(dev())
    y_eager.backward(gy)
    xf = x.clone().requires_grad_(True)
    y = q(xf)
    y.backward(gy)
    a, b = y.detach().cpu().numpy(), y_eager.detach().cpu().numpy()
    assert np.mean(a != b) < 2e-3, (scheme, np.mean(a != b))
    ga, gb = xf.grad.cpu().numpy(), xr.grad.cpu().numpy()
    assert np.mean(~np.isclose(ga, gb, rtol=1e-5, atol=1e-8)) < 2e-3, scheme
    # on-grid: every output is (k - zp) * scale for an integer k in [qmin, qmax]
    qmin, qmax = q.qdesc.qrange
    s = q.scale.detach().reshape([-1] + [1] * (len(shape) - 1)).cpu().numpy() if q.scale.numel() > 1 else float(q.scale)
    z = q.zero_point.detach().reshape([-1] + [1] * (len(shape) - 1)).cpu().numpy() if q.scale.numel() > 1 else float(q.zero_point)
    k = a / s + np.rint(z)
    assert np.abs(k - np.rint(k)).max() < 1e-3 and k.min() >= qmin - 1e-3 and k.max() <= qmax + 1e-3
    # the numpy restatement of the reference chain (oracle.qdq.dorefa_*, pinned to the reference's own DoReFa output):
    # numpy's tanh may differ from libdevice's by an ulp, so a few values may sit on the neighbouring grid point
    sc_np, zp_np = q.scale.detach().reshape(-1).cpu().numpy(), q.zero_point.detach().reshape(-1).cpu().numpy()
    exp = oqdq.dorefa_forward(x.cpu().numpy(), sc_np, zp_np, qmin, qmax, ch_axis=0)
    assert np.mean(a != exp) < 5e-3, (scheme, np.mean(a != exp))
    egx = oqdq.dorefa_grad_x(x.cpu().numpy(), sc_np, zp_np, gy.cpu().numpy(), qmin, qmax, ch_axis=0)
    assert np.mean(~np.isclose(ga, egx, rtol=1e-4, atol=1e-6)) < 5e-3, scheme


def test_dorefa_nan_and_ragged_inputs():
    from sparsebit_b200 import ops

    x = torch.randn(1025, device=dev())[1:]  # 4-byte aligned only, odd length: scalar paths
    m = ops.dorefa_absmax(x)
    assert abs(float(m) - float(x.tanh().abs().max())) <= 1.2e-7
    s, z = torch.tensor([0.125], device=dev()), torch.tensor([0.0], device=dev())
    xc = x.contiguous()
    y = ops.dorefa_forward(xc, m, s, z, -8, 7)
    ref = torch.clamp(torch.round((xc.tanh() / m) / s), -8, 7) * s
    assert np.mean(y.cpu().numpy() != ref.cpu().numpy()) < 2e-3
    xb = xc.clone()
    xb[5] = float("nan")
    mb = ops.dorefa_absmax(xb)
    assert torch.isnan(mb).all()  # torch.max propagates NaN; every normalised value is then NaN, like the reference
    assert torch.isnan(ops.dorefa_forward(xb, mb, s, z, -8, 7)).all()
    gx = ops.dorefa_backward(xc, m, s, z, torch.ones_like(xc), -8, 7)
    t_ = xc.tanh()
    vq = torch.round((t_ / m) / s)
    exp = torch.where((vq >= -8) & (vq <= 7), torch.ones_like(xc), torch.zeros_like(xc)) / m * (1 - t_ * t_)
    assert np.mean(~np.isclose(gx.cpu().numpy(), exp.cpu().numpy(), rtol=1e-5, atol=1e-8)) < 2e-3
