"""Gradients of the learnable quantizers in a QAT step: LSQ (|s| and GradScale), LSQ+ (plus a learned zero point through
clamp), PACT (learnable alpha, the grid built from [lower, alpha]) and DoReFa (tanh / abs-max), each chaining the STE
backward kernels into autograd.  Compared with the unmodified reference (tests/golden/qat.npz) and with the fp64
restatement in oracle/qdq.py (lsq_grads, pact_grads, dorefa_grads).

Tolerances.  y and x.grad are elementwise selections and single-rounded fp32 operations, the same IEEE operations as
the reference: bit-exact.  A parameter gradient is a sum of n terms; the kernels and the reference sum them in
different orders, and any order of n fp32 additions stays within (n - 1) u L1 of the exact sum (u = 2^-24, L1 the norm
of the terms).  The reductions here are trees or fp64, whose error grows with log2(n) <= 23 levels instead of n, so
1e-5 L1 (168 levels of u) bounds them with room to spare, while a wrong term (a dropped mask, a missing scale path)
moves a gradient by a whole term, far beyond it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import bits_equal, dev, seed_of, t
# TF32 off on every test: the module-step bounds assume fp32 products and sums in the conv / linear
from gpu_util import no_tf32_autouse  # noqa: F401
from oracle import qdq as oqdq
from qat_ref import GRAD_KEYS, case_geometry, oracle_case, plant_grid_edges, plant_pact_bounds, within_l1
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization import build_quantizer
from sparsebit_b200.quantization.common import Backend
from sparsebit_b200.quantization.modules import QConv2d, QLinear

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _quantizer(qtype, scheme, bit, target, layout, x, alpha=10.0):
    q = build_quantizer(sbcfg.quantizer_config(scheme, bit, target, "minmax", layout, qtype=qtype, pact_alpha=alpha)).to(dev())
    q.set_backend(Backend.VIRTUAL)
    q.update_observer(x)
    q.calc_qparams()
    q.enable_quant()
    return q


def _set(q, scale=None, zero_point=None, alpha=None):
    with torch.no_grad():
        if alpha is not None:
            q.alpha.fill_(float(np.asarray(alpha).reshape(-1)[0]))
        if scale is not None:
            q.scale.copy_(t(np.asarray(scale, np.float32)).reshape(q.scale.shape))
        if zero_point is not None:
            q.zero_point.copy_(t(np.asarray(zero_point, np.float32)).reshape(q.zero_point.shape))


def _learnable(q):
    if q.TYPE == "PACT":
        return {"alpha": q.alpha}
    return {k: p for k, p in (("scale", q.scale), ("zero_point", q.zero_point)) if isinstance(p, torch.nn.Parameter)}


def _step(q, x, gy):
    """One train-mode forward / backward with loss sum(y * gy): (y, x.grad, {param: grad}) on the host."""
    xr = x.clone().requires_grad_(True)
    y = q(xr)
    (y * gy).sum().backward()
    grads = {k: p.grad.reshape(-1).cpu().numpy() for k, p in _learnable(q).items()}
    return y.detach().cpu().numpy(), xr.grad.cpu().numpy(), grads


def _zero_grad(q):
    for p in _learnable(q).values():
        p.grad = None


def _check(name, got, want, dorefa=False):
    """got = (y, gx, grads) of the kernels, want = (y, gx, {param: (grad, l1)}) of the oracle."""
    (y, gx, grads), (ey, egx, egrads) = got, want
    if dorefa:  # libdevice tanhf vs numpy's tanh: an ulp apart, which can move a value across a rounding boundary
        assert np.mean(y != ey) < 5e-3, name
        assert np.mean(~np.isclose(gx, egx, rtol=1e-4, atol=1e-6)) < 5e-3, name
    else:
        assert bits_equal(y, ey), (name, int(np.sum(y != ey)))
        assert bits_equal(gx, egx), (name, int(np.sum(gx != egx)))
    assert set(grads) == set(egrads), (name, set(grads), set(egrads))
    for k, (eg, l1) in egrads.items():
        assert within_l1(grads[k], eg, l1), (name, k, grads[k][:4], eg[:4])


# ---------------------------------------------------------------------------------------------------- golden replay
def test_qat_golden_replay(golden):
    """Every case of qat.npz through the port's quantizer with the recorded parameters: y and x.grad bit for bit, every
    parameter gradient within 1e-5 L1 of the reference's."""
    g = golden("qat")
    for name in g["cases"]:
        qtype, scheme, target, layout, qmin, qmax, ch_axis, perch, bit = case_geometry(g, name)
        x, gy = g[name + "_x"], g[name + "_gy"]
        if qtype == "pact":
            q = _quantizer(qtype, scheme, bit, target, layout, t(x), alpha=float(g[name + "_alpha"][0]))
        else:
            q = _quantizer(qtype, scheme, bit, target, layout, t(x))
            _set(q, g[name + "_scale"], g[name + "_zp"])
        y, gx, grads = _step(q, t(x), t(gy))
        _, _, egrads = oracle_case(g, name)  # the L1 norms of the summed terms
        want = (g[name + "_y"], g[name + "_gx"], {k: (g[name + GRAD_KEYS[k]], l1) for k, (_, l1) in egrads.items()})
        _check(name, (y, gx, grads), want, dorefa=qtype == "dorefa")
    # the worked example of SURVEY Q19 (signed 8-bit, alpha 1.5, seed 0): the reference's alpha.grad = 45.153
    q = _quantizer("pact", "per-tensor-symmetric", 8, "feature", "NCHW", t(g["pact_s8_a15_x"]), alpha=1.5)
    _, _, grads = _step(q, t(g["pact_s8_a15_x"]), t(g["pact_s8_a15_gy"]))
    assert abs(float(grads["alpha"][0]) - 45.1534) < 1e-5 * oracle_case(g, "pact_s8_a15")[2]["alpha"][1][0]


# ---------------------------------------------------------------------------------------------------- oracle matrix
SCHEME = {"lsq": "per-tensor-symmetric", "lsq+": "per-tensor-affine", "pact_s": "per-tensor-symmetric",
          "pact_u": "per-tensor-affine"}


def _oracle(qtype, x, gy, qmin, qmax, ch_axis, **params):
    if qtype == "pact":
        return oqdq.pact_grads(x, params["alpha"], gy, qmin, qmax)
    return oqdq.lsq_grads(x, params["scale"], params["zero_point"], gy, qmin, qmax, ch_axis,
                          learn_zero_point=qtype == "lsq+" and ch_axis is None)


def _run_case(kind, bit, shape, target="feature", layout="NCHW", per_channel=False, tag=""):
    """Calibrate on planted data, run one step on the kernels and compare with the oracle at the port's parameters."""
    rng = np.random.default_rng(seed_of(kind, bit, shape, tag))
    qtype = "pact" if kind.startswith("pact") else kind
    scheme = ("per-channel-symmetric" if per_channel else SCHEME[kind])
    ch_axis = (0 if target == "weight" else (2 if layout == "NLC" else 1)) if per_channel else None
    x = (rng.standard_normal(shape) * (0.2 if target == "weight" else 1.5)).astype(np.float32)
    gy = rng.standard_normal(shape).astype(np.float32)
    alpha = np.float32(1.5 if kind == "pact_s" else 3.0)
    q = _quantizer(qtype, scheme, bit, target, layout, t(x), alpha=float(alpha))
    qmin, qmax = q.qdesc.qrange
    with torch.no_grad():
        if qtype == "lsq+" and not per_channel:
            _set(q, zero_point=float(torch.round(q.zero_point).reshape(-1)[0]) + 0.5)  # a learned, fractional zero point
        s, z = (v.detach().reshape(-1).cpu().numpy() for v in q._qparams_preprocess(t(x)))
    plant_grid_edges(x, s, z, qmin, qmax, ch_axis)
    if qtype == "pact":
        plant_pact_bounds(x, alpha, qmin < 0)
    params = {"alpha": alpha} if qtype == "pact" else {k: p.detach().reshape(-1).cpu().numpy() for k, p in
                                                       (("scale", q.scale), ("zero_point", q.zero_point))}
    got = _step(q, t(x), t(gy))
    _check(f"{kind} {bit}b {shape}", got, _oracle(qtype, x, gy, qmin, qmax, ch_axis, **params))


@pytest.mark.parametrize("n", [5, 100_003, 2_000_003])
@pytest.mark.parametrize("bit", [2, 4, 8])
@pytest.mark.parametrize("kind", ["lsq", "lsq+", "pact_s", "pact_u"])
def test_per_tensor_matrix(kind, bit, n):
    """n = 5 stays in one CTA; 100 003 and 2 000 003 reach the STE backward's multi-CTA and multi-tile finish paths."""
    _run_case(kind, bit, (1, n))


@pytest.mark.parametrize("bit", [2, 4, 8])
@pytest.mark.parametrize("kind,shape,target,layout", [("lsq", (512, 256, 3, 3), "weight", "NCHW"),
                                                      ("lsq+", (512, 256, 3, 3), "weight", "NCHW"),
                                                      ("lsq", (4096, 1024), "weight", "NCHW"),
                                                      ("lsq+", (4096, 1024), "weight", "NCHW"),
                                                      ("lsq", (8, 197, 768), "feature", "NLC")])
def test_per_channel_matrix(kind, shape, target, layout, bit):
    _run_case(kind, bit, shape, target, layout, per_channel=True)


@pytest.mark.parametrize("bit", [2, 4, 8])
@pytest.mark.parametrize("kind", ["lsq+", "pact_s", "pact_u"])
def test_nlc_activations(kind, bit):
    _run_case(kind, bit, (8, 197, 768), layout="NLC")


# ---------------------------------------------------------------------------------------------------- parameter edges
def _feature_step(qtype, scheme, bit, x, gy, alpha=10.0, **params):
    q = _quantizer(qtype, scheme, bit, "feature", "NCHW", t(x), alpha=alpha)
    _set(q, **params)
    return q, _step(q, t(x), t(gy))


def test_negative_lsq_scale():
    """|s| in the forward; the scale gradient changes sign with s (d|s|/ds = sign s), per tensor and per channel."""
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((4, 3, 9, 9)) * 1.5).astype(np.float32)
    gy = rng.standard_normal(x.shape).astype(np.float32)
    for s in (np.float32(-0.21), np.float32(0.21)):
        q, got = _feature_step("lsq", "per-tensor-symmetric", 4, x, gy, scale=[s], zero_point=[0.0])
        _check(f"lsq s={s}", got, oqdq.lsq_grads(x, [s], [0.0], gy, -8, 7))
    w = (rng.standard_normal((6, 5, 3, 3)) * 0.2).astype(np.float32)
    gw = rng.standard_normal(w.shape).astype(np.float32)
    q = _quantizer("lsq", "per-channel-symmetric", 4, "weight", "NCHW", t(w))
    s = q.scale.detach().reshape(-1).cpu().numpy() * np.array([-1, 1, -1, 1, 1, -1], np.float32)
    _set(q, scale=s)
    got = _step(q, t(w), t(gw))
    _check("lsq per-channel mixed signs", got, oqdq.lsq_grads(w, s, np.zeros(6, np.float32), gw, -8, 7, 0))
    assert np.all(np.sign(got[2]["scale"]) == -np.sign(oqdq.lsq_grads(w, -s, np.zeros(6, np.float32), gw, -8, 7, 0)[2]["scale"][0]))


@pytest.mark.parametrize("zp", [-3.0, 0.0, 0.25, 17.5, 18.5, 255.0, 257.75])
def test_lsq_plus_zero_point_edges(zp):
    """The learned zero point below, on, fractionally inside (incl. .5 ties, rounded half to even) and above [0, 255]:
    the clamp passes its gradient on the closed interval only."""
    rng = np.random.default_rng(seed_of("zp", zp))
    x = (rng.standard_normal((2, 4, 11, 11)) * 1.5).astype(np.float32)
    gy = rng.standard_normal(x.shape).astype(np.float32)
    s = np.float32(0.013)
    plant_grid_edges(x, s, np.clip(zp, 0, 255), 0, 255)
    _, got = _feature_step("lsq+", "per-tensor-affine", 8, x, gy, scale=[s], zero_point=[zp])
    want = oqdq.lsq_grads(x, [s], [zp], gy, 0, 255, learn_zero_point=True)
    _check(f"lsq+ zp={zp}", got, want)
    if not 0 <= zp <= 255:
        assert got[2]["zero_point"][0] == 0.0


def _alpha_near_tie(bit, rounds_past_qmax):
    """An alpha whose bound alpha / scale, (qmax - qmin) / 2 in exact arithmetic, rounds to qmax + 1 or to qmax in fp32."""
    span = np.float32(2 ** bit - 1)
    qmax = 2 ** (bit - 1) - 1
    for a in np.linspace(1.0, 2.0, 4001, dtype=np.float32):
        if (np.rint(a / ((a * np.float32(2)) / span)) > qmax) == rounds_past_qmax:
            return a
    raise AssertionError("no alpha found")


@pytest.mark.parametrize("bit", [4, 8])
@pytest.mark.parametrize("past_qmax", [True, False])
def test_pact_alpha_on_both_sides_of_the_tie(bit, past_qmax):
    """Signed PACT: when +alpha rounds to qmax + 1 the STE masks every element clamped to it; when it rounds to qmax,
    -alpha rounds to qmin + 1 and the clamp narrows the forward grid.  x sits on +-alpha and one ulp either side."""
    alpha = _alpha_near_tie(bit, past_qmax)
    rng = np.random.default_rng(seed_of("tie", bit, past_qmax))
    x = (rng.standard_normal((3, 4, 13, 13)) * 1.5).astype(np.float32)
    gy = rng.standard_normal(x.shape).astype(np.float32)
    qmin, qmax = -2 ** (bit - 1), 2 ** (bit - 1) - 1
    s = (alpha * np.float32(2)) / np.float32(qmax - qmin)
    plant_grid_edges(x, s, 0.0, qmin, qmax)
    plant_pact_bounds(x, alpha, True)
    _, got = _feature_step("pact", "per-tensor-symmetric", bit, x, gy, alpha=float(alpha))
    want = oqdq.pact_grads(x, alpha, gy, qmin, qmax)
    _check(f"pact {bit}b alpha={alpha}", got, want)
    lowest = np.rint(got[0].min() / s)
    assert lowest == (qmin if past_qmax else qmin + 1)


@pytest.mark.parametrize("signed", [True, False])
def test_pact_bounds_and_neighbours(signed):
    """x exactly on the clamp bounds goes to x (closed interval); one ulp outside goes to alpha."""
    alpha = np.float32(1.5)
    x = np.zeros((1, 64), np.float32)
    plant_pact_bounds(x, alpha, signed, at=0)
    gy = np.arange(1, 65, dtype=np.float32).reshape(1, 64)
    scheme = "per-tensor-symmetric" if signed else "per-tensor-affine"
    qmin, qmax = (-128, 127) if signed else (0, 255)
    _, got = _feature_step("pact", scheme, 8, x, gy, alpha=float(alpha))
    _check(f"pact bounds signed={signed}", got, oqdq.pact_grads(x, alpha, gy, qmin, qmax))
    # +alpha rounds past qmax on the signed grid (alpha 1.5): its own gradient and alpha's share from above are masked
    assert got[1][0, 0] == (0.0 if signed else gy[0, 0]) and got[1][0, 1] == gy[0, 1]


# ---------------------------------------------------------------------------------------------------- dtype, repeats
@pytest.mark.parametrize("kind", ["lsq", "lsq+", "pact_s", "pact_u"])
def test_fp16_input(kind):
    """fp16 x: y stays fp32 (SURVEY Q3) and equals the fp32 run; x.grad is fp16, the fp32 gradient cast."""
    rng = np.random.default_rng(seed_of("fp16", kind))
    x16 = (rng.standard_normal((2, 3, 17, 17)) * 1.5).astype(np.float16)
    gy = rng.standard_normal(x16.shape).astype(np.float32)
    qtype = "pact" if kind.startswith("pact") else kind
    q = _quantizer(qtype, SCHEME[kind], 8, "feature", "NCHW", t(x16.astype(np.float32)), alpha=1.5)
    y32, gx32, g32 = _step(q, t(x16.astype(np.float32)), t(gy))
    _zero_grad(q)
    xr = t(x16).requires_grad_(True)
    y = q(xr)
    (y * t(gy)).sum().backward()
    assert y.dtype == torch.float32 and xr.grad.dtype == torch.float16
    assert bits_equal(y.detach().cpu().numpy(), y32)
    assert np.array_equal(xr.grad.cpu().numpy(), gx32.astype(np.float16))
    for k, p in _learnable(q).items():
        assert np.array_equal(p.grad.reshape(-1).cpu().numpy(), g32[k]), k


@pytest.mark.parametrize("kind", ["lsq", "lsq+", "pact_s"])
def test_repeat_is_bit_identical_and_grads_accumulate(kind):
    rng = np.random.default_rng(seed_of("repeat", kind))
    x = (rng.standard_normal((4, 8, 31, 31)) * 1.5).astype(np.float32)
    gy = rng.standard_normal(x.shape).astype(np.float32)
    qtype = "pact" if kind.startswith("pact") else kind
    q = _quantizer(qtype, SCHEME[kind], 4, "feature", "NCHW", t(x), alpha=1.5)
    _, gx1, g1 = _step(q, t(x), t(gy))
    _zero_grad(q)
    _, gx2, g2 = _step(q, t(x), t(gy))
    assert np.array_equal(gx1, gx2)
    for k in g1:
        assert np.array_equal(g1[k], g2[k]), k
    _, _, g3 = _step(q, t(x), t(gy))  # no zero_grad: .grad holds g + g
    for k in g1:
        assert np.array_equal(g3[k], (g1[k] + g1[k]).astype(np.float32)), k


# ---------------------------------------------------------------------------------------------------- module step
class _OracleQuantizer(torch.autograd.Function):
    """A quantizer node of the fp64 graph: forward and backward are the oracle's (``fn(x, params, gy)`` returning
    (y, gx, [(grad, l1)] in the order of ``params``))."""

    @staticmethod
    def forward(ctx, fn, x, *params):
        ctx.fn, ctx.x, ctx.params = fn, x.detach().float().cpu().numpy(), [p.detach().cpu().numpy() for p in params]
        ctx.shapes = [p.shape for p in params]
        y, _, _ = fn(ctx.x, ctx.params, np.zeros_like(ctx.x))
        return torch.from_numpy(np.asarray(y, np.float64)).to(x.device)

    @staticmethod
    def backward(ctx, gy):
        _, gx, grads = ctx.fn(ctx.x, ctx.params, gy.detach().float().cpu().numpy())
        dev_ = gy.device
        return (None, torch.from_numpy(np.asarray(gx, np.float64)).to(dev_),
                *(torch.from_numpy(np.asarray(g, np.float64)).reshape(shp).to(dev_) for (g, _), shp in zip(grads, ctx.shapes)))


def _oracle_fn(q):
    """The oracle chain of the port's quantizer q, for _OracleQuantizer."""
    qmin, qmax = q.qdesc.qrange
    if q.TYPE == "PACT":
        return lambda x, p, gy: _ordered(oqdq.pact_grads(x, p[0], gy, qmin, qmax), ["alpha"])
    ch_axis = q.qdesc.ch_axis if q.qdesc.is_perchannel else None
    if isinstance(q.zero_point, torch.nn.Parameter):
        return lambda x, p, gy: _ordered(oqdq.lsq_grads(x, p[0], p[1], gy, qmin, qmax, ch_axis, learn_zero_point=True),
                                         ["scale", "zero_point"])
    zp = q.zero_point.detach().reshape(-1).cpu().numpy()
    return lambda x, p, gy: _ordered(oqdq.lsq_grads(x, p[0], zp, gy, qmin, qmax, ch_axis), ["scale"])


def _ordered(res, names):
    y, gx, grads = res
    return y, gx, [grads[k] for k in names]


def _l1_of(fn, x, params, weight):
    """L1 norms of the oracle's summed parameter terms for the incoming gradient ``weight``."""
    return [l1 for _, l1 in fn(x, params, weight)[2]]


@pytest.mark.parametrize("op", ["conv", "linear"])
def test_module_step_matches_fp64_autograd(op):
    """One QAT step of QConv2d (LSQ 4-bit per-channel weights, LSQ+ 8-bit per-tensor affine inputs) and QLinear (LSQ
    8-bit per-channel weights, signed 8-bit PACT inputs with alpha 1.5) against fp64 autograd over the same graph:
    conv / linear in fp64, quantizer nodes from the oracle.

    Bounds.  The quantized operands are bit-identical on both sides (the forward tests above), so the only differences
    are the fp32 sums of the conv / linear backward.  dL/d(quantized input) and dL/d(quantized weight) are sums of K
    products each; in fp32 each stays within (K + 2) u of the same sum of absolute products, A = |gout| (x) |w| or
    |x| (x) |gout| (the backward of the op applied to absolute values, in fp64).  The STE passes them through or zeroes
    them, so x.grad and weight.grad inherit that bound.  A parameter gradient sums terms t_i dL/dy_i: its error is
    within (K + 2) u sum |t_i| A_i (the oracle's L1 with A as the incoming gradient) plus 1e-5 L1 for its own sum.
    The bias gradient sums n = N H W outputs: (n + 2) u sum |gout|."""
    torch.manual_seed(seed_of("module", op))
    if op == "conv":
        mod = torch.nn.Conv2d(8, 16, 3, padding=1).to(dev())
        x = torch.randn(2, 8, 10, 10, device=dev()) * 1.5
        a_cfg = sbcfg.quantizer_config("per-tensor-affine", 8, "feature", qtype="lsq+")
        w_cfg = sbcfg.quantizer_config("per-channel-symmetric", 4, "weight", qtype="lsq")
        qmod = QConv2d(mod)
    else:
        mod = torch.nn.Linear(64, 32).to(dev())
        x = torch.randn(6, 64, device=dev()) * 1.5
        a_cfg = sbcfg.quantizer_config("per-tensor-symmetric", 8, "feature", qtype="pact", pact_alpha=1.5)
        w_cfg = sbcfg.quantizer_config("per-channel-symmetric", 8, "weight", qtype="lsq")
        qmod = QLinear(mod)
    qmod.build_quantizer(a_cfg, w_cfg)
    qmod.to(dev())
    qmod.input_quantizer.update_observer(x)
    qmod.weight_quantizer.update_observer(qmod.weight.detach())
    qmod.input_quantizer.calc_qparams()
    qmod.weight_quantizer.calc_qparams()
    if op == "conv":  # a learned, fractional zero point
        _set(qmod.input_quantizer, zero_point=float(torch.round(qmod.input_quantizer.zero_point.detach()).reshape(-1)[0]) + 0.5)
    qmod.set_quant(w_quant=True, a_quant=True)
    xr = x.clone().requires_grad_(True)
    out = qmod(xr)
    gout = torch.randn_like(out)
    (out * gout).sum().backward()

    # the fp64 graph
    aq, wq = qmod.input_quantizer, qmod.weight_quantizer
    a_fn, w_fn = _oracle_fn(aq), _oracle_fn(wq)
    a_params = [p.detach().double().clone().requires_grad_(True) for p in _learnable(aq).values()]
    w_params = [p.detach().double().clone().requires_grad_(True) for p in _learnable(wq).values()]
    x64 = x.double().requires_grad_(True)
    w64 = qmod.weight.detach().double().requires_grad_(True)
    b64 = qmod.bias.detach().double().requires_grad_(True)
    ya = _OracleQuantizer.apply(a_fn, x64, *a_params)
    yw = _OracleQuantizer.apply(w_fn, w64, *w_params)
    ya.retain_grad()
    yw.retain_grad()
    fwd = (lambda a, w, b: F.conv2d(a, w, b, padding=1)) if op == "conv" else F.linear
    ref = fwd(ya, yw, b64)
    (ref * gout.double()).sum().backward()

    # the sums of absolute products behind each backward sum, and their lengths
    g_abs = gout.double().abs()
    ya_d, yw_d = ya.detach().requires_grad_(True), yw.detach().requires_grad_(True)
    A_in = torch.autograd.grad(fwd(ya_d, yw.detach().abs(), None), ya_d, g_abs)[0]
    A_w = torch.autograd.grad(fwd(ya.detach().abs(), yw_d, None), yw_d, g_abs)[0]
    if op == "conv":
        k_in, k_w = qmod.weight.shape[0] * qmod.weight[0, 0].numel(), x.shape[0] * out.shape[2] * out.shape[3]
    else:
        k_in, k_w = qmod.weight.shape[0], x.shape[0]
    bound_in = (k_in + 2) * U * A_in.cpu().numpy()
    bound_w = (k_w + 2) * U * A_w.cpu().numpy()
    assert np.all(np.abs(xr.grad.double().cpu().numpy() - x64.grad.cpu().numpy()) <= bound_in), op
    assert np.all(np.abs(qmod.weight.grad.double().cpu().numpy() - w64.grad.cpu().numpy()) <= bound_w), op
    n_b = gout.numel() // gout.shape[1]
    bias_bound = (n_b + 2) * U * g_abs.sum(dim=[d for d in range(gout.dim()) if d != 1]).cpu().numpy()
    assert np.all(np.abs(qmod.bias.grad.double().cpu().numpy() - b64.grad.cpu().numpy()) <= bias_bound), op
    for quant, params, fn, xin, y64, A, k in ((aq, a_params, a_fn, x, ya, A_in, k_in), (wq, w_params, w_fn, qmod.weight, yw, A_w, k_w)):
        xn = xin.detach().float().cpu().numpy()
        pn = [p.detach().cpu().numpy() for p in params]
        ref_l1 = _l1_of(fn, xn, pn, y64.grad.float().cpu().numpy())
        prop = _l1_of(fn, xn, pn, A.float().cpu().numpy())
        for (name, p), p64, l1, a_l1 in zip(_learnable(quant).items(), params, ref_l1, prop):
            got = p.grad.double().reshape(-1).cpu().numpy()
            want = p64.grad.reshape(-1).cpu().numpy()
            tol = 1e-5 * np.asarray(l1) + (k + 2) * U * np.asarray(a_l1)
            assert np.all(np.abs(got - want) <= tol), (op, name, got[:4], want[:4])
