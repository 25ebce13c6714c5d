"""GPU: the integer-grid linear (sb200_int8_quantize_rows, sb200_int8_linear, QLinearInt8, to_integer_linears).

* The integer grid equals oracle.qdq.quantize_int bit for bit (stored with the 128 offset for unsigned ranges), with
  ties, +-inf, NaN, +-0, subnormals, ragged K (zero padding), row sums and NaN flags.
* Exact mode: with power-of-two scales and zero bias, every output whose integer sum I is exact in fp32 equals the
  fp64 truth bit for bit -- symmetric and affine ranges with the zero points at qmin / qmax, 2 / 4 / 8 bits, ragged M
  and N, K from 16 to 11008, and the int32 edge K = 2^17 - 1 with every operand -128.
* General data with MinMax qparams: |y - T| <= 2^-21 (sum |fx fw| + |bias|) elementwise (tests/int8_linear_ref.py);
  NaN rows, inf inputs, determinism, CUDA graph replay, K = 2^17 unsupported.
* Modules: calibrated models converted by to_integer_linears meet the same bound per layer."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from gpu_util import dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from int8_harness import calibrated, cfg, check_converted, layer_qparams, qrange, stored_rows
from int8_linear_ref import grid_offset, truth
from oracle import observers as oobs
from oracle import qdq as oqdq
from sparsebit_b200 import SparsebitB200Error, ops
from sparsebit_b200.quantization.modules import QConv2d, QLinear, QLinearInt8, QReLU
from sparsebit_b200.quantization.tools import to_integer_linears

pytestmark = pytest.mark.gpu

F32 = np.float32


# ---------------------------------------------------------------------------------------------- the integer grid
def _specials(rng, x, s):
    """Ties (k + 1/2) s, +-inf, NaN (row 1 only), +-0 and subnormals spread over the rows."""
    rows, k = x.shape
    s = np.broadcast_to(np.asarray(s, F32).reshape(-1, 1), (rows, 1))
    ties = rng.integers(-140, 140, (rows, k)).astype(F32) + F32(0.5)
    pick = rng.random((rows, k)) < 0.25
    x = np.where(pick, (ties * s).astype(F32), x)
    special = np.array([np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39], F32)
    for r in range(rows):
        cols = rng.choice(k, size=min(k, len(special)), replace=False)
        x[r, cols] = special[: len(cols)]
    if rows > 1:
        x[1, rng.integers(0, k)] = np.nan
    return x


@pytest.mark.parametrize("qrange", [(-128, 127), (0, 255), (-8, 7), (0, 15), (-2, 1)])
@pytest.mark.parametrize("per_row", [False, True])
@pytest.mark.parametrize("k", [16, 33, 768, 1001])
def test_grid_is_the_oracle_grid(qrange, per_row, k):
    qmin, qmax = qrange
    rng = np.random.default_rng(k * 7 + qmin + 200 + per_row)
    rows = 37
    x = (rng.standard_normal((rows, k)) * 40).astype(F32)
    if per_row:
        s = (rng.uniform(0.05, 2.0, rows)).astype(F32)
        z = rng.integers(qmin, qmax + 1, rows).astype(F32) + F32(0.3) * rng.integers(-1, 2, rows).astype(F32)
    else:
        s = np.array([0.37], F32)
        z = np.array([(qmin + qmax) // 2 + 0.5], F32)  # a tie of rint: half-to-even
    x = _specials(rng, x, s)
    q, row_sum, nan = ops.int8_quantize_rows(t(x), t(s), t(z), qmin, qmax)
    kp = (k + 15) // 16 * 16
    assert q.shape == (rows, kp) and q.dtype == torch.int8
    q, row_sum, nan = q.cpu().numpy(), row_sum.cpu().numpy(), nan.cpu().numpy()
    exp = oqdq.quantize_int(x, s if per_row else s[0], z if per_row else z[0], qmin, qmax)
    exp_nan = np.isnan(exp)
    stored = np.where(exp_nan, 0, np.nan_to_num(exp) - grid_offset(qmin)).astype(np.int64)
    assert np.array_equal(q[:, :k].astype(np.int64), stored)
    assert not q[:, k:].any()  # zero padding
    assert np.array_equal(row_sum.astype(np.int64), stored.sum(axis=1))
    assert np.array_equal(nan, exp_nan.any(axis=1))
    assert nan[1] and nan.sum() == 1


def test_grid_matches_the_qdq_kernel_values():
    """The grid the integer path stores is the one the fake-quant kernel dequantizes: (g - Z) s == qdq(x)."""
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((64, 300)) * 3).astype(F32)
    s, z = np.array([0.021], F32), np.array([7.0], F32)
    q, _, _ = ops.int8_quantize_rows(t(x), t(s), t(z), 0, 255)
    v = (q[:, :300].cpu().numpy().astype(F32) + F32(128) - z[0]).astype(F32)
    from sparsebit_b200 import fake_quant
    y = fake_quant.quant_pertensor_forward(t(x), t(s), t(z), 0, 255, 0).cpu().numpy()
    assert np.array_equal((v * s[0]).astype(F32), y)


# ---------------------------------------------------------------------------------------------- the GEMM
def _run(x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax, bias=None):
    w_q, w_sum, w_scale, w_zero = stored_rows(w, ws, wz, wqmin, wqmax)
    y = ops.int8_linear(t(x), t(np.array([xs], F32)), t(np.array([xz], F32)), xqmin, xqmax, w_q, w_sum, w_scale, w_zero,
                        None if bias is None else t(bias))
    return y.cpu().numpy().reshape(-1, w.shape[0])


def _exact_case(rng, m, k, n, xr, wr, zx_at=None, zw_at=None):
    (xqmin, xqmax), (wqmin, wqmax) = xr, wr
    xs, ws = F32(2.0 ** -4), (2.0 ** -rng.integers(3, 8, n)).astype(F32)
    zx = {None: 0 if xqmin < 0 else (xqmin + xqmax) // 2, "min": xqmin, "max": xqmax}[zx_at]
    zw = {None: np.zeros(n) if wqmin < 0 else rng.integers(wqmin, wqmax + 1, n), "min": np.full(n, wqmin),
          "max": np.full(n, wqmax)}[zw_at].astype(F32)
    # values spread over (and beyond) the whole grid, so that both clamps are hit
    span_x = (xqmax - xqmin) * float(xs)
    x = rng.uniform(-0.7 * span_x, 0.7 * span_x, (m, k)).astype(F32)
    w = (rng.uniform(-0.7, 0.7, (n, k)) * (wqmax - wqmin) * ws[:, None]).astype(F32)
    return x, xs, F32(zx), xqmin, xqmax, w, ws, zw, wqmin, wqmax


def _assert_exact(y, args, bias=None):
    t_, _ = truth(*args, bias=bias)
    xs, ws = float(args[1]), np.broadcast_to(np.asarray(args[6], np.float64).reshape(-1), (y.shape[1],))
    i = t_ / (xs * ws[None, :])
    exact = i.astype(F32).astype(np.float64) == i  # I is exactly representable in fp32
    assert exact.mean() > 0.5
    assert np.array_equal(y.astype(np.float64)[exact], t_[exact])


EXACT = [
    # (m, k, n, x range, w range, zx, zw)
    (1, 16, 8, (-128, 127), (-128, 127), None, None),
    (7, 33, 100, (-128, 127), (-128, 127), None, None),
    (591, 768, 2304, (-128, 127), (-128, 127), None, None),
    (7, 3072, 100, (-128, 127), (-128, 127), None, None),
    (591, 11008, 100, (-128, 127), (-128, 127), None, None),
    (1, 11008, 2304, (-128, 127), (-128, 127), None, None),
    (7, 768, 8, (0, 255), (0, 255), "min", "min"),
    (7, 768, 100, (0, 255), (0, 255), "max", "max"),
    (591, 33, 100, (0, 255), (0, 255), "min", "max"),
    (7, 3072, 2304, (0, 255), (-128, 127), "max", None),
    (7, 768, 100, qrange(4, False), qrange(4, False), None, None),
    (7, 768, 100, qrange(4, True), qrange(4, True), "max", "min"),
    (7, 768, 100, qrange(2, False), qrange(2, True), None, "max"),
    (7, 768, 100, qrange(2, True), qrange(2, False), "min", None),
    (1, 33, 8, qrange(2, True), qrange(4, True), "max", "max"),
]


@pytest.mark.parametrize("m,k,n,xr,wr,zx_at,zw_at", EXACT)
def test_exact_mode(m, k, n, xr, wr, zx_at, zw_at):
    rng = np.random.default_rng(m * 131 + k + n)
    args = _exact_case(rng, m, k, n, xr, wr, zx_at, zw_at)
    y = _run(*args, bias=np.zeros(n, F32))
    _assert_exact(y, args)


def test_int32_edge():
    """K = 2^17 - 1 with every operand at -128: sum a b = (2^17 - 1) 2^14, the largest the accumulator meets."""
    k, m, n = (1 << 17) - 1, 3, 24
    x = np.full((m, k), -1000.0, F32)
    w = np.full((n, k), -1000.0, F32)
    args = (x, F32(0.5), F32(0), -128, 127, w, np.full(n, 0.25, F32), np.zeros(n, F32), -128, 127)
    y = _run(*args)
    assert np.all(y == F32(k * 2 ** 14 * 0.125))


def _minmax_case(rng, m, k, n, affine_x, per_channel_w):
    x = (rng.standard_normal((m, k)) * 2 + (0.8 if affine_x else 0)).astype(F32)
    w = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(F32)
    xqmin, xqmax = (0, 255) if affine_x else (-128, 127)
    xs, xz = oobs.calc_qparams_with_minmax(*oobs.minmax([x]), xqmin, xqmax, not affine_x)
    ws, wz = oobs.calc_qparams_with_minmax(*oobs.minmax([w], per_channel=per_channel_w), -128, 127, True)
    bias = rng.standard_normal(n).astype(F32)
    return (x, F32(xs), F32(xz), xqmin, xqmax, w, ws, wz, -128, 127), bias


@pytest.mark.parametrize("m,k,n,affine_x,per_channel_w", [(197 * 3, 768, 2304, False, True), (64, 3072, 768, True, True),
                                                          (7, 33, 100, True, False), (300, 11008, 264, False, True)])
def test_general_data_meets_the_bound(m, k, n, affine_x, per_channel_w):
    rng = np.random.default_rng(m + k + n)
    args, bias = _minmax_case(rng, m, k, n, affine_x, per_channel_w)
    y = _run(*args, bias=bias)
    t_, bound = truth(*args, bias=bias)
    err = np.abs(y - t_)
    assert np.all(err <= bound), float((err / bound).max())


def test_nan_rows_and_inf_inputs():
    rng = np.random.default_rng(11)
    args, bias = _minmax_case(rng, 40, 200, 72, False, True)
    x = args[0].copy()
    x[3, 17] = np.nan
    x[5, 0], x[6, 199], x[7, 100] = np.inf, -np.inf, np.inf
    args = (x,) + args[1:]
    y = _run(*args, bias=bias)
    t_, bound = truth(*args, bias=bias)
    assert np.isnan(y[3]).all() and np.isnan(y).sum() == y.shape[1]
    ok = np.arange(40) != 3
    assert np.isfinite(y[ok]).all() and np.all(np.abs(y[ok] - t_[ok]) <= bound[ok])


def test_deterministic_and_graph_replay():
    rng = np.random.default_rng(12)
    (x, xs, xz, xqmin, xqmax, w, ws, wz, wqmin, wqmax), bias = _minmax_case(rng, 517, 768, 300, True, True)
    w_q, w_sum, w_scale, w_zero = stored_rows(w, ws, wz, wqmin, wqmax)
    xt, xst, xzt, bt = t(x), t(np.array([xs], F32)), t(np.array([xz], F32)), t(bias)

    def call():
        return ops.int8_linear(xt, xst, xzt, xqmin, xqmax, w_q, w_sum, w_scale, w_zero, bt)

    y1, y2 = call(), call()
    assert torch.equal(y1, y2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()  # warm the per-stream workspace outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            yg = call()
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        xt.copy_(t(x))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, y1)


def test_k_limit_is_unsupported():
    k = 1 << 17
    x = torch.zeros(2, k, device=dev())
    one = torch.ones(1, device=dev())
    w_q = torch.zeros(8, k, dtype=torch.int8, device=dev())
    i32 = torch.zeros(8, dtype=torch.int32, device=dev())
    with pytest.raises(SparsebitB200Error, match=r"K < 2\^17.*status -3"):
        ops.int8_linear(x, one, one * 0, -128, 127, w_q, i32, torch.ones(8, device=dev()), i32)


# ---------------------------------------------------------------------------------------------- modules
class CnnHead(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = QConv2d(nn.Conv2d(3, 16, 3, stride=2)).build_quantizer(cfg("per-tensor-symmetric", "feature"),
                                                                           cfg("per-channel-symmetric", "weight"))
        self.relu = QReLU().build_quantizer(cfg("per-tensor-symmetric", "feature", disable=True))
        self.fc1 = QLinear(nn.Linear(16 * 7 * 7, 120)).build_quantizer(cfg("per-tensor-affine", "feature"),
                                                                        cfg("per-channel-symmetric", "weight"))
        self.fc2 = QLinear(nn.Linear(120, 10)).build_quantizer(cfg("per-tensor-symmetric", "feature"),
                                                                cfg("per-tensor-symmetric", "weight"))

    def forward(self, x):
        x = torch.flatten(self.relu(self.conv(x)), 1)
        return self.fc2(torch.relu(self.fc1(x)))


class DeitMlp(nn.Module):
    """The MLP of a DeiT-base block plus an ineligible projection (per-channel activations)."""

    def __init__(self):
        super().__init__()
        self.fc1 = QLinear(nn.Linear(768, 3072)).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"),
                                                                  cfg("per-channel-symmetric", "weight"))
        self.fc2 = QLinear(nn.Linear(3072, 768)).build_quantizer(cfg("per-tensor-affine", "feature", layout="NLC"),
                                                                  cfg("per-channel-symmetric", "weight"))
        self.proj = QLinear(nn.Linear(768, 64)).build_quantizer(cfg("per-channel-symmetric", "feature", layout="NLC"),
                                                                 cfg("per-channel-symmetric", "weight"))

    def forward(self, x):
        return self.proj(self.fc2(nn.functional.gelu(self.fc1(x))))


def _truth_of(qlinear, x):
    return truth(**layer_qparams(qlinear, x))


def test_cnn_head_converts_and_meets_the_bound():
    torch.manual_seed(0)
    batches = [torch.randn(8, 3, 16, 16, device=dev()) for _ in range(3)]
    model = calibrated(CnnHead(), batches, streaming=True, record_inputs=None)
    originals = {"fc1": model.fc1, "fc2": model.fc2}
    names = to_integer_linears(model)
    assert names == ["fc1", "fc2"]
    assert isinstance(model.fc1, QLinearInt8) and isinstance(model.fc2, QLinearInt8) and isinstance(model.conv, QConv2d)
    check_converted(model, originals, batches[:2], names, expected_cls=QLinearInt8, layer_truth=_truth_of,
                    compare_fake_quant=True)


def test_deit_mlp_converts_and_meets_the_bound():
    torch.manual_seed(1)
    batches = [torch.randn(2, 197, 768, device=dev()) for _ in range(2)]
    model = calibrated(DeitMlp(), batches, streaming=True, record_inputs=None)
    originals = {"fc1": model.fc1, "fc2": model.fc2}
    assert to_integer_linears(model) == ["fc1", "fc2"]
    assert isinstance(model.proj, QLinear)  # per-channel activations: not eligible, left alone
    check_converted(model, originals, batches[:1], ["fc1", "fc2"], expected_cls=QLinearInt8, layer_truth=_truth_of,
                    compare_fake_quant=True)


def test_module_input_forms():
    torch.manual_seed(2)
    batches = [torch.randn(4, 197, 768, device=dev())]
    model = calibrated(DeitMlp(), batches, streaming=True, record_inputs=None)
    to_integer_linears(model)
    fc1 = model.fc1
    x = batches[0]
    with torch.no_grad():
        y3 = fc1(x)
        assert y3.shape == (4, 197, 3072) and y3.dtype == torch.float32
        assert torch.equal(y3.reshape(-1, 3072), fc1(x.reshape(-1, 768)))
        x16 = x.half()
        assert torch.equal(fc1(x16), fc1(x16.float()))
    xg = x.clone().requires_grad_()
    with pytest.raises(RuntimeError, match="no backward"):
        fc1(xg)
    with torch.no_grad():
        fc1(xg)  # no graph to cut under no_grad


def test_weight_nan_row_gives_a_nan_column():
    torch.manual_seed(3)
    model = calibrated(CnnHead(), [torch.randn(8, 3, 16, 16, device=dev())], streaming=True, record_inputs=None)
    with torch.no_grad():
        model.fc2.weight[4, 7] = float("nan")
    conv = QLinearInt8.from_qlinear(model.fc2)
    with torch.no_grad():
        y = conv(torch.randn(5, 120, device=dev())).cpu().numpy()
    assert np.isnan(y[:, 4]).all() and np.isfinite(np.delete(y, 4, axis=1)).all()
