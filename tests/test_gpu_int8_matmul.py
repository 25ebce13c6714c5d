"""GPU: the integer-grid matmul (sb200_int8_quantize_cols, sb200_int8_matmul, QMatMulInt8, to_integer_matmuls).

* The column quantizer equals the oracle's integer grid, transposed, bit for bit (tests/int8_matmul_ref.py): K not a
  multiple of 16, N not a multiple of 4 and a misaligned base (the scalar loads), signed / unsigned / 4- and 2-bit
  ranges, zero points away from 0, ties, +-inf and NaN, several batch entries.
* The matmul is exact for power-of-two scales and within 2^-21 (|fa| @ |fb|) otherwise: DeiT-tiny / -base head shapes
  (both products, both layouts of b), M / N around 64 and 128, K from 1 to 1000, broadcast leading dimensions.
* Batch entries are isolated: extreme and NaN neighbours change nothing; NaN rows / columns stay inside their entry.
* It equals QLinearInt8's arithmetic when b is a weight matrix with the same per-tensor qparams.
* CUDA graph replay with new inputs; two streams use two workspaces.
* An attention block calibrated by CalibrationRunner (streaming and the fx replay), converted by to_integer_linears +
  to_integer_matmuls: no QMatMul / QLinear is left, every matmul meets the bound, and a forward launches exactly the
  library's 10 kernels, no ATen matmul and no foreign GEMM kernel."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from gpu_util import dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from int8_harness import calibrated, cfg, qrange, scalar
from int8_matmul_ref import grid_offset, integer_form, quantize_cols, truth
from sparsebit_b200 import SparsebitB200Error, launch_count, ops
from sparsebit_b200.quantization.modules import QLinear, QLinearInt8, QMatMul, QMatMulInt8
from sparsebit_b200.quantization.tools import to_integer_linears, to_integer_matmuls

pytestmark = pytest.mark.gpu

F32 = np.float32


# ---------------------------------------------------------------------------------------------- the column quantizer
def _specials(rng, x, s):
    """Ties (k + 1/2) s, +-inf, +-0, subnormals; one NaN in batch entry 0."""
    ties = (rng.integers(-140, 140, x.shape).astype(F32) + F32(0.5)) * F32(s)
    x = np.where(rng.random(x.shape) < 0.25, ties.astype(F32), x)
    flat = x.reshape(-1)
    special = np.array([np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39], F32)
    flat[rng.choice(flat.size, size=min(len(special), flat.size), replace=False)] = special[:flat.size]
    x = flat.reshape(x.shape)
    x[0, rng.integers(0, x.shape[1]), rng.integers(0, x.shape[2])] = np.nan
    return x


COLS = [(1, 16, 4), (3, 15, 7), (2, 17, 64), (2, 129, 197), (4, 197, 64), (1, 1000, 130), (2, 64, 128), (5, 1, 1), (2, 260, 68)]
COL_RANGES = [((-128, 127), 0), ((0, 255), 131), ((-8, 7), 0), ((0, 15), 6), ((-2, 1), 0)]


@pytest.mark.parametrize("qrange,z", COL_RANGES)
@pytest.mark.parametrize("batch,k,n", COLS)
@pytest.mark.parametrize("misaligned", [False, True])
def test_cols_grid_is_the_transposed_oracle_grid(batch, k, n, qrange, z, misaligned):
    if misaligned and (n % 4 != 0 or qrange != (0, 255)):
        pytest.skip("the misaligned base matters where the vector loads would otherwise run")
    rng = np.random.default_rng(batch * 7919 + k * 31 + n + qrange[1])
    s = F32(0.037)
    x = _specials(rng, (rng.standard_normal((batch, k, n)) * 0.4 * (qrange[1] - qrange[0]) * s).astype(F32), s)
    if misaligned:  # base pointer 4 bytes past a 16-byte boundary
        xt = torch.empty(x.size + 1, device=dev())[1:].view(x.shape)
        xt.copy_(t(x))
        assert xt.data_ptr() % 16 == 4 and xt.is_contiguous()
    else:
        xt = t(x)
        assert xt.data_ptr() % 16 == 0
    q, col_sum, nan = ops.int8_quantize_cols(xt, scalar(s), scalar(z), *qrange)
    eq, esum, enan = quantize_cols(x, s, z, *qrange)
    assert enan.sum() == 1 and enan[0].any()
    assert q.shape == eq.shape and np.array_equal(q.cpu().numpy(), eq)
    assert np.array_equal(col_sum.cpu().numpy(), esum)
    assert np.array_equal(nan.cpu().numpy(), enan)


def test_cols_equals_rows_of_the_transpose():
    rng = np.random.default_rng(3)
    x = (rng.standard_normal((3, 2, 197, 64)) * 2).astype(F32)
    s, z = scalar(0.02), scalar(117)
    q, col_sum, nan = ops.int8_quantize_cols(t(x), s, z, 0, 255)
    qr, row_sum, rnan = ops.int8_quantize_rows(t(np.swapaxes(x, -1, -2)).reshape(-1, 197), s, z, 0, 255)
    assert torch.equal(q.reshape(-1, q.shape[-1]), qr) and torch.equal(col_sum.reshape(-1), row_sum)
    assert torch.equal(nan.reshape(-1), rnan)


# ---------------------------------------------------------------------------------------------- the matmul
def _operand(rng, shape, qrange, pow2, z_at=None):
    qmin, qmax = qrange
    z = {None: 0 if qmin < 0 else (qmin + qmax) // 2 + 3, "min": qmin, "max": qmax}[z_at]
    if pow2:  # values spread over (and beyond) the whole grid, so that both clamps are hit
        s = F32(2.0 ** -4)
        x = rng.uniform(-0.7, 0.7, shape) * (qmax - qmin) * float(s)
    else:
        x = rng.standard_normal(shape) * 1.7 + (0.0 if qmin < 0 else 1.1)
        s = F32((x.max() - x.min()) / (qmax - qmin) * 0.93)
        if qmin >= 0:
            z = int(np.clip(np.rint(qmin - x.min() / s), qmin, qmax))
    return x.astype(F32), s, F32(z), qmin, qmax


def _matmul(a, b, k_major):
    """ops.int8_matmul of two operand tuples; ``k_major``: b reaches the op as the transposed view of a contiguous
    [..., N, K] tensor."""
    bt = t(np.swapaxes(b[0], -1, -2)).transpose(-2, -1) if k_major else t(b[0])
    assert bt.shape == b[0].shape and bt.is_contiguous() == (not k_major or min(b[0].shape[-2:]) == 1)
    y = ops.int8_matmul(t(a[0]), scalar(a[1]), scalar(a[2]), a[3:], bt, scalar(b[1]), scalar(b[2]), b[3:])
    return y.cpu().numpy()


def _check(a, b, pow2, k_major):
    y = _matmul(a, b, k_major)
    t_, bound = truth(a, b)
    assert y.shape == t_.shape and y.dtype == F32
    if pow2:
        i = integer_form(a, b)[4].astype(np.float64)
        exact = i.astype(F32).astype(np.float64) == i  # I is exactly representable in fp32
        assert exact.mean() > 0.5
        assert np.array_equal(y.astype(np.float64)[exact], t_[exact])
    err = np.abs(y - t_)
    assert np.all(err <= bound), float((err / np.maximum(bound, 1e-300)).max())
    # and it is the integer form, rounded once
    assert np.array_equal(y, integer_form(a, b)[-1].astype(F32))


DEIT = [((4, 3, 197, 64), (4, 3, 64, 197)),     # DeiT-tiny q @ k^T
        ((4, 3, 197, 197), (4, 3, 197, 64)),    # DeiT-tiny p @ v
        ((2, 12, 197, 64), (2, 12, 64, 197)),   # DeiT-base q @ k^T
        ((2, 12, 197, 197), (2, 12, 197, 64))]  # DeiT-base p @ v


@pytest.mark.parametrize("ashape,bshape", DEIT)
@pytest.mark.parametrize("k_major", [True, False])
@pytest.mark.parametrize("pow2", [True, False])
def test_deit_head_shapes(ashape, bshape, k_major, pow2):
    rng = np.random.default_rng(ashape[1] * 1000 + ashape[3] + 2 * k_major + pow2)
    a = _operand(rng, ashape, (0, 255) if ashape[3] == 197 else (-128, 127), pow2)  # softmax output: unsigned
    b = _operand(rng, bshape, (-128, 127), pow2)
    _check(a, b, pow2, k_major)


EDGES = [(63, 64, 63), (64, 64, 64), (65, 64, 65), (127, 64, 129), (128, 64, 128), (129, 64, 127),
         (65, 1, 130), (130, 15, 63), (5, 16, 5), (64, 17, 128), (70, 128, 3), (1, 129, 1), (129, 197, 66), (67, 1000, 131)]


@pytest.mark.parametrize("m,k,n", EDGES)
@pytest.mark.parametrize("batch", [(), (5,)])
@pytest.mark.parametrize("k_major", [True, False])
def test_tile_and_k_edges(m, k, n, batch, k_major):
    rng = np.random.default_rng(m * 131 + k * 7 + n + len(batch))
    pow2 = (m + k) % 2 == 0
    ar, br = [((-128, 127), (0, 255)), ((0, 255), (-128, 127)), ((0, 15), (-8, 7))][(m + n) % 3]
    a = _operand(rng, batch + (m, k), ar, pow2, z_at=[None, "min", "max"][k % 3] if ar[0] >= 0 else None)
    b = _operand(rng, batch + (k, n), br, pow2, z_at=[None, "max", "min"][n % 3] if br[0] >= 0 else None)
    _check(a, b, pow2, k_major)


@pytest.mark.parametrize("ashape,bshape", [((3, 1, 40, 24), (1, 4, 24, 50)), ((40, 24), (2, 3, 24, 50)), ((2, 3, 40, 24), (24, 50)),
                                           ((4, 40, 24), (3, 1, 24, 50))])
@pytest.mark.parametrize("k_major", [True, False])
def test_leading_dimensions_broadcast(ashape, bshape, k_major):
    rng = np.random.default_rng(len(ashape) * 10 + len(bshape))
    _check(_operand(rng, ashape, (-128, 127), False), _operand(rng, bshape, (0, 255), False), False, k_major)


def test_non_contiguous_operands_are_taken():
    """The q, k, v of a fused qkv projection are strided views: neither contiguous nor a plain transpose."""
    rng = np.random.default_rng(11)
    qkv = (rng.standard_normal((2, 50, 3, 4, 32))).astype(F32)
    a, b = (None, F32(0.031), F32(0), -128, 127), (None, F32(0.027), F32(0), -128, 127)
    q, k = np.transpose(qkv[:, :, 0], (0, 2, 1, 3)), np.transpose(qkv[:, :, 1], (0, 2, 1, 3))
    qt, kt = t(qkv)[:, :, 0].permute(0, 2, 1, 3), t(qkv)[:, :, 1].permute(0, 2, 1, 3)
    assert not qt.is_contiguous() and not kt.is_contiguous()
    y = ops.int8_matmul(qt, scalar(a[1]), scalar(a[2]), a[3:], kt.transpose(-2, -1), scalar(b[1]), scalar(b[2]), b[3:])
    an, bn = (q,) + a[1:], (np.swapaxes(k, -1, -2),) + b[1:]
    assert np.array_equal(y.cpu().numpy(), integer_form(an, bn)[-1].astype(F32))


def test_int32_edge():
    """K = 2^17 - 1 with every operand at -128: sum a b = (2^17 - 1) 2^14, the largest the accumulator meets."""
    k = (1 << 17) - 1
    a = (np.full((2, 3, k), -1000.0, F32), F32(1.0), F32(0), -128, 127)
    b = (np.full((2, k, 5), -1000.0, F32), F32(0.5), F32(0), -128, 127)
    for k_major in (True, False):
        y = _matmul(a, b, k_major)
        assert np.all(y == F32(k * 16384 * 0.5))


def test_argument_errors():
    one = torch.ones(1, device=dev())
    x = torch.zeros(1, 2, 1 << 17, device=dev())
    with pytest.raises(SparsebitB200Error, match=r"K < 2\^17.*status -3"):
        ops.int8_matmul(x, one, one * 0, (-128, 127), x.transpose(-2, -1), one, one * 0, (-128, 127))
    with pytest.raises(SparsebitB200Error, match=r"K < 2\^17.*status -3"):
        ops.int8_quantize_cols(x.transpose(-2, -1).contiguous(), one, one * 0, -128, 127)
    a, b = torch.zeros(2, 3, 4, device=dev()), torch.zeros(2, 5, 6, device=dev())
    with pytest.raises(SparsebitB200Error, match="inner dimensions differ"):
        ops.int8_matmul(a, one, one * 0, (-128, 127), b, one, one * 0, (-128, 127))
    with pytest.raises(SparsebitB200Error, match="at least 2 dimensions"):
        ops.int8_matmul(a[0, 0], one, one * 0, (-128, 127), b, one, one * 0, (-128, 127))
    with pytest.raises(SparsebitB200Error, match="per-tensor"):
        ops.int8_matmul(a, torch.ones(2, device=dev()), one, (-128, 127), a.transpose(-2, -1), one, one, (-128, 127))
    with pytest.raises(SparsebitB200Error, match=r"wider than 8 bits.*status -1"):
        ops.int8_matmul(a, one, one * 0, (-128, 127), a.transpose(-2, -1), one, one * 0, (0, 256))


# ---------------------------------------------------------------------------------------------- batch isolation, NaN
@pytest.mark.parametrize("k_major", [True, False])
@pytest.mark.parametrize("poison", ["extreme", "nan"])
def test_batch_entries_are_isolated(k_major, poison):
    rng = np.random.default_rng(17)
    m, k, n = 70, 40, 50  # partial tiles: a 128-row box starting in entry 1 covers rows of entry 2 in memory
    a = _operand(rng, (3, m, k), (-128, 127), False)
    b = _operand(rng, (3, k, n), (0, 255), False)
    alone = _matmul((a[0][1:2],) + a[1:], (b[0][1:2],) + b[1:], k_major)
    fill = np.nan if poison == "nan" else 1e30
    for x in (a[0], b[0]):
        x[0], x[2] = fill, -fill
    y = _matmul(a, b, k_major)
    assert np.array_equal(y[1], alone[0]) and np.isfinite(y[1]).all()
    if poison == "nan":
        assert np.isnan(y[0]).all() and np.isnan(y[2]).all()
    else:  # every element at the end of its range
        za, zb = int(a[2]), int(b[2])
        assert np.all(y[0] == F32(np.float64(k * (127 - za) * (255 - zb)) * (np.float64(a[1]) * np.float64(b[1]))))


@pytest.mark.parametrize("k_major", [True, False])
def test_nan_rows_and_columns_stay_inside_their_entry(k_major):
    rng = np.random.default_rng(19)
    a = _operand(rng, (3, 130, 33), (-128, 127), False)
    b = _operand(rng, (3, 33, 140), (-128, 127), False)
    a[0][0, 129, 32] = np.nan
    a[0][2, 0, 0] = np.inf
    b[0][1, 7, 139] = np.nan
    b[0][2, 32, 0] = -np.inf
    y = _matmul(a, b, k_major)
    expect = np.zeros(y.shape, bool)
    expect[0, 129, :] = True
    expect[1, :, 139] = True
    assert np.array_equal(np.isnan(y), expect)
    assert np.array_equal(np.isnan(truth(a, b)[0]), expect)  # the product of the fake-quant operands has the same NaNs
    assert np.array_equal(y, integer_form(a, b)[-1].astype(F32), equal_nan=True)


# ---------------------------------------------------------------------------------------------- ties to the merged paths
@pytest.mark.parametrize("affine", [False, True])
def test_equals_the_integer_linear_for_a_per_tensor_weight(affine):
    rng = np.random.default_rng(23)
    m, k, n = 197, 192, 100
    x = _operand(rng, (m, k), qrange(8, affine), False)
    w = _operand(rng, (n, k), (-128, 127), False)
    ws, wz = t(np.full(n, w[1], F32)), t(np.full(n, w[2], F32))
    w_q, w_sum, _ = ops.int8_quantize_rows(t(w[0]), ws, wz, -128, 127)
    w_zero = t(np.full(n, int(w[2]) - grid_offset(-128), np.int32))
    lin = ops.int8_linear(t(x[0]), scalar(x[1]), scalar(x[2]), x[3], x[4], w_q, w_sum, ws, w_zero)
    wt = t(w[0])
    for b in (wt.t(), wt.t().contiguous()):  # K-major as the weight lies, and N-major
        y = ops.int8_matmul(t(x[0]), scalar(x[1]), scalar(x[2]), x[3:], b, scalar(w[1]), scalar(w[2]), w[3:])
        assert torch.equal(y, lin)


def test_graph_replay_with_new_inputs_and_two_streams():
    rng = np.random.default_rng(29)
    a = _operand(rng, (6, 197, 64), (-128, 127), False)
    b = _operand(rng, (6, 64, 197), (0, 255), False)
    a2, b2 = (rng.permutation(a[0].reshape(-1)).reshape(a[0].shape), rng.permutation(b[0].reshape(-1)).reshape(b[0].shape))
    at, bt = t(a[0]), t(b[0])
    qp = [scalar(a[1]), scalar(a[2]), a[3:], None, scalar(b[1]), scalar(b[2]), b[3:]]

    def call(x, y):
        return ops.int8_matmul(x, qp[0], qp[1], qp[2], y, qp[4], qp[5], qp[6])

    y1 = call(at, bt)
    assert torch.equal(y1, call(at, bt))  # deterministic
    y2 = call(t(a2), t(b2))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call(at, bt)  # warm the per-stream workspace outside the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            yg = call(at, bt)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y1)
    at.copy_(t(a2)), bt.copy_(t(b2))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y2)
    # two streams, two workspaces: different problems in flight at once do not disturb each other
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    big_a, big_b = at.repeat(8, 1, 1), bt.repeat(8, 1, 1)
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        o1 = [call(big_a, big_b) for _ in range(3)]
    with torch.cuda.stream(s2):
        o2 = [call(at[:3], bt[:3]) for _ in range(3)]
    torch.cuda.synchronize()
    ws = ops._int8_ws
    assert ws[(at.device, s1.cuda_stream)].data_ptr() != ws[(at.device, s2.cuda_stream)].data_ptr()
    assert all(torch.equal(o, y2.repeat(8, 1, 1)) for o in o1) and all(torch.equal(o, y2[:3]) for o in o2)


# ---------------------------------------------------------------------------------------------- modules
class Attention(nn.Module):
    """The attention of a DeiT-tiny block: fused qkv projection, q @ k^T, softmax, p @ v, output projection."""

    def __init__(self, dim=192, heads=3):
        super().__init__()
        self.heads, self.head_dim = heads, dim // heads
        self.qkv = QLinear(nn.Linear(dim, 3 * dim)).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"),
                                                                     cfg("per-channel-symmetric", "weight"))
        self.qk = QMatMul().build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"))
        # softmax output: unsigned, Z = 0 ... 255
        self.pv = QMatMul().build_quantizer(cfg("per-tensor-affine", "feature", layout="NLC"))
        self.proj = QLinear(nn.Linear(dim, dim)).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"),
                                                                 cfg("per-channel-symmetric", "weight"))

    def forward(self, x):
        qkv = self.qkv(x).reshape(x.shape[0], x.shape[1], 3, self.heads, self.head_dim).permute(2, 0, 3, 1, 4)
        attn = self.qk(qkv[0] * self.head_dim ** -0.5, qkv[1].transpose(-2, -1)).softmax(dim=-1)
        out = self.pv(attn, qkv[2]).transpose(1, 2).reshape(x.shape[0], x.shape[1], -1)
        return self.proj(out)


def _matmul_truth(qmatmul, xl, xr):
    ops_ = []
    for carrier, x in ((qmatmul.left, xl), (qmatmul.right, xr)):
        q = carrier.input_quantizer
        s, z = (v.detach().reshape(-1).cpu().numpy() for v in q._qparams_preprocess(x))
        ops_.append((x.cpu().numpy(), s[0], z[0], *q.qdesc.qrange))
    return truth(*ops_)


@pytest.mark.parametrize("replay", [False, True])
def test_attention_block_converts_and_meets_the_bound(replay):
    torch.manual_seed(0)
    batches = [torch.randn(4, 197, 192, device=dev()) for _ in range(3)]
    model = calibrated(Attention(), batches, streaming=not replay, record_inputs=None, replay=replay)
    originals = {nm: getattr(model, nm) for nm in ("qk", "pv")}
    for nm, qm in originals.items():  # calibration reached both carriers of both matmuls
        for q in (qm.left.input_quantizer, qm.right.input_quantizer):
            assert float(q.scale.reshape(-1)[0]) > 0 and float(q.scale.reshape(-1)[0]) != 1.0, nm
    assert to_integer_linears(model) == ["qkv", "proj"]
    assert to_integer_matmuls(model) == ["qk", "pv"]
    assert isinstance(model.qkv, QLinearInt8) and isinstance(model.qk, QMatMulInt8) and isinstance(model.pv, QMatMulInt8)
    assert not any(isinstance(m, (QMatMul, QLinear)) for m in model.modules())
    assert model.pv.left_qrange == (0, 255) and model.qk.left_qrange == (-128, 127)
    seen = {}
    hooks = [model.get_submodule(nm).register_forward_hook(lambda mod, i, o, nm=nm: seen.__setitem__(nm, (i, o)))
             for nm in originals]
    with torch.no_grad():
        for x in batches[:2]:
            model(x)
            for nm, original in originals.items():
                (xl, xr), y = seen[nm]
                t_, bound = _matmul_truth(original, xl, xr)
                err = np.abs(y.cpu().numpy() - t_)
                assert np.all(err <= bound), (nm, float((err / bound).max()))
                ref_err = np.abs(original(xl, xr).cpu().numpy() - t_)  # QDQ + QDQ + fp32 torch.matmul, TF32 off
                assert err.max() <= ref_err.max(), (nm, err.max(), ref_err.max())
                print(f"{nm}: int8 max |y - T| = {err.max():.3e}, fake-quant max |y - T| = {ref_err.max():.3e}")
    for h in hooks:
        h.remove()
    # No GEMM but the library's own runs in the converted block.  What runs is established without relying on the
    # profiler's device trace, whose per-kernel records CUPTI can miss: the library counts its own launches (qkv and
    # proj: row quantizer + GEMM each; qk and pv: the row quantizer of a, the column or row quantizer of b, the GEMM
    # each), and the operator trace, recorded on the host for every call, holds no ATen matmul.  The kernels the device
    # trace does record are checked too.
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    before = launch_count()
    with torch.no_grad(), profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        model(batches[0])
        torch.cuda.synchronize()
    assert launch_count() - before == 2 + 3 + 3 + 2
    events = prof.events()
    aten = {e.name for e in events if e.name.startswith("aten::")}
    assert "aten::softmax" in aten, sorted(aten)  # the host trace is there
    forbidden = {"aten::matmul", "aten::bmm", "aten::mm", "aten::addmm", "aten::baddbmm", "aten::linear"}
    assert not aten & forbidden, sorted(aten & forbidden)
    kernels = {e.name for e in events if e.device_type == DeviceType.CUDA}
    foreign = [n for n in kernels if "sb200" not in n and any(w in n.lower() for w in ("gemm", "cutlass", "xmma", "gemv"))]
    assert not foreign, foreign


def test_module_input_forms():
    torch.manual_seed(1)
    qm = QMatMul().build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC")).to(dev())
    xl, xr = torch.randn(2, 3, 20, 16, device=dev()), torch.randn(2, 3, 16, 24, device=dev())
    for carrier, x in ((qm.left, xl), (qm.right, xr)):
        carrier.input_quantizer.update_observer(x)
        carrier.input_quantizer.calc_qparams()
    qm.set_quant(a_quant=True)
    mod = QMatMulInt8.from_qmatmul(qm)
    with torch.no_grad():
        y = mod(xl, xr)
        assert y.dtype == torch.float32 and y.shape == (2, 3, 20, 24)
        t_, bound = _matmul_truth(qm, xl, xr)
        assert np.all(np.abs(y.cpu().numpy() - t_) <= bound)
        yh = mod(xl.half(), xr.half())  # fp16 operands are up-cast, the result is fp32
        assert yh.dtype == torch.float32 and torch.equal(yh, mod(xl.half().float(), xr.half().float()))
        assert torch.equal(mod(xl[0, 0], xr), mod(xl[0, 0].expand(2, 3, 20, 16), xr))  # 2-D left operand broadcasts
    with pytest.raises(ValueError, match="1-D operands are not supported"):
        mod(xl[0, 0, 0], xr)
    with pytest.raises(RuntimeError, match="inference-only"):
        mod(xl.clone().requires_grad_(), xr)
    assert "left_qrange=[-128, 127]" in repr(mod)
