"""GPU: the fused integer-grid attention (sb200_int8_attention, ops.int8_attention, QAttentionInt8,
to_integer_attentions) against tests/int8_attention_ref.py.

* Over a geometry matrix (Tq, Tk in 1, 31, 64, 65, 197, >= 1000; d, dv in 8, 40, 64, 128; signed and unsigned p; with
  and without a scale; power-of-two and general operand scales):
  - stage 3 is exact: out equals the integer form of p @ v built on the kernel's own p grid, bit for bit;
  - every p grid value is admissible under the contract |p - p64| <= EPS p64 + ALPHA;
  - |y - T| <= 2^-21 (|f_p64| @ |f_v|) + s_p s_v sum_j |g - g64| |v_v - Z_v| elementwise.
* The scores equal QMatMulInt8's q @ k^T: the fused output equals int8_matmul(softmax grid, v) built from them.
* NaN placement, batch isolation, determinism, CUDA-graph replay (also after the workspace grows).
* Tq = Tk = 16384: no T^2 allocation, a handful of rows checked against the reference.
* A DeiT-tiny attention block calibrated by streaming and by the fx replay, converted by to_integer_linears +
  to_integer_attentions: within the bounds; the library launches exactly its 8 kernels per forward and no ATen
  softmax or matmul runs."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_attention_ref as ref
from gpu_util import dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from int8_harness import attention_operand, calibrated, cfg, operands_of, p_qparams, scalar
from sparsebit_b200 import SparsebitB200Error, launch_count, ops
from sparsebit_b200.quantization.modules import QAttention, QAttentionInt8, QLinear, QLinearInt8, QMatMul
from sparsebit_b200.quantization.tools import to_integer_attentions, to_integer_linears, to_integer_matmuls

pytestmark = pytest.mark.gpu

F32 = np.float32


def _run(q, k, v, p, scale=None, return_p=True):
    qp = [(scalar(o[1]), scalar(o[2]), o[3:]) for o in (q, k)]
    pp = (scalar(p[0]), scalar(p[1]), p[2:])
    vp = (scalar(v[1]), scalar(v[2]), v[3:])
    return ops.int8_attention(t(q[0]), t(k[0]), t(v[0]), qp[0], qp[1], pp, vp, scale=scale, return_p=return_p)


def _check(q, k, v, p, scale, label):
    y, pq = _run(q, k, v, p, scale)
    y, pq = y.cpu().numpy(), pq.cpu().numpy()
    tk = k[0].shape[-2]
    assert pq.shape[-1] == ref.padded(tk) and not pq[..., tk:].any(), label
    # stage 3 exact on the kernel's own grid
    exp = ref.expected(pq, q, k, v, p, scale)
    assert np.array_equal(y, exp, equal_nan=True), (label, float(np.nanmax(np.abs(y - exp))))
    # p admissible
    s, bad = ref.scores(q, k, scale)
    p64 = ref.softmax64(s)
    lo, hi = ref.admissible_range(p64, p)
    g = pq[..., :tk].astype(np.int64)
    ok = (g >= lo) & (g <= hi)
    assert ok[~bad].all(), (label, int((~ok[~bad]).sum()))
    T, g64, mm, _ = ref.truth(q, k, v, p, scale)
    diff = float((g != g64)[~bad].mean())
    # truth bound
    bound = ref.truth_bound(g, g64, p, v, mm)
    err = np.abs(y.astype(np.float64) - T)
    good = ~bad[..., None] & np.isfinite(T)
    assert np.all(err[good] <= bound[good]), (label, float(np.max((err - bound)[good])))
    print(f"{label}: p grid differs from g64 at {diff:.2e} of elements, max |y - T| = {err[good].max():.3e}")
    return y, pq


# (batch, Tq, Tk, d, dv)
GEOMS = [(2, 1, 1, 8, 8), (3, 31, 64, 40, 8), (2, 64, 31, 64, 40), (2, 65, 65, 8, 128), (2, 197, 197, 64, 64),
         (1, 1000, 65, 128, 128), (1, 65, 1031, 40, 64), (1, 31, 1000, 128, 40), (2, 197, 1, 64, 128),
         (1, 1, 197, 128, 8)]


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("unsigned_p,scaled,pow2", [(True, True, False), (False, False, True), (True, False, True),
                                                    (False, True, False)])
def test_geometry_matrix(geom, unsigned_p, scaled, pow2):
    b, tq, tk, d, dv = geom
    rng = np.random.default_rng(abs(hash((geom, unsigned_p, scaled, pow2))) % 2**32)
    q = attention_operand(rng, (b, tq, d), pow2, 2.0)
    k = attention_operand(rng, (b, tk, d), pow2, 2.0, (0, 255) if d == 40 else (-128, 127))
    v = attention_operand(rng, (b, tk, dv), pow2, 1.0, (0, 255) if dv == 64 else (-128, 127))
    scale = (2.0 ** -3 if pow2 else d ** -0.5) if scaled else None
    _check(q, k, v, p_qparams(unsigned_p, pow2), scale, f"{geom} unsigned_p={unsigned_p} scale={scale} pow2={pow2}")


def test_scores_are_those_of_the_integer_matmul():
    """With the kernel's p grid fed to int8_matmul as an exact operand, the fused output is int8_matmul's p @ v."""
    rng = np.random.default_rng(3)
    q, k, v = (attention_operand(rng, (4, 197, 64), False, 2.0) for _ in range(3))
    p = p_qparams(True, False)
    y, pq = _run(q, k, v, p, 0.125)
    s_mm = ops.int8_matmul(t(q[0]), scalar(q[1]), scalar(q[2]), q[3:], t(k[0]).transpose(-2, -1), scalar(k[1]),
                           scalar(k[2]), k[3:])
    s_ref, _ = ref.scores(q, k)
    assert np.array_equal(s_mm.cpu().numpy(), s_ref)  # the reference's scores are QMatMulInt8's, bit for bit
    # p @ v through int8_matmul on the kernel's grid dequantized to g s_p, which int8_matmul quantizes back to g
    fp = ((pq[..., :197].float() + 128 - p[1]) * float(p[0]))
    y_mm = ops.int8_matmul(fp, scalar(p[0]), scalar(p[1]), p[2:], t(v[0]), scalar(v[1]), scalar(v[2]), v[3:])
    assert torch.equal(y, y_mm)


def test_nan_placement_and_batch_isolation():
    rng = np.random.default_rng(4)
    b, tq, tk, d, dv = 4, 70, 150, 64, 40
    q, k, v = (attention_operand(rng, shape, False) for shape in ((b, tq, d), (b, tk, d), (b, tk, dv)))
    p = p_qparams(True, False)
    clean = _run(q, k, v, p, 0.125, return_p=False).cpu().numpy()
    assert np.isfinite(clean).all()
    q[0][1, 5, 3] = np.nan  # row 5 of entry 1
    k[0][2, 149, 0] = np.nan  # all of entry 2
    v[0][3, 17, 11] = np.nan  # column 11 of entry 3
    q[0][0, 0, 0], k[0][0, 3, 1], v[0][0, 2, 2] = np.inf, -np.inf, np.inf  # clamped: entry 0 stays finite
    y = _run(q, k, v, p, 0.125, return_p=False).cpu().numpy()
    expect = np.zeros(y.shape, bool)
    expect[1, 5, :] = True
    expect[2] = True
    expect[3, :, 11] = True
    assert np.array_equal(np.isnan(y), expect)
    for e in (1, 3):  # the NaN rows / columns of an entry touch nothing else
        assert np.array_equal(y[e][~expect[e]], clean[e][~expect[e]])
    # extreme and NaN-filled neighbours change nothing in entry 0's neighbour-free twin
    q2, k2, v2 = (list(o) for o in (q, k, v))
    for o in (q2, k2, v2):
        o[0] = o[0].copy()
        o[0][1] = np.nan
        o[0][2] = 1e30
    y2 = _run(tuple(q2), tuple(k2), tuple(v2), p, 0.125, return_p=False).cpu().numpy()
    assert np.array_equal(y2[0], y[0]) and np.array_equal(y2[3], y[3], equal_nan=True)


def test_determinism_and_graph_replay_after_growth():
    rng = np.random.default_rng(5)
    q, k, v = (attention_operand(rng, (6, 197, 64), False) for _ in range(3))
    p = p_qparams(True, False)
    qt, kt, vt = t(q[0]), t(k[0]), t(v[0])
    qp = [(scalar(o[1]), scalar(o[2]), o[3:]) for o in (q, k)]
    pp, vp = (scalar(p[0]), scalar(p[1]), p[2:]), (scalar(v[1]), scalar(v[2]), v[3:])

    def call(x, y, z):
        return ops.int8_attention(x, y, z, qp[0], qp[1], pp, vp, scale=0.125)

    y1 = call(qt, kt, vt)
    assert all(torch.equal(y1, call(qt, kt, vt)) for _ in range(3))
    perm = [t(rng.permutation(o[0].reshape(-1)).reshape(o[0].shape)) for o in (q, k, v)]
    y2 = call(*perm)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call(qt, kt, vt)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            yg = call(qt, kt, vt)
        # grow the stream's workspace after the capture, then fill the freed-size allocations
        big = [o.repeat(8, 1, 1) for o in (qt, kt, vt)]
        call(*big)
        old_bytes = ops._int8_workspaces.retired[(qt.device, s.cuda_stream)][-1].numel()
        fill = [torch.full((old_bytes,), 7, dtype=torch.uint8, device=qt.device) for _ in range(12)]
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y1)
    for x, src in zip((qt, kt, vt), perm):
        x.copy_(src)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y2)
    assert all(bool((f == 7).all()) for f in fill)


def test_16k_tokens_without_a_t_squared_allocation():
    b, tq, d = 2, 16384, 64
    g = torch.Generator(device=dev()).manual_seed(6)
    q, k, v = (torch.randn(b, tq, d, device=dev(), generator=g) for _ in range(3))
    s1 = float(q.abs().max()) / 127
    one = lambda x: torch.tensor([x], dtype=torch.float32, device=dev())
    qp = (one(s1), one(0.0), (-128, 127))
    pp = (one(1 / 255), one(0.0), (0, 255))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    y = ops.int8_attention(q, k, v, qp, qp, pp, qp, scale=d ** -0.5)
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    assert grew <= 4 * b * tq * (d + d) * 4, grew  # O(B T (d + dv)); one fp32 score tensor would be 2 GiB
    print(f"Tq = Tk = {tq}: peak allocation grew by {grew / 2**20:.1f} MiB")
    rows = [0, 1, 8191, 16383]
    kk, vv = k.cpu().numpy(), v.cpu().numpy()
    for e in range(b):
        qo = (q[e, rows].cpu().numpy(), F32(s1), F32(0), -128, 127)
        ko, vo = (kk[e], F32(s1), F32(0), -128, 127), (vv[e], F32(s1), F32(0), -128, 127)
        p = (F32(1 / 255), F32(0), 0, 255)
        T, g64, mm, _ = ref.truth(qo, ko, vo, p, d ** -0.5)
        s, _ = ref.scores(qo, ko, d ** -0.5)
        lo, hi = ref.admissible_range(ref.softmax64(s), p)
        # the kernel's rows are within the truth bound of some admissible grid: bound by the widest admissible gap
        g_far = np.where(np.abs(lo - g64) > np.abs(hi - g64), lo, hi)
        bound = ref.truth_bound(g_far, g64, p, vo, mm)
        assert np.all(np.abs(y[e, rows].cpu().numpy() - T) <= bound), e


# ---------------------------------------------------------------------------------------------- the DeiT-tiny block
class Attention(nn.Module):
    """The attention of a DeiT-tiny block around QAttention: fused qkv projection, the quantized attention, output
    projection."""

    def __init__(self, dim=192, heads=3):
        super().__init__()
        self.heads, self.head_dim = heads, dim // heads
        self.qkv = QLinear(nn.Linear(dim, 3 * dim)).build_quantizer(
            cfg("per-tensor-symmetric", "feature", layout="NLC"), cfg("per-channel-symmetric", "weight"))
        self.attn = QAttention(scale=self.head_dim ** -0.5).build_quantizer(  # p: unsigned, Z = 0 ... 255
            cfg("per-tensor-symmetric", "feature", layout="NLC"), cfg("per-tensor-affine", "feature", layout="NLC"))
        self.proj = QLinear(nn.Linear(dim, dim)).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"),
                                                                 cfg("per-channel-symmetric", "weight"))

    def forward(self, x):
        qkv = self.qkv(x).reshape(x.shape[0], x.shape[1], 3, self.heads, self.head_dim).permute(2, 0, 3, 1, 4)
        out = self.attn(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(x.shape[0], x.shape[1], -1)
        return self.proj(out)


@pytest.mark.parametrize("replay", [False, True])
def test_deit_tiny_block_converts_and_meets_the_bounds(replay):
    torch.manual_seed(0)
    batches = [torch.randn(4, 197, 192, device=dev()) for _ in range(3)]
    model = calibrated(Attention(), batches, streaming=not replay, record_inputs=None, replay=replay)
    original = model.attn
    for carrier in (original.qk.left, original.qk.right, original.pv.left, original.pv.right):
        s = float(carrier.input_quantizer.scale.reshape(-1)[0])
        assert s > 0 and s != 1.0  # calibration reached all four carriers
    assert original.pv.left.input_quantizer.qdesc.qrange == (0, 255)
    assert to_integer_linears(model) == ["qkv", "proj"]
    assert to_integer_attentions(model) == ["attn"]
    assert to_integer_matmuls(model) == []
    assert isinstance(model.attn, QAttentionInt8) and isinstance(model.qkv, QLinearInt8)
    assert not any(isinstance(m, (QAttention, QMatMul, QLinear)) for m in model.modules())
    seen = {}
    hook = model.attn.register_forward_hook(lambda mod, i, o: seen.__setitem__("attn", (i, o)))
    with torch.no_grad():
        for x in batches[:2]:
            model(x)
            (qx, kx, vx), y = seen["attn"]
            (q, k, v), p = operands_of(original, qx, kx, vx)
            T, g64, mm, _ = ref.truth(q, k, v, p, original.scale)
            s, _ = ref.scores(q, k, original.scale)
            lo, hi = ref.admissible_range(ref.softmax64(s), p)
            g_far = np.where(np.abs(lo - g64) > np.abs(hi - g64), lo, hi)
            err = np.abs(y.cpu().numpy() - T)
            assert np.all(err <= ref.truth_bound(g_far, g64, p, v, mm))
            fq_err = np.abs(original(qx, kx, vx).cpu().numpy() - T)
            print(f"attention: fused max |y - T| = {err.max():.3e}, fake-quant max |y - T| = {fq_err.max():.3e}")
    hook.remove()
    # What runs is established without relying on the profiler's device trace, whose per-kernel records CUPTI can
    # miss: the library counts its own launches (qkv and proj: row quantizer + GEMM each; the attention: two row
    # quantizers, the column quantizer and the fused kernel), and the operator trace, recorded on the host for every
    # call, holds no ATen softmax and no ATen matmul.  The kernels the device trace does record are checked too.
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    before = launch_count()
    with torch.no_grad(), profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        model(batches[0])
        torch.cuda.synchronize()
    assert launch_count() - before == 8
    events = prof.events()
    aten = {e.name for e in events if e.name.startswith("aten::")}
    assert "aten::permute" in aten, sorted(aten)  # the host trace is there
    forbidden = {"aten::softmax", "aten::_softmax", "aten::matmul", "aten::bmm", "aten::mm", "aten::addmm",
                 "aten::baddbmm", "aten::linear"}
    assert not aten & forbidden, sorted(aten & forbidden)
    kernels = {e.name for e in events if e.device_type == DeviceType.CUDA}
    foreign = [n for n in kernels if "sb200" not in n and any(w in n.lower() for w in ("softmax", "gemm", "cutlass",
                                                                                        "xmma", "gemv"))]
    assert not foreign, foreign


def test_module_input_forms_and_errors():
    torch.manual_seed(1)
    qa = QAttention(scale=0.25).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC")).to(dev())
    xs = [torch.randn(2, 3, 20, 16, device=dev()) for _ in range(3)]
    for carrier, x in ((qa.qk.left, xs[0]), (qa.qk.right, xs[1].transpose(-2, -1)), (qa.pv.right, xs[2]),
                       (qa.pv.left, torch.rand(2, 3, 20, 20, device=dev()))):
        carrier.input_quantizer.update_observer(x)
        carrier.input_quantizer.calc_qparams()
    qa.set_quant(a_quant=True)
    mod = QAttentionInt8.from_qattention(qa)
    with torch.no_grad():
        y = mod(*xs)
        assert y.dtype == torch.float32 and y.shape == (2, 3, 20, 16)
        yh = mod(*(x.half() for x in xs))
        assert yh.dtype == torch.float32 and torch.equal(yh, mod(*(x.half().float() for x in xs)))
        assert torch.equal(mod(xs[0].transpose(-2, -1).contiguous().transpose(-2, -1), xs[1], xs[2]), y)  # non-contiguous
        with pytest.raises(SparsebitB200Error, match="leading dimensions"):
            mod(xs[0][:1], xs[1], xs[2])
        with pytest.raises(SparsebitB200Error, match="d <= 128"):
            big = torch.randn(1, 4, 130, device=dev())
            mod(big, big, big)
    with pytest.raises(RuntimeError, match="inference-only"):
        mod(xs[0].requires_grad_(), xs[1], xs[2])
