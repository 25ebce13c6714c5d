"""GPU: the masked and causal fused attention (sb200_int8_attention_masked, ops.int8_attention with attn_mask /
causal, QAttentionInt8) against tests/int8_attention_mask_ref.py.

* Over a geometry matrix (Tq, Tk not multiples of 128, Tq < Tk, Tq > Tk, Tq = 1; d, dv <= 128) and five masks (key
  padding with -10000 and with -inf, a full random mask, causal, causal + padding), signed and unsigned p, power-of-two
  and general scales: out is exact on the kernel's own p grid, every p value is admissible, out is within the truth
  bound, and p_q holds the grid of 0 wherever the composition's p is 0, the skipped blocks included.
* Mask identities: an all-zero mask is the unmasked call bit for bit; with Tq = Tk, causal is the masked kernel given
  the explicit -inf triangle, bit for bit.
* NaN placement, batch isolation through a broadcast mask, determinism, CUDA-graph replay after the workspace grows,
  a 16384-token causal + padded run without a T^2 allocation.
* A BERT-style (key padding) and a GPT-2-style (causal) block, calibrated by streaming and by the fx replay and
  converted: within the bounds; the library launches the expected kernels and no ATen softmax, matmul, where or add
  runs on the attention path."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_attention_mask_ref as mref
import int8_attention_ref as ref
from gpu_util import dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from int8_harness import attention_operand, calibrated, cfg, check_p, operands_of, p_qparams, scalar
from int8_matmul_ref import BOUND
from oracle import qdq as oqdq
from sparsebit_b200 import launch_count, ops
from sparsebit_b200.quantization.modules import QAttention, QAttentionInt8, QLinear, QLinearInt8
from sparsebit_b200.quantization.tools import to_integer_attentions, to_integer_linears

pytestmark = pytest.mark.gpu

F32 = np.float32


def _run(q, k, v, p, scale=None, mask=None, causal=False, return_p=True):
    qp = [(scalar(o[1]), scalar(o[2]), o[3:]) for o in (q, k)]
    pp = (scalar(p[0]), scalar(p[1]), p[2:])
    vp = (scalar(v[1]), scalar(v[2]), v[3:])
    m = None if mask is None else (mask if isinstance(mask, torch.Tensor) else t(mask))
    return ops.int8_attention(t(q[0]), t(k[0]), t(v[0]), qp[0], qp[1], pp, vp, scale=scale, return_p=return_p,
                              attn_mask=m, causal=causal)


def _mask(kind, rng, lead, tq, tk):
    """(mask or None, causal) of a mask kind; padding masks are [B, 1, 1, Tk] over lead = (B, H)."""
    causal = kind.startswith("causal")
    if kind in ("pad_1e4", "pad_inf", "causal_pad"):
        keep = np.ones((lead[0], 1, 1, tk), F32)
        for b in range(lead[0]):
            keep[b, ..., max(1, tk - b * tk // 3):] = 0  # entry b pads its last b / 3 of the keys (never all)
        fill = F32(-np.inf) if kind == "pad_inf" else F32(-10000)
        return np.where(keep == 0, fill, F32(0)).astype(F32), causal
    if kind == "full":
        m = (rng.standard_normal(lead + (tq, tk)) * 3).astype(F32)
        m[rng.random(m.shape) < 0.1] = -np.inf
        return m, causal
    return None, causal


def _check(q, k, v, p, scale, mask, causal, label):
    y, pq = _run(q, k, v, p, scale, mask, causal)
    y, g = y.cpu().numpy(), pq.cpu().numpy()
    tq, tk = q[0].shape[-2], k[0].shape[-2]
    exp = mref.expected(g, q, k, v, p, scale, mask, causal)
    assert np.array_equal(y, exp, equal_nan=True), (label, float(np.nanmax(np.abs(y - exp))))
    s, bad = mref.scores(q, k, scale, mask, causal)
    check_p(g, s, bad, p, tq, tk, causal, label)
    T, g64, mm, _ = mref.truth(q, k, v, p, scale, mask, causal)
    bound = ref.truth_bound(g[..., :tk], g64, p, v, mm)
    err = np.abs(y.astype(np.float64) - T)
    good = ~bad[..., None] & np.isfinite(T)
    assert np.all(err[good] <= bound[good]), (label, float(np.max((err - bound)[good])))
    diff = float((g[..., :tk] != g64)[~bad].mean()) if (~bad).any() else 0.0
    print(f"{label}: p grid differs from g64 at {diff:.2e} of elements, max |y - T| = {err[good].max():.3e}")
    return y, g


# (lead, Tq, Tk, d, dv)
GEOMS = [((2, 2), 1, 1, 8, 8), ((2, 2), 31, 64, 40, 8), ((2, 1), 64, 31, 64, 40), ((1, 2), 65, 65, 8, 128),
         ((2, 2), 197, 197, 64, 64), ((1, 1), 1000, 65, 128, 128), ((1, 1), 65, 1031, 40, 64),
         ((2, 1), 300, 300, 128, 40), ((1, 2), 1, 197, 128, 8), ((3, 1), 260, 700, 32, 64)]
MASKS = ["pad_1e4", "pad_inf", "full", "causal", "causal_pad"]


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("kind", MASKS)
@pytest.mark.parametrize("unsigned_p,pow2", [(True, False), (False, True)])
def test_geometry_matrix(geom, kind, unsigned_p, pow2):
    lead, tq, tk, d, dv = geom
    rng = np.random.default_rng(abs(hash((geom, kind, unsigned_p, pow2))) % 2**32)
    q = attention_operand(rng, lead + (tq, d), pow2, 2.0)
    k = attention_operand(rng, lead + (tk, d), pow2, 2.0, (0, 255) if d == 40 else (-128, 127))
    v = attention_operand(rng, lead + (tk, dv), pow2, 1.0, (0, 255) if dv == 64 else (-128, 127))
    scale = 2.0 ** -3 if pow2 else d ** -0.5
    mask, causal = _mask(kind, rng, lead, tq, tk)
    _check(q, k, v, p_qparams(unsigned_p, pow2), scale, mask, causal, f"{geom} {kind} unsigned_p={unsigned_p}")


def test_mask_identities():
    rng = np.random.default_rng(11)
    lead, tq, tk = (2, 3), 300, 300
    q, k, v = (attention_operand(rng, lead + (tq, 64), False, 2.0) for _ in range(3))
    p = p_qparams(True, False)
    y0, g0 = _run(q, k, v, p, 0.125)
    yz, gz = _run(q, k, v, p, 0.125, mask=np.zeros((lead[0], 1, 1, tk), F32))  # the masked kernel with a zero mask
    assert torch.equal(y0, yz) and torch.equal(g0, gz)
    yz, gz = _run(q, k, v, p, 0.125, mask=np.zeros(lead + (tq, tk), F32))
    assert torch.equal(y0, yz) and torch.equal(g0, gz)
    tri = np.where(mref.visible(tq, tk, True), F32(0), F32(-np.inf)).astype(F32)
    yc, gc = _run(q, k, v, p, 0.125, causal=True)  # skips blocks, sums v over the visited prefix
    yt, gt = _run(q, k, v, p, 0.125, mask=tri)     # visits every block
    assert torch.equal(yc, yt) and torch.equal(gc, gt)
    # and a zero point off p's range: the skipped keys' (g_0 - Z_p) terms are added exactly
    poff = (F32(1 / 255), F32(-3), 0, 255)
    yc, gc = _run(q, k, v, poff, 0.125, causal=True)
    yt, gt = _run(q, k, v, poff, 0.125, mask=tri)
    assert torch.equal(yc, yt) and torch.equal(gc, gt)
    assert np.array_equal(yc.cpu().numpy(), mref.expected(gc.cpu().numpy(), q, k, v, poff, 0.125, None, True))


def test_nan_placement():
    rng = np.random.default_rng(12)
    lead, tq, tk, d, dv = (3,), 260, 260, 64, 40
    q, k, v = (attention_operand(rng, shape, False) for shape in (lead + (tq, d), lead + (tk, d), lead + (tk, dv)))
    p = p_qparams(True, False)
    clean = _run(q, k, v, p, 0.125, causal=True, return_p=False).cpu().numpy()
    assert np.isfinite(clean).all()
    k[0][0, 150, 2] = np.nan  # entry 0: rows >= 150 see key 150
    v[0][1, 250, 7] = np.nan  # entry 1: key 250 is hidden from rows < 250, column 7 is NaN everywhere
    q[0][2, 9, 0] = np.nan    # entry 2: row 9
    y = _run(q, k, v, p, 0.125, causal=True, return_p=False).cpu().numpy()
    expect = np.zeros(y.shape, bool)
    expect[0, 150:] = True
    expect[1, :, 7] = True
    expect[2, 9] = True
    assert np.array_equal(np.isnan(y), expect)
    assert np.array_equal(y[~expect], clean[~expect])
    # rows without a visible key: causal with Tq > Tk, and an all -inf mask row
    q2 = attention_operand(rng, (2, 200, d), False)
    k2, v2 = attention_operand(rng, (2, 50, d), False), attention_operand(rng, (2, 50, dv), False)
    m = np.zeros((2, 1, 50), F32)
    m[1, 0, :] = -np.inf
    y2 = _run(q2, k2, v2, p, 0.125, mask=m, return_p=False).cpu().numpy()
    assert np.isnan(y2[1]).all() and np.isfinite(y2[0]).all()
    y3 = _run(q2, k2, v2, p, 0.125, causal=True, return_p=False).cpu().numpy()
    assert np.isnan(y3[:, :150]).all() and np.isfinite(y3[:, 150:]).all()


def test_batch_isolation_through_a_broadcast_mask():
    rng = np.random.default_rng(13)
    b, h, tq, tk, d = 4, 3, 128, 333, 64
    q, k, v = (attention_operand(rng, (b, h, n, d), False) for n in (tq, tk, tk))
    p = p_qparams(True, False)
    lens = [333, 200, 1, 129]
    m = np.zeros((b, 1, 1, tk), F32)
    for e, n in enumerate(lens):
        m[e, ..., n:] = -10000.0
    y = _run(q, k, v, p, 0.125, mask=m, causal=True, return_p=False).cpu().numpy()
    for e in range(b):  # each entry alone, with its own padding
        one = [(o[0][e:e + 1],) + o[1:] for o in (q, k, v)]
        ye = _run(*one, p, 0.125, mask=m[e:e + 1], causal=True, return_p=False).cpu().numpy()
        assert np.array_equal(y[e:e + 1], ye), e


def test_determinism_and_graph_replay_after_growth():
    rng = np.random.default_rng(15)
    lead = (2, 3)
    q, k, v = (attention_operand(rng, lead + (300, 64), False) for _ in range(3))
    p = p_qparams(True, False)
    qt, kt, vt = t(q[0]), t(k[0]), t(v[0])
    mask = torch.zeros(2, 1, 1, 300, device=dev())
    mask[1, ..., 250:] = -10000.0
    qp = [(scalar(o[1]), scalar(o[2]), o[3:]) for o in (q, k)]
    pp, vp = (scalar(p[0]), scalar(p[1]), p[2:]), (scalar(v[1]), scalar(v[2]), v[3:])

    def call(x, y, z, m=mask):
        return ops.int8_attention(x, y, z, qp[0], qp[1], pp, vp, scale=0.125, attn_mask=m, causal=True)

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
        big = [o.repeat(8, 1, 1, 1) for o in (qt, kt, vt)]
        call(*big, m=mask.repeat(8, 1, 1, 1))  # grows the stream's workspace
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


def test_16k_tokens_causal_padded_without_a_t_squared_allocation():
    b, h, tq, d = 1, 2, 16384, 64
    gen = torch.Generator(device=dev()).manual_seed(16)
    q, k, v = (torch.randn(b, h, tq, d, device=dev(), generator=gen) for _ in range(3))
    mask = torch.zeros(b, 1, 1, tq, device=dev())
    mask[..., 15000:] = -10000.0
    s1 = float(q.abs().max()) / 127
    one = lambda x: torch.tensor([x], dtype=torch.float32, device=dev())
    qp, pp = (one(s1), one(0.0), (-128, 127)), (one(1 / 255), one(0.0), (0, 255))
    ops.int8_attention(q[:, :, :256], k[:, :, :256], v[:, :, :256], qp, qp, pp, qp, attn_mask=mask[..., :256],
                       causal=True)  # the library is loaded, the kernel attribute set
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    y = ops.int8_attention(q, k, v, qp, qp, pp, qp, scale=d ** -0.5, attn_mask=mask, causal=True)
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    operands = 3 * q.numel() * 4
    assert grew <= operands, grew  # workspace + out; a copy of the expanded mask alone would be 2 GiB
    print(f"Tq = Tk = {tq} causal + padded: peak allocation grew by {grew / 2**20:.1f} MiB")
    rows = [0, 1, 8191, 15500, 16383]
    for e in range(h):
        qo = (q[0, e, rows].cpu().numpy(), F32(s1), F32(0), -128, 127)
        ko, vo = ((x[0, e].cpu().numpy(), F32(s1), F32(0), -128, 127) for x in (k, v))
        p = (F32(1 / 255), F32(0), 0, 255)
        s, _ = ref.scores(qo, ko, d ** -0.5)
        vis = np.arange(tq)[None, :] <= np.array(rows)[:, None]
        s = (np.where(vis, s, F32(-np.inf)) + mask[0, 0].cpu().numpy()).astype(F32)
        p64 = mref.softmax64(s)
        g64 = ref.p_grid(p64.astype(F32), p)
        lo, hi = ref.admissible_range(p64, p)
        fv = oqdq.qdq(*vo).astype(np.float64)
        fp = oqdq.qdq(p64.astype(F32), *p).astype(np.float64)
        T = fp @ fv
        g_far = np.where(np.abs(lo - g64) > np.abs(hi - g64), lo, hi)
        bound = ref.truth_bound(g_far, g64, p, vo, BOUND * (np.abs(fp) @ np.abs(fv)))
        assert np.all(np.abs(y[0, e, rows].cpu().numpy() - T) <= bound), e


# ---------------------------------------------------------------------------------------------- the synthetic blocks
class Block(nn.Module):
    """A transformer attention around QAttention: fused qkv projection, the quantized attention with a mask, output
    projection.  ``causal=False``: BERT-style, a [B, 1, 1, T] key-padding mask (1 - m) * -10000; ``causal=True``:
    GPT-2-style, the causal band plus the same additive padding mask."""

    def __init__(self, causal, dim=192, heads=3):
        super().__init__()
        self.causal, self.heads, self.head_dim = causal, heads, dim // heads
        self.qkv = QLinear(nn.Linear(dim, 3 * dim)).build_quantizer(
            cfg("per-tensor-symmetric", "feature", layout="NLC"), cfg("per-channel-symmetric", "weight"))
        self.attn = QAttention(scale=self.head_dim ** -0.5).build_quantizer(
            cfg("per-tensor-symmetric", "feature", layout="NLC"), cfg("per-tensor-affine", "feature", layout="NLC"))
        self.proj = QLinear(nn.Linear(dim, dim)).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC"),
                                                                 cfg("per-channel-symmetric", "weight"))

    def forward(self, x, keep):
        mask = (1.0 - keep[:, None, None, :]) * -10000.0
        qkv = self.qkv(x).reshape(x.shape[0], x.shape[1], 3, self.heads, self.head_dim).permute(2, 0, 3, 1, 4)
        out = self.attn(qkv[0], qkv[1], qkv[2], attn_mask=mask, causal=self.causal)
        return self.proj(out.transpose(1, 2).reshape(x.shape[0], x.shape[1], -1))


@pytest.mark.parametrize("causal", [False, True], ids=["bert_padding", "gpt2_causal"])
@pytest.mark.parametrize("replay", [False, True])
def test_synthetic_block_converts_and_meets_the_bounds(causal, replay):
    torch.manual_seed(0)
    t_len = 128 if not causal else 256
    batches = []
    for _ in range(3):
        keep = torch.ones(4, t_len, device=dev())
        keep[1, t_len - 40:] = 0
        keep[3, t_len // 2:] = 0
        batches.append((torch.randn(4, t_len, 192, device=dev()), keep))
    model = calibrated(Block(causal), batches, streaming=not replay, record_inputs=None, replay=replay)
    original = model.attn
    for carrier in (original.qk.left, original.qk.right, original.pv.left, original.pv.right):
        s = float(carrier.input_quantizer.scale.reshape(-1)[0])
        assert s > 0 and s != 1.0  # calibration reached all four carriers
    assert to_integer_linears(model) == ["qkv", "proj"]
    assert to_integer_attentions(model) == ["attn"]
    assert isinstance(model.attn, QAttentionInt8) and isinstance(model.qkv, QLinearInt8)
    seen = {}
    hook = model.attn.register_forward_hook(lambda mod, i, kw, o: seen.__setitem__("attn", (i, kw, o)),
                                            with_kwargs=True)
    with torch.no_grad():
        for x, keep in batches[:2]:
            model(x, keep)
            (qx, kx, vx), kw, y = seen["attn"]
            mask = kw["attn_mask"]
            assert kw["causal"] == causal
            (q, k, v), p = operands_of(original, qx, kx, vx)
            m = mask.cpu().numpy()
            T, g64, mm, _ = mref.truth(q, k, v, p, original.scale, m, causal)
            s, bad = mref.scores(q, k, original.scale, m, causal)
            assert not bad.any()
            lo, hi = ref.admissible_range(mref.softmax64(s), p)
            g_far = np.where(np.abs(lo - g64) > np.abs(hi - g64), lo, hi)
            err = np.abs(y.cpu().numpy() - T)
            assert np.all(err <= ref.truth_bound(g_far, g64, p, v, mm))
            fq_err = np.abs(original(qx, kx, vx, attn_mask=mask, causal=causal).cpu().numpy() - T)
            print(f"attention: fused max |y - T| = {err.max():.3e}, fake-quant max |y - T| = {fq_err.max():.3e}")
    hook.remove()
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    before = launch_count()
    with torch.no_grad():
        model(*batches[0])
    torch.cuda.synchronize()
    # qkv and proj: row quantizer + GEMM each; the attention: two row quantizers, the column quantizer, (causal) the
    # column sums of v, the fused kernel
    assert launch_count() - before == 4 + (5 if causal else 4)
    with torch.no_grad(), profile(activities=[ProfilerActivity.CPU]) as prof:
        model.attn(qx, kx, vx, attn_mask=mask, causal=causal)
        torch.cuda.synchronize()
    aten = {e.name for e in prof.events() if e.name.startswith("aten::")}
    forbidden = {"aten::softmax", "aten::_softmax", "aten::matmul", "aten::bmm", "aten::mm", "aten::where",
                 "aten::add", "aten::add_", "aten::masked_fill", "aten::masked_fill_", "aten::baddbmm"}
    assert not aten & forbidden, sorted(aten & forbidden)


def test_module_masks():
    torch.manual_seed(1)
    qa = QAttention(scale=0.25).build_quantizer(cfg("per-tensor-symmetric", "feature", layout="NLC")).to(dev())
    xs = [torch.randn(2, 3, 20, 16, device=dev()) for _ in range(3)]
    for carrier, x in ((qa.qk.left, xs[0]), (qa.qk.right, xs[1].transpose(-2, -1)), (qa.pv.right, xs[2]),
                       (qa.pv.left, torch.rand(2, 3, 20, 20, device=dev()))):
        carrier.input_quantizer.update_observer(x)
        carrier.input_quantizer.calc_qparams()
    qa.set_quant(a_quant=True)
    mod = QAttentionInt8.from_qattention(qa)
    m = torch.zeros(2, 1, 1, 20, device=dev())
    m[1, ..., 15:] = -10000.0
    with torch.no_grad():
        y = mod(*xs, attn_mask=m, causal=True)
        assert torch.equal(mod(*xs, attn_mask=m.half(), causal=True), y)  # fp16 masks are up-cast exactly
        assert torch.equal(mod(*xs, attn_mask=m.expand(2, 3, 20, 20).transpose(-2, -1).contiguous().transpose(-2, -1),
                               causal=True), y)  # a key stride != 1 is copied
        assert torch.equal(mod(*xs), ops.int8_attention(*xs, *[(getattr(mod, f"{r}_scale"), getattr(mod, f"{r}_zero_point"),
                                                                 mod.qranges[r]) for r in mod.ROLES], scale=0.25))
        with pytest.raises(TypeError, match="bool mask"):
            mod(*xs, attn_mask=m == 0)
        with pytest.raises(Exception, match="does not broadcast"):
            mod(*xs, attn_mask=torch.zeros(3, 1, 1, 20, device=dev()))
