"""GPU: the int8 key/value cache (ops.Int8KVCache, ops.int8_kv_append, ops.int8_attention_cached and
QAttentionInt8.forward(..., cache=)) against the uncached fused attention and tests/int8_attention_ref.py /
int8_attention_mask_ref.py.

* After appends of uneven sizes every cache buffer is what int8_quantize_rows / int8_quantize_cols write for the
  concatenated keys and values, NaN flags included, and every byte past the stored keys is 0.
* Tq > 16: bit-identical to ops.int8_attention on the concatenated operands (plain, a [B, 1, 1, Tk] padding view,
  causal), p_q included.
* Tq <= 16 (the split-key decode kernels): out is exact on the kernel's own p grid, every p is admissible, NaN rows and
  columns follow the fused kernel's rules, and against the fused kernel every p grid value is within one step (the
  mismatches are counted and reported).
* NaN placement, batch isolation, determinism, launches per decode step, and a two-block mini GPT-2 decoding through
  the caches of its converted attentions."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_attention_mask_ref as mref
import int8_attention_ref as ref
from gpu_util import dev, t
from gpu_util import no_tf32_autouse  # noqa: F401 -- TF32 off on every test
from int8_harness import attention_operand, calibrated, cfg, check_p, p_qparams, scalar
from sparsebit_b200 import SparsebitB200Error, launch_count, ops
from sparsebit_b200.quantization.modules import QAttention, QAttentionInt8, QLinear
from sparsebit_b200.quantization.tools import to_integer_attentions, to_integer_linears

pytestmark = pytest.mark.gpu

F32 = np.float32


def qparams(o):
    return (scalar(o[1]), scalar(o[2]), o[3:])


def pparams(p):
    return (scalar(p[0]), scalar(p[1]), p[2:])


def fill(q, k, v, chunks, capacity):
    """A cache of ``capacity`` with k, v appended in ``chunks`` (token counts), as ops.int8_kv_append does."""
    lead, d, dv = k[0].shape[:-2], k[0].shape[-1], v[0].shape[-1]
    cache = ops.Int8KVCache(None, lead, capacity, d, dv, dev())
    at = 0
    for n in chunks:
        ops.int8_kv_append(cache, t(np.ascontiguousarray(k[0][..., at:at + n, :])),
                           t(np.ascontiguousarray(v[0][..., at:at + n, :])), qparams(k), qparams(v))
        at += n
    assert cache.length == at == k[0].shape[-2]
    return cache


def cached(q, cache, k, v, p, scale=None, mask=None, causal=False):
    m = None if mask is None else (mask if isinstance(mask, torch.Tensor) else t(mask))
    return ops.int8_attention_cached(t(q[0]), cache, qparams(q), qparams(k), pparams(p), qparams(v), scale=scale,
                                     return_p=True, attn_mask=m, causal=causal)


def fused(q, k, v, p, scale=None, mask=None, causal=False):
    m = None if mask is None else (mask if isinstance(mask, torch.Tensor) else t(mask))
    return ops.int8_attention(t(q[0]), t(k[0]), t(v[0]), qparams(q), qparams(k), pparams(p), qparams(v), scale=scale,
                              return_p=True, attn_mask=m, causal=causal)


def operands(seed, lead, tq, tk, d, dv, kq=(-128, 127), vq=(0, 255)):
    rng = np.random.default_rng(seed)
    q = attention_operand(rng, lead + (tq, d), False, 2.0)
    k = attention_operand(rng, lead + (tk, d), False, 2.0, kq)
    v = attention_operand(rng, lead + (tk, dv), False, 1.0, vq)
    return rng, q, k, v


def check_decode(q, k, v, p, scale, mask, causal, cache, label):
    """Contract (b)-(e) of the decode kernels; returns (out, p_q, mismatched p entries)."""
    y, pq = cached(q, cache, k, v, p, scale, mask, causal)
    y, g = y.cpu().numpy(), pq.cpu().numpy()
    tq, tk = q[0].shape[-2], k[0].shape[-2]
    exp = mref.expected(g, q, k, v, p, scale, mask, causal)
    assert np.array_equal(y, exp, equal_nan=True), label                       # (c) (d)
    s, bad = mref.scores(q, k, scale, mask, causal)                            # (a) the exact scores, restated
    check_p(g, s, bad, p, tq, tk, False, label)                                # (b)
    _, gf = fused(q, k, v, p, scale, mask, causal)
    gf = gf.cpu().numpy()
    diff = np.abs(g.astype(np.int64) - gf)
    assert diff.max() <= 1, label                                              # (e)
    print(f"{label}: {int((diff != 0).sum())} of {diff.size} p grid entries differ from the fused kernel (by one step)")
    return y, g, int((diff != 0).sum())


def test_append_matches_the_quantizers():
    _, q, k, v = operands(1, (2, 3), 1, 349, 80, 40)
    k[0][1, 2, 20, 5] = np.nan
    v[0][0, 1, 300, 7] = np.nan
    cache = fill(q, k, v, (1, 15, 16, 17, 300), 400)
    kt, vt = t(k[0]), t(v[0])
    rq, rs, rn = ops.int8_quantize_rows(kt.reshape(-1, 80), qparams(k)[0], qparams(k)[1], -128, 127)
    cq, cs, cn = ops.int8_quantize_cols(vt, qparams(v)[0], qparams(v)[1], 0, 255)
    L = 349
    assert torch.equal(cache.k_q[..., :L, :].reshape(-1, 80), rq)
    assert torch.equal(cache.k_sum[..., :L].reshape(-1), rs) and torch.equal(cache.k_nan[..., :L].reshape(-1), rn)
    assert torch.equal(cache.v_t[..., :ref.padded(L)], cq)
    assert torch.equal(cache.v_sum, cs) and torch.equal(cache.v_nan, cn)
    assert bool(cache.k_nan[1, 2, 20]) and bool(cache.v_nan[0, 1, 7])
    assert not cache.k_q[..., L:, :].any() and not cache.k_sum[..., L:].any() and not cache.k_nan[..., L:].any()
    assert not cache.v_t[..., L:].any()


@pytest.mark.parametrize("kind", ["plain", "pad", "causal"])
@pytest.mark.parametrize("unsigned_p", [True, False])
def test_long_query_blocks_are_the_fused_kernel(kind, unsigned_p):
    lead, tq, tk = (2, 3), 40, 300
    rng, q, k, v = operands(2, lead, tq, tk, 64, 64)
    p = p_qparams(unsigned_p, False)
    mask = None
    if kind == "pad":
        keep = np.ones((lead[0], 1, 1, tk), F32)
        keep[1, ..., 250:] = 0
        mask = t(np.where(keep == 0, F32(-10000), F32(0)).astype(F32))
    causal = kind == "causal"
    cache = fill(q, k, v, (17, 243, 40), 333)
    y, g = cached(q, cache, k, v, p, 0.125, mask, causal)
    yf, gf = fused(q, k, v, p, 0.125, mask, causal)
    assert torch.equal(y, yf) and torch.equal(g, gf)


@pytest.mark.parametrize("tq", [1, 2, 16])
@pytest.mark.parametrize("kind", ["plain", "pad", "causal"])
def test_decode_contract(tq, kind):
    lead, tk = (2, 3), 700
    rng, q, k, v = operands(3 + tq, lead, tq, tk, 64, 40)
    p = p_qparams(True, False)
    mask, causal = None, kind == "causal"
    if kind == "pad":
        keep = np.ones((lead[0], 1, 1, tk), F32)
        keep[0, ..., 500:] = 0
        mask = np.where(keep == 0, F32(-np.inf), F32(0)).astype(F32)
    cache = fill(q, k, v, (tk - 1, 1), 1000)
    check_decode(q, k, v, p, 0.125, mask, causal, cache, f"tq={tq} {kind}")


def test_nan_placement_and_batch_isolation():
    lead, tq, tk = (3,), 4, 300
    rng, q, k, v = operands(5, lead, tq, tk, 64, 40)
    p = p_qparams(True, False)
    clean = cached(q, fill(q, k, v, (tk,), 512), k, v, p, 0.125, None, True)[0].cpu().numpy()
    assert np.isfinite(clean).all()
    k[0][0, 298, 2] = np.nan  # entry 0: rows 2, 3 see key 298 (row i sees keys <= i + 296)
    v[0][1, 299, 7] = np.nan  # entry 1: column 7 NaN in every row
    q[0][2, 1, 0] = np.nan    # entry 2: row 1
    y = check_decode(q, k, v, p, 0.125, None, True, fill(q, k, v, (150, 150), 512), "nan")[0]
    expect = np.zeros(y.shape, bool)
    expect[0, 2:] = True
    expect[1, :, 7] = True
    expect[2, 1] = True
    assert np.array_equal(np.isnan(y), expect)
    assert np.array_equal(y[~expect], clean[~expect])
    # without causal a NaN key poisons the whole entry; a row that sees no key (causal with Tq > Tk) is NaN
    y = check_decode(q, k, v, p, 0.125, None, False, fill(q, k, v, (tk,), 512), "nan plain")[0]
    assert np.isnan(y[0]).all()
    _, q2, k2, v2 = operands(6, (2,), 8, 5, 64, 40)
    y = check_decode(q2, k2, v2, p, None, None, True, fill(q2, k2, v2, (5,), 64), "rows without keys")[0]
    assert np.isnan(y[:, :3]).all() and np.isfinite(y[:, 3:]).all()


def test_determinism_and_launches_per_step():
    lead, tq, tk = (8, 12), 1, 1024
    _, q, k, v = operands(7, lead, tq, tk, 64, 64)
    p = p_qparams(True, False)
    cache = fill(q, k, v, (tk,), 2048)
    runs = [cached(q, cache, k, v, p, 0.125, None, True) for _ in range(3)]
    for y, g in runs[1:]:
        assert torch.equal(y, runs[0][0]) and torch.equal(g, runs[0][1])
    attn = QAttentionInt8(dev(), 0.125)
    c = attn.new_cache(lead, 64, 64, 64)
    x = torch.randn(lead + (1, 64), device=dev())
    with torch.no_grad():
        attn(x, x, x, causal=True, cache=c)
        torch.cuda.synchronize()
        before = launch_count()
        attn(x, x, x, causal=True, cache=c)  # append, q's quantizer, scores, p @ v, combine
        torch.cuda.synchronize()
        assert launch_count() - before == 5
        before = launch_count()
        attn(torch.randn(lead + (17, 64), device=dev()), *(torch.randn(lead + (17, 64), device=dev()),) * 2,
             causal=True, cache=c)  # append, q's quantizer, the column sums of v, the fused kernel
        torch.cuda.synchronize()
        assert launch_count() - before == 4


def test_module_errors():
    attn, other = QAttentionInt8(dev()), QAttentionInt8(dev())
    c = attn.new_cache((2,), 8, 16, 16)
    x = torch.randn(2, 3, 16, device=dev())
    with torch.no_grad():
        with pytest.raises(ValueError, match="new_cache"):
            other(x, x, x, cache=c)
        with pytest.raises(ValueError, match="lead"):
            attn(x[:1], x[:1], x[:1], cache=c)
        with pytest.raises(ValueError, match="dv"):
            attn(x, x, torch.randn(2, 3, 8, device=dev()), cache=c)
        attn(x, x, x, cache=c)
        attn(x, x, x, cache=c)
        with pytest.raises(SparsebitB200Error, match="capacity"):
            attn(x, x, x, cache=c)
        assert c.length == 6
    with pytest.raises(RuntimeError, match="inference-only"):
        attn(x.requires_grad_(), x, x, cache=c)


# ---------------------------------------------------------------------------------------------- a mini GPT-2
class Block(nn.Module):
    def __init__(self, dim=128, heads=4):
        super().__init__()
        self.heads, self.hd = heads, dim // heads
        act, wt = cfg("per-tensor-symmetric", "feature", layout="NLC"), cfg("per-channel-symmetric", "weight")
        self.q, self.k, self.v, self.proj = (QLinear(nn.Linear(dim, dim)).build_quantizer(act, wt) for _ in range(4))
        self.attn = QAttention(scale=self.hd ** -0.5).build_quantizer(act, cfg("per-tensor-affine", "feature",
                                                                                  layout="NLC"))
        self.fc, self.out = QLinear(nn.Linear(dim, 2 * dim)).build_quantizer(act, wt), \
            QLinear(nn.Linear(2 * dim, dim)).build_quantizer(act, wt)

    def heads_of(self, x):
        return x.reshape(x.shape[0], x.shape[1], self.heads, self.hd).transpose(1, 2)

    def forward(self, x, cache=None):
        q, k, v = (self.heads_of(m(x)) for m in (self.q, self.k, self.v))
        a = self.attn(q, k, v, causal=True) if cache is None else self.attn(q, k, v, causal=True, cache=cache)
        x = x + self.proj(a.transpose(1, 2).reshape(x.shape))
        return x + self.out(torch.relu(self.fc(x)))


class MiniGPT(nn.Module):
    def __init__(self):
        super().__init__()
        self.blocks = nn.ModuleList([Block(), Block()])

    def forward(self, x, caches=None):
        for i, b in enumerate(self.blocks):
            x = b(x) if caches is None else b(x, caches[i])
        return x


def _layer_operands(mod, q, k, v):
    """The reference operand tuples of q, k, v and p's qparams under a converted attention's qparams."""
    def op(x, role):
        return (x.cpu().numpy(), F32(getattr(mod, f"{role}_scale").item()),
                F32(getattr(mod, f"{role}_zero_point").item()), *mod.qranges[role])
    p = (F32(mod.p_scale.item()), F32(mod.p_zero_point.item()), *mod.qranges["p"])
    return op(q, "q"), op(k, "k"), op(v, "v"), p


def test_mini_gpt2_decodes_through_the_cache():
    """A 200-token prefill, 40 one-token steps and two 4-token steps.  Per attention layer and step, the cached call is
    compared with the fused kernel on the concatenated fp32 keys and values that layer appended: the prefill bit for
    bit; a decode step's p grid within one step of the fused kernel's (mismatches counted and reported), its rows
    without a mismatch bit-identical, and every row within truth_bound of the fp64 attention on its own p grid.  The
    model output equals the uncached converted model's run on the full sequence when no p grid entry differs."""
    torch.manual_seed(0)
    batches = [torch.randn(2, 248, 128, device=dev()) for _ in range(2)]
    model = calibrated(MiniGPT(), batches, streaming=True, record_inputs=None)
    assert len(to_integer_linears(model)) == 12 and len(to_integer_attentions(model)) == 2
    attns = [b.attn for b in model.blocks]
    past = [None, None]  # per layer: the fp32 (k, v) appended so far
    mismatched = [0, 0]

    def hook(i):
        def check(mod, args, kwargs, out):
            if kwargs.get("cache") is None:
                return
            q, k, v = args
            past[i] = (k, v) if past[i] is None else tuple(torch.cat((a, b), -2) for a, b in zip(past[i], (k, v)))
            pk, pv = past[i]
            qp = [(getattr(mod, f"{r}_scale"), getattr(mod, f"{r}_zero_point"), mod.qranges[r]) for r in mod.ROLES]
            y, g = ops.int8_attention_cached(q, kwargs["cache"], *qp, scale=mod.scale, return_p=True, causal=True)
            yf, gf = ops.int8_attention(q, pk, pv, *qp, scale=mod.scale, return_p=True, causal=True)
            assert torch.equal(y, out)  # deterministic: the forward's own output
            if q.shape[-2] > 16:
                assert torch.equal(y, yf) and torch.equal(g, gf)
                return
            diff = (g.long() - gf.long()).abs()
            assert int(diff.max()) <= 1
            mismatched[i] += int((diff != 0).sum())
            same = ~(diff != 0).any(-1)
            assert torch.equal(y[same], yf[same])
            qo, ko, vo, p = _layer_operands(mod, q, pk, pv)
            T, g64, mm, _ = mref.truth(qo, ko, vo, p, mod.scale, None, True)
            tk = pk.shape[-2]
            bound = ref.truth_bound(g.cpu().numpy()[..., :tk], g64, p, vo, mm)
            err = np.abs(y.cpu().numpy().astype(np.float64) - T)
            good = np.isfinite(T)
            assert np.all(err[good] <= bound[good])
        return check

    hooks = [a.register_forward_hook(hook(i), with_kwargs=True) for i, a in enumerate(attns)]
    x = batches[0]
    caches = [a.new_cache((2, 4), 256, 32, 32) for a in attns]
    steps = [200] + [1] * 40 + [4, 4]
    at = 0
    with torch.no_grad():
        for n in steps:
            before = list(mismatched)
            y = model(x[:, at:at + n], caches)
            full = model(x[:, :at + n])[:, at:]
            if mismatched == before:
                assert torch.equal(y, full), at
            else:
                assert float((y - full).abs().max() / full.abs().max()) < 2e-2, at
            at += n
        assert all(c.length == 248 for c in caches)
    for h in hooks:
        h.remove()
    print(f"mini GPT-2: 42 decode steps, p grid entries differing from the fused kernel per layer: {mismatched}")
