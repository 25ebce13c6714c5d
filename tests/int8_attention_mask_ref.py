"""numpy restatement of the masked and causal fused attention (sb200_int8_attention_masked, csrc/int8_attention.cu,
int8_attention_kernel<true>), on top of tests/int8_attention_ref.py.

Scores, per batch entry, after the unmasked kernel's s (and its scale):
    causal:  s[i, j] = -inf where j > i + (Tk - Tq)       (bottom-right band, QAttention / the reference's GPT-2)
    mask:    s[i, j] = RN32(s[i, j] + mask[i, j])          (one fp32 add)
NaN rules of the composition: a NaN in q row i makes row i NaN; a NaN in k at key j makes NaN the rows that see key j
(all rows without causal); a NaN in column n of v makes column n NaN in every row; a row without a visible key, or with
a NaN score, is NaN.  The launch plan: a CTA of 128 rows visits the key blocks up to the last key its last row sees;
the skipped keys hold p = 0 (their grid in p_q).  ``branches`` names the kernel paths of the masked instantiation a call
reaches (the unmasked kernel's list stays in tests/int8_attention_geometry.py)."""
import numpy as np

import int8_attention_ref as ref
from int8_geometry import cdiv
from int8_matmul_ref import BOUND, stored_grid
from oracle import qdq as oqdq

F32, F64 = np.float32, np.float64
ROWS = KEYS = 128

ALL = ("masked", "mask_row_broadcast", "mask_full", "mask_two_level_batch", "causal_diagonal_block",
       "causal_skipped_blocks", "causal_no_skip", "rows_without_keys", "cta_without_keys", "p_q_fill", "nan_k_hidden",
       "nan_v_hidden")


def visible(tq, tk, causal):
    """[Tq, Tk] bool: key j is visible to query row i."""
    if not causal:
        return np.ones((tq, tk), bool)
    return np.arange(tk)[None, :] <= np.arange(tq)[:, None] + (tk - tq)


def visited_blocks(tq, tk, causal):
    """Per row tile, the number of 128-key blocks the CTA visits (at_visible_blocks)."""
    nkb = cdiv(tk, KEYS)
    if not causal:
        return [nkb] * cdiv(tq, ROWS)
    out = []
    for m0 in range(0, tq, ROWS):
        last = min(m0 + ROWS, tq) - 1 + tk - tq
        out.append(0 if last < 0 else min(nkb, last // KEYS + 1))
    return out


def skipped(tq, tk, causal):
    """[Tq, Tk] bool: the keys the kernel never visits for each row."""
    tkp = cdiv(tk, KEYS) * KEYS
    out = np.zeros((tq, tkp), bool)
    for t, nvb in enumerate(visited_blocks(tq, tk, causal)):
        out[t * ROWS:(t + 1) * ROWS, nvb * KEYS:] = True
    return out[:, :tk]


def masked(s, mask=None, causal=False):
    """The masked fp32 scores of QAttention: -inf outside the band, then one fp32 add of the mask."""
    tq, tk = s.shape[-2:]
    s = np.where(visible(tq, tk, causal), s, F32(-np.inf)).astype(F32)
    if mask is not None:
        with np.errstate(invalid="ignore"):
            s = (s + np.asarray(mask, F32)).astype(F32)
    return s


def scores(q, k, scale=None, mask=None, causal=False):
    """(masked fp32 scores [..., Tq, Tk], NaN rows [..., Tq])."""
    s, _ = ref.scores(q, k, scale)
    s = masked(s, mask, causal)
    tq, tk = s.shape[-2:]
    _, nq = stored_grid(*q)
    _, nk = stored_grid(*k)
    kn = nk.any(-1)  # [..., Tk]
    bad = nq.any(-1) | (kn[..., None, :] & visible(tq, tk, causal)).any(-1)
    with np.errstate(invalid="ignore"):
        bad = bad | np.isnan(s).any(-1) | (np.where(np.isnan(s), F32(0), s).max(-1) == -np.inf)
    return s, bad


def softmax64(s):
    """The fp64 softmax of the masked scores; NaN rows where no key is visible."""
    s = s.astype(F64)
    with np.errstate(invalid="ignore"):
        e = np.exp(s - s.max(-1, keepdims=True))
        return e / e.sum(-1, keepdims=True)


def expected(pq, q, k, v, p, scale=None, mask=None, causal=False):
    """What the kernel must write given its own p grid: the exact integer p @ v with the NaN rows and columns."""
    _, bad = scores(q, k, scale, mask, causal)
    y = ref.stage3(pq, k[0].shape[-2], p, v)
    return np.where(bad[..., None], F32(np.nan), y)


def truth(q, k, v, p, scale=None, mask=None, causal=False):
    """(T, g64, the matmul bound term, f_v) as ref.truth, on the masked scores."""
    s, _ = scores(q, k, scale, mask, causal)
    p64 = softmax64(s)
    fp = oqdq.qdq(p64.astype(F32), F32(p[0]), F32(p[1]), p[2], p[3]).astype(F64)
    fv = oqdq.qdq(*v).astype(F64)
    with np.errstate(all="ignore"):
        return np.matmul(fp, fv), ref.p_grid(p64.astype(F32), p), BOUND * np.matmul(np.abs(fp), np.abs(fv)), fv


def p_zero_grid(p):
    """The stored grid of p = 0."""
    return int(ref.p_grid(np.zeros(1, F32), p)[0])


def branches(batch, tq, tk, mask_kind=None, causal=False, p_q=True, nan=()):
    """The masked-kernel branches a call reaches.  ``mask_kind``: None, "row" (a [B, 1, 1, Tk]-style mask with row
    stride 0), "full" (a row stride > 0), each "two_level" when the batch offset uses both levels; ``nan``: "k_hidden"
    (a NaN key that causal hides from some rows) and / or "v_hidden" (a NaN v at such a key)."""
    out = {"masked"}
    if mask_kind is not None:
        out.add("mask_row_broadcast" if mask_kind.startswith("row") else "mask_full")
        if mask_kind.endswith("two_level"):
            out.add("mask_two_level_batch")
    if causal:
        nvb = visited_blocks(tq, tk, True)
        nkb = cdiv(tk, KEYS)
        out.add("causal_skipped_blocks" if min(nvb) < nkb else "causal_no_skip")
        if any((t * ROWS + tk - tq) // KEYS < n for t, n in enumerate(nvb)):
            out.add("causal_diagonal_block")  # a visited block holds keys some row of the CTA does not see
        if tq > tk:
            out.add("rows_without_keys")
        if min(nvb) == 0:
            out.add("cta_without_keys")
        if p_q and min(nvb) < nkb:
            out.add("p_q_fill")
    out.update(f"nan_{n}" for n in nan)
    return out
