"""CPU: the host side of sb200_int8_kv_append and sb200_int8_attention_cached and of their Python wrappers.

* Every bad argument of either entry point is rejected on the host before any CUDA call (there is no device here).
* The workspace query is a pure function and 0 for arguments the attention rejects.
* The branch cases of tests/test_gpu_int8_attention_cache_branches.py reach every branch of the launch plan."""
import numpy as np
import pytest
import torch

import int8_attention_cache_geometry as geo
from int8_harness import E_INVALID, E_UNSUPPORTED, E_WORKSPACE, buf, rejector
from sparsebit_b200 import SparsebitB200Error, _lib, ops
from sparsebit_b200.quantization.modules import QAttentionInt8
from test_gpu_int8_attention_cache_branches import CASES, case_branches


# k v | k: s z lo hi | v: s z lo hi | k_q k_sum k_nan v_t v_sum v_nan | batch capacity length t d dv | stream
def _append_args(p):
    return [p, p, p, p, -128, 127, p, p, 0, 255, p, p, p, p, p, p, 6, 100, 90, 10, 64, 32, None]


def test_append_rejects_bad_arguments_on_the_host():
    lib = _lib.load()
    keep, p = buf()
    rejected = rejector(lib.sb200_int8_kv_append, _append_args(p), prefix=b"sb200_int8_kv_append")
    for i in (0, 1, 2, 3, 6, 7, 10, 11, 12, 13, 14, 15):
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    for i in (16, 17, 19, 20, 21):
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
    rejected(E_INVALID, b"negative length", a18=-1)
    rejected(E_INVALID, b"do not fit", a19=11)                    # 90 + 11 > 100
    rejected(E_UNSUPPORTED, b"capacity < 2^17", a17=1 << 17, a18=0)
    rejected(E_UNSUPPORTED, b"d <= 128", a20=129)
    rejected(E_UNSUPPORTED, b"dv <= 128", a21=129)
    rejected(E_INVALID, b"batch capacity", a16=1 << 15, a17=1 << 16, a18=0)
    rejected(E_INVALID, b"16-byte aligned", a10=p + 4)
    rejected(E_INVALID, b"16-byte aligned", a13=p + 8)
    rejected(E_INVALID, b"wider than 8 bits", a4=-128, a5=128)
    rejected(E_INVALID, b"neither signed", a8=-5, a9=200)


# q | q: s z lo hi | k: s z lo hi | p: s z lo hi | v: s z lo hi | has_scale scale | mask so si inner sr causal |
# k_q k_sum k_nan v_t v_sum v_nan | capacity length | out p_q | batch tq d dv | ws ws_bytes stream
def _cached_args(p, ws_bytes, tq=5, causal=1):
    return [p, p, p, -128, 127, p, p, -128, 127, p, p, 0, 255, p, p, -128, 127, 1, 0.125,
            p, 7, 0, 3, 0, causal, p, p, p, p, p, p, 100, 90, p, p, 6, tq, 64, 32, p, ws_bytes, None]


@pytest.mark.parametrize("tq", [5, 17])
def test_cached_attention_rejects_bad_arguments_on_the_host(tq):
    lib = _lib.load()
    keep, p = buf()
    ws_ok = int(lib.sb200_int8_attention_cached_workspace_bytes(6, tq, 100, 90, 64, 32, 1))
    assert ws_ok > 0
    rejected = rejector(lib.sb200_int8_attention_cached, _cached_args(p, ws_ok, tq), prefix=b"sb200_int8_attention_cached")
    for i in (0, 1, 2, 5, 6, 9, 10, 13, 14, 25, 26, 27, 28, 29, 30, 33, 39):  # the mask (19) and p_q (34) may be null
        rejected(E_INVALID, b"null pointer", **{f"a{i}": None})
    rejected(E_INVALID, b"empty cache", a31=0)
    for i in (32, 35, 36, 37, 38):
        rejected(E_INVALID, b"empty operand", **{f"a{i}": 0})
    rejected(E_INVALID, b"do not fit", a32=101)
    rejected(E_UNSUPPORTED, b"capacity < 2^17", a31=1 << 17)
    rejected(E_UNSUPPORTED, b"d <= 128", a37=129)
    rejected(E_UNSUPPORTED, b"dv <= 128", a38=129)
    rejected(E_INVALID, b"batch capacity", a35=1 << 15, a31=1 << 16)
    rejected(E_INVALID, b"16-byte aligned", a25=p + 4)
    rejected(E_INVALID, b"16-byte aligned", a28=p + 1)
    rejected(E_INVALID, b"16-byte aligned", a34=p + 2)            # p_q
    rejected(E_INVALID, b"wider than 8 bits", a11=-128, a12=128)
    rejected(E_INVALID, b"not finite", a18=float("inf"))
    rejected(E_INVALID, b"causal must be 0 or 1", a24=2)
    rejected(E_INVALID, b"negative mask stride", a20=-1)
    rejected(E_INVALID, b"mask_inner", a22=4)
    rejected(E_INVALID, b"4-byte aligned", a19=p + 1)
    rejected(E_WORKSPACE, b"workspace too small", a40=ws_ok - 1)


def test_workspace_query_is_pure():
    lib = _lib.load()
    q = lib.sb200_int8_attention_cached_workspace_bytes
    for tq in (1, 16, 17, 300):
        for causal in (0, 1):
            a = q(8, tq, 4096, 1000, 64, 64, causal)
            assert a > 0 and a == q(8, tq, 4096, 1000, 64, 64, causal)
            assert a == q(8, tq, 2048, 1000, 64, 64, causal)  # the capacity is not workspace
    assert q(8, 17, 4096, 1000, 64, 64, 1) > q(8, 17, 4096, 1000, 64, 64, 0)  # causal: the column sums of v
    assert q(8, 1, 4096, 2000, 64, 64, 0) > q(8, 1, 4096, 1000, 64, 64, 0)    # decode: the scores
    for bad in ((0, 1, 8, 4, 16, 16, 0), (1, 0, 8, 4, 16, 16, 0), (1, 1, 0, 0, 16, 16, 0), (1, 1, 8, 0, 16, 16, 0),
                (1, 1, 8, 9, 16, 16, 0), (1, 1, 1 << 17, 4, 16, 16, 0), (1, 1, 8, 4, 129, 16, 0),
                (1, 1, 8, 4, 16, 129, 0), (1, 1, 8, 4, 16, 16, 2), (1 << 15, 1, 1 << 16, 4, 16, 16, 0)):
        assert q(*bad) == 0, bad


def test_split_plan():
    assert geo.split(96, 512) == (128, 4)       # GPT-2 small at batch 8: 4 splits of 128 keys per (batch, head)
    assert geo.split(32, 4096) == (256, 16)     # LLaMA-7B heads at batch 1
    assert geo.split(1000, 100000) == (2048, 49)
    for e, n in ((1, 1), (7, 129), (528, 2177), (3, 131071)):
        s, ns = geo.split(e, n)
        assert s % 128 == 0 and s <= geo.MAX_SPLIT and (ns - 1) * s < n <= ns * s


def test_cases_reach_every_branch():
    reached = set()
    for name in CASES:
        reached |= case_branches(name)
    assert reached == set(geo.ALL), sorted(set(geo.ALL) - reached)


def test_python_errors_before_any_launch():
    cache = ops.Int8KVCache(None, (2,), 8, 16, 16, torch.device("cpu"))
    assert cache.k_q.shape == (2, 8, 16) and cache.v_t.shape == (2, 16, 16) and cache.length == 0
    one = (torch.ones(1), torch.zeros(1), (-128, 127))
    x = torch.zeros(2, 9, 16)
    with pytest.raises(SparsebitB200Error, match="overflow"):
        ops.int8_kv_append(cache, x, x, one, one)
    with pytest.raises(SparsebitB200Error, match="do not match"):
        ops.int8_kv_append(cache, x[:1, :2], x[:1, :2], one, one)
    with pytest.raises(SparsebitB200Error, match="empty"):
        ops.int8_attention_cached(x[:, :1], cache, one, one, one, one)
    with pytest.raises(SparsebitB200Error, match="positive"):
        ops.Int8KVCache(None, (2,), 0, 16, 16, torch.device("cpu"))
    attn = QAttentionInt8(torch.device("cpu"))
    c = attn.new_cache((2,), 8, 16, 16)
    assert c.layer is attn
    with pytest.raises(ValueError, match="new_cache"):
        QAttentionInt8(torch.device("cpu"))(x, x, x, cache=c)
    with pytest.raises(ValueError, match="do not match"):
        attn(x[:1], x[:1], x[:1], cache=c)
    with pytest.raises(SparsebitB200Error, match="attn_mask"):  # [2, 3, 4] does not broadcast to [2, 9, 3]
        attn(x, x[:, :3], x[:, :3], attn_mask=torch.zeros(2, 3, 4), cache=c)
    with pytest.raises(SparsebitB200Error, match="causal must be a bool"):
        attn(x, x[:, :3], x[:, :3], causal="yes", cache=c)
    assert c.length == 0  # nothing was appended
