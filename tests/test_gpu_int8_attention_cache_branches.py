"""GPU: one case per launch branch of the attention over an int8 key/value cache (tests/int8_attention_cache_geometry.py
names the branches; tests/test_int8_attention_cache_host.py checks on the CPU that together the cases reach all of
them).  Decode cases meet the contract of the split-key kernels (test_gpu_int8_attention_cache.check_decode); routed
cases with Tq > 16 are bit-identical to the fused kernel on the concatenated operands."""
import numpy as np
import pytest
import torch

import int8_attention_cache_geometry as geo
from int8_harness import p_qparams
from test_gpu_int8_attention_cache import cached, check_decode, fill, fused, operands

pytestmark = pytest.mark.gpu

F32 = np.float32
P_OFF = (F32(1 / 255), F32(-3), 0, 255)  # p's zero point off its range: the grid of p = 0 is not Z_p

# name: (lead, Tq, capacity, length, d, dv, p_signed, zp_off, causal)
CASES = {
    "one_split_tail_1": ((1, 1), 1, 16, 1, 16, 16, False, False, False),
    "two_splits_full_cache": ((2, 132), 2, 256, 256, 64, 64, True, False, False),
    "many_splits_tail_127_causal": ((1, 1), 4, 1000, 767, 80, 80, False, False, True),
    "split_capped_tail_129": ((4, 132), 1, 2200, 2177, 32, 16, False, False, False),
    "route_16_decode": ((2, 2), 16, 300, 300, 128, 128, False, True, True),
    "route_17_fused": ((2, 2), 17, 300, 300, 128, 128, False, True, True),
}


def case_branches(name):
    lead, tq, cap, length, d, dv, p_signed, zp_off, causal = CASES[name]
    return geo.branches(int(np.prod(lead)), tq, cap, length, d, dv, p_signed, zp_off, causal)


@pytest.mark.parametrize("name", sorted(CASES))
def test_branch_case(name):
    lead, tq, cap, length, d, dv, p_signed, zp_off, causal = CASES[name]
    _, q, k, v = operands(sum(map(ord, name)), lead, tq, length, d, dv)
    p = P_OFF if zp_off else p_qparams(not p_signed, False)
    chunks = (length,) if length < 3 else (length - 2, 1, 1)
    cache = fill(q, k, v, chunks, cap)
    if tq > geo.DEC_ROWS:
        y, g = cached(q, cache, k, v, p, d ** -0.5, None, causal)
        yf, gf = fused(q, k, v, p, d ** -0.5, None, causal)
        assert torch.equal(y, yf) and torch.equal(g, gf)
    else:
        check_decode(q, k, v, p, d ** -0.5, None, causal, cache, name)
