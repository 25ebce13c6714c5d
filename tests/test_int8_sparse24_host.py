"""CPU: the numpy restatement of the 2:4 mask and weight format (tests/int8_sparse24_ref.py) on crafted cases, its
round trip to the dense centred grid, the ineligibility rules that need no device, and the argument errors of the
2:4 entry points, which are reported before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch.nn as nn

import int8_sparse24_ref as ref
from sparsebit_b200 import _lib
from sparsebit_b200.quantization.modules import QLinear, int8_sparse24_ineligibility

F32 = np.float32
NAN, INF = np.float32(np.nan), np.float32(np.inf)


@pytest.mark.parametrize("row, keep", [
    ([1, 2, 3, 4], [0, 0, 1, 1]),
    ([4, 3, 2, 1], [1, 1, 0, 0]),
    ([-5, 1, 5, 0], [1, 0, 1, 0]),            # |w| ties the sign
    ([2, 2, 2, 2], [1, 1, 0, 0]),             # ties go to the lower index
    ([1, 3, 3, 3], [0, 1, 1, 0]),
    ([0.0, -0.0, 0.0, -0.0], [1, 1, 0, 0]),   # +-0 rank as 0
    ([-0.0, 0.0, 1e-45, 0.0], [1, 0, 1, 0]),  # a subnormal beats zero
    ([1, NAN, 2, 3], [0, 1, 0, 1]),           # NaN above every number
    ([NAN, INF, -INF, 7], [1, 1, 0, 0]),
    ([INF, 1, -INF, 2], [1, 0, 1, 0]),
    ([NAN, 1, NAN, NAN], [1, 0, 1, 0]),       # NaNs tie among themselves
    ([1, 2, 3, 4, 9], [0, 0, 1, 1, 1]),       # tail of 1 keeps it
    ([1, 2, 3, 4, 9, 8], [0, 0, 1, 1, 1, 1]), # tail of 2 keeps both
    ([1, 2, 3, 4, 9, 8, 10], [0, 0, 1, 1, 1, 0, 1]),  # tail of 3 keeps 2
    ([5], [1]),
    ([5, 6, 7], [0, 1, 1]),
])
def test_mask_rule(row, keep):
    w = np.array([row], F32)
    assert np.array_equal(ref.mask24(w)[0], np.array(keep, bool))


def test_mask_keeps_half_of_every_full_group_and_rows_are_independent():
    rng = np.random.default_rng(0)
    w = rng.standard_normal((5, 3, 3, 3)).astype(F32)  # conv weight: K = 27, tail of 3
    m = ref.mask24(w).reshape(5, -1)
    assert m.shape == (5, 27)
    assert (m[:, :24].reshape(5, 6, 4).sum(2) == 2).all() and (m[:, 24:].sum(1) == 2).all()
    for r in range(5):
        assert np.array_equal(ref.mask24(w[r:r + 1]).reshape(-1), m[r])


def _sparse_grid(rng, n, k, lo=-128, hi=127, zero=0):
    """A stored grid w_q [N, Kp] whose centred values (w_q - zero) are 2:4 sparse."""
    kp = (k + 15) // 16 * 16
    d = rng.integers(lo, hi + 1, (n, k)).astype(np.int64)
    d[~ref.mask24(rng.standard_normal((n, k)).astype(F32))] = 0
    d[:, rng.random(k) < 0.1] = 0  # some groups with fewer than two nonzeros
    w_q = np.zeros((n, kp), np.int64)
    w_q[:, :k] = d + zero
    return w_q.astype(np.int8), d


@pytest.mark.parametrize("n, k", [(1, 1), (3, 16), (37, 33), (130, 100), (64, 192), (257, 77)])
def test_pack_round_trips_to_the_dense_grid(n, k):
    rng = np.random.default_rng(n * 1000 + k)
    w_q, d = _sparse_grid(rng, n, k)
    zero = np.zeros(n, np.int32)
    scale = np.full(n, 0.01, F32)
    vals, meta, dsum, bad = ref.pack(w_q, zero, scale, k)
    assert vals.shape == (n, ref.k64(k) // 2) and meta.shape == ((n + 127) // 128, ref.k64(k) // 64, 2, 128)
    assert not bad.any()
    back = ref.unpack(vals, meta, n, k)
    assert np.array_equal(back[:, :k], d) and not back[:, k:].any()
    assert np.array_equal(dsum, d.sum(1))
    # every group's indices are a valid increasing pair, padding features hold the padding word
    words = meta.astype(np.uint64)
    for q in range(8):
        nib = (words >> np.uint64(4 * q)) & np.uint64(15)
        assert ((nib & np.uint64(3)) < (nib >> np.uint64(2))).all()
    t = np.arange(128)
    f = 16 * (t >> 5) + ((t & 31) >> 2) + 8 * (t & 1)
    for b in range(meta.shape[0]):
        for h in range(2):
            pad = 128 * b + 64 * h + f >= n
            assert (meta[b, :, h, pad] == ref.PAD_WORD).all()


def test_pack_zero_points_nan_rows_and_bad_groups():
    rng = np.random.default_rng(5)
    n, k = 6, 40
    w_q, d = _sparse_grid(rng, n, k, lo=-100, hi=100, zero=20)
    zero = np.full(n, 20, np.int32)
    scale = np.full(n, 0.5, F32)
    scale[2] = np.nan
    w_q[4, 8:12] = [21, 22, 23, 20]     # three nonzeros in group 2 of row 4
    w_q[5, :4] = [-128, 20, 20, 20]     # d = -148 leaves s8
    vals, meta, dsum, bad = ref.pack(w_q, zero, scale, k)
    assert list(bad) == [0, 0, 0, 0, 1, 1]
    assert dsum[2] == 0 and not vals[2].any()
    back = ref.unpack(vals, meta, n, k)
    assert np.array_equal(back[[0, 1, 3], :k], d[[0, 1, 3]])
    # groups with fewer than two nonzeros keep their lowest zeros: an all-zero group is (0, 1)
    i0, i1, _ = ref.kept(np.array([[0, 0, 0, 0, 0, 0, 5, 0]]))
    assert i0.tolist() == [[0, 0]] and i1.tolist() == [[1, 2]]


def test_ineligibility_rules_without_a_device():
    assert "expected a QLinear" in int8_sparse24_ineligibility(nn.Linear(4, 4))
    q = QLinear(nn.Linear(8, 4))
    assert int8_sparse24_ineligibility(q) == "the input quantizer is missing"


def test_argument_errors_come_before_any_cuda_call():
    lib = _lib.load()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    p16 = (p + 15) // 16 * 16
    err = lambda: lib.sb200_last_error().decode()
    assert lib.sb200_sparse24_mask(None, p, 4, 4, None) == -1 and "null" in err()
    assert lib.sb200_sparse24_mask(p, p, 0, 4, None) == -1 and "empty" in err()
    assert lib.sb200_int8_sparse24_pack(p, p, p, p16, p, p, p, 0, 16, None) == -1 and "empty" in err()
    assert lib.sb200_int8_sparse24_pack(p, p, p, p16 + 1, p, p, p, 4, 16, None) == -1 and "aligned" in err()
    assert lib.sb200_int8_sparse24_pack(p, p, p, p16, p, p, p, 4, 1 << 17, None) != 0 and "2^17" in err()
    lin = lambda qmin=-128, qmax=127, vals=p16, meta=p16, m=4, k=16, n=4, ws=1 << 20: lib.sb200_int8_sparse24_linear(
        p, p, p, qmin, qmax, vals, meta, p, p, None, p, m, k, n, p, ws, None)
    assert lin(m=0) == -1 and "empty" in err()
    assert lin(n=1 << 31) == -1 and "too large" in err()
    assert lin(qmin=0, qmax=256) == -1 and "8 bits" in err()
    assert lin(qmin=-100, qmax=200) != 0
    assert lin(vals=p16 + 8) == -1 and "aligned" in err()
    assert lin(meta=p16 + 4) == -1 and "aligned" in err()
    st = lin(k=1 << 17)
    assert st != 0 and st != -1 and "2^17" in err()
    st = lin(ws=16)
    assert st != 0 and "workspace" in err()
    assert lib.sb200_int8_sparse24_linear(p, p, p, -128, 127, p16, p16, p, p, None, None, 4, 16, 4, p, 1 << 20, None) == -1
