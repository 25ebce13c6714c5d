"""Every launch branch and in-kernel path of csrc/int8_sparse24.cu, as tests/int8_sparse24_geometry.py names them: one
case per branch, run through the C-ABI into sentinel-filled outputs.  The mask is compared with the numpy rule, the
packed operand with the numpy restatement, and the sparse GEMM, bit for bit, with sb200_int8_linear on the same stored
weight -- every element written, none left at the sentinel.

Cases: mask_grid (full groups, partial CTA), mask_tail (a tail group), pack_pad (padding features, a K tail, a NaN
row, zero points), gemm_one_stage, gemm_pad_steps, gemm_short_tail, gemm_ring, gemm_partial, gemm_idle_wg,
gemm_scalar_store, gemm_unsigned_nan."""
import numpy as np
import pytest
import torch

import int8_sparse24_geometry as geo
import int8_sparse24_ref as ref
from branch_cases import C, assert_table_covers, check_reach, params
from gpu_util import dev, t
from sparsebit_b200 import _lib, ops

F32 = np.float32
SENTINEL = 1234.5

CASES = [
    C("mask_grid", "mask", {"mask_full_group", "mask_grid_tail"}, rows=37, cols=64),
    C("mask_tail", "mask", {"mask_full_group", "mask_tail_group", "mask_grid_tail"}, rows=5, cols=27),
    C("pack_pad", "pack", {"pack_word", "pack_pad_feature", "pack_k_tail"}, ("(data) pack_nan_row", "(data) pack_zero_point"),
      n=70, k=100),
    C("gemm_one_stage", "gemm", {"gemm_one_stage", "gemm_store_vec4", "gemm_bias", "gemm_x_signed", "gemm_pad_steps",
                                 "gemm_no_second_box"}, m=128, k=64, n=128),
    C("gemm_pad_steps", "gemm", {"gemm_multi_stage", "gemm_pad_steps"}, m=128, k=448, n=256),
    C("gemm_short_tail", "gemm", {"gemm_multi_stage", "gemm_no_second_box", "gemm_no_bias"}, m=64, k=320, n=128, bias=False),
    C("gemm_ring", "gemm", {"gemm_ring_wraps", "gemm_multi_stage"}, m=256, k=2304, n=128),
    C("gemm_partial", "gemm", {"gemm_partial_m", "gemm_partial_n"}, m=201, k=768, n=200),
    C("gemm_idle_wg", "gemm", {"gemm_partial_n", "gemm_idle_warpgroup"}, m=130, k=256, n=164),
    C("gemm_scalar_store", "gemm", {"gemm_store_scalar", "gemm_partial_n"}, m=33, k=1001, n=131),
    C("gemm_unsigned_nan", "gemm", {"gemm_x_unsigned"}, ("(data) gemm_nan_row",), m=77, k=520, n=96, unsigned=True),
]


def covers(case):
    if case.op == "mask":
        reached = geo.mask_branches(case.get("rows"), case.get("cols"))
    elif case.op == "pack":
        reached = geo.pack_branches(case.get("n"), case.get("k"))
    else:
        reached = geo.gemm_branches(case.get("m"), case.get("k"), case.get("n"), bias=case.get("bias", True),
                                    unsigned_x=case.get("unsigned", False))
    return check_reach(case, reached)


def test_case_table_covers_every_branch():
    assert_table_covers(CASES, geo.REQUIRED, covers, __doc__, doc_branches=False)


def _stored(rng, n, k, wz=0, nan_row=None):
    ws = (2.0 ** -rng.integers(3, 8, n)).astype(F32)
    w = (rng.uniform(-0.45, 0.45, (n, k)) * 255 * ws[:, None]).astype(F32)
    w = np.where(ref.mask24(rng.standard_normal((n, k)).astype(F32)), w, F32(0))
    if nan_row is not None:
        w[nan_row, 3] = np.nan
    z = np.full(n, wz, F32)
    w_q, w_sum, w_nan = ops.int8_quantize_rows(t(w), t(ws), t(z), -128, 127)
    w_scale = torch.where(w_nan, torch.full_like(t(ws), float("nan")), t(ws))
    return w_q, w_sum, w_scale, t(np.rint(z).astype(np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("case", params(CASES))
def test_branch_case(case):
    lib = _lib.load()
    rng = np.random.default_rng(sum(map(ord, case.name)))
    stream = torch.cuda.current_stream().cuda_stream
    if case.op == "mask":
        w = rng.standard_normal((case.get("rows"), case.get("cols"))).astype(F32)
        w[0, :4] = [1.0, -1.0, np.nan, 0.0]
        mask = torch.full(w.shape, 7, dtype=torch.uint8, device=dev())
        _lib.check(lib.sb200_sparse24_mask(t(w).data_ptr(), mask.data_ptr(), w.shape[0], w.shape[1], stream))
        assert np.array_equal(mask.cpu().numpy(), ref.mask24(w).astype(np.uint8))
        return
    if case.op == "pack":
        n, k = case.get("n"), case.get("k")
        w_q, _, w_scale, w_zero = _stored(rng, n, k, wz=3, nan_row=2)
        vshape, mshape = ops.int8_sparse24_shapes(n, k)
        vals = torch.full(vshape, 99, dtype=torch.int8, device=dev())
        meta = torch.full(mshape, 0x5A5A5A5A, dtype=torch.int32, device=dev())
        dsum = torch.full((n,), 12345, dtype=torch.int32, device=dev())
        bad = torch.full((n,), 777, dtype=torch.int32, device=dev())
        _lib.check(lib.sb200_int8_sparse24_pack(w_q.data_ptr(), w_zero.data_ptr(), w_scale.data_ptr(), vals.data_ptr(),
                                                meta.data_ptr(), dsum.data_ptr(), bad.data_ptr(), n, k, stream))
        ev, em, ed, eb = ref.pack(w_q.cpu().numpy(), w_zero.cpu().numpy(), w_scale.cpu().numpy(), k)
        assert np.array_equal(vals.cpu().numpy(), ev) and np.array_equal(meta.cpu().numpy().view(np.uint32), em)
        assert np.array_equal(dsum.cpu().numpy(), ed) and np.array_equal(bad.cpu().numpy(), eb)
        assert ed[2] == 0 and not ev[2].any()  # the NaN row is packed as zeros
        return
    m, k, n = case.get("m"), case.get("k"), case.get("n")
    unsigned = case.get("unsigned", False)
    qmin, qmax = (0, 255) if unsigned else (-128, 127)
    w_q, w_sum, w_scale, w_zero = _stored(rng, n, k)
    vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero, w_scale, k)
    assert not bad.any()
    x = (rng.uniform(-6, 6, (m, k)) + (8 if unsigned else 0)).astype(F32)
    if unsigned:
        x[m // 2, k // 3] = np.nan
    xs = t(np.array([2.0 ** -4], F32))
    xz = t(np.array([131 if unsigned else 0], F32))
    bias = t(rng.standard_normal(n).astype(F32)) if case.get("bias", True) else None
    out = torch.full((m, n), SENTINEL, dtype=torch.float32, device=dev())
    ws_bytes = int(lib.sb200_int8_linear_workspace_bytes(m, k))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
    xt = t(x)
    _lib.check(lib.sb200_int8_sparse24_linear(xt.data_ptr(), xs.data_ptr(), xz.data_ptr(), qmin, qmax, vals.data_ptr(),
                                              meta.data_ptr(), dsum.data_ptr(), w_scale.data_ptr(),
                                              bias.data_ptr() if bias is not None else None, out.data_ptr(), m, k, n,
                                              ws.data_ptr(), ws_bytes, stream))
    dense = ops.int8_linear(xt, xs, xz, qmin, qmax, w_q, w_sum, w_scale, w_zero, bias)
    y = out.cpu().numpy()
    assert not (y == F32(SENTINEL)).any()
    assert np.array_equal(y.view(np.uint32), dense.cpu().numpy().view(np.uint32))
    if unsigned:
        assert np.isnan(y[m // 2]).all()
