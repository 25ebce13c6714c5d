"""The channels-last (NHWC) integer-grid convs against their NCHW counterparts: the lowered matrix, row sums and NaN
flags byte for byte, and the dense, 2:4-sparse and grouped / depthwise conv outputs bit for bit (NaNs included), each
NHWC result written into a sentinel-filled buffer through the C-ABI; determinism and CUDA graph replay; and the conv
modules, which route a channels-last input to these kernels and give the same values as on the NCHW input."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_sparse24_ref as ref
from gpu_util import bits_equal, dev, on_device, t
from int8_harness import calibrated, cfg, stored_rows, wrap_quantized
from sparsebit_b200 import _lib, ops
from sparsebit_b200.quantization.modules import QConv2d, QConv2dInt8
from sparsebit_b200.quantization.tools import to_integer_convs, to_integer_group_convs

pytestmark = pytest.mark.gpu

F32 = np.float32
SIGNED, UNSIGNED = (-128, 127), (0, 255)
SENTINEL = 1234.5

# (n, c, h, w, kernel, stride, padding, dilation): ResNet-18 / 50 convs at small spatial sizes, the stem, odd C,
# dilation, asymmetric and 'same' padding, strided and unit-stride 1 x 1
LOWER_GEOMS = [
    (2, 3, 40, 40, 7, 2, 3, 1),                # stem, C = 3
    (2, 64, 14, 14, 3, 1, 1, 1),               # ResNet 3x3 p1
    (2, 128, 15, 15, 3, 2, 1, 1),              # 3x3 s2
    (2, 256, 7, 7, 1, 1, 0, 1),                # 1x1 s1 (row quantizer)
    (2, 256, 14, 14, 1, 2, 0, 1),              # 1x1 s2 downsample
    (2, 512, 4, 4, 3, 1, 1, 1),                # deep 3x3, K = 4608
    (3, 5, 9, 11, 3, 1, 1, 1),                 # odd C
    (2, 6, 10, 10, 3, 1, 2, 2),                # C % 4 != 0, dilation 2
    (1, 12, 11, 10, 3, 2, (1, 0, 2, 1), 1),    # asymmetric padding
    (2, 8, 9, 9, 4, 1, (1, 2, 1, 2), 1),       # 'same' padding of an even kernel
    (1, 16, 6, 6, (1, 3), 1, (0, 0, 1, 1), 1),  # 1 x 3
    (1, 20, 5, 5, 1, 1, (1, 0, 0, 1), 1),      # padded 1x1 takes the lowering
]


def _cl(x):
    """x [N, C, H, W] numpy -> a channels-last device tensor (values as given)."""
    return t(x).to(memory_format=torch.channels_last)


def _cl_misaligned(x):
    """A channels-last device tensor whose storage starts 4 bytes past a 16-byte boundary."""
    v = on_device(np.ascontiguousarray(x.transpose(0, 2, 3, 1)), 1)
    return v.permute(0, 3, 1, 2)


def _geom(shape, kernel, stride, padding, dilation):
    return ops.conv2d_geometry(shape, kernel, stride, padding, dilation)


def _x(rng, shape, xr, nan=0):
    span = (xr[1] - xr[0]) * 2.0 ** -4
    x = rng.uniform(-0.7 * span, 0.7 * span, shape).astype(F32) + (F32(0.4 * span) if xr[0] >= 0 else F32(0))
    for _ in range(nan):
        x[tuple(rng.integers(0, d) for d in shape)] = np.nan
    if nan:
        x[0, shape[1] // 2, 0, 0] = np.nan  # inside the first window of every geometry here
    return x


def _lower_nhwc(xc, kernel, s, z, xr, stride, padding, dilation):
    g = _geom(xc.shape, kernel, stride, padding, dilation)
    oh, ow = ops.conv2d_output_hw(g)
    m, kp = g.n * oh * ow, ops.int8_padded_k(g.c * g.kh * g.kw)
    q = torch.full((m, kp), 77, dtype=torch.int8, device=dev())
    rs = torch.full((m,), -5, dtype=torch.int32, device=dev())
    nan = torch.full((m,), 9, dtype=torch.uint8, device=dev())
    lib = _lib.load()
    rc = lib.sb200_int8_im2col_quantize_nhwc(xc.data_ptr(), ctypes.byref(g), s.data_ptr(), z.data_ptr(), *xr,
                                             q.data_ptr(), rs.data_ptr(), nan.data_ptr(), None)
    assert rc == 0, lib.sb200_last_error()
    return q, rs, nan


@pytest.mark.parametrize("geom", LOWER_GEOMS)
@pytest.mark.parametrize("xr", [SIGNED, UNSIGNED])
@pytest.mark.parametrize("misaligned", [False, True])
def test_lowered_matrix_equals_the_nchw_lowering(geom, xr, misaligned):
    n, c, h, w, kernel, stride, padding, dilation = geom
    rng = np.random.default_rng(abs(hash((geom, xr))) % 2**32)
    x = _x(rng, (n, c, h, w), xr, nan=2)
    s, z = t(np.array([2.0 ** -4], F32)), t(np.array([0.0 if xr[0] < 0 else 131.0], F32))
    q0, rs0, nan0 = ops.int8_im2col_quantize(t(x), kernel, s, z, *xr, stride, padding, dilation)
    xc = _cl_misaligned(x) if misaligned else _cl(x)
    assert xc.is_contiguous(memory_format=torch.channels_last)
    q1, rs1, nan1 = _lower_nhwc(xc, kernel, s, z, xr, stride, padding, dilation)
    torch.cuda.synchronize()
    assert torch.equal(q0, q1) and torch.equal(rs0, rs1) and torch.equal(nan0.to(torch.uint8), nan1)
    assert nan1.any()
    if not misaligned:
        q2, rs2, nan2 = ops.int8_im2col_quantize_nhwc(xc, kernel, s, z, *xr, stride, padding, dilation)
        assert torch.equal(q0, q2) and torch.equal(rs0, rs2) and torch.equal(nan0, nan2)


# (n, c, h, kernel, padding): M Kp >= 2^31 bytes of lowered workspace through the NHWC lowering (C = 1, 7x7, Kp = 64,
# M = 700 * 224^2) and through the row quantizer of a stride-1 unpadded 1x1 (C = 256, M = 133 * 252^2)
FAR_END = [(700, 1, 224, 7, 3), (133, 256, 252, 1, 0)]


@pytest.mark.parametrize("n,c,h,kernel,padding", FAR_END)
def test_lowering_far_end_of_a_workspace_past_2_31(n, c, h, kernel, padding):
    """The rows of the first and the last image equal the NCHW lowering of those images alone."""
    g = torch.Generator(device=dev()).manual_seed(11 + c)
    xc = (torch.randn(n, h, h, c, generator=g, device=dev()) * 3).permute(0, 3, 1, 2)
    xc[-1, c // 2, h - 3, 7] = float("nan")
    assert xc.is_contiguous(memory_format=torch.channels_last)
    s, z = t(np.array([0.05], F32)), t(np.array([131.0], F32))
    q, row_sum, nan = ops.int8_im2col_quantize_nhwc(xc, kernel, s, z, 0, 255, 1, padding, 1)
    p = h * h
    assert q.shape == (n * p, ops.int8_padded_k(c * kernel * kernel)) and q.numel() >= 2**31
    for img, sl in ((0, slice(0, p)), (n - 1, slice((n - 1) * p, n * p))):
        eq, esum, enan = ops.int8_im2col_quantize(xc[img:img + 1].contiguous(), kernel, s, z, 0, 255, 1, padding, 1)
        assert torch.equal(q[sl], eq) and torch.equal(row_sum[sl], esum) and torch.equal(nan[sl], enan)
    assert nan[-p:].any()
    del q, row_sum, nan, xc
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- dense and 2:4 conv
def _nhwc_into_sentinel(fn, xc, g, args, c_out, oh, ow, workspace=True):
    out = torch.full((g.n, c_out, oh, ow), SENTINEL, device=dev()).to(memory_format=torch.channels_last)
    lib = _lib.load()
    if workspace:
        nb = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
        ws = torch.empty(nb, dtype=torch.uint8, device=dev())
        rc = getattr(lib, fn)(xc.data_ptr(), ctypes.byref(g), *args, out.data_ptr(), c_out, ws.data_ptr(), nb, None)
    else:
        rc = getattr(lib, fn)(xc.data_ptr(), ctypes.byref(g), *args, out.data_ptr(), c_out, None)
    assert rc == 0, lib.sb200_last_error()
    torch.cuda.synchronize()
    return out


CONV_GEOMS = [
    # (n, c, h, w, c_out, kernel, stride, padding, dilation, x range)
    (2, 3, 40, 40, 64, 7, 2, 3, 1, SIGNED),
    (2, 64, 14, 14, 64, 3, 1, 1, 1, UNSIGNED),
    (2, 128, 15, 15, 128, 3, 2, 1, 1, SIGNED),
    (2, 256, 7, 7, 1024, 1, 1, 0, 1, UNSIGNED),
    (2, 256, 14, 14, 512, 1, 2, 0, 1, SIGNED),
    (2, 512, 4, 4, 512, 3, 1, 1, 1, SIGNED),
    (3, 5, 9, 11, 12, 3, 1, 1, 1, UNSIGNED),
    (2, 6, 10, 10, 20, 3, 1, 2, 2, SIGNED),
    (1, 12, 11, 10, 1, 3, 2, (1, 0, 2, 1), 1, SIGNED),
    (2, 8, 9, 9, 24, 4, 1, (1, 2, 1, 2), 1, UNSIGNED),
]


@pytest.mark.parametrize("geom", CONV_GEOMS)
def test_dense_and_sparse_conv_equal_the_nchw_entry_points(geom):
    n, c, h, w, c_out, kernel, stride, padding, dilation, xr = geom
    rng = np.random.default_rng(abs(hash(geom)) % 2**32)
    kh, kw = (kernel, kernel) if isinstance(kernel, int) else kernel
    wr = SIGNED
    x = _x(rng, (n, c, h, w), xr, nan=2)
    ws = (rng.uniform(0.5, 2.0, c_out) * 2.0 ** -6).astype(F32)
    wt = (rng.uniform(-0.45, 0.45, (c_out, c, kh, kw)) * 255 * ws[:, None, None, None]).astype(F32)
    wt = np.where(ref.mask24(rng.standard_normal(wt.shape).astype(F32)), wt, F32(0))
    wt[c_out // 2, 0, 0, 0] = np.nan  # a NaN weight row
    bias = rng.standard_normal(c_out).astype(F32)
    s, z = t(np.array([2.0 ** -4], F32)), t(np.array([0.0 if xr[0] < 0 else 131.0], F32))
    w_q, w_sum, w_scale, w_zero = stored_rows(wt, ws, np.zeros_like(ws), *wr)
    bt = t(bias)
    y0 = ops.int8_conv2d(t(x), s, z, *xr, w_q, w_sum, w_scale, w_zero, (kh, kw), bt, stride, padding, dilation)
    g = _geom(x.shape, (kh, kw), stride, padding, dilation)
    oh, ow = ops.conv2d_output_hw(g)
    xc = _cl(x)
    for xv in (xc, _cl_misaligned(x)):  # 16-byte and scalar loads of the lowering
        y1 = _nhwc_into_sentinel("sb200_int8_conv2d_nhwc", xv, g, [s.data_ptr(), z.data_ptr(), *xr, w_q.data_ptr(),
                                 w_sum.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(), bt.data_ptr()], c_out, oh, ow)
        assert bits_equal(y1.cpu().numpy(), y0.cpu().numpy())
    assert np.isnan(y0.cpu().numpy()).any()
    y2 = ops.int8_conv2d_nhwc(xc, s, z, *xr, w_q, w_sum, w_scale, w_zero, (kh, kw), bt, stride, padding, dilation)
    assert y2.is_contiguous(memory_format=torch.channels_last) and bits_equal(y2.cpu().numpy(), y0.cpu().numpy())

    # the 2:4 operand of the same stored weight (the NaN row is marked through w_scale, its vals are finite)
    vals, meta, dsum, bad = ops.int8_sparse24_pack(w_q, w_zero, w_scale, c * kh * kw)
    assert not bad.any()
    ys0 = ops.int8_sparse24_conv2d(t(x), s, z, *xr, vals, meta, dsum, w_scale, (kh, kw), bt, stride, padding, dilation)
    for xv in (xc, _cl_misaligned(x)):
        ys1 = _nhwc_into_sentinel("sb200_int8_sparse24_conv2d_nhwc", xv, g, [s.data_ptr(), z.data_ptr(), *xr,
                                  vals.data_ptr(), meta.data_ptr(), dsum.data_ptr(), w_scale.data_ptr(),
                                  bt.data_ptr()], c_out, oh, ow)
        assert bits_equal(ys1.cpu().numpy(), ys0.cpu().numpy())
    ys2 = ops.int8_sparse24_conv2d_nhwc(xc, s, z, *xr, vals, meta, dsum, w_scale, (kh, kw), bt, stride, padding,
                                        dilation)
    assert ys2.is_contiguous(memory_format=torch.channels_last) and bits_equal(ys2.cpu().numpy(), ys0.cpu().numpy())


# ---------------------------------------------------------------------------------------------- grouped / depthwise
GROUP_GEOMS = [
    # (n, c, h, w, c_out, groups, kernel, stride, padding, dilation, x range)
    (2, 32, 28, 28, 32, 32, 3, 1, 1, 1, SIGNED),        # MobileNetV2 depthwise
    (2, 144, 14, 14, 144, 144, 3, 2, 1, 1, UNSIGNED),   # MobileNetV2 depthwise s2
    (2, 240, 7, 7, 240, 240, 5, 1, 2, 1, SIGNED),       # EfficientNet-B0 5x5 depthwise
    (2, 18, 9, 9, 18, 18, 3, 1, 1, 1, SIGNED),          # C % 4 != 0 depthwise
    (2, 6, 10, 12, 18, 6, 3, 1, 1, 1, UNSIGNED),        # channel multiplier 3
    (2, 8, 9, 9, 32, 8, 3, 1, 1, 1, SIGNED),            # channel multiplier 4
    (2, 16, 9, 9, 16, 8, 3, 1, 1, 1, SIGNED),           # C_g = 2
    (2, 12, 9, 9, 12, 4, 3, 2, 1, 1, UNSIGNED),         # C_g = 3
    (2, 16, 9, 9, 16, 4, 3, 1, 1, 1, SIGNED),           # C_g = 4
    (2, 64, 14, 14, 64, 8, 3, 1, 1, 1, UNSIGNED),       # C_g = 8
    (2, 128, 14, 14, 128, 8, 3, 2, 1, 1, SIGNED),       # C_g = 16 (RegNetX-400MF)
    (2, 256, 8, 8, 256, 8, 3, 1, 1, 1, SIGNED),         # C_g = 32 (ResNeXt-50 32x4d, stage 2: 256 / 8)
    (2, 128, 14, 14, 128, 32, 3, 1, 1, 1, UNSIGNED),    # ResNeXt-50 32x4d stage 1, C_g = 4
    (1, 12, 9, 9, 6, 3, 3, 1, (0, 1, 2, 0), 2, SIGNED),  # M_g = 2, asymmetric padding, dilation
]


@pytest.mark.parametrize("geom", GROUP_GEOMS)
def test_group_conv_equals_the_nchw_entry_point(geom):
    n, c, h, w, c_out, groups, kernel, stride, padding, dilation, xr = geom
    rng = np.random.default_rng(abs(hash(geom)) % 2**32)
    wr = SIGNED
    x = _x(rng, (n, c, h, w), xr, nan=2)
    ws = (rng.uniform(0.5, 2.0, c_out) * 2.0 ** -6).astype(F32)
    wt = (rng.uniform(-0.45, 0.45, (c_out, c // groups, kernel, kernel)) * 255 * ws[:, None, None, None]).astype(F32)
    s, z = t(np.array([2.0 ** -4], F32)), t(np.array([0.0 if xr[0] < 0 else 131.0], F32))
    w_q, w_sum, w_scale, w_zero = stored_rows(wt, ws, np.zeros_like(ws), *wr)
    for bt in (t(rng.standard_normal(c_out).astype(F32)), None):
        y0 = ops.int8_group_conv2d(t(x), s, z, *xr, w_q, w_sum, w_scale, w_zero, kernel, groups, bt, stride, padding,
                                   dilation)
        g = _geom(x.shape, kernel, stride, padding, dilation)
        oh, ow = ops.conv2d_output_hw(g)
        for xc in (_cl(x), _cl_misaligned(x)):
            y1 = _nhwc_into_sentinel("sb200_int8_group_conv2d_nhwc", xc, g, [groups, s.data_ptr(), z.data_ptr(), *xr,
                                     w_q.data_ptr(), w_sum.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(),
                                     bt.data_ptr() if bt is not None else None], c_out, oh, ow, workspace=False)
            assert bits_equal(y1.cpu().numpy(), y0.cpu().numpy())
        assert np.isnan(y0.cpu().numpy()).any()
        y2 = ops.int8_group_conv2d_nhwc(_cl(x), s, z, *xr, w_q, w_sum, w_scale, w_zero, kernel, groups, bt, stride,
                                        padding, dilation)
        assert y2.is_contiguous(memory_format=torch.channels_last) and bits_equal(y2.cpu().numpy(), y0.cpu().numpy())


# ---------------------------------------------------------------------------------------------- determinism, graphs
def test_deterministic_and_graph_replay():
    rng = np.random.default_rng(7)
    x = _cl(_x(rng, (2, 64, 14, 14), SIGNED))
    s, z = t(np.array([2.0 ** -4], F32)), t(np.array([0.0], F32))
    ws = np.full(64, 2.0 ** -6, F32)
    wd = (rng.uniform(-0.45, 0.45, (64, 64, 3, 3)) * 255 * 2.0 ** -6).astype(F32)
    wd = np.where(ref.mask24(rng.standard_normal(wd.shape).astype(F32)), wd, F32(0))
    wg = (rng.uniform(-0.45, 0.45, (64, 1, 3, 3)) * 255 * 2.0 ** -6).astype(F32)
    dq, dsm, dsc, dz = stored_rows(wd, ws, np.zeros_like(ws), *SIGNED)
    vals, meta, dsum, _ = ops.int8_sparse24_pack(dq, dz, dsc, 64 * 9)
    gq, gsm, gsc, gz = stored_rows(wg, ws, np.zeros_like(ws), *SIGNED)
    calls = [
        lambda: ops.int8_im2col_quantize_nhwc(x, 3, s, z, -128, 127, 1, 1)[0],
        lambda: ops.int8_conv2d_nhwc(x, s, z, -128, 127, dq, dsm, dsc, dz, 3, None, 1, 1),
        lambda: ops.int8_sparse24_conv2d_nhwc(x, s, z, -128, 127, vals, meta, dsum, dsc, 3, None, 1, 1),
        lambda: ops.int8_group_conv2d_nhwc(x, s, z, -128, 127, gq, gsm, gsc, gz, 3, 64, None, 1, 1),
    ]
    for call in calls:
        first = call().clone()
        assert torch.equal(call(), first)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            call()  # warm the stream's workspace before capture
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                out = call()
        torch.cuda.current_stream().wait_stream(side)
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, first)


# ---------------------------------------------------------------------------------------------- modules and models
def _outputs(model, x, names):
    seen = {}
    hooks = [model.get_submodule(nm).register_forward_hook(lambda mod, i, o, nm=nm: seen.__setitem__(nm, o))
             for nm in names]
    with torch.no_grad():
        y = model(x)
    for h in hooks:
        h.remove()
    return y, seen


@pytest.mark.parametrize("arch", ["resnet18", "mobilenet_v2"])
def test_converted_model_channels_last_equals_nchw(arch):
    import torchvision

    torch.manual_seed(3)
    qnet = wrap_quantized(getattr(torchvision.models, arch)(weights=None).eval(), cfg("per-tensor-affine", "feature"),
                          cfg("per-channel-symmetric", "weight"))
    batches = [torch.randn(2, 3, 96, 96, device=dev()) for _ in range(2)]
    qnet = calibrated(qnet, batches, streaming=True, record_inputs=False)
    names = to_integer_convs(qnet) + to_integer_group_convs(qnet)
    assert len(names) == (20 if arch == "resnet18" else 52)
    x = batches[0]
    y0, seen0 = _outputs(qnet, x, names)
    y1, seen1 = _outputs(qnet, x.to(memory_format=torch.channels_last), names)
    for nm in names:
        assert seen1[nm].is_contiguous(memory_format=torch.channels_last), nm
        assert bits_equal(seen1[nm].cpu().numpy(), seen0[nm].cpu().numpy()), nm
    assert bits_equal(y1.cpu().numpy(), y0.cpu().numpy())


def test_module_routes_by_memory_format():
    torch.manual_seed(4)
    q = QConv2d(nn.Conv2d(16, 32, 3, padding=1)).build_quantizer(cfg("per-tensor-affine", "feature"),
                                                                 cfg("per-channel-symmetric", "weight"))
    q = calibrated(q, [torch.randn(4, 16, 12, 12, device=dev())], streaming=True, record_inputs=False)
    conv = QConv2dInt8.from_qconv2d(q)
    x = torch.randn(3, 16, 12, 12, device=dev())
    with torch.no_grad():
        y = conv(x)
        ycl = conv(x.to(memory_format=torch.channels_last))
        assert ycl.is_contiguous(memory_format=torch.channels_last) and torch.equal(ycl, y)
        y16 = conv(x.half().to(memory_format=torch.channels_last))
        assert y16.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(y16, conv(x.half().float()))
        assert conv(x[1]).is_contiguous() and torch.equal(conv(x[1]), y[1])  # unbatched: NCHW
        hwc = x[1].permute(1, 2, 0).contiguous().permute(2, 0, 1)  # unbatched, stored HWC (an image's permute)
        yu = conv(hwc)
        assert yu.is_contiguous() and torch.equal(yu, y[1])
        x1 = torch.randn(2, 16, 1, 1, device=dev())  # contiguous in both formats: today's path
        q1 = conv(x1.to(memory_format=torch.channels_last))
        assert q1.is_contiguous() and torch.equal(q1, conv(x1))


def test_nhwc_ops_refuse_nchw_and_strided_tensors():
    s = torch.ones(1, device=dev())
    w = torch.zeros(8, 80, dtype=torch.int8, device=dev())
    i32 = torch.zeros(8, dtype=torch.int32, device=dev())
    calls = [
        lambda x: ops.int8_im2col_quantize_nhwc(x, 3, s, s, -128, 127),
        lambda x: ops.int8_conv2d_nhwc(x, s, s, -128, 127, w, i32, s, i32, 3),
        lambda x: ops.int8_sparse24_conv2d_nhwc(x, s, s, -128, 127, w, i32, i32, s, 3),
        lambda x: ops.int8_group_conv2d_nhwc(x, s, s, -128, 127, w, i32, s, i32, 3, 2),
    ]
    x = torch.zeros(2, 8, 6, 6, device=dev())
    for call in calls:
        for bad in (x, x.to(memory_format=torch.channels_last)[:, :, ::2]):
            with pytest.raises(ops.SparsebitB200Error, match="channels-last"):
                call(bad)
    with pytest.raises(ops.SparsebitB200Error, match="contiguous"):  # the NCHW ops still refuse channels-last
        ops.int8_conv2d(x.to(memory_format=torch.channels_last), s, s, -128, 127, w, i32, s, i32, 3)
