"""The fake-quant op as the quantizers see it: ``STE`` autograd function and the per-backend
forward functions (reference: sparsebit/quantization/quantizers/quant_tensor.py:74-249).

Tensor math runs in libsparsebit_b200.so through ``sparsebit_b200.fake_quant`` (CUDA tensors) or
through the host-buffer C-ABI entry points (CPU tensors: the library stages them through the GPU;
there is no eager CPU implementation here).
"""
import ctypes

import numpy as np
import torch

from ... import _lib
from ... import fake_quant as fake_quant_kernel
from ..common import Backend


def _host_forward(x_f, scale, zero_point, qdesc):
    """CPU tensors: sb200_qdq_*_fwd_host (H2D -> sm_90a kernel -> D2H inside the library)."""
    lib = _lib.load()
    x = x_f.detach().float().contiguous()
    out = torch.empty_like(x)
    qmin, qmax = qdesc.qrange
    s = scale.detach().float().reshape(-1).contiguous()
    z = zero_point.detach().float().reshape(-1).contiguous()
    if x.numel() == 0:
        raise _lib.SparsebitB200Error("Kernel Failure, Tensor is empty: data")
    if qdesc.is_perchannel and s.numel() > 1:
        ch_axis = qdesc.ch_axis
        outer = int(np.prod(x.shape[:ch_axis], dtype=np.int64))
        c = x.shape[ch_axis]
        inner = int(np.prod(x.shape[ch_axis + 1 :], dtype=np.int64))
        _lib.check(lib.sb200_qdq_perchannel_fwd_host(x.data_ptr(), s.data_ptr(), z.data_ptr(), out.data_ptr(),
                                                     outer, c, inner, qmin, qmax, 0))
    else:
        _lib.check(lib.sb200_qdq_pertensor_fwd_host(x.data_ptr(), ctypes.c_float(float(s[0])), ctypes.c_float(float(z[0])),
                                                    out.data_ptr(), None, x.numel(), qmin, qmax, 0))
    return out


def ort_fake_quant(x_f, scale, zero_point, qdesc):
    """quant_tensor.py:159-185.  fp16 input is up-cast and the result stays fp32 (Q3)."""
    assert x_f.device == scale.device == zero_point.device, \
        "input, scale and zero_point of quantizer must be on same device!"
    qmin, qmax = qdesc.qrange
    if not x_f.is_cuda:
        return _host_forward(x_f, scale, zero_point, qdesc)
    if x_f.dtype != torch.float32:
        x_f = x_f.float()
    if qdesc.is_perchannel:
        return fake_quant_kernel.quant_perchannel_forward(
            x_f.contiguous(), scale.contiguous(), zero_point.float().contiguous(), qmin, qmax, qdesc.ch_axis, 0)
    return fake_quant_kernel.quant_pertensor_forward(x_f.contiguous(), scale.contiguous(),
                                                     zero_point.float().contiguous(), qmin, qmax, 0)


def trt_fake_quant(x_f, scale, zero_point, qdesc):
    """quant_tensor.py:128-156: TensorRT only supports symmetric quantisation.  The reference
    asserts ``abs(zero_point).sum() == 0`` with a device sync on every call (:132-134); here the
    check is done once per zero_point tensor version."""
    check_trt_symmetric(zero_point)
    return ort_fake_quant(x_f, scale, zero_point, qdesc)


def check_trt_symmetric(zero_point):
    key = (zero_point.data_ptr(), zero_point._version)
    if getattr(trt_fake_quant, "_ok_key", None) != key:
        assert float(zero_point.abs().sum()) == 0, "tensorrt only support symmetric quant, but zp={}".format(zero_point)
        trt_fake_quant._ok_key = key


fake_quant_factory = {
    Backend.VIRTUAL: ort_fake_quant,
    Backend.ONNXRUNTIME: ort_fake_quant,
    Backend.TENSORRT: trt_fake_quant,
}


def ort_dqrange(scale, zero_point, qdesc):
    qmin, qmax = qdesc.qrange
    return (qmin - zero_point) * scale, (qmax - zero_point) * scale


def trt_dqrange(scale, zero_point, qdesc):
    qmin, qmax = qdesc.qrange
    return scale * qmin, scale * qmax


fake_qrange_factory = {
    Backend.VIRTUAL: ort_dqrange,
    Backend.ONNXRUNTIME: ort_dqrange,
    Backend.TENSORRT: trt_dqrange,
}


class STE(torch.autograd.Function):
    """Straight-through estimator around the fake-quant op (quant_tensor.py:74-125)."""

    @staticmethod
    def forward(ctx, x, scale, zero_point, qdesc, backend):
        ctx.save_for_backward(x, scale, zero_point)
        ctx.qdesc = qdesc
        return fake_quant_factory[backend](x, scale, zero_point, qdesc)

    @staticmethod
    def backward(ctx, gout):
        x, scale, zero_point = ctx.saved_tensors
        qdesc = ctx.qdesc
        qmin, qmax = qdesc.qrange
        if not x.is_cuda:
            # same restriction as the reference (quant_tensor.py:113-116)
            raise NotImplementedError("We recommended that use cuda to speedup when training")
        if x.dtype != torch.float32:
            x = x.float()
        gout = gout.float().contiguous()
        if qdesc.is_perchannel:
            gx, gs, gzp = fake_quant_kernel.quant_perchannel_backward(
                x.contiguous(), scale.contiguous(), zero_point.float().contiguous(), gout, qmin, qmax, qdesc.ch_axis, 0)
        else:
            gx, gs, gzp = fake_quant_kernel.quant_pertensor_backward(
                x.contiguous(), scale.contiguous(), zero_point.float().contiguous(), gout, qmin, qmax, 0)
        return gx, (gs if scale.requires_grad else None), (gzp if zero_point.requires_grad else None), None, None


def torch_fake_quant(x_f, scale, zero_point, qdesc):
    """ONNX-export branch (quant_tensor.py:220-249): must stay on stock ATen fake_quantize ops so
    the exporter emits QuantizeLinear / DequantizeLinear; the custom kernels are NOT used here."""
    lower, upper = (0, 255) if qdesc._type.startswith("uint") else (-128, 127)
    if scale.numel() > 1:
        ch_axis = int(np.argmax(list(scale.shape)))
        return torch.fake_quantize_per_channel_affine(
            x_f, scale.reshape(-1).detach().to(x_f.device), zero_point.reshape(-1).int().to(x_f.device), ch_axis, lower, upper)
    if scale.numel() == 1:
        return torch.fake_quantize_per_tensor_affine(x_f, scale.item(), zero_point.int().item(), lower, upper)
    raise TypeError("scale / zeropoint is not allowed to be an empty tensor")
