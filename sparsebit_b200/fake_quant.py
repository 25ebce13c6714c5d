"""Drop-in for the reference's JIT-built pybind module ``fake_quant``
(sparsebit/quantization/torch_extensions/export.cc:3-8): same four names, argument order and
return conventions, backed by the sm_90a C-ABI library instead of the PPQ-derived kernels.

    import sparsebit_b200.fake_quant as fake_quant_kernel
    y = fake_quant_kernel.quant_pertensor_forward(x, scale, zero_point, qmin, qmax, 0)

``sparsebit_b200.install()`` rebinds ``sparsebit.quantization.quantizers.quant_tensor
.fake_quant_kernel`` to this module so an unmodified Sparsebit runs on these kernels.
"""
from . import ops


def quant_pertensor_forward(data, scale, zero_point, qmin, qmax, rounding):
    """QuantizePerTensorForward (fake_quant_tensor.cu:69-94)."""
    return ops.qdq_pertensor(data, scale, zero_point, qmin, qmax, rounding)


def quant_perchannel_forward(data, scale, zero_point, qmin, qmax, ch_axis, rounding):
    """QuantizePerChannelForward (fake_quant_tensor.cu:191-224)."""
    return ops.qdq_perchannel(data, scale, zero_point, qmin, qmax, ch_axis, rounding)


def quant_pertensor_backward(data, scale, zero_point, grad_y, qmin, qmax, rounding):
    """QuantizePerTensorBackward (fake_quant_tensor.cu:135-167): [gx, gs, gzp]; gs / gzp are only
    reduced when the corresponding tensor requires grad (:164-165), zeros otherwise."""
    gx, gs, gzp = ops.qdq_backward(data, scale, zero_point, grad_y, qmin, qmax, None, rounding,
                                   need_gs=scale.requires_grad, need_gzp=zero_point.requires_grad)
    return [gx, gs, gzp]


def quant_perchannel_backward(data, scale, zero_point, grad_y, qmin, qmax, ch_axis, rounding, gzp_closed=False):
    """QuantizePerChannelBackward (fake_quant_tensor.cu:273-314).  The zero-point gradient follows the
    reference kernel (vq == qmax counts as clipped, :264); ``gzp_closed=True`` (an extension, not part of
    the reference signature) switches to MySTE.backward's closed interval (quant_tensor.py:62-69)."""
    gx, gs, gzp = ops.qdq_backward(data, scale, zero_point, grad_y, qmin, qmax, ch_axis, rounding,
                                   need_gs=scale.requires_grad, need_gzp=zero_point.requires_grad,
                                   gzp_closed=gzp_closed)
    return [gx, gs, gzp]
