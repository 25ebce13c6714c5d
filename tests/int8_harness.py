"""What the integer-grid accuracy suites (tests/test_gpu_int8_*.py) and host suites (tests/test_int8_*_host.py) share:
quantizer configs, calibration, weight rows on the stored grid, model wrapping, the per-layer check of a converted
model, the operands of the attention suites and the C-ABI rejection helpers.  Importing it launches nothing; only
calling the device helpers does."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_attention_mask_ref as mref
import int8_attention_ref as aref
from gpu_util import dev, t
from int8_linear_ref import BOUND, grid_offset
from sparsebit_b200 import _lib, ops
from sparsebit_b200 import config as sbcfg
from sparsebit_b200.quantization.modules import QConv2d, QLinear, resolve_conv_padding
from sparsebit_b200.quantization.tools import CalibrationRunner, trace_quant_model

F32 = np.float32


# ---------------------------------------------------------------------------------------------- configs and models
def cfg(scheme, target, bit=8, layout="NCHW", **kw):
    return sbcfg.quantizer_config(scheme, bit, target, layout=layout, **kw)


def qrange(bits, affine):
    return (0, (1 << bits) - 1) if affine else (-(1 << (bits - 1)), (1 << (bits - 1)) - 1)


def calibrated(model, batches, *, streaming, record_inputs, replay=False):
    """``model`` on the device, calibrated by CalibrationRunner over ``batches`` (each a tensor or a tuple of forward
    arguments), with every quantizer enabled.  ``replay``: the runner drives the fx trace of ``model``, which shares
    its operators, so the calibration reaches ``model``."""
    model = model.to(dev())
    driven = trace_quant_model(model) if replay else model
    runner = CalibrationRunner(driven, streaming=streaming, record_inputs=record_inputs)
    runner.prepare_calibration()
    with torch.no_grad():
        for b in batches:
            driven(*b) if isinstance(b, tuple) else driven(b)
    runner.layerwise_calibration(dev())
    for m in model.modules():
        if hasattr(m, "set_quant") and callable(m.set_quant) and getattr(m, "input_quantizer", None) is not None:
            m.set_quant(w_quant=True, a_quant=True)
    return model


def wrap_quantized(net, act_cfg, weight_cfg):
    """``net`` with every nn.Conv2d and nn.Linear, at any depth, replaced by a QConv2d / QLinear of these configs."""
    for name, child in list(net.named_children()):
        if isinstance(child, nn.Conv2d):
            setattr(net, name, QConv2d(child).build_quantizer(act_cfg, weight_cfg))
        elif isinstance(child, nn.Linear):
            setattr(net, name, QLinear(child).build_quantizer(act_cfg, weight_cfg))
        else:
            wrap_quantized(child, act_cfg, weight_cfg)
    return net


# ---------------------------------------------------------------------------------------------- weights and layers
def stored_rows(w, ws, wz, qmin, qmax):
    """The rows of w.reshape(n, -1) on the stored grid, as int8_quantize_rows stores them with the per-row (or one)
    qparams ws, wz: (w_q, w_rowsum, w_scale, w_zero), the scale NaN on a row that holds a NaN."""
    n = w.shape[0]
    ws = np.broadcast_to(np.asarray(ws, F32).reshape(-1), (n,)).copy()
    wz = np.broadcast_to(np.asarray(wz, F32).reshape(-1), (n,)).copy()
    w_q, w_sum, w_nan = ops.int8_quantize_rows(t(w.reshape(n, -1)), t(ws), t(wz), qmin, qmax)
    w_scale = torch.where(w_nan, torch.full_like(t(ws), float("nan")), t(ws))
    w_zero = t((np.rint(wz) - grid_offset(qmin)).astype(np.int32))
    return w_q, w_sum, w_scale, w_zero


def layer_qparams(qmod, x):
    """The keyword arguments of the fp64 truth (int8_linear_ref / int8_conv_ref / int8_group_conv_ref) of a calibrated
    QLinear or QConv2d on its input ``x``: the operands with the qparams its quantizers give them, the bias and, for a
    conv, stride, dilation and the padding resolved to four sides."""
    aq, wq = qmod.input_quantizer, qmod.weight_quantizer
    xs, xz = (v.detach().reshape(-1).cpu().numpy() for v in aq._qparams_preprocess(x))
    ws, wz = (v.detach().reshape(-1).cpu().numpy() for v in wq._qparams_preprocess(qmod.weight))
    (xqmin, xqmax), (wqmin, wqmax) = aq.qdesc.qrange, wq.qdesc.qrange
    kw = dict(x=x.cpu().numpy(), xs=xs[0], xz=xz[0], xqmin=xqmin, xqmax=xqmax, w=qmod.weight.detach().cpu().numpy(),
              ws=ws, wz=wz, wqmin=wqmin, wqmax=wqmax,
              bias=qmod.bias.detach().cpu().numpy() if qmod.bias is not None else None)
    if isinstance(qmod, QConv2d):
        f = qmod.fwd_kwargs
        kw.update(stride=f["stride"], dilation=f["dilation"],
                  padding=resolve_conv_padding(f["padding"], qmod.weight.shape[2:], f["dilation"], f["stride"]))
    return kw


def _as_truth(y, t_):
    """A layer output in the truth's shape: the linear truth is [M, N], the output's leading dimensions flattened."""
    return y if y.shape == t_.shape else y.reshape(-1, y.shape[-1])


def check_converted(model, originals, inputs, names, *, expected_cls, layer_truth, compare_fake_quant):
    """Run the converted ``model`` on each of ``inputs``; every layer in ``names`` meets |y - T| <= bound elementwise on
    the input it saw, (T, bound) = ``layer_truth(originals[name], input)``.  ``expected_cls``: the class each converted
    layer has (None: not checked).  ``compare_fake_quant``: the fake-quant original, QDQ + an fp32 layer, is within its
    own fp32 accumulation error of T, 2^-22 K bound / BOUND."""
    seen = {}
    hooks = [model.get_submodule(nm).register_forward_hook(lambda mod, i, o, nm=nm: seen.__setitem__(nm, (i[0], o)))
             for nm in names]
    with torch.no_grad():
        for x in inputs:
            model(x)
            for nm in names:
                xin, y = seen[nm]
                if expected_cls is not None:
                    assert isinstance(model.get_submodule(nm), expected_cls)
                t_, bound = layer_truth(originals[nm], xin)
                err = np.abs(_as_truth(y.cpu().numpy(), t_) - t_)
                assert np.all(err <= bound), (nm, float((err / bound).max()))
                if compare_fake_quant:
                    ref_err = np.abs(_as_truth(originals[nm](xin).cpu().numpy(), t_) - t_)
                    k = originals[nm].weight[0].numel()
                    assert np.all(ref_err <= 2.0 ** -22 * k * bound / BOUND), nm
                    print(f"{nm}: int8 max |y - T| = {err.max():.3e}, fake-quant max |y - T| = {ref_err.max():.3e}")
    for h in hooks:
        h.remove()


# ---------------------------------------------------------------------------------------------- attention operands
def scalar(v):
    return t(np.array([v], F32))


def attention_operand(rng, shape, pow2, spread=1.0, qrange=(-128, 127)):
    """(x, s, z, qmin, qmax): standard normal x times ``spread``; a power-of-two scale or one from max |x|, and an
    unsigned range's zero point drawn from its first 20 steps."""
    x = (rng.standard_normal(shape) * spread).astype(F32)
    qmin, qmax = qrange
    s = F32(2.0 ** np.round(np.log2(spread * 4 / (qmax - qmin)))) if pow2 else F32(np.abs(x).max() / (0.49 * (qmax - qmin)))
    z = F32(0 if qmin < 0 else rng.integers(qmin, qmin + 20))
    return x, s, z, qmin, qmax


def p_qparams(unsigned, pow2):
    if unsigned:
        return (F32(2.0 ** -8) if pow2 else F32(1.0 / 255 * 1.37), F32(0), 0, 255)
    return (F32(2.0 ** -7) if pow2 else F32(1.0 / 127 * 0.93), F32(0), -128, 127)


def operands_of(qattn, q, k, v):
    """The reference operand tuples of q, k, v and p's qparams under a calibrated QAttention's quantizers."""
    out = []
    for carrier, x in ((qattn.qk.left, q), (qattn.qk.right, k), (qattn.pv.right, v)):
        qz = carrier.input_quantizer
        s, z = (w.detach().reshape(-1).cpu().numpy() for w in qz._qparams_preprocess(x))
        out.append((x.float().cpu().numpy(), F32(s[0]), F32(z[0]), *qz.qdesc.qrange))
    pq = qattn.pv.left.input_quantizer
    s, z = (w.detach().reshape(-1).cpu().numpy() for w in pq._qparams_preprocess(None))
    return out, (F32(s[0]), F32(z[0]), *pq.qdesc.qrange)


def check_p(g, s, bad, p, tq, tk, causal, label):
    """g [..., Tq, >= Tk] the kernel's stored p grid: admissible on the rows without NaN, the grid of 0 where the
    composition's p is exactly 0 (a -inf score, which covers the skipped keys), 0 (the grid of NaN) on rows without a
    visible key, the padding 0."""
    assert not g[..., tk:].any(), label
    gg = g[..., :tk].astype(np.int64)
    lo, hi = aref.admissible_range(mref.softmax64(s), p)
    assert np.all(((gg >= lo) & (gg <= hi))[~bad]), label
    zero = (s == -np.inf) & ~bad[..., None]
    assert np.all(gg[zero] == mref.p_zero_grid(p)), label
    with np.errstate(invalid="ignore"):
        empty = np.where(np.isnan(s), F32(0), s).max(-1) == -np.inf
    assert not gg[empty].any(), label
    sk = np.broadcast_to(mref.skipped(tq, tk, causal), gg.shape)
    assert np.all(gg[sk & ~empty[..., None]] == mref.p_zero_grid(p)), label


# ---------------------------------------------------------------------------------------------- the C-ABI on the host
E_INVALID, E_UNSUPPORTED, E_WORKSPACE = -1, -3, -4


def buf(nbytes=4096):
    """(the buffer, its first 16-byte aligned address): ``nbytes`` of host memory to pass where a pointer must be valid."""
    b = ctypes.create_string_buffer(nbytes + 16)
    return b, (ctypes.addressof(b) + 15) // 16 * 16


def rejector(call, ok, *, prefix=b""):
    """``rejected(code, text, aN=v, ...)``: ``call`` on the arguments ``ok`` with argument N set to v returns ``code``,
    and the library's last error holds ``text`` and starts with ``prefix``."""
    lib = _lib.load()

    def rejected(code, text, **changes):
        args = list(ok)
        for i, v in changes.items():
            args[int(i[1:])] = v
        assert call(*args) == code, changes
        assert text in lib.sb200_last_error(), (changes, lib.sb200_last_error())
        assert lib.sb200_last_error().startswith(prefix), (changes, lib.sb200_last_error())

    return rejected


def refusal(ineligibility, build):
    """``reason(q)``: ``ineligibility(q)``, which must name a reason that ``build(q)`` raises its ValueError with."""
    def reason(q):
        r = ineligibility(q)
        assert r is not None
        with pytest.raises(ValueError) as e:
            build(q)
        assert r in str(e.value)
        return r

    return reason


def conv_geom(**kw):
    g = dict(n=2, c=4, h=8, w=8, kh=3, kw=3, stride_h=1, stride_w=1, dilation_h=1, dilation_w=1, pad_top=1, pad_bottom=1,
             pad_left=1, pad_right=1)
    g.update(kw)
    return _lib.Conv2dGeom(**g)


BAD_GEOMS = [dict(n=0), dict(c=-1), dict(h=0), dict(w=0), dict(kh=0), dict(kw=-3), dict(stride_h=0), dict(stride_w=-1),
             dict(dilation_h=0), dict(dilation_w=0), dict(pad_top=-1), dict(pad_right=-2), dict(h=1 << 31)]


def check_geometry_rules(rejected, at):
    """The geometry checks of the dense conv entry points, the geometry passed as argument ``at``."""
    for bad in BAD_GEOMS:
        rejected(E_INVALID, b"non-positive geometry", **{f"a{at}": ctypes.byref(conv_geom(**bad))})
    rejected(E_INVALID, b"empty output", **{f"a{at}": ctypes.byref(conv_geom(kh=11))})
    rejected(E_INVALID, b"empty output", **{f"a{at}": ctypes.byref(conv_geom(kw=5, dilation_w=3))})
    rejected(E_INVALID, b"too many output pixels", **{f"a{at}": ctypes.byref(conv_geom(n=1 << 20, h=64, w=64, c=1))})
    rejected(E_UNSUPPORTED, b"K < 2^17", **{f"a{at}": ctypes.byref(conv_geom(c=1 << 17, kh=1, kw=1, pad_top=0, pad_bottom=0,
                                                                              pad_left=0, pad_right=0))})
    rejected(E_UNSUPPORTED, b"K < 2^17", **{f"a{at}": ctypes.byref(conv_geom(c=(1 << 17) // 9 + 1))})
