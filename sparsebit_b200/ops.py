"""Tensor-level wrappers over the C-ABI: torch is used for device memory and streams only.

Every function takes CUDA fp32 tensors, launches on ``torch.cuda.current_stream()`` of the
tensor's device and never synchronises the host.  Non-fp32 / empty / CPU inputs raise
``RuntimeError`` like the reference's pybind modules do (torch_extensions/common.cuh:45-55).
"""
import ctypes

import torch

from . import _lib
from ._lib import SparsebitB200Error, check


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _req(t, name, dtype=torch.float32, memory_format=torch.contiguous_format):
    if not isinstance(t, torch.Tensor):
        raise SparsebitB200Error(f"{name}: expected a torch.Tensor")
    if not t.is_cuda:
        raise SparsebitB200Error(f"{name}: expected a CUDA tensor (sparsebit_b200 has no CPU fallback)")
    if t.dtype != dtype:
        raise SparsebitB200Error(f"Kernel Failure, Invalid dtype of Input tensor: {name}(Expect to be {dtype})")
    if t.numel() == 0:
        raise SparsebitB200Error(f"Kernel Failure, Tensor is empty: {name}")
    if not t.is_contiguous(memory_format=memory_format):
        if memory_format == torch.channels_last:
            raise SparsebitB200Error(f"{name}: expected a 4-D channels-last (NHWC) contiguous tensor")
        raise SparsebitB200Error(f"{name}: expected a contiguous tensor")
    return t


def channel_geometry(shape, ch_axis):
    """[outer, C, inner] view used by the per-channel kernels (fake_quant_tensor.cu:203-208)."""
    ch_axis = ch_axis % len(shape)
    outer = 1
    for d in shape[:ch_axis]:
        outer *= int(d)
    inner = 1
    for d in shape[ch_axis + 1 :]:
        inner *= int(d)
    return outer, int(shape[ch_axis]), inner


# ----------------------------------------------------------------------------- QDQ forward
def qdq_pertensor(x, scale, zero_point, qmin, qmax, rounding=0, out=None):
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale"), _req(zero_point, "zero_point")
    out = torch.empty_like(x) if out is None else out
    with torch.cuda.device(x.device):
        check(lib.sb200_qdq_pertensor_fwd(x.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), out.data_ptr(),
                                          x.numel(), int(qmin), int(qmax), int(rounding), _stream(x)))
    return out


def qdq_perchannel(x, scale, zero_point, qmin, qmax, ch_axis, rounding=0, out=None):
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale"), _req(zero_point, "zero_point")
    outer, c, inner = channel_geometry(x.shape, ch_axis)
    if scale.numel() != c or zero_point.numel() != c:
        raise SparsebitB200Error(f"per-channel qparams need {c} elements (got {scale.numel()}, {zero_point.numel()})")
    out = torch.empty_like(x) if out is None else out
    with torch.cuda.device(x.device):
        check(lib.sb200_qdq_perchannel_fwd(x.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), out.data_ptr(),
                                           outer, c, inner, int(qmin), int(qmax), int(rounding), _stream(x)))
    return out


def qdq_stats_pertensor(x, scale, zero_point, qmin, qmax, state, rounding=0, out=None):
    """Fused QDQ + running min/max of x.  ``state``: int32[2] tensor from ``minmax_new(1)``."""
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale"), _req(zero_point, "zero_point")
    out = torch.empty_like(x) if out is None else out
    with torch.cuda.device(x.device):
        check(lib.sb200_qdq_stats_pertensor_fwd(x.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), out.data_ptr(),
                                                state.data_ptr(), x.numel(), int(qmin), int(qmax), int(rounding), _stream(x)))
    return out


# ----------------------------------------------------------------------------- STE backward
def clamp_backward(x, grad_y, lo, hi):
    """Backward of ``clamp(x, lo, hi)`` with tensor bounds: (gx, g_hi, g_lo) -- sb200_clamp_bwd (PACT)."""
    lib = _lib.load()
    _req(x, "data"), _req(grad_y, "grad"), _req(lo, "lower"), _req(hi, "alpha")
    if grad_y.shape != x.shape:
        raise SparsebitB200Error("grad_y must have the shape of data")
    gx = torch.empty_like(x)
    g_hi = torch.zeros(1, dtype=torch.float32, device=x.device)
    g_lo = torch.zeros(1, dtype=torch.float32, device=x.device)
    ws_bytes = int(lib.sb200_clamp_bwd_workspace_bytes(x.numel()))
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.sb200_clamp_bwd(x.data_ptr(), grad_y.data_ptr(), lo.data_ptr(), hi.data_ptr(), gx.data_ptr(), g_hi.data_ptr(),
                                  g_lo.data_ptr(), x.numel(), ws.data_ptr(), ws_bytes, _stream(x)))
    return gx, g_hi, g_lo


BWD_GZP_CLOSED = 1  # include/sparsebit_b200.h SB200_BWD_GZP_CLOSED


def qdq_backward(x, scale, zero_point, grad_y, qmin, qmax, ch_axis=None, rounding=0, need_gs=True, need_gzp=True,
                 gzp_closed=False):
    """Returns (gx, gs, gzp); gs / gzp shaped like scale / zero_point (zeros when not requested,
    like the reference which returns zeros_like, fake_quant_tensor.cu:147-149).  Per-channel zero-point
    gradient: by default the reference kernel's rule (vq == qmax counts as clipped, fake_quant_tensor.cu:264);
    ``gzp_closed=True`` selects MySTE.backward's closed interval (quant_tensor.py:62-69)."""
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale"), _req(zero_point, "zero_point"), _req(grad_y, "grad")
    if grad_y.shape != x.shape:
        raise SparsebitB200Error("grad_y must have the shape of data")
    gx = torch.empty_like(x)
    gs = torch.zeros_like(scale)
    gzp = torch.zeros_like(zero_point)
    if ch_axis is None:
        outer, c, inner = 1, 1, x.numel()
    else:
        outer, c, inner = channel_geometry(x.shape, ch_axis)
        if scale.numel() != c or zero_point.numel() != c:
            raise SparsebitB200Error(f"per-channel qparams need {c} elements (got {scale.numel()}, {zero_point.numel()})")
    need = need_gs or need_gzp
    ws_bytes = int(lib.sb200_qdq_bwd_workspace_bytes(outer, c, inner)) if need else 0
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
    with torch.cuda.device(x.device):
        if ch_axis is None:
            check(lib.sb200_qdq_pertensor_bwd(x.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), grad_y.data_ptr(),
                                              gx.data_ptr(), gs.data_ptr() if need_gs else None,
                                              gzp.data_ptr() if need_gzp else None, x.numel(), int(qmin), int(qmax),
                                              int(rounding), ws.data_ptr(), ws_bytes, _stream(x)))
        else:
            check(lib.sb200_qdq_perchannel_bwd_ex(x.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), grad_y.data_ptr(),
                                                  gx.data_ptr(), gs.data_ptr() if need_gs else None,
                                                  gzp.data_ptr() if need_gzp else None, outer, c, inner, int(qmin),
                                                  int(qmax), int(rounding), BWD_GZP_CLOSED if gzp_closed else 0,
                                                  ws.data_ptr(), ws_bytes, _stream(x)))
    return gx, gs, gzp


# ----------------------------------------------------------------------------- multi-tensor weight QDQ
class _QdqTensorDesc(ctypes.Structure):  # include/sparsebit_b200.h sb200_qdq_tensor_desc
    _fields_ = [("x", ctypes.c_void_p), ("mask", ctypes.c_void_p), ("scale", ctypes.c_void_p), ("zero_point", ctypes.c_void_p),
                ("out", ctypes.c_void_p), ("outer", ctypes.c_int64), ("channels", ctypes.c_int64), ("inner", ctypes.c_int64),
                ("qmin", ctypes.c_int), ("qmax", ctypes.c_int)]


class QdqMulti:
    """(mask-apply +) per-channel QDQ of many tensors in ONE launch (sb200_qdq_multi_plan / _run).

    ``items``: iterable of dicts ``x, scale, zero_point, qmin, qmax`` and optional ``mask`` (bool / uint8),
    ``out`` (default: a new tensor), ``ch_axis`` (default 0).  The plan keeps references to every tensor; ``run()``
    re-reads their CURRENT contents (the weights of a training step), one kernel launch per call."""

    def __init__(self, items):
        lib = _lib.load()
        self.items = []
        descs = []
        for it in items:
            x = _req(it["x"], "data")
            scale = _req(it["scale"].reshape(-1), "scale")
            zp = _req(it["zero_point"].reshape(-1), "zero_point")
            outer, c, inner = channel_geometry(x.shape, it.get("ch_axis", 0))
            if scale.numel() != c or zp.numel() != c:
                raise SparsebitB200Error(f"per-channel qparams need {c} elements (got {scale.numel()}, {zp.numel()})")
            mask = it.get("mask")
            if mask is not None:
                if mask.dtype not in (torch.bool, torch.uint8) or mask.shape != x.shape or not mask.is_contiguous():
                    raise SparsebitB200Error("mask must be a contiguous bool / uint8 tensor shaped like the data")
            out = it.get("out")
            out = torch.empty_like(x) if out is None else _req(out, "out")
            self.items.append((x, mask, scale, zp, out))
            descs.append(_QdqTensorDesc(x.data_ptr(), mask.data_ptr() if mask is not None else None, scale.data_ptr(),
                                        zp.data_ptr(), out.data_ptr(), outer, c, inner, int(it["qmin"]), int(it["qmax"])))
        if not descs:
            raise SparsebitB200Error("QdqMulti: no tensors")
        self.device = self.items[0][0].device
        self.count = len(descs)
        arr = (_QdqTensorDesc * self.count)(*descs)
        self.table = torch.empty(int(lib.sb200_qdq_multi_table_bytes(self.count)), dtype=torch.uint8, device=self.device)
        rows = ctypes.c_int64(0)
        with torch.cuda.device(self.device):
            check(lib.sb200_qdq_multi_plan(arr, self.count, self.table.data_ptr(), self.table.numel(), ctypes.byref(rows),
                                           torch.cuda.current_stream(self.device).cuda_stream))
        self.total_rows = rows.value
        self.outputs = [it[4] for it in self.items]

    def run(self):
        with torch.cuda.device(self.device):
            check(_lib.load().sb200_qdq_multi_run(self.table.data_ptr(), self.count, self.total_rows,
                                                  torch.cuda.current_stream(self.device).cuda_stream))
        return self.outputs


# ----------------------------------------------------------------------------- row moments
MOMENTS = 5  # sum x, sum x^2, sum |x|, sum |x - c|, sum (x - c)^2


def moments_new(rows, device):
    return torch.zeros(rows, MOMENTS, dtype=torch.float64, device=device)


def moments_update(x2d, out, centre=None):
    """Accumulate the fp64 row moments of x2d [rows, row_len] into ``out`` [rows, 5] (deterministic order)."""
    lib = _lib.load()
    _req(x2d, "data")
    if x2d.dim() != 2 or out.shape != (x2d.shape[0], MOMENTS) or out.dtype != torch.float64:
        raise SparsebitB200Error("moments_update: x2d must be [rows, row_len] and out float64 [rows, 5]")
    if centre is not None and (centre.dtype != torch.float64 or centre.numel() != x2d.shape[0]):
        raise SparsebitB200Error("moments_update: centre must hold one float64 per row")
    rows, row_len = x2d.shape
    ws_bytes = int(lib.sb200_moments_workspace_bytes(rows, row_len))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x2d.device)
    with torch.cuda.device(x2d.device):
        check(lib.sb200_observe_moments(x2d.data_ptr(), rows, row_len, centre.data_ptr() if centre is not None else None,
                                        out.data_ptr(), ws.data_ptr(), ws_bytes, _stream(x2d)))
    return out


# ----------------------------------------------------------------------------- DoReFa
def dorefa_absmax(x):
    """max |tanh(x)| as a one-element float tensor (dorefa.py:16-17), one 4 B/elem pass."""
    lib = _lib.load()
    _req(x, "data")
    m = torch.zeros(1, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.sb200_dorefa_absmax(x.data_ptr(), x.numel(), m.data_ptr(), _stream(x)))
    return m


def dorefa_forward(x, absmax, scale=None, zero_point=None, qmin=0, qmax=0, ch_axis=None):
    """tanh(x) / absmax, fake-quantised when qparams are given (dorefa.py:15-20); without them the normalised tensor
    the observer sees (dorefa.py:22-26)."""
    lib = _lib.load()
    _req(x, "data"), _req(absmax, "absmax")
    quantize = scale is not None
    if quantize:
        _req(scale, "scale"), _req(zero_point, "zero_point")
        outer, c, inner = _adaround_geometry(x, scale, ch_axis)
        if zero_point.numel() != c:
            raise SparsebitB200Error(f"dorefa: qparams need {c} elements (got {zero_point.numel()})")
    else:
        outer, c, inner = 1, 1, x.numel()
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.sb200_dorefa_fwd(x.data_ptr(), absmax.data_ptr(), scale.data_ptr() if quantize else None,
                                   zero_point.data_ptr() if quantize else None, out.data_ptr(), outer, c, inner,
                                   int(qmin), int(qmax), int(quantize), _stream(x)))
    return out


def dorefa_backward(x, absmax, scale, zero_point, grad_y, qmin, qmax, ch_axis=None):
    """Gradient of dorefa_forward with respect to x (STE mask -> / absmax -> tanh'), one 12 B/elem pass."""
    lib = _lib.load()
    _req(x, "data"), _req(absmax, "absmax"), _req(scale, "scale"), _req(zero_point, "zero_point"), _req(grad_y, "grad")
    if grad_y.shape != x.shape:
        raise SparsebitB200Error("dorefa: grad_y must have the shape of data")
    outer, c, inner = _adaround_geometry(x, scale, ch_axis)
    if zero_point.numel() != c:
        raise SparsebitB200Error(f"dorefa: qparams need {c} elements (got {zero_point.numel()})")
    gx = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.sb200_dorefa_bwd(x.data_ptr(), absmax.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), grad_y.data_ptr(),
                                   gx.data_ptr(), outer, c, inner, int(qmin), int(qmax), _stream(x)))
    return gx


# ----------------------------------------------------------------------------- AdaRound
def _adaround_geometry(x, scale, ch_axis):
    if ch_axis is None:
        outer, c, inner = 1, 1, x.numel()
    else:
        outer, c, inner = channel_geometry(x.shape, ch_axis)
    if scale.numel() != c:
        raise SparsebitB200Error(f"adaround: qparams need {c} elements (got {scale.numel()})")
    return outer, c, inner


def adaround_forward(x, v, scale, zero_point, qmin, qmax, ch_axis=None, soft=False, out=None):
    """adaround.py:46-54; soft=True is the training branch, soft=False the (exact) eval branch."""
    lib = _lib.load()
    _req(x, "data"), _req(v, "v"), _req(scale, "scale"), _req(zero_point, "zero_point")
    if v.shape != x.shape:
        raise SparsebitB200Error("adaround: v must have the shape of data")
    outer, c, inner = _adaround_geometry(x, scale, ch_axis)
    out = torch.empty_like(x) if out is None else out
    with torch.cuda.device(x.device):
        check(lib.sb200_adaround_fwd(x.data_ptr(), v.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), out.data_ptr(),
                                     outer, c, inner, int(qmin), int(qmax), int(bool(soft)), _stream(x)))
    return out


def adaround_backward(x, v, scale, zero_point, grad_y, qmin, qmax, ch_axis=None):
    lib = _lib.load()
    _req(x, "data"), _req(v, "v"), _req(scale, "scale"), _req(zero_point, "zero_point"), _req(grad_y, "grad")
    if v.shape != x.shape or grad_y.shape != x.shape:
        raise SparsebitB200Error("adaround: v and grad_y must have the shape of data")
    outer, c, inner = _adaround_geometry(x, scale, ch_axis)
    gv = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.sb200_adaround_bwd(x.data_ptr(), v.data_ptr(), scale.data_ptr(), zero_point.data_ptr(),
                                     grad_y.data_ptr(), gv.data_ptr(), outer, c, inner, int(qmin), int(qmax), _stream(x)))
    return gv


def adaround_init(x, scale, ch_axis=None):
    """adaround.py:26-32."""
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale")
    outer, c, inner = _adaround_geometry(x, scale, ch_axis)
    v = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib.sb200_adaround_init(x.data_ptr(), scale.data_ptr(), v.data_ptr(), outer, c, inner, _stream(x)))
    return v


# ----------------------------------------------------------------------------- MinMax
def minmax_new(channels, device):
    """Fresh running min/max state: int32[2*C] (bit pattern of the uint32 ordered keys)."""
    lib = _lib.load()
    st = torch.empty(2 * channels, dtype=torch.int32, device=device)
    with torch.cuda.device(st.device):
        check(lib.sb200_minmax_init(st.data_ptr(), channels, _stream(st)))
    return st


def minmax_update(x, state, ch_axis=None):
    lib = _lib.load()
    _req(x, "data")
    with torch.cuda.device(x.device):
        if ch_axis is None:
            check(lib.sb200_observe_minmax(x.data_ptr(), x.numel(), state.data_ptr(), _stream(x)))
        else:
            outer, c, inner = channel_geometry(x.shape, ch_axis)
            if state.numel() != 2 * c:
                raise SparsebitB200Error(f"minmax state holds {state.numel() // 2} channels, data has {c}")
            check(lib.sb200_observe_minmax_perchannel(x.data_ptr(), outer, c, inner, state.data_ptr(), _stream(x)))


def minmax_read(state):
    lib = _lib.load()
    c = state.numel() // 2
    mn = torch.empty(c, dtype=torch.float32, device=state.device)
    mx = torch.empty(c, dtype=torch.float32, device=state.device)
    with torch.cuda.device(state.device):
        check(lib.sb200_minmax_read(state.data_ptr(), c, mn.data_ptr(), mx.data_ptr(), _stream(state)))
    return mn, mx


class _QparamsDesc(ctypes.Structure):  # include/sparsebit_b200.h sb200_minmax_qparams_desc
    _fields_ = [("state", ctypes.c_void_p), ("out_min", ctypes.c_void_p), ("out_max", ctypes.c_void_p), ("out_scale", ctypes.c_void_p),
                ("out_zero_point", ctypes.c_void_p), ("channels", ctypes.c_int64), ("qmin", ctypes.c_int), ("qmax", ctypes.c_int),
                ("symmetric", ctypes.c_int)]


def minmax_qparams_multi(requests):
    """``requests``: [(state int32[2C], qmin, qmax, symmetric)] -> [(min, max, scale, zero_point)] float32[C] views of one
    buffer, computed by ONE launch (sb200_minmax_qparams_multi)."""
    lib = _lib.load()
    if not requests:
        return []
    dev = requests[0][0].device
    chans = [r[0].numel() // 2 for r in requests]
    total = sum(chans)
    flat = torch.empty(4, total, dtype=torch.float32, device=dev)
    table = torch.empty(64 * len(requests), dtype=torch.uint8, device=dev)
    descs, outs, off = [], [], 0
    base, plane = flat.data_ptr(), total * 4
    for (state, qmin, qmax, sym), c in zip(requests, chans):
        p = base + off * 4
        descs.append(_QparamsDesc(state.data_ptr(), p, p + plane, p + 2 * plane, p + 3 * plane, c, int(qmin), int(qmax), int(bool(sym))))
        outs.append(tuple(flat[k, off:off + c] for k in range(4)))
        off += c
    arr = (_QparamsDesc * len(descs))(*descs)
    with torch.cuda.device(dev):
        check(lib.sb200_minmax_qparams_multi(arr, len(descs), table.data_ptr(), table.numel(), torch.cuda.current_stream(dev).cuda_stream))
    return outs


# ----------------------------------------------------------------------------- histogram / MSE
def hist_update(x, range_lo_hi, counts):
    """counts (int64[bins]) += histc(x, bins, lo, hi); ``range_lo_hi``: device float32[2]."""
    lib = _lib.load()
    _req(x, "data"), _req(range_lo_hi, "range")
    with torch.cuda.device(x.device):
        check(lib.sb200_observe_hist(x.data_ptr(), x.numel(), range_lo_hi.data_ptr(), counts.numel(), counts.data_ptr(), _stream(x)))


def mse_sweep(x2d, cand_scale, cand_zp, qmin, qmax, sse):
    """sse[rows, ncand] (fp64) += sum_j (x - qdq_i(x))^2 for every candidate i; x2d: [rows, row_len]."""
    lib = _lib.load()
    _req(x2d, "data"), _req(cand_scale, "cand_scale"), _req(cand_zp, "cand_zp")
    rows, row_len = x2d.shape
    ncand = cand_scale.numel() // rows
    ws_bytes = int(lib.sb200_mse_workspace_bytes(rows, row_len, ncand))
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x2d.device)
    with torch.cuda.device(x2d.device):
        check(lib.sb200_observe_mse_sweep(x2d.data_ptr(), rows, row_len, cand_scale.data_ptr(), cand_zp.data_ptr(), ncand,
                                          int(qmin), int(qmax), sse.data_ptr(), ws.data_ptr(), ws_bytes, _stream(x2d)))


# ----------------------------------------------------------------------------- radix select
class RadixSelect:
    """Exact order statistics over one or more device tensors (3 passes x 4 B/elem).

    rows x ntargets_per_row independent selections; ``add_pass(p, tensors)`` accumulates the
    digit histograms of pass p for every tensor (each viewed as [rows, row_len]); an optional
    ``reduce`` callback (SUM all-reduce across GPUs) runs between histogram and scan."""

    def __init__(self, rows, ntargets_per_row, device, key_mode=0):
        self.lib = _lib.load()
        self.rows, self.ntpr, self.key_mode = rows, ntargets_per_row, key_mode
        n = rows * ntargets_per_row
        self.sel = torch.zeros(n * _lib.SELECT_STATE_WORDS, dtype=torch.int64, device=device)
        self.hist = torch.zeros(n * _lib.SELECT_BINS, dtype=torch.int64, device=device)
        self.counts = torch.zeros(rows * 2, dtype=torch.int64, device=device)
        with torch.cuda.device(device):
            check(self.lib.sb200_select_init(self.sel.data_ptr(), self.hist.data_ptr(), n, None, _stream(self.sel)))

    def set_ranks(self, ranks):
        """ranks: int64 device tensor [rows * ntpr] of 0-based ranks."""
        self.sel.view(-1, _lib.SELECT_STATE_WORDS)[:, 1] = ranks.to(torch.int64)

    def hist_pass(self, p, x2d, with_counts=False):
        _req(x2d, "data")
        rows, row_len = x2d.shape
        with torch.cuda.device(x2d.device):
            if with_counts and p == 0:
                check(self.lib.sb200_select_hist_counts(x2d.data_ptr(), rows, row_len, self.ntpr, self.sel.data_ptr(),
                                                        self.hist.data_ptr(), p, self.key_mode, self.counts.data_ptr(), _stream(x2d)))
            else:
                check(self.lib.sb200_select_hist(x2d.data_ptr(), rows, row_len, self.ntpr, self.sel.data_ptr(),
                                                 self.hist.data_ptr(), p, self.key_mode, _stream(x2d)))

    def percentile_ranks(self, total, alpha):
        """total: int64 device tensor [rows] (elements per row incl. NaN)."""
        with torch.cuda.device(self.sel.device):
            check(self.lib.sb200_percentile_ranks(self.counts.data_ptr(), total.data_ptr(), self.rows, float(alpha),
                                                  self.sel.data_ptr(), _stream(self.sel)))

    def scan(self, p):
        with torch.cuda.device(self.sel.device):
            check(self.lib.sb200_select_scan(self.sel.data_ptr(), self.hist.data_ptr(), self.rows, self.ntpr, p, _stream(self.sel)))

    def values(self):
        n = self.rows * self.ntpr
        out = torch.empty(n, dtype=torch.float32, device=self.sel.device)
        with torch.cuda.device(self.sel.device):
            check(self.lib.sb200_select_read(self.sel.data_ptr(), n, self.key_mode, out.data_ptr(), _stream(self.sel)))
        return out


def kth_value(x, k, key_mode=0):
    """k-th smallest (0-based) of a flat tensor, exact; key_mode 1 ranks |x|."""
    rs = RadixSelect(1, 1, x.device, key_mode)
    rs.set_ranks(torch.tensor([k], dtype=torch.int64, device=x.device))
    x2 = x.reshape(1, -1)
    for p in range(3):
        rs.hist_pass(p, x2)
        rs.scan(p)
    return rs.values()


# ----------------------------------------------------------------------------- sparser
def mask_gt(w, thresh):
    lib = _lib.load()
    _req(w, "weight"), _req(thresh, "thresh")
    mask = torch.empty(w.shape, dtype=torch.bool, device=w.device)
    with torch.cuda.device(w.device):
        check(lib.sb200_mask_gt(w.data_ptr(), thresh.data_ptr(), mask.data_ptr(), w.numel(), _stream(w)))
    return mask


def mask_rows_gt(score, thresh, shape):
    """Float mask of ``shape`` = [rows, ...]: row r is all ones if score[r] > thresh else all zeros."""
    lib = _lib.load()
    _req(score, "score"), _req(thresh, "thresh")
    rows = int(shape[0])
    if score.numel() != rows:
        raise SparsebitB200Error("mask_rows_gt: one score per row expected")
    mask = torch.empty(tuple(shape), dtype=torch.float32, device=score.device)
    with torch.cuda.device(score.device):
        check(lib.sb200_mask_rows_gt(score.data_ptr(), thresh.data_ptr(), mask.data_ptr(), rows, mask.numel() // rows,
                                     _stream(score)))
    return mask


def mask_apply(w, mask, out=None):
    lib = _lib.load()
    _req(w, "weight")
    if mask.shape != w.shape or not mask.is_cuda or not mask.is_contiguous():
        raise SparsebitB200Error("mask must be a contiguous CUDA tensor of the weight's shape")
    out = torch.empty_like(w) if out is None else out
    with torch.cuda.device(w.device):
        if mask.dtype in (torch.bool, torch.uint8):
            check(lib.sb200_mask_apply(w.data_ptr(), mask.data_ptr(), out.data_ptr(), w.numel(), _stream(w)))
        elif mask.dtype == torch.float32:
            check(lib.sb200_mask_apply_f32(w.data_ptr(), mask.data_ptr(), out.data_ptr(), w.numel(), _stream(w)))
        else:
            raise SparsebitB200Error(f"unsupported mask dtype {mask.dtype}")
    return out


def mask_apply_qdq_perchannel(w, mask, scale, zero_point, qmin, qmax, ch_axis=0, rounding=0, out=None):
    lib = _lib.load()
    _req(w, "weight"), _req(scale, "scale"), _req(zero_point, "zero_point")
    if mask.dtype not in (torch.bool, torch.uint8) or mask.shape != w.shape or not mask.is_contiguous():
        raise SparsebitB200Error("fused mask+QDQ needs a contiguous bool mask of the weight's shape")
    outer, c, inner = channel_geometry(w.shape, ch_axis)
    out = torch.empty_like(w) if out is None else out
    with torch.cuda.device(w.device):
        check(lib.sb200_mask_apply_qdq_perchannel(w.data_ptr(), mask.data_ptr(), scale.data_ptr(), zero_point.data_ptr(),
                                                  out.data_ptr(), outer, c, inner, int(qmin), int(qmax), int(rounding), _stream(w)))
    return out


# ----------------------------------------------------------------------------- per-stream workspaces
class _StreamWorkspaces:
    """Scratch buffers of one family of entry points, one per key (device, stream[, kind]), grown on demand.

    A CUDA graph captured on a stream keeps the raw address of the workspace its kernels used.  So a workspace used
    while its stream is capturing is pinned: when a later, larger call outgrows it, it moves to ``retired`` and stays
    allocated for the life of the process instead of going back to the caching allocator, which would hand it to the
    next allocation on the stream for every replay to overwrite.  An unpinned workspace is replaced and freed as
    before, so eager-only use holds one workspace per key."""

    def __init__(self):
        self.live = {}     # key -> uint8 tensor
        self.pinned = set()  # keys whose live workspace a captured graph holds
        self.retired = {}  # key -> [outgrown workspaces captured graphs hold]

    def get(self, key, device, nbytes):
        ws = self.live.get(key)
        if ws is None or ws.numel() < nbytes:
            if key in self.pinned:
                self.retired.setdefault(key, []).append(ws)
                self.pinned.discard(key)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
            self.live[key] = ws
        with torch.cuda.device(device):
            if torch.cuda.is_current_stream_capturing():
                self.pinned.add(key)
        return ws


# ----------------------------------------------------------------------------- GPTQ
_gptq_workspaces = _StreamWorkspaces()
_gptq_ws = _gptq_workspaces.live


class _Gptq4Options(ctypes.Structure):  # include/sparsebit_b200.h sb200_gptq4_options
    _fields_ = [("impl", ctypes.c_int), ("chunk_k", ctypes.c_int), ("flags", ctypes.c_int), ("reserved", ctypes.c_int * 5)]


GPTQ4_STATIC_WEIGHTS = 1  # include/sparsebit_b200.h SB200_GPTQ4_STATIC_WEIGHTS


def gptq4_matmul(x, qweight, out, scales, zeros, group_size=0, impl=None, chunk_k=0, static_weights=False):
    """In-place ``out += x @ dequant(qweight)`` (vecquant4matmul contract, cuda_kernel.cpp:10-23).
    ``impl``: per-call kernel selection (sb200_gptq4_matmul_ex); None = the library default.
    ``chunk_k``: the reserved ``sb200_gptq4_options.chunk_k``; only 0 is valid, anything else raises.
    ``static_weights``: qweight / scales / zeros are constants of the model (not written by the kernel just in front on
    the stream), so the decode kernel may fetch them while its predecessor is still draining."""
    lib = _lib.load()
    _req(x, "inp1"), _req(out, "out"), _req(scales, "scales"), _req(zeros, "zeros")
    _req(qweight, "inp2", torch.int32)
    if x.dim() < 2:
        raise SparsebitB200Error("input1 must be with dimension >= 2")  # cuda_kernel_4bit.cu:44
    if qweight.dim() != 2:
        raise SparsebitB200Error("input2 must be with dimension == 2")  # cuda_kernel_4bit.cu:48
    k = x.shape[-1]
    m = x.numel() // k
    n = qweight.shape[1]
    if out.shape[-1] != n:
        raise SparsebitB200Error("output channel must be the same with input2 out_channel")  # :52
    ws_bytes = int(lib.sb200_gptq4_workspace_bytes(m, k, n, int(group_size)))
    ws = None
    if ws_bytes:
        ws = _gptq_workspaces.get((x.device, torch.cuda.current_stream(x.device).cuda_stream), x.device, ws_bytes)
    with torch.cuda.device(x.device):
        if impl is None and not chunk_k and not static_weights:
            check(lib.sb200_gptq4_matmul(x.data_ptr(), qweight.data_ptr(), out.data_ptr(), scales.data_ptr(), zeros.data_ptr(),
                                         m, k, n, qweight.shape[0], int(group_size), ws.data_ptr() if ws is not None else None,
                                         ws_bytes, _stream(x)))
        else:
            opts = _Gptq4Options(int(impl or 0), int(chunk_k), GPTQ4_STATIC_WEIGHTS if static_weights else 0)
            check(lib.sb200_gptq4_matmul_ex(x.data_ptr(), qweight.data_ptr(), out.data_ptr(), scales.data_ptr(),
                                            zeros.data_ptr(), m, k, n, qweight.shape[0], int(group_size), ctypes.byref(opts),
                                            ws.data_ptr() if ws is not None else None, ws_bytes, _stream(x)))
    return out


class _Gptq4Problem(ctypes.Structure):  # include/sparsebit_b200.h sb200_gptq4_problem
    _fields_ = [("x", ctypes.c_void_p), ("qweight", ctypes.c_void_p), ("out", ctypes.c_void_p), ("scales", ctypes.c_void_p),
                ("zeros", ctypes.c_void_p), ("k", ctypes.c_int64), ("n", ctypes.c_int64), ("qweight_rows", ctypes.c_int64),
                ("group_size", ctypes.c_int)]


def gptq4_matmul_batch(problems, group_size=0, static_weights=False):
    """Up to 4 decode-sized linears sharing M in ONE launch (q / k / v, gate / up): ``problems`` = [(x, qweight, out, scales,
    zeros)], every ``out`` pre-initialised and accumulated in place (sb200_gptq4_matmul_batch[_ex])."""
    lib = _lib.load()
    m = None
    arr = (_Gptq4Problem * len(problems))()
    for i, (x, qw, out, sc, zr) in enumerate(problems):
        _req(x, "inp1"), _req(out, "out"), _req(sc, "scales"), _req(zr, "zeros"), _req(qw, "inp2", torch.int32)
        k = x.shape[-1]
        mi = x.numel() // k
        if m is None:
            m = mi
        elif mi != m:
            raise SparsebitB200Error("gptq4_matmul_batch: all problems must have the same number of tokens")
        if out.shape[-1] != qw.shape[1]:
            raise SparsebitB200Error("output channel must be the same with input2 out_channel")
        arr[i] = _Gptq4Problem(x.data_ptr(), qw.data_ptr(), out.data_ptr(), sc.data_ptr(), zr.data_ptr(), k, qw.shape[1], qw.shape[0],
                               int(group_size))
    dev = problems[0][0].device
    with torch.cuda.device(dev):
        check(lib.sb200_gptq4_matmul_batch_ex(arr, len(problems), m, GPTQ4_STATIC_WEIGHTS if static_weights else 0,
                                              torch.cuda.current_stream(dev).cuda_stream))
    return [p[2] for p in problems]


_gptq_state = {}  # (device, stream) -> zero-initialised, self-resetting arrival counters of the single-launch decode path


def gptq4_linear_f16(x, qweight, scales, zeros, bias=None, group_size=0, static_weights=False, single_launch=True):
    """fp16 activations in, fp16 ``bias + x @ dequant(qweight)`` out, no eager casts (sb200_gptq4_linear_f16_ex).
    Decode-sized M (<= 32) is ONE kernel launch; ``single_launch=False`` keeps the staged path (cast, bias, kernel, cast).
    ``static_weights``: see ``gptq4_matmul``."""
    lib = _lib.load()
    _req(x, "inp1", torch.float16), _req(scales, "scales"), _req(zeros, "zeros"), _req(qweight, "inp2", torch.int32)
    if bias is not None:
        _req(bias, "bias")
    k = x.shape[-1]
    m = x.numel() // k
    n = qweight.shape[1]
    out = torch.empty(x.shape[:-1] + (n,), dtype=torch.float16, device=x.device)
    ws_bytes = int(lib.sb200_gptq4_linear_f16_workspace_bytes(m, k, n, int(group_size)))
    key = (x.device, torch.cuda.current_stream(x.device).cuda_stream, "f16")
    ws = _gptq_workspaces.get(key, x.device, ws_bytes)
    state = None
    if single_launch and m <= 32:
        skey = key[:2]
        state = _gptq_state.get(skey)
        if state is None:
            state = torch.zeros(int(lib.sb200_gptq4_linear_f16_state_bytes()), dtype=torch.uint8, device=x.device)
            _gptq_state[skey] = state
    with torch.cuda.device(x.device):
        check(lib.sb200_gptq4_linear_f16_ex(x.data_ptr(), qweight.data_ptr(), out.data_ptr(), bias.data_ptr() if bias is not None else None,
                                            scales.data_ptr(), zeros.data_ptr(), m, k, n, qweight.shape[0], int(group_size),
                                            state.data_ptr() if state is not None else None,
                                            GPTQ4_STATIC_WEIGHTS if static_weights else 0, ws.data_ptr(), ws_bytes, _stream(x)))
    return out


def gptq_matmul(x, qweight, out, scales, zeros, bits, group_size=0):
    """In-place ``out += x @ dequant(qweight)`` for 2 / 3 / 4-bit GPTQ weights
    (vecquant{2,3,4}matmul / vecgroupquant{2,3,4}matmul, cuda_kernel.cpp:10-57)."""
    if int(bits) == 4:
        return gptq4_matmul(x, qweight, out, scales, zeros, group_size)
    lib = _lib.load()
    _req(x, "inp1"), _req(out, "out"), _req(scales, "scales"), _req(zeros, "zeros")
    _req(qweight, "inp2", torch.int32)
    if x.dim() < 2:
        raise SparsebitB200Error("input1 must be with dimension >= 2")  # cuda_kernel_3bit.cu:40
    if qweight.dim() != 2:
        raise SparsebitB200Error("input2 must be with dimension == 2")  # cuda_kernel_3bit.cu:44
    k = x.shape[-1]
    m = x.numel() // k
    n = qweight.shape[1]
    if out.shape[-1] != n:
        raise SparsebitB200Error("output channel must be the same with input2 out_channel")  # :48
    with torch.cuda.device(x.device):
        check(lib.sb200_gptq_matmul(x.data_ptr(), qweight.data_ptr(), out.data_ptr(), scales.data_ptr(), zeros.data_ptr(),
                                    m, k, n, qweight.shape[0], int(bits), int(group_size), None, 0, _stream(x)))
    return out


def int8_grid_offset(qmin):
    """What the integer path subtracts from a grid value to store it as s8: 128 for unsigned ranges, else 0."""
    return 128 if int(qmin) >= 0 else 0


def int8_padded_k(k):
    return (int(k) + 15) // 16 * 16


def _check_per_tensor(fn, *qparams):
    """The activation operands of the integer path are per-tensor: one scale and one zero point each."""
    if any(t.numel() != 1 for t in qparams):
        raise SparsebitB200Error(f"{fn}: the qparams are per-tensor (1 element each)")


def _req_int8_operands(x, x_scale, x_zero_point, w_scale, bias, x_format=torch.contiguous_format, **weight):
    """The dtypes of a per-tensor fp32 activation (contiguous in ``x_format``), the fp32 ``w_scale`` and ``bias``, and the
    integer tensors of the weight operand by name: int8 ``w_q`` / ``vals``, the others int32."""
    _req(x, "data", memory_format=x_format), _req(x_scale, "x_scale"), _req(x_zero_point, "x_zero_point"), _req(w_scale, "w_scale")
    for name, t in weight.items():
        _req(t, name, torch.int8 if name in ("w_q", "vals") else torch.int32)
    if bias is not None:
        _req(bias, "bias")


def _int8_weight_rows(fn, n, bias, **per_row):
    """``n``, the rows of the weight operand, which each per-row term (by name) and the bias must match."""
    if any(t.numel() != n for t in per_row.values()) or (bias is not None and bias.numel() != n):
        raise SparsebitB200Error(f"{fn}: {' / '.join(per_row)} / bias need {n} elements")
    return n


def _x_absmax_args(fn, x, x_absmax):
    """The entry-point suffix and extra argument of an integer-grid op's optional DoReFa input: ``("", [])`` without
    ``x_absmax``, else ``("_dorefa", [pointer])`` once it is checked to be the one-element fp32 tensor on x's device that
    ``dorefa_absmax(x)`` returns (max |tanh(x)|; the kernels quantize tanh(x) / x_absmax)."""
    if x_absmax is None:
        return "", []
    _req(x_absmax, "x_absmax")
    if x_absmax.numel() != 1 or x_absmax.device != x.device:
        raise SparsebitB200Error(f"{fn}: x_absmax must be one fp32 element on x's device, as dorefa_absmax(x) returns "
                                 f"(got {x_absmax.numel()} on {x_absmax.device})")
    return "_dorefa", [x_absmax.data_ptr()]


def int8_quantize_rows(x, scale, zero_point, qmin, qmax):
    """Integer grid of every row of ``x`` [rows, K] (sb200_int8_quantize_rows): returns ``(q, row_sum, nan)`` with
    q int8 [rows, Kp] = clamp(round(x / s) + rint(zp), qmin, qmax) - int8_grid_offset(qmin), the padding to
    Kp = round_up(K, 16) zero; row_sum int32 [rows]; nan bool [rows].  ``scale`` / ``zero_point``: one value for all
    rows or one per row."""
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale"), _req(zero_point, "zero_point")
    if x.dim() != 2:
        raise SparsebitB200Error("int8_quantize_rows: data must be [rows, K]")
    rows, k = x.shape
    if scale.numel() != zero_point.numel() or scale.numel() not in (1, rows):
        raise SparsebitB200Error(f"int8_quantize_rows: qparams need 1 or {rows} elements (got {scale.numel()}, {zero_point.numel()})")
    q = torch.empty(rows, int8_padded_k(k), dtype=torch.int8, device=x.device)
    row_sum = torch.empty(rows, dtype=torch.int32, device=x.device)
    nan = torch.empty(rows, dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.sb200_int8_quantize_rows(x.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), int(scale.numel() > 1),
                                           int(qmin), int(qmax), q.data_ptr(), row_sum.data_ptr(), nan.data_ptr(), rows, k,
                                           _stream(x)))
    return q, row_sum, nan


_int8_workspaces = _StreamWorkspaces()
_int8_ws = _int8_workspaces.live


def _int8_workspace(device, nbytes):
    """The integer path's workspace of (device, current stream), grown on demand and shared by its entry points.

    A workspace used during CUDA graph capture is pinned: a captured graph keeps writing the lowered activations to its
    address on every replay, so when a larger eager call outgrows it (a prefill after a captured decode step) it is
    retired, kept allocated, rather than freed to the caching allocator.  Workspaces never used under capture are
    simply replaced (see _StreamWorkspaces)."""
    return _int8_workspaces.get((device, torch.cuda.current_stream(device).cuda_stream), device, nbytes)


def int8_linear(x, x_scale, x_zero_point, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, bias=None, k=None, x_absmax=None):
    """``y = s_x s_w[n] sum_k v_x v_w + bias`` on the int8 tensor cores (sb200_int8_linear): the fake-quant linear of
    per-tensor activations [qmin, qmax] with the weights stored by ``int8_quantize_rows`` (w_q int8 [N, Kp], w_rowsum
    int32 [N], w_scale fp32 [N], w_zero int32 [N] = rint(zero point) - int8_grid_offset).  ``x`` [..., K] fp32; returns
    fp32 [..., N].  ``k`` defaults to x.shape[-1].  ``x_absmax``: ``dorefa_absmax(x)`` of a DoReFa input, whose
    tanh(x) / x_absmax is quantized (sb200_int8_linear_dorefa; the plain op on ``dorefa_forward(x, x_absmax)``, bit for
    bit)."""
    lib = _lib.load()
    _req_int8_operands(x, x_scale, x_zero_point, w_scale, bias, w_q=w_q, w_rowsum=w_rowsum, w_zero=w_zero)
    k = x.shape[-1] if k is None else int(k)
    if x.shape[-1] != k or w_q.dim() != 2 or w_q.shape[1] != int8_padded_k(k):
        raise SparsebitB200Error(f"int8_linear: x has {x.shape[-1]} features, w_q is {tuple(w_q.shape)} (need [N, {int8_padded_k(k)}])")
    n = _int8_weight_rows("int8_linear", w_q.shape[0], bias, w_rowsum=w_rowsum, w_scale=w_scale, w_zero=w_zero)
    m = x.numel() // k
    out = torch.empty(x.shape[:-1] + (n,), dtype=torch.float32, device=x.device)
    sfx, am = _x_absmax_args("int8_linear", x, x_absmax)
    ws_bytes = int(lib.sb200_int8_linear_workspace_bytes(m, k))
    ws = _int8_workspace(x.device, ws_bytes)
    with torch.cuda.device(x.device):
        check(getattr(lib, "sb200_int8_linear" + sfx)(x.data_ptr(), x_scale.data_ptr(), x_zero_point.data_ptr(), *am,
                                    int(qmin), int(qmax), w_q.data_ptr(), w_rowsum.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(),
                                    bias.data_ptr() if bias is not None else None, out.data_ptr(), m, k, n, ws.data_ptr(),
                                    ws_bytes, _stream(x)))
    return out


def sparse24_mask(w):
    """2:4 keep-mask of ``w`` (sb200_sparse24_mask): bool, shaped like ``w``.  Each row of ``w.reshape(w.shape[0], -1)``
    keeps the two largest |w| of every aligned group of 4 (ties to the lower index, NaN kept, a tail of r < 4 keeps
    min(2, r))."""
    lib = _lib.load()
    _req(w, "weight")
    rows = int(w.shape[0]) if w.dim() > 0 else 1
    mask = torch.empty(w.shape, dtype=torch.bool, device=w.device)
    with torch.cuda.device(w.device):
        check(lib.sb200_sparse24_mask(w.data_ptr(), mask.data_ptr(), rows, w.numel() // rows, _stream(w)))
    return mask


def int8_sparse24_shapes(n, k):
    """Shapes of the packed 2:4 weight (see sb200_int8_sparse24_pack): vals [N, K64 / 2], meta [ceil(N / 128), K64 / 64,
    2, 128], K64 = round_up(K, 64)."""
    k64 = (int(k) + 63) // 64 * 64
    return (int(n), k64 // 2), ((int(n) + 127) // 128, k64 // 64, 2, 128)


def int8_sparse24_pack(w_q, w_zero, w_scale, k):
    """Compress a weight stored by ``int8_quantize_rows`` (w_q int8 [N, Kp], w_zero int32 [N], w_scale fp32 [N]) into
    the 2:4 operand of ``int8_sparse24_linear``: returns ``(vals, meta, dsum, bad)`` with vals int8 [N, K64 / 2], meta
    int32 [ceil(N / 128), K64 / 64, 2, 128] (uint32 words), dsum int32 [N] = sum_k (w_q - w_zero) and bad int32 [N] =
    the groups of each row that are not 2:4 on the centred grid or leave s8 (a nonzero row cannot be used)."""
    lib = _lib.load()
    _req(w_q, "w_q", torch.int8), _req(w_zero, "w_zero", torch.int32), _req(w_scale, "w_scale")
    k = int(k)
    if w_q.dim() != 2 or w_q.shape[1] != int8_padded_k(k):
        raise SparsebitB200Error(f"int8_sparse24_pack: w_q is {tuple(w_q.shape)} (need [N, {int8_padded_k(k)}])")
    n = w_q.shape[0]
    if w_zero.numel() != n or w_scale.numel() != n:
        raise SparsebitB200Error(f"int8_sparse24_pack: w_zero / w_scale need {n} elements")
    vshape, mshape = int8_sparse24_shapes(n, k)
    vals = torch.empty(vshape, dtype=torch.int8, device=w_q.device)
    meta = torch.empty(mshape, dtype=torch.int32, device=w_q.device)
    dsum = torch.empty(n, dtype=torch.int32, device=w_q.device)
    bad = torch.empty(n, dtype=torch.int32, device=w_q.device)
    with torch.cuda.device(w_q.device):
        check(lib.sb200_int8_sparse24_pack(w_q.data_ptr(), w_zero.data_ptr(), w_scale.data_ptr(), vals.data_ptr(),
                                           meta.data_ptr(), dsum.data_ptr(), bad.data_ptr(), n, k, _stream(w_q)))
    return vals, meta, dsum, bad


def int8_sparse24_linear(x, x_scale, x_zero_point, qmin, qmax, vals, meta, dsum, w_scale, bias=None, k=None):
    """``int8_linear`` of a 2:4-sparse weight on the sparse int8 tensor cores (sb200_int8_sparse24_linear), from the
    operand ``int8_sparse24_pack`` made (vals, meta, dsum; every ``bad`` entry 0) and w_scale fp32 [N].  The output
    equals ``int8_linear`` on the dense stored weight bit for bit.  ``x`` [..., K] fp32; returns fp32 [..., N]."""
    lib = _lib.load()
    _req_int8_operands(x, x_scale, x_zero_point, w_scale, bias, vals=vals, meta=meta, dsum=dsum)
    k = x.shape[-1] if k is None else int(k)
    n = vals.shape[0] if vals.dim() == 2 else -1
    vshape, mshape = int8_sparse24_shapes(max(n, 1), k)
    if x.shape[-1] != k or tuple(vals.shape) != vshape or tuple(meta.shape) != mshape:
        raise SparsebitB200Error(f"int8_sparse24_linear: x has {x.shape[-1]} features, vals is {tuple(vals.shape)} and meta "
                                 f"{tuple(meta.shape)} (need {vshape} and {mshape})")
    _int8_weight_rows("int8_sparse24_linear", n, bias, dsum=dsum, w_scale=w_scale)
    m = x.numel() // k
    out = torch.empty(x.shape[:-1] + (n,), dtype=torch.float32, device=x.device)
    ws_bytes = int(lib.sb200_int8_linear_workspace_bytes(m, k))
    ws = _int8_workspace(x.device, ws_bytes)
    with torch.cuda.device(x.device):
        check(lib.sb200_int8_sparse24_linear(x.data_ptr(), x_scale.data_ptr(), x_zero_point.data_ptr(), int(qmin), int(qmax),
                                             vals.data_ptr(), meta.data_ptr(), dsum.data_ptr(), w_scale.data_ptr(),
                                             bias.data_ptr() if bias is not None else None, out.data_ptr(), m, k, n,
                                             ws.data_ptr(), ws_bytes, _stream(x)))
    return out


def int8_quantize_cols(x, scale, zero_point, qmin, qmax):
    """Transposed integer grid of ``x`` [..., K, N] (sb200_int8_quantize_cols): returns ``(q, col_sum, nan)`` with q int8
    [..., N, Kp], q[..., n, k] = the ``int8_quantize_rows`` grid value of x[..., k, n], the padding to Kp =
    round_up(K, 16) zero; col_sum int32 [..., N]; nan bool [..., N].  ``scale`` / ``zero_point``: 1 element."""
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale"), _req(zero_point, "zero_point")
    if x.dim() < 2:
        raise SparsebitB200Error("int8_quantize_cols: data must be [..., K, N]")
    _check_per_tensor("int8_quantize_cols", scale, zero_point)
    lead, (k, n) = tuple(x.shape[:-2]), x.shape[-2:]
    batch = x.numel() // (k * n)
    q = torch.empty(lead + (n, int8_padded_k(k)), dtype=torch.int8, device=x.device)
    col_sum = torch.empty(lead + (n,), dtype=torch.int32, device=x.device)
    nan = torch.empty(lead + (n,), dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.sb200_int8_quantize_cols(x.data_ptr(), scale.data_ptr(), zero_point.data_ptr(), int(qmin), int(qmax),
                                           q.data_ptr(), col_sum.data_ptr(), nan.data_ptr(), batch, k, n, _stream(x)))
    return q, col_sum, nan


def _is_k_major(b):
    """``b`` [..., K, N] is the transposed view of a contiguous [..., N, K] tensor."""
    return b.stride(-2) == 1 and b.transpose(-2, -1).is_contiguous()


def int8_matmul(a, a_scale, a_zero_point, a_qrange, b, b_scale, b_zero_point, b_qrange):
    """``y = s_a s_b sum_k v_a v_b`` on the int8 tensor cores (sb200_int8_matmul): the ``torch.matmul`` of two per-tensor
    fake-quantized activations, ``a`` [..., M, K] with ``(a_scale, a_zero_point, a_qrange = (qmin, qmax))`` and ``b``
    [..., K, N] likewise, both fp32 and quantized on the fly.  Leading dimensions broadcast as in ``torch.matmul``
    (copied only where they really broadcast).  A ``b`` that is the transposed view of a contiguous [..., N, K] tensor
    (``k.transpose(-2, -1)``) is read as it lies; any other non-contiguous operand is made contiguous.  Returns fp32
    [..., M, N]."""
    lib = _lib.load()
    for t, name in ((a, "a"), (b, "b")):
        if not isinstance(t, torch.Tensor) or t.dim() < 2:
            raise SparsebitB200Error(f"int8_matmul: {name} must be a tensor with at least 2 dimensions")
    _req(a_scale, "a_scale"), _req(a_zero_point, "a_zero_point"), _req(b_scale, "b_scale"), _req(b_zero_point, "b_zero_point")
    _check_per_tensor("int8_matmul", a_scale, a_zero_point, b_scale, b_zero_point)
    (m, k), (kb, n) = a.shape[-2:], b.shape[-2:]
    if k != kb:
        raise SparsebitB200Error(f"int8_matmul: a is {tuple(a.shape)}, b is {tuple(b.shape)} (inner dimensions differ)")
    lead = torch.broadcast_shapes(a.shape[:-2], b.shape[:-2])
    a = a.expand(lead + (m, k)).reshape(-1, m, k).contiguous()
    b = b.expand(lead + (k, n)).reshape(-1, k, n)
    k_major = _is_k_major(b)
    b = b.transpose(-2, -1) if k_major else b.contiguous()  # [batch, N, K] as it lies, or [batch, K, N]
    _req(a, "a"), _req(b, "b")
    batch = a.shape[0]
    out = torch.empty(lead + (m, n), dtype=torch.float32, device=a.device)
    ws_bytes = int(lib.sb200_int8_matmul_workspace_bytes(batch, m, k, n))
    ws = _int8_workspace(a.device, max(ws_bytes, 16))
    with torch.cuda.device(a.device):
        check(lib.sb200_int8_matmul(a.data_ptr(), b.data_ptr(), int(k_major), a_scale.data_ptr(), a_zero_point.data_ptr(),
                                    int(a_qrange[0]), int(a_qrange[1]), b_scale.data_ptr(), b_zero_point.data_ptr(),
                                    int(b_qrange[0]), int(b_qrange[1]), out.data_ptr(), batch, m, k, n, ws.data_ptr(),
                                    ws.numel(), _stream(a)))
    return out


def attention_mask_check(attn_mask):
    """``attn_mask`` as the fp32 additive mask the attention adds to its scores: float32 as is, float16 / bfloat16
    up-cast (exact); a bool or any other mask raises ``TypeError``, since a bool mask has two conventions (True = keep in
    ``scaled_dot_product_attention``, True = hide elsewhere) and the reference's models use additive masks."""
    if not isinstance(attn_mask, torch.Tensor):
        raise TypeError(f"attn_mask must be a tensor, got {type(attn_mask).__name__}")
    if attn_mask.dtype == torch.bool:
        raise TypeError("attn_mask is a bool mask; pass an additive float mask instead: 0 where a key is seen, -inf (or a "
                        "large negative value such as -10000) where it is not, e.g. (1 - keep.float()) * -10000")
    if attn_mask.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise TypeError(f"attn_mask must be an additive float32, float16 or bfloat16 mask, got {attn_mask.dtype}")
    return attn_mask.float()


def attention_mask_strides(shape, strides, lead, tq, tk):
    """How sb200_int8_attention_masked addresses a mask of ``shape`` and ``strides`` (in elements) broadcast to
    ``lead + (tq, tk)``, the batch entries flattened: ``(stride_outer, stride_inner, inner, stride_row)`` with entry b at
    ``(b // inner) stride_outer + (b % inner) stride_inner``, or None when the broadcast view cannot be addressed so (a
    key stride other than 1, or batch dimensions that do not fold into two).  Raises ``ValueError`` when ``shape`` does
    not broadcast to ``lead + (tq, tk)``."""
    full = tuple(int(n) for n in lead) + (int(tq), int(tk))
    shape, strides = tuple(int(n) for n in shape), tuple(int(s) for s in strides)
    if len(shape) > len(full):
        raise ValueError(f"a mask of shape {shape} does not broadcast to {full}")
    pad = len(full) - len(shape)
    shape, strides = (1,) * pad + shape, (0,) * pad + strides
    es = []
    for n, m, st in zip(full, shape, strides):
        if m != n and m != 1:
            raise ValueError(f"a mask of shape {shape[pad:]} does not broadcast to {full}")
        es.append(st if m == n and n > 1 else 0)
    if tk > 1 and es[-1] != 1:
        return None
    dims = []  # the batch dimensions of size > 1, adjacent ones folded where their strides allow
    for n, st in zip(full[:-2], es[:-2]):
        if n == 1:
            continue
        if dims and dims[-1][1] == st * n:
            dims[-1] = (dims[-1][0] * n, st)
        else:
            dims.append((n, st))
    if len(dims) > 2:
        return None
    if len(dims) < 2:
        return (dims[0][1] if dims else 0, 0, 1, es[-2])
    return (dims[0][1], dims[1][1], dims[1][0], es[-2])


def _attention_qparams(fn, *qparams):
    """The C-ABI arguments of (q, k, p, v) qparams: ``(scale, zero_point, (qmin, qmax))`` each, per-tensor fp32."""
    qp = []
    for (s, z, qrange), name in zip(qparams, ("q", "k", "p", "v")):
        _req(s, f"{name}_scale"), _req(z, f"{name}_zero_point")
        _check_per_tensor(fn, s, z)
        qp += [s.data_ptr(), z.data_ptr(), int(qrange[0]), int(qrange[1])]
    return qp


def _attention_mask(fn, attn_mask, causal, device, lead, tq, tk):
    """(fp32 mask or None, its ``attention_mask_strides`` plan) of an attention call over ``lead + (tq, tk)``; a mask
    whose broadcast cannot be addressed in place is copied (batch dimensions and keys, a broadcast row kept)."""
    if causal not in (False, True):
        raise SparsebitB200Error(f"{fn}: causal must be a bool, got {causal!r}")
    if attn_mask is None:
        return None, None
    mask = attention_mask_check(attn_mask)
    if mask.device != device:
        raise SparsebitB200Error(f"{fn}: attn_mask is on {mask.device}, q on {device}")
    try:
        plan = attention_mask_strides(mask.shape, mask.stride(), lead, tq, tk)
    except ValueError as e:
        raise SparsebitB200Error(f"{fn}: attn_mask: {e}") from None
    if plan is None:  # materialise the batch dimensions and the keys, keep a broadcast row
        shape = (1,) * (len(lead) + 2 - mask.dim()) + tuple(mask.shape)
        mask = mask.reshape(shape).expand(lead + (shape[-2], tk)).contiguous()
        plan = attention_mask_strides(mask.shape, mask.stride(), lead, tq, tk)
    return mask, plan


def _mask_args(mask, plan):
    return [mask.data_ptr(), *plan[:3], plan[3]] if mask is not None else [None, 0, 0, 1, 0]


def int8_attention(q, k, v, q_qparams, k_qparams, p_qparams, v_qparams, scale=None, return_p=False, attn_mask=None,
                   causal=False):
    """``softmax(q @ k^T [* scale] [masked]) @ v`` with q, k, the softmax output p and v each on a per-tensor int8 grid,
    in one fused kernel (sb200_int8_attention, or sb200_int8_attention_masked with a mask or ``causal``) that never
    writes the [Tq, Tk] scores: the scores are bit-identical to ``int8_matmul(q, k^T)``, p is the fp32 softmax
    quantized with ``p_qparams``, and ``p @ v`` is exact on the grid.
    ``q`` [..., Tq, d], ``k`` [..., Tk, d], ``v`` [..., Tk, dv] fp32 with equal leading dimensions (no broadcasting);
    non-contiguous operands are made contiguous.  Each ``*_qparams`` is ``(scale, zero_point, (qmin, qmax))`` with
    1-element fp32 tensors.  ``causal`` hides key j from row i when j > i + (Tk - Tq) (bottom-right, as
    ``QAttention``); ``attn_mask`` is an additive float mask broadcastable to [..., Tq, Tk], added after the scale and
    the causal band, read in place as a strided view when its broadcast can be addressed so (``attention_mask_strides``)
    and copied otherwise.  Returns fp32 [..., Tq, dv], and with ``return_p`` also the stored int8 grid of p
    [..., Tq, round_up(Tk, 16)]."""
    lib = _lib.load()
    for x, name in ((q, "q"), (k, "k"), (v, "v")):
        if not isinstance(x, torch.Tensor) or x.dim() < 2:
            raise SparsebitB200Error(f"int8_attention: {name} must be a tensor with at least 2 dimensions")
    qp = _attention_qparams("int8_attention", q_qparams, k_qparams, p_qparams, v_qparams)
    lead = tuple(q.shape[:-2])
    if tuple(k.shape[:-2]) != lead or tuple(v.shape[:-2]) != lead:
        raise SparsebitB200Error(f"int8_attention: q {tuple(q.shape)}, k {tuple(k.shape)} and v {tuple(v.shape)} need equal "
                                 "leading dimensions (no broadcasting)")
    (tq, d), (tk, dk), (tkv, dv) = q.shape[-2:], k.shape[-2:], v.shape[-2:]
    if dk != d or tkv != tk:
        raise SparsebitB200Error(f"int8_attention: q {tuple(q.shape)}, k {tuple(k.shape)} and v {tuple(v.shape)} do not "
                                 "chain (q and k need the same d, k and v the same Tk)")
    mask, plan = _attention_mask("int8_attention", attn_mask, causal, q.device, lead, tq, tk)
    q, k, v = (x.reshape(-1, *x.shape[-2:]).contiguous() for x in (q, k, v))
    _req(q, "q"), _req(k, "k"), _req(v, "v")
    batch = q.shape[0]
    out = torch.empty(lead + (tq, dv), dtype=torch.float32, device=q.device)
    p_q = torch.empty(lead + (tq, int8_padded_k(tk)), dtype=torch.int8, device=q.device) if return_p else None
    tail = [out.data_ptr(), p_q.data_ptr() if p_q is not None else None, batch, tq, tk, d, dv]
    scl = [int(scale is not None), float(scale) if scale is not None else 1.0]
    if mask is None and not causal:
        ws_bytes = int(lib.sb200_int8_attention_workspace_bytes(batch, tq, tk, d, dv))
        ws = _int8_workspace(q.device, max(ws_bytes, 16))
        with torch.cuda.device(q.device):
            check(lib.sb200_int8_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), *qp, *scl, *tail, ws.data_ptr(),
                                           ws.numel(), _stream(q)))
    else:
        mk = _mask_args(mask, plan)
        ws_bytes = int(lib.sb200_int8_attention_masked_workspace_bytes(batch, tq, tk, d, dv, int(causal)))
        ws = _int8_workspace(q.device, max(ws_bytes, 16))
        with torch.cuda.device(q.device):
            check(lib.sb200_int8_attention_masked(q.data_ptr(), k.data_ptr(), v.data_ptr(), *qp, *scl, *mk, int(causal),
                                                  *tail, ws.data_ptr(), ws.numel(), _stream(q)))
    return (out, p_q) if return_p else out


class Int8KVCache:
    """An int8 key/value cache of ``int8_attention_cached``: keys and values quantized once, on append, with the
    qparams of the layer that owns the cache (``QAttentionInt8.new_cache``).  For ``lead`` entries (the leading
    dimensions of q / k / v), ``capacity`` keys of width ``d`` and values of width ``dv``, zero-initialised:

    * ``k_q`` int8 [*lead, capacity, round_up(d, 16)], ``k_sum`` int32 / ``k_nan`` bool [*lead, capacity]: key j's
      stored grid, its sum and NaN flag, as ``int8_quantize_rows`` writes them;
    * ``v_t`` int8 [*lead, dv, round_up(capacity, 16)], ``v_sum`` int32 / ``v_nan`` bool [*lead, dv]: v^T as
      ``int8_quantize_cols`` writes it, the column sums over the stored keys and a sticky NaN flag.

    ``length`` (a host integer) keys are stored; every byte past them is 0."""

    def __init__(self, layer, lead, capacity, d, dv, device):
        lead, capacity, d, dv = tuple(int(n) for n in lead), int(capacity), int(d), int(dv)
        if min(lead + (capacity, d, dv), default=1) <= 0:
            raise SparsebitB200Error(f"Int8KVCache: lead {lead}, capacity {capacity}, d {d} and dv {dv} must be positive")
        self.layer, self.lead, self.capacity, self.d, self.dv, self.length = layer, lead, capacity, d, dv, 0
        z = dict(device=device)
        self.k_q = torch.zeros(lead + (capacity, int8_padded_k(d)), dtype=torch.int8, **z)
        self.k_sum = torch.zeros(lead + (capacity,), dtype=torch.int32, **z)
        self.k_nan = torch.zeros(lead + (capacity,), dtype=torch.bool, **z)
        self.v_t = torch.zeros(lead + (dv, int8_padded_k(capacity)), dtype=torch.int8, **z)
        self.v_sum = torch.zeros(lead + (dv,), dtype=torch.int32, **z)
        self.v_nan = torch.zeros(lead + (dv,), dtype=torch.bool, **z)

    def buffers(self):
        return (self.k_q, self.k_sum, self.k_nan, self.v_t, self.v_sum, self.v_nan)

    def __repr__(self):
        return f"Int8KVCache(lead={self.lead}, length={self.length}, capacity={self.capacity}, d={self.d}, dv={self.dv})"


def int8_kv_append(cache, k, v, k_qparams, v_qparams):
    """Quantize ``k`` [*lead, t, d] and ``v`` [*lead, t, dv] (fp32) into ``cache`` at positions [length, length + t)
    in one launch (sb200_int8_kv_append), then advance ``cache.length``.  ``k_qparams`` / ``v_qparams`` are
    ``(scale, zero_point, (qmin, qmax))`` and must be the same at every call on a cache."""
    lib = _lib.load()
    fn = "int8_kv_append"
    for x, name in ((k, "k"), (v, "v")):
        if not isinstance(x, torch.Tensor) or x.dim() < 2:
            raise SparsebitB200Error(f"{fn}: {name} must be a tensor with at least 2 dimensions")
    (t, d), (tv, dv) = k.shape[-2:], v.shape[-2:]
    if tuple(k.shape[:-2]) != cache.lead or tuple(v.shape[:-2]) != cache.lead or tv != t or d != cache.d or dv != cache.dv:
        raise SparsebitB200Error(f"{fn}: k {tuple(k.shape)} and v {tuple(v.shape)} do not match the cache's lead "
                                 f"{cache.lead}, d = {cache.d} and dv = {cache.dv}")
    if cache.length + t > cache.capacity:
        raise SparsebitB200Error(f"{fn}: {cache.length} + {t} keys overflow the cache's capacity {cache.capacity}")
    qp = []
    for (s, z, qrange), name in ((k_qparams, "k"), (v_qparams, "v")):
        _req(s, f"{name}_scale"), _req(z, f"{name}_zero_point")
        _check_per_tensor(fn, s, z)
        qp.append([s.data_ptr(), z.data_ptr(), int(qrange[0]), int(qrange[1])])
    k, v = (x.reshape(-1, *x.shape[-2:]).contiguous() for x in (k, v))
    _req(k, "k"), _req(v, "v")
    if k.device != cache.k_q.device:
        raise SparsebitB200Error(f"{fn}: k is on {k.device}, the cache on {cache.k_q.device}")
    with torch.cuda.device(k.device):
        check(lib.sb200_int8_kv_append(k.data_ptr(), v.data_ptr(), *qp[0], *qp[1], *(b.data_ptr() for b in cache.buffers()),
                                       k.shape[0], cache.capacity, cache.length, t, d, dv, _stream(k)))
    cache.length += int(t)


def int8_attention_cached(q, cache, q_qparams, k_qparams, p_qparams, v_qparams, scale=None, return_p=False,
                          attn_mask=None, causal=False):
    """``int8_attention`` of ``q`` [*lead, Tq, d] over the ``cache.length`` keys and values stored in ``cache``
    (sb200_int8_attention_cached), with the same arguments, mask broadcasting over [*lead, Tq, length], ``return_p``
    and workspace.  Tq > 16 runs the fused kernel over the cache: bit-identical to ``int8_attention`` on the
    concatenated fp32 keys and values.  Tq <= 16 runs the split-key decode kernels: the same scores bit for bit, every p
    within the bound of the fused kernel, out exact on the returned p grid; a p grid value can differ from the fused
    kernel's by one step where its fp64 denominator rounds differently."""
    lib = _lib.load()
    fn = "int8_attention_cached"
    if not isinstance(q, torch.Tensor) or q.dim() < 2:
        raise SparsebitB200Error(f"{fn}: q must be a tensor with at least 2 dimensions")
    lead, (tq, d) = tuple(q.shape[:-2]), q.shape[-2:]
    if lead != cache.lead or d != cache.d:
        raise SparsebitB200Error(f"{fn}: q {tuple(q.shape)} does not match the cache's lead {cache.lead} and d = {cache.d}")
    tk, dv = cache.length, cache.dv
    if tk == 0:
        raise SparsebitB200Error(f"{fn}: the cache is empty")
    qp = _attention_qparams(fn, q_qparams, k_qparams, p_qparams, v_qparams)
    mask, plan = _attention_mask(fn, attn_mask, causal, q.device, lead, tq, tk)
    q = q.reshape(-1, tq, d).contiguous()
    _req(q, "q")
    batch = q.shape[0]
    out = torch.empty(lead + (tq, dv), dtype=torch.float32, device=q.device)
    p_q = torch.empty(lead + (tq, int8_padded_k(tk)), dtype=torch.int8, device=q.device) if return_p else None
    scl = [int(scale is not None), float(scale) if scale is not None else 1.0]
    ws_bytes = int(lib.sb200_int8_attention_cached_workspace_bytes(batch, tq, cache.capacity, tk, d, dv, int(causal)))
    ws = _int8_workspace(q.device, max(ws_bytes, 16))
    with torch.cuda.device(q.device):
        check(lib.sb200_int8_attention_cached(q.data_ptr(), *qp, *scl, *_mask_args(mask, plan), int(causal),
                                              *(b.data_ptr() for b in cache.buffers()), cache.capacity, tk,
                                              out.data_ptr(), p_q.data_ptr() if p_q is not None else None, batch, tq,
                                              d, dv, ws.data_ptr(), ws.numel(), _stream(q)))
    return (out, p_q) if return_p else out


def _pair(v):
    return (int(v), int(v)) if isinstance(v, int) else tuple(int(e) for e in v)


def conv2d_geometry(x_shape, kernel_size, stride=1, padding=0, dilation=1):
    """``sb200_conv2d_geom`` of an [N, C, H, W] input.  ``padding``: an int, (pad_h, pad_w) or
    (top, bottom, left, right)."""
    n, c, h, w = (int(d) for d in x_shape)
    kh, kw = _pair(kernel_size)
    sh, sw = _pair(stride)
    dh, dw = _pair(dilation)
    pad = _pair(padding)
    if len(pad) == 2:
        pad = (pad[0], pad[0], pad[1], pad[1])
    if len(pad) != 4:
        raise SparsebitB200Error(f"conv2d padding must be an int, 2 or 4 ints (got {padding!r})")
    return _lib.Conv2dGeom(n, c, h, w, kh, kw, sh, sw, dh, dw, *pad)


def conv2d_output_hw(g):
    """(OH, OW) of a ``Conv2dGeom`` (may be < 1 for a kernel that does not fit)."""
    oh = (g.h + g.pad_top + g.pad_bottom - g.dilation_h * (g.kh - 1) - 1) // g.stride_h + 1
    ow = (g.w + g.pad_left + g.pad_right - g.dilation_w * (g.kw - 1) - 1) // g.stride_w + 1
    return oh, ow


def _int8_conv_rows(fn, k, w_scale, bias, w_q, w_rowsum, w_zero):
    """C_out of the weight operand ``int8_quantize_rows`` stores, for K = C / groups KH KW."""
    kp = int8_padded_k(k)
    if w_q.dim() != 2 or w_q.shape[1] != kp:
        raise SparsebitB200Error(f"{fn}: w_q is {tuple(w_q.shape)}, the geometry needs [C_out, {kp}]")
    return _int8_weight_rows(fn, w_q.shape[0], bias, w_rowsum=w_rowsum, w_scale=w_scale, w_zero=w_zero)


def _sparse24_conv_rows(fn, k, w_scale, bias, vals, meta, dsum):
    """C_out of the 2:4 operand ``int8_sparse24_pack`` made, for K = C KH KW."""
    n = vals.shape[0] if vals.dim() == 2 else -1
    vshape, mshape = int8_sparse24_shapes(max(n, 1), k)
    if tuple(vals.shape) != vshape or tuple(meta.shape) != mshape:
        raise SparsebitB200Error(f"{fn}: vals is {tuple(vals.shape)} and meta {tuple(meta.shape)}, the geometry (K = {k}) "
                                 f"needs {vshape} and {mshape}")
    return _int8_weight_rows(fn, n, bias, dsum=dsum, w_scale=w_scale)


def _int8_conv_prelude(fn, x, x_scale, x_zero_point, w_scale, bias, weight_rows, weight, kernel_size, groups, stride,
                       padding, dilation, memory_format=torch.contiguous_format):
    """The argument checks of the integer-grid conv wrappers, ``weight`` being the integer tensors of the weight
    operand by name and ``weight_rows`` its ``_int8_conv_rows`` / ``_sparse24_conv_rows``: returns the
    ``Conv2dGeom``, C_out and the fp32 [N, C_out, OH, OW] output in ``memory_format``, the layout x must have (one
    pixel when the kernel does not fit, which the C entry points reject)."""
    if memory_format == torch.channels_last and isinstance(x, torch.Tensor) and x.dim() != 4:
        raise SparsebitB200Error(f"{fn}: data must be [N, C, H, W] stored channels-last")
    _req_int8_operands(x, x_scale, x_zero_point, w_scale, bias, x_format=memory_format, **weight)
    if x.dim() != 4:
        raise SparsebitB200Error(f"{fn}: data must be [N, C, H, W]")
    groups = int(groups)
    g = conv2d_geometry(x.shape, kernel_size, stride, padding, dilation)
    if groups < 1 or g.c % groups:
        raise SparsebitB200Error(f"{fn}: groups = {groups} does not divide C = {g.c}")
    n = weight_rows(fn, g.c // groups * g.kh * g.kw, w_scale, bias, **weight)
    oh, ow = conv2d_output_hw(g)
    return g, n, torch.empty(g.n, n, max(oh, 1), max(ow, 1), dtype=torch.float32, device=x.device,
                             memory_format=memory_format)


def int8_im2col_quantize(x, kernel_size, scale, zero_point, qmin, qmax, stride=1, padding=0, dilation=1):
    """The lowered integer grid of a conv input (sb200_int8_im2col_quantize): ``x`` [N, C, H, W] fp32 -> ``(q, row_sum,
    nan)`` with q int8 [M, Kp], M = N OH OW (m = (n OH + oh) OW + ow), K = C KH KW (k = (c KH + kh) KW + kw), Kp =
    round_up(K, 16); element (m, k) is the stored grid value of the tap, padding taps store rint(zp) - offset, the K
    padding is zero; row_sum int32 [M]; nan bool [M] (the window holds a NaN).  ``scale`` / ``zero_point``: 1 element."""
    lib = _lib.load()
    _req(x, "data"), _req(scale, "scale"), _req(zero_point, "zero_point")
    if x.dim() != 4:
        raise SparsebitB200Error("int8_im2col_quantize: data must be [N, C, H, W]")
    _check_per_tensor("int8_im2col_quantize", scale, zero_point)
    g = conv2d_geometry(x.shape, kernel_size, stride, padding, dilation)
    oh, ow = conv2d_output_hw(g)
    m = g.n * max(oh, 0) * max(ow, 0)
    q = torch.empty(max(m, 1), int8_padded_k(g.c * g.kh * g.kw), dtype=torch.int8, device=x.device)
    row_sum = torch.empty(max(m, 1), dtype=torch.int32, device=x.device)
    nan = torch.empty(max(m, 1), dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.sb200_int8_im2col_quantize(x.data_ptr(), ctypes.byref(g), scale.data_ptr(), zero_point.data_ptr(),
                                             int(qmin), int(qmax), q.data_ptr(), row_sum.data_ptr(), nan.data_ptr(),
                                             _stream(x)))
    return q, row_sum, nan


def int8_conv2d(x, x_scale, x_zero_point, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, kernel_size, bias=None, stride=1,
                padding=0, dilation=1, x_absmax=None):
    """The fake-quant conv2d (groups = 1) on the int8 tensor cores (sb200_int8_conv2d): ``x`` [N, C, H, W] fp32 is
    lowered to its integer grid and multiplied with the weights stored by ``int8_quantize_rows`` from
    ``weight.reshape(C_out, -1)`` (w_q int8 [C_out, Kp], w_rowsum int32, w_scale fp32, w_zero int32 [C_out]), as in
    ``int8_linear``.  Returns fp32 [N, C_out, OH, OW].  ``padding``: an int, (pad_h, pad_w) or (top, bottom, left,
    right).  ``x_absmax``: a DoReFa input's ``dorefa_absmax(x)``, as ``int8_linear`` takes it
    (sb200_int8_conv2d_dorefa)."""
    lib = _lib.load()
    g, n, out = _int8_conv_prelude("int8_conv2d", x, x_scale, x_zero_point, w_scale, bias, _int8_conv_rows,
                                   dict(w_q=w_q, w_rowsum=w_rowsum, w_zero=w_zero), kernel_size, 1, stride, padding,
                                   dilation)
    sfx, am = _x_absmax_args("int8_conv2d", x, x_absmax)
    ws_bytes = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    ws = _int8_workspace(x.device, max(ws_bytes, 16))
    with torch.cuda.device(x.device):
        check(getattr(lib, "sb200_int8_conv2d" + sfx)(x.data_ptr(), ctypes.byref(g), x_scale.data_ptr(),
                                    x_zero_point.data_ptr(), *am, int(qmin), int(qmax), w_q.data_ptr(), w_rowsum.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(),
                                    bias.data_ptr() if bias is not None else None, out.data_ptr(), n, ws.data_ptr(),
                                    ws.numel(), _stream(x)))
    return out


def int8_sparse24_conv2d(x, x_scale, x_zero_point, qmin, qmax, vals, meta, dsum, w_scale, kernel_size, bias=None,
                         stride=1, padding=0, dilation=1):
    """``int8_conv2d`` of a 2:4-sparse weight on the sparse int8 tensor cores (sb200_int8_sparse24_conv2d): ``x`` [N, C,
    H, W] fp32 is lowered as ``int8_conv2d`` lowers it and multiplied with the operand ``int8_sparse24_pack`` made from
    the stored rows of ``weight.reshape(C_out, -1)`` (K = C KH KW; vals, meta, dsum, every ``bad`` entry 0) and w_scale
    fp32 [C_out].  The output equals ``int8_conv2d`` on the dense stored weight bit for bit.  Returns fp32 [N, C_out, OH,
    OW].  ``padding``: an int, (pad_h, pad_w) or (top, bottom, left, right)."""
    lib = _lib.load()
    g, n, out = _int8_conv_prelude("int8_sparse24_conv2d", x, x_scale, x_zero_point, w_scale, bias, _sparse24_conv_rows,
                                   dict(vals=vals, meta=meta, dsum=dsum), kernel_size, 1, stride, padding, dilation)
    ws_bytes = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    ws = _int8_workspace(x.device, max(ws_bytes, 16))
    with torch.cuda.device(x.device):
        check(lib.sb200_int8_sparse24_conv2d(x.data_ptr(), ctypes.byref(g), x_scale.data_ptr(), x_zero_point.data_ptr(),
                                             int(qmin), int(qmax), vals.data_ptr(), meta.data_ptr(), dsum.data_ptr(),
                                             w_scale.data_ptr(), bias.data_ptr() if bias is not None else None,
                                             out.data_ptr(), n, ws.data_ptr(), ws.numel(), _stream(x)))
    return out


def int8_group_conv2d(x, x_scale, x_zero_point, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, kernel_size, groups, bias=None,
                      stride=1, padding=0, dilation=1, x_absmax=None):
    """The fake-quant grouped / depthwise conv2d (groups >= 2) on the integer grid (sb200_int8_group_conv2d): one direct
    int8 kernel that quantizes its input tile on the fly.  ``x`` [N, C, H, W] fp32; the weights as ``int8_conv2d``
    takes them, stored by ``int8_quantize_rows`` from ``weight.reshape(C_out, -1)`` (w_q int8 [C_out, Kp] with Kp =
    round_up(C / groups KH KW, 16), w_rowsum int32, w_scale fp32, w_zero int32 [C_out]).  Returns fp32 [N, C_out, OH,
    OW].  ``padding``: an int, (pad_h, pad_w) or (top, bottom, left, right).  No workspace.  ``x_absmax``: a DoReFa
    input's ``dorefa_absmax(x)``, as ``int8_linear`` takes it (sb200_int8_group_conv2d_dorefa)."""
    lib = _lib.load()
    g, n, out = _int8_conv_prelude("int8_group_conv2d", x, x_scale, x_zero_point, w_scale, bias, _int8_conv_rows,
                                   dict(w_q=w_q, w_rowsum=w_rowsum, w_zero=w_zero), kernel_size, groups, stride, padding,
                                   dilation)
    sfx, am = _x_absmax_args("int8_group_conv2d", x, x_absmax)
    with torch.cuda.device(x.device):
        check(getattr(lib, "sb200_int8_group_conv2d" + sfx)(x.data_ptr(), ctypes.byref(g), int(groups), x_scale.data_ptr(),
                                          x_zero_point.data_ptr(), *am, int(qmin), int(qmax), w_q.data_ptr(),
                                          w_rowsum.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(),
                                          bias.data_ptr() if bias is not None else None, out.data_ptr(), n, _stream(x)))
    return out


# ----------------------------------------------------------------------------- channels-last (NHWC) convs
def int8_im2col_quantize_nhwc(x, kernel_size, scale, zero_point, qmin, qmax, stride=1, padding=0, dilation=1):
    """``int8_im2col_quantize`` of a channels-last ``x`` (sb200_int8_im2col_quantize_nhwc): ``x`` [N, C, H, W] fp32
    with ``x.is_contiguous(memory_format=torch.channels_last)``; the same ``(q, row_sum, nan)`` byte for byte."""
    lib = _lib.load()
    if isinstance(x, torch.Tensor) and x.dim() != 4:
        raise SparsebitB200Error("int8_im2col_quantize_nhwc: data must be [N, C, H, W] stored channels-last")
    _req(x, "data", memory_format=torch.channels_last), _req(scale, "scale"), _req(zero_point, "zero_point")
    _check_per_tensor("int8_im2col_quantize_nhwc", scale, zero_point)
    g = conv2d_geometry(x.shape, kernel_size, stride, padding, dilation)
    oh, ow = conv2d_output_hw(g)
    m = g.n * max(oh, 0) * max(ow, 0)
    q = torch.empty(max(m, 1), int8_padded_k(g.c * g.kh * g.kw), dtype=torch.int8, device=x.device)
    row_sum = torch.empty(max(m, 1), dtype=torch.int32, device=x.device)
    nan = torch.empty(max(m, 1), dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.sb200_int8_im2col_quantize_nhwc(x.data_ptr(), ctypes.byref(g), scale.data_ptr(), zero_point.data_ptr(),
                                                  int(qmin), int(qmax), q.data_ptr(), row_sum.data_ptr(), nan.data_ptr(),
                                                  _stream(x)))
    return q, row_sum, nan


def int8_conv2d_nhwc(x, x_scale, x_zero_point, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, kernel_size, bias=None,
                     stride=1, padding=0, dilation=1, x_absmax=None):
    """``int8_conv2d`` of a channels-last ``x`` (sb200_int8_conv2d_nhwc), with the same stored weights: returns a
    channels-last fp32 [N, C_out, OH, OW] whose values equal ``int8_conv2d`` on ``x.contiguous()`` bit for bit.
    ``x_absmax``: as ``int8_conv2d`` takes it (sb200_int8_conv2d_nhwc_dorefa)."""
    lib = _lib.load()
    g, n, out = _int8_conv_prelude("int8_conv2d_nhwc", x, x_scale, x_zero_point, w_scale, bias, _int8_conv_rows,
                                   dict(w_q=w_q, w_rowsum=w_rowsum, w_zero=w_zero), kernel_size, 1, stride, padding,
                                   dilation, torch.channels_last)
    sfx, am = _x_absmax_args("int8_conv2d_nhwc", x, x_absmax)
    ws_bytes = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    ws = _int8_workspace(x.device, max(ws_bytes, 16))
    with torch.cuda.device(x.device):
        check(getattr(lib, "sb200_int8_conv2d_nhwc" + sfx)(x.data_ptr(), ctypes.byref(g), x_scale.data_ptr(),
                                         x_zero_point.data_ptr(), *am, int(qmin), int(qmax), w_q.data_ptr(), w_rowsum.data_ptr(), w_scale.data_ptr(),
                                         w_zero.data_ptr(), bias.data_ptr() if bias is not None else None, out.data_ptr(),
                                         n, ws.data_ptr(), ws.numel(), _stream(x)))
    return out


def int8_sparse24_conv2d_nhwc(x, x_scale, x_zero_point, qmin, qmax, vals, meta, dsum, w_scale, kernel_size, bias=None,
                              stride=1, padding=0, dilation=1):
    """``int8_sparse24_conv2d`` of a channels-last ``x`` (sb200_int8_sparse24_conv2d_nhwc): returns a channels-last fp32
    [N, C_out, OH, OW] whose values equal ``int8_sparse24_conv2d`` on ``x.contiguous()`` bit for bit."""
    lib = _lib.load()
    g, n, out = _int8_conv_prelude("int8_sparse24_conv2d_nhwc", x, x_scale, x_zero_point, w_scale, bias,
                                   _sparse24_conv_rows, dict(vals=vals, meta=meta, dsum=dsum), kernel_size, 1, stride,
                                   padding, dilation, torch.channels_last)
    ws_bytes = int(lib.sb200_int8_conv2d_workspace_bytes(ctypes.byref(g)))
    ws = _int8_workspace(x.device, max(ws_bytes, 16))
    with torch.cuda.device(x.device):
        check(lib.sb200_int8_sparse24_conv2d_nhwc(x.data_ptr(), ctypes.byref(g), x_scale.data_ptr(),
                                                  x_zero_point.data_ptr(), int(qmin), int(qmax), vals.data_ptr(),
                                                  meta.data_ptr(), dsum.data_ptr(), w_scale.data_ptr(),
                                                  bias.data_ptr() if bias is not None else None, out.data_ptr(), n,
                                                  ws.data_ptr(), ws.numel(), _stream(x)))
    return out


def int8_group_conv2d_nhwc(x, x_scale, x_zero_point, qmin, qmax, w_q, w_rowsum, w_scale, w_zero, kernel_size, groups,
                           bias=None, stride=1, padding=0, dilation=1, x_absmax=None):
    """``int8_group_conv2d`` of a channels-last ``x`` (sb200_int8_group_conv2d_nhwc), with the same stored weights:
    returns a channels-last fp32 [N, C_out, OH, OW] whose values equal ``int8_group_conv2d`` on ``x.contiguous()`` bit
    for bit.  No workspace.  ``x_absmax``: as ``int8_group_conv2d`` takes it (sb200_int8_group_conv2d_nhwc_dorefa)."""
    lib = _lib.load()
    g, n, out = _int8_conv_prelude("int8_group_conv2d_nhwc", x, x_scale, x_zero_point, w_scale, bias, _int8_conv_rows,
                                   dict(w_q=w_q, w_rowsum=w_rowsum, w_zero=w_zero), kernel_size, groups, stride, padding,
                                   dilation, torch.channels_last)
    sfx, am = _x_absmax_args("int8_group_conv2d_nhwc", x, x_absmax)
    with torch.cuda.device(x.device):
        check(getattr(lib, "sb200_int8_group_conv2d_nhwc" + sfx)(x.data_ptr(), ctypes.byref(g), int(groups),
                                               x_scale.data_ptr(), x_zero_point.data_ptr(), *am, int(qmin), int(qmax), w_q.data_ptr(),
                                               w_rowsum.data_ptr(), w_scale.data_ptr(), w_zero.data_ptr(),
                                               bias.data_ptr() if bias is not None else None, out.data_ptr(), n,
                                               _stream(x)))
    return out


def gptq_matmul_dgrad(grad_out, qweight, grad_in, scales, zeros, bits, group_size=0, impl=None):
    """In-place ``grad_in += grad_out @ dequant(qweight).T``: the input gradient of ``gptq_matmul`` for 2 / 3 / 4-bit
    weights (sb200_gptq_matmul_dgrad).  ``grad_out`` [..., N], ``grad_in`` [..., K] fp32.  ``impl``: per-call kernel
    selection, None / 0 = auto, 1 = SIMT, 2 = 4-bit wgmma kernel (an error on shapes it does not take).
    Deterministic: identical calls give bit-identical results."""
    lib = _lib.load()
    _req(grad_out, "grad_out"), _req(grad_in, "grad_in"), _req(scales, "scales"), _req(zeros, "zeros")
    _req(qweight, "qweight", torch.int32)
    if qweight.dim() != 2:
        raise SparsebitB200Error("qweight must be with dimension == 2")
    n = qweight.shape[1]
    if grad_out.shape[-1] != n:
        raise SparsebitB200Error(f"grad_out has {grad_out.shape[-1]} features, qweight {n}")
    k = grad_in.shape[-1]
    m = grad_out.numel() // n
    if grad_in.numel() // k != m:
        raise SparsebitB200Error("grad_in and grad_out must have the same number of rows")
    ws_bytes = int(lib.sb200_gptq_dgrad_workspace_bytes(m, k, n, int(bits), int(group_size)))
    key = (grad_out.device, torch.cuda.current_stream(grad_out.device).cuda_stream, "dgrad")
    ws = _gptq_workspaces.get(key, grad_out.device, ws_bytes)
    with torch.cuda.device(grad_out.device):
        check(lib.sb200_gptq_matmul_dgrad(grad_out.data_ptr(), qweight.data_ptr(), grad_in.data_ptr(), scales.data_ptr(),
                                          zeros.data_ptr(), m, k, n, qweight.shape[0], int(bits), int(group_size), int(impl or 0),
                                          ws.data_ptr(), ws_bytes, _stream(grad_out)))
    return grad_in
