"""Oracle: observer calibration reductions (numpy restatement of the reference observers)."""
import numpy as np

from . import qdq as _qdq

F32 = np.float32


def calc_qparams_with_minmax(min_val, max_val, qmin, qmax, symmetric):
    """sparsebit/quantization/observers/base.py:63-79 (all arithmetic in fp32, like the torch ops)."""
    min_val = np.asarray(min_val, dtype=F32)
    max_val = np.asarray(max_val, dtype=F32)
    min_neg = np.minimum(min_val, F32(0))
    max_pos = np.maximum(max_val, F32(0))
    denom = F32(float(qmax - qmin))
    if symmetric:
        max_pos = np.maximum(-min_neg, max_pos)
        scale = np.maximum(((max_pos * F32(2)).astype(F32) / denom).astype(F32), F32(1e-6))
        zero_point = np.zeros_like(scale)
    else:
        scale = np.maximum(((max_pos - min_neg).astype(F32) / denom).astype(F32), F32(1e-6))
        zero_point = np.rint((-min_neg / scale).astype(F32)).astype(F32)
    return scale.astype(F32), zero_point.astype(F32)


def channel_first(batches, ch_axis):
    """DataCache.get_data_for_calibration(CHANNELWISE) -- observers/base.py:27-31: cat along
    ch_axis (Q16), move ch_axis first, flatten the rest."""
    data = np.concatenate([np.asarray(b, dtype=F32) for b in batches], axis=ch_axis)
    if ch_axis != 0:
        data = np.swapaxes(data, 0, ch_axis)
    return np.ascontiguousarray(data).reshape(data.shape[0], -1)


def layerwise(batches):
    """DataCache.get_data_for_calibration(LAYERWISE) -- observers/base.py:32-33."""
    return np.concatenate([np.asarray(b, dtype=F32).reshape(-1) for b in batches])


def minmax(batches, per_channel=False, ch_axis=0):
    """observers/minmax.py:14-25."""
    if per_channel:
        d = channel_first(batches, ch_axis)
        return d.min(axis=1), d.max(axis=1)
    d = layerwise(batches)
    return d.min(), d.max()


def mse(batches, qmin, qmax, symmetric, per_channel=False, ch_axis=0, steps=80):
    """observers/mse.py:28-63: sweep (min, max) * (1 - 0.01 i), keep the strict minimum of
    mean((x - qdq(x))^2) (first wins).  Per-channel is only meaningful for ch_axis == 0 rows (Q7).
    Loss accumulated in fp64.  Returns (scale, zero_point, losses[steps] or [steps, C])."""
    d = channel_first(batches, ch_axis)
    if per_channel:
        mn, mx = d.min(axis=1), d.max(axis=1)
    else:
        mn, mx = d.min(), d.max()
    best_s = best_z = None
    loss_min = None
    losses = []
    for i in range(steps):
        f = F32(1.0 - (i * 0.01))
        s, z = calc_qparams_with_minmax(mn * f, mx * f, qmin, qmax, symmetric)
        if per_channel:
            xdq = _qdq.qdq(d, s, z, qmin, qmax, ch_axis=0)
            loss = ((d.astype(np.float64) - xdq.astype(np.float64)) ** 2).mean(axis=1)
            if loss_min is None:
                loss_min = np.full(d.shape[0], 1e10)
                best_s = np.ones(d.shape[0], dtype=F32)
                best_z = np.zeros(d.shape[0], dtype=F32)
            upd = loss < loss_min
            best_s = np.where(upd, s, best_s)
            best_z = np.where(upd, z, best_z)
            loss_min = np.where(upd, loss, loss_min)
        else:
            xdq = _qdq.qdq(d, s.reshape(1), z.reshape(1), qmin, qmax)
            loss = float(((d.astype(np.float64) - xdq.astype(np.float64)) ** 2).mean())
            if loss_min is None:
                loss_min = 1e10
            if loss < loss_min:
                loss_min, best_s, best_z = loss, s, z
        losses.append(loss)
    return best_s, best_z, np.array(losses)


def _kth(row, k):
    """torch.kthvalue(row, k).values with 1-based k (NaN sorts last)."""
    return np.partition(row, k - 1)[k - 1]


def percentile(batches, alpha, per_channel=False, ch_axis=0):
    """observers/percentile.py:16-46 (Python round() = half-to-even on the double product)."""
    d = channel_first(batches, ch_axis) if per_channel else layerwise(batches).reshape(1, -1)
    c = d.shape[0]
    mx = np.zeros(c, dtype=F32)
    mn = np.zeros(c, dtype=F32)
    for i in range(c):
        neg = int((d[i] < 0).sum())
        pos = int((d[i] >= 0).sum())
        if pos > 0:
            mx[i] = _kth(d[i], d[i].size - max(round(pos * alpha), 0))
        if neg > 0:
            mn[i] = _kth(d[i], max(round(neg * alpha), 1))
    return mn, mx


def histc(x, bins, lo, hi):
    """torch.histc on CPU (what observers/kl_histogram.py:48 calls after ``.cpu()``).  ATen
    (aten/src/ATen/native/cpu/HistogramKernel.cpp, linear interpolation without local search):
        pos = int64(((x - lo) * bins) / (hi - lo))   in fp32;   pos == bins -> bins - 1
    elements outside [lo, hi] (and NaN) are dropped.  Verified against torch.histc on 6e6 random
    and on-edge values (tests/golden/make_golden.py, tests/test_oracle_golden.py).
    An empty range (lo == hi) is widened first, as ATen's histc_select_outer_bin_edges does: to the
    data's own min and max, and if those are equal too, to [lo - 1, hi + 1].  Like ATen, a range
    that is not finite after this (an infinite bound, or NaN data in an empty range) raises."""
    x = np.asarray(x, dtype=F32).reshape(-1)
    lo = F32(lo)
    hi = F32(hi)
    if lo == hi and x.size:
        lo, hi = x.min(), x.max()
    if lo == hi:
        lo, hi = F32(lo - F32(1)), F32(hi + F32(1))
    if not (np.isfinite(lo) and np.isfinite(hi)):
        raise ValueError(f"histc: range of [{lo}, {hi}] is not finite")
    xs = x[(x >= lo) & (x <= hi)]
    with np.errstate(all="ignore"):
        pos = (((xs - lo).astype(F32) * F32(bins)).astype(F32) / F32(hi - lo)).astype(F32).astype(np.int64)
    pos = np.minimum(pos, bins - 1)
    return np.bincount(pos, minlength=bins).astype(np.int64)


def calibrate_entropy(distribution, bin_width, src_bins, dst_bins=255):
    """observers/kl_histogram.py:54-94, restated loop for loop INCLUDING its index quirks (Q6):
    ``divergence[i - dst_bins]`` wraps for i < dst_bins and leaves one slot at 0; the last slice
    element of p is overwritten (not accumulated); the last q segment stops one short."""
    from scipy import stats

    distribution = np.asarray(distribution)
    zero_idx = src_bins // 2
    half_q = dst_bins // 2
    divergence = np.zeros([src_bins // 2 + 1 - dst_bins // 2])
    for i in range(half_q, zero_idx):
        a, b = zero_idx - i, zero_idx + i + 1
        p = distribution[a:b].copy()
        p[0] += sum(distribution[:a])
        p[b - a - 1] = sum(distribution[b:])
        sliced = distribution[a:b].copy()
        nm = sliced.size // dst_bins
        qb = np.zeros([dst_bins])
        for j in range(dst_bins):
            qb[j] = sliced[j * nm : j * nm + nm].sum()
        qb[-1] += sliced[dst_bins * nm :].sum()
        nz = (p != 0).astype(np.int64)
        q = np.zeros(sliced.size, dtype=np.float64)
        for j in range(dst_bins):
            s0 = j * nm
            s1 = -1 if j == dst_bins - 1 else s0 + nm
            norm = nz[s0:s1].sum()
            if norm != 0:
                q[s0:s1] = float(qb[j]) / float(norm)
        q[p == 0] = 0
        p[p == 0] = 0.0001
        q[q == 0] = 0.0001
        divergence[i - dst_bins] = stats.entropy(p, q)
    return bin_width * np.argmin(divergence)


def kl_histogram(batches, bit, bins=2048):
    """observers/kl_histogram.py:130-151 (per-tensor): abs_max, histc(2048, -absmax, absmax),
    entropy threshold; min = -th if any negative else 0."""
    d = layerwise(batches)
    abs_max = np.abs(d).max()
    hist = histc(d, bins, -abs_max, abs_max).astype(F32)
    bin_width = (F32(abs_max) - F32(-abs_max)) / bins
    th = calibrate_entropy(hist, bin_width, bins, 2**bit - 1)
    th = F32(th)
    return (F32(-th) if d.min() < 0 else F32(0)), th
