"""The reference's own CPU path, op for op, as it runs when tensors live on the CPU -- a chain of
ATen elementwise ops (sparsebit/quantization/quantizers/quant_tensor.py:181-184), torch.min/max
(observers/minmax.py:22) and ``weight * w_mask`` (sparse/modules/conv.py:40).

TEST / BASELINE INFRASTRUCTURE ONLY: ``bench.py`` times these functions on the GPU machine's host
cores (``cpu_baseline`` and ``--impl reference``), where the reference itself need not be installed.  Validated bit-for-bit against the unmodified reference through the
golden vectors (tests/test_oracle_golden.py::test_torch_port_matches_reference).
"""
import torch


def ort_fake_quant_cpu(x_f, scale, zero_point, qmin, qmax):
    zp = zero_point.round()
    x_q = torch.clamp((x_f / scale).round() + zp, qmin, qmax)
    return (x_q - zp) * scale


def minmax_cpu(x):
    return x.min(), x.max()


def mask_apply_cpu(weight, mask):
    return weight * mask


# ------------------------------------------------------------------------------------------------------------
# Observer / sparser CPU paths of the reference as torch op chains (per-tensor forms), for bench.py's
# ``cpu_baselines`` (BASELINE.md section 3.1).  Same ops in the same order as the cited lines; pinned to the
# reference's outputs through tests/golden/observers.npz and sparse.npz (tests/test_oracle_golden.py).
def calc_qparams_with_minmax_cpu(min_val, max_val, qmin, qmax, symmetric):
    """observers/base.py:63-79."""
    min_val_neg = torch.min(min_val, torch.zeros_like(min_val))
    max_val_pos = torch.max(max_val, torch.zeros_like(max_val))
    if symmetric:
        max_val_pos = torch.max(-min_val_neg, max_val_pos)
        scale = max_val_pos * 2 / float(qmax - qmin)
        zero_point = torch.zeros(max_val_pos.size())
    else:
        scale = (max_val_pos - min_val_neg) / float(qmax - qmin)
        zero_point = torch.round(-min_val_neg / scale)
    return torch.max(scale, torch.tensor(1e-6)), zero_point


def minmax_observer_cpu(batches):
    """observers/base.py:28 (torch.cat of the cached batches) + minmax.py:22-25, layer-wise."""
    data = torch.cat([b.reshape(-1) for b in batches], dim=0)
    return data.min(), data.max()


def mse_observer_cpu(batches, qmin, qmax, symmetric, steps=80):
    """observers/mse.py:28-63, per tensor: 80 clipping candidates, each a full QDQ (the CPU branch of
    ort_fake_quant, quant_tensor.py:181-184) and a mean squared error (observers/utils.py:1-5)."""
    x_f = torch.cat([b.reshape(-1) for b in batches], dim=0).reshape(1, -1)
    min_val, max_val = x_f.min(), x_f.max()
    best, loss_min = None, 1e10
    for i in range(steps):
        scale, zero_point = calc_qparams_with_minmax_cpu(min_val * (1.0 - (i * 0.01)), max_val * (1.0 - (i * 0.01)), qmin, qmax, symmetric)
        x_dq = ort_fake_quant_cpu(x_f, scale, zero_point, qmin, qmax)
        loss = ((x_f - x_dq) ** 2).mean()
        if loss < loss_min:
            loss_min, best = loss, (scale, zero_point)
    return best


def percentile_observer_cpu(batches, alpha):
    """observers/percentile.py:16-46, per tensor: two torch.kthvalue calls on the concatenated data."""
    data = torch.cat([b.reshape(-1) for b in batches], dim=0)
    neg_length, pos_length = int((data < 0).sum()), int((data >= 0).sum())
    max_val = torch.kthvalue(data, data.numel() - max(round(pos_length * alpha), 0)).values if pos_length > 0 else torch.zeros(())
    min_val = torch.kthvalue(data, max(round(neg_length * alpha), 1)).values if neg_length > 0 else torch.zeros(())
    return min_val, max_val


def kl_observer_cpu(batches, bit, bins=2048):
    """observers/kl_histogram.py:47-50,131-147, per tensor: abs-max, torch.histc, then the entropy search
    (calibrate_entropy :54-94, restated index-exactly in oracle/observers.py)."""
    from . import observers as oobs

    data = torch.cat([b.reshape(-1) for b in batches], dim=0)
    abs_max = data.abs().max()
    hist = torch.histc(data, bins=bins, min=float(-abs_max), max=float(abs_max))
    bin_width = (abs_max - (-abs_max)) / bins
    th = oobs.calibrate_entropy(hist.numpy(), float(bin_width), bins, 2**bit - 1)
    return (-th if bool(data.min() < 0) else 0.0), th


def l1_unstructured_mask_cpu(w, ratio):
    """sparse/sparsers/l1norm.py:17-26: full sort of |w| for one order statistic, strict > mask."""
    data = torch.abs(w.detach()).flatten()
    sorted_data, _ = torch.sort(data)
    thresh = sorted_data[min(int(data.numel() * ratio), data.numel() - 1)]
    return (data > thresh).reshape(w.shape)
