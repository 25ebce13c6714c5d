"""``STRATEGY = "l1norm"`` (sparsebit/sparse/sparsers/l1norm.py:14-42).

unstructed: the reference fully sorts |w| to read ONE order statistic (``sorted[min(int(n*ratio),
n-1)]``) and masks ``|w| > thresh`` (strict: ties at the threshold are pruned, Q12).  Here the
threshold is the exact k-th smallest |w| from a 3-pass radix select on the device
(``sb200_select_*`` with key = |x|) followed by ``sb200_mask_gt`` -- same element, same mask, no
sort.  structed (:27-40): the per-filter L1 norms are one pass of the row-moments kernel (``sb200_observe_moments``,
fp64 sums), the cut is the exact (pruned - 1)-th smallest norm from the same radix select, and the float mask is
written by ``sb200_mask_rows_gt`` -- no ``abs().sum()`` / ``torch.sort`` / per-index CPU round trips.  The ranking
equals the reference's whenever two filters' norms differ by more than its fp32 summation error; filters that tie
with the cut are pruned together.  2:4 (not in the reference): every aligned group of 4 along a row of
``w.reshape(C_out, -1)`` keeps its two largest |w| (``sb200_sparse24_mask``), the pattern the sparse tensor cores run;
RATIO is 0 (all ones) or 0.5.
"""
import torch

from ... import ops
from . import Sparser as BaseSparser
from . import register_sparser


@register_sparser
class Sparser(BaseSparser):
    STRATEGY = "l1norm"

    def calc_mask(self, x):
        if self.ratio == 0.0:
            return torch.ones_like(x)
        if self.type == "2:4" and self.ratio != 0.5:
            raise ValueError(f"the 2:4 sparser prunes half of every group of 4: RATIO must be 0 or 0.5, got {self.ratio}")
        w = x.detach()
        if not w.is_cuda:
            if not torch.cuda.is_available():
                raise ops.SparsebitB200Error("sparsebit_b200 sparsers need a CUDA device (no CPU fallback)")
            w = w.cuda()
        w = w.float().contiguous()
        if self.type == "unstructed":
            n = w.numel()
            k = min(int(n * self.ratio), n - 1)
            thresh = ops.kth_value(w.reshape(-1), k, key_mode=1)
            mask = ops.mask_gt(w, thresh)
        elif self.type == "2:4":
            mask = ops.sparse24_mask(w)
        elif self.type == "structed":
            pruned = int(w.shape[0] * self.ratio)
            if pruned == 0:
                return torch.ones_like(x)
            rows = w.reshape(w.shape[0], -1)
            l1 = ops.moments_update(rows, ops.moments_new(rows.shape[0], w.device))[:, 2].to(torch.float32).contiguous()
            thresh = ops.kth_value(l1, pruned - 1, key_mode=0)
            mask = ops.mask_rows_gt(l1, thresh, w.shape)
        else:
            raise NotImplementedError(self.type)
        return mask.to(x.device)
