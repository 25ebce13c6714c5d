"""Sparser plugin contract (the interface sparsebit/sparse/sparsers/base.py:6-25 exposes to SparseOpr):
a module built from ``(config, opr)`` that turns a weight into a keep-mask via ``calc_mask``; the owning
operator multiplies by that mask on every forward."""
from torch import nn

_KNOWN_TYPES = ("unstructed", "structed", "2:4")  # the reference's two config values, and 2:4 (N:M) sparsity


class Sparser(nn.Module):
    STRATEGY = "base"

    def __init__(self, config, opr):
        super().__init__()
        sparser_cfg = config.SPARSER
        self.config = config
        # The owning operator registers this sparser as a submodule; registering the operator back as a submodule
        # of the sparser would make the module tree cyclic (eval() / to() / state_dict() recurse forever).  The
        # reference passes a repr string here (sparse/modules/base.py:23-24); keep the object, unregistered.
        object.__setattr__(self, "opr", opr)
        self.type, self.strategy = sparser_cfg.TYPE, sparser_cfg.STRATEGY
        self.set_ratio(sparser_cfg.RATIO)

    # -- plugin hook ---------------------------------------------------------------------------
    def calc_mask(self, x):
        """Return a tensor shaped like ``x``: nonzero = keep.  Implemented by the registered strategies."""
        raise NotImplementedError(f"{type(self).__name__} does not implement calc_mask")

    # -- knobs the pruning schedules of the reference drive ---------------------------------------
    def set_ratio(self, ratio):
        ratio = float(ratio)
        if not 0.0 <= ratio <= 1.0:
            raise ValueError(f"sparsity ratio must be in [0, 1], got {ratio}")
        self.ratio = ratio

    @property
    def is_structured(self):
        return self.type == _KNOWN_TYPES[1]

    def __repr__(self):
        return ", ".join(str(v) for v in (self.type, self.strategy, self.ratio))
