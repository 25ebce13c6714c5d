"""sparsebit_b200 -- H100-native (sm_90a) fake-quantisation / observer / sparser / GPTQ-int4 hot
path behind Sparsebit's own plugin and kernel-module interfaces.

Layout
  include/sparsebit_b200.h            the C-ABI drop-in boundary
  sparsebit_b200/csrc/                hand-written CUDA kernels + the C-ABI (libsparsebit_b200.so)
  sparsebit_b200/_lib.py, ops.py      ctypes binding, tensor-level wrappers
  sparsebit_b200/fake_quant.py        mirror of the reference's ``fake_quant`` pybind module
  sparsebit_b200/gptq/cuda_kernel.py  mirror of the reference's GPTQ ``cuda_kernel`` pybind module
  sparsebit_b200/quantization/        register_quantizer / register_observer plugin classes
  sparsebit_b200/sparse/              register_sparser plugin classes, mask-apply modules
  sparsebit_b200/distributed.py       sharded-calibration statistic all-reduce (NCCL)

There is no CPU or eager fallback: without the built library every op raises.
"""
from ._lib import LIB_PATH, SparsebitB200Error, launch_count  # noqa: F401

__version__ = "0.1.0"


def install():
    """Drop-in mode for an importable, unmodified ``sparsebit``: rebind its native fake-quant
    module to the sm_90a kernels and register the streaming observers / radix-select sparser
    under their reference TYPE / STRATEGY names.  See INTEGRATION.md."""
    import importlib

    from . import fake_quant

    qt = importlib.import_module("sparsebit.quantization.quantizers.quant_tensor")
    qt.fake_quant_kernel = fake_quant
    ref_obs = importlib.import_module("sparsebit.quantization.observers")
    from .quantization import observers as my_obs

    for name in ("minmax", "mse", "percentile", "kl_histogram", "moving_average", "aciq"):
        ref_obs.OBSERVERS_MAP[name] = my_obs.OBSERVERS_MAP[name]
    # The reference's own LSQ / LSQ+ quantizers stay in place and read the calibration batches themselves
    # (data_cache.get_data_for_calibration, lsq.py:36, lsq_plus.py:26): their observers must retain the batches.
    for modname in ("lsq", "lsq_plus"):
        cls = importlib.import_module(f"sparsebit.quantization.quantizers.{modname}").Quantizer
        if not getattr(cls, "_sb200_keep_data", False):
            def _init(self, config, _orig=cls.__init__):
                _orig(self, config)
                self.observer.keep_data = True

            cls.__init__ = _init
            cls._sb200_keep_data = True
    # QuantModel.prepare_calibration imports CalibrationRunner at call time (quant_model.py:185-189)
    ref_cal = importlib.import_module("sparsebit.quantization.tools.calibration")
    from .quantization.tools import CalibrationRunner

    ref_cal.CalibrationRunner = CalibrationRunner
    try:
        ref_sp = importlib.import_module("sparsebit.sparse.sparsers")
        from .sparse import sparsers as my_sp

        ref_sp.SPARSERS_MAP["l1norm"] = my_sp.SPARSERS_MAP["l1norm"]
    except ImportError:
        pass
    return qt
