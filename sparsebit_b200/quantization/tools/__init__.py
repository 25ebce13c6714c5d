from .calibration import CalibrationRunner, trace_quant_model  # noqa: F401
from .integer_linear import (to_integer_attentions, to_integer_convs, to_integer_dorefa_adaround,  # noqa: F401
                             to_integer_group_convs, to_integer_linears, to_integer_matmuls, to_sparse24_integer_convs,
                             to_sparse24_integer_linears)
