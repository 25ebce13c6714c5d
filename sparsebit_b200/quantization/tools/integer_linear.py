"""Turn a calibrated model into an integer-inference model: every eligible ``QLinear`` becomes a ``QLinearInt8``
(``to_integer_linears``), every eligible ``QConv2d`` a ``QConv2dInt8`` (``to_integer_convs``)."""
from ..modules import QConv2d, QConv2dInt8, QLinear, QLinearInt8, int8_conv_ineligibility, int8_ineligibility


def to_integer_linears(model):
    """Swap, in place, every ``QLinear`` of ``model`` that ``QLinearInt8.from_qlinear`` accepts; the others stay
    ``QLinear``.  Returns the qualified names of the converted modules, in ``named_modules`` order."""
    targets = [(name, m) for name, m in model.named_modules() if isinstance(m, QLinear) and name]
    converted = []
    for name, m in targets:
        if int8_ineligibility(m) is not None:
            continue
        parent_name, _, attr = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        setattr(parent, attr, QLinearInt8.from_qlinear(m))
        converted.append(name)
    return converted


def to_integer_convs(model):
    """Swap, in place, every ``QConv2d`` of ``model`` that ``QConv2dInt8.from_qconv2d`` accepts; the others stay
    ``QConv2d``.  Returns the qualified names of the converted modules, in ``named_modules`` order."""
    targets = [(name, m) for name, m in model.named_modules() if isinstance(m, QConv2d) and name]
    converted = []
    for name, m in targets:
        if int8_conv_ineligibility(m) is not None:
            continue
        parent_name, _, attr = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        setattr(parent, attr, QConv2dInt8.from_qconv2d(m))
        converted.append(name)
    return converted
