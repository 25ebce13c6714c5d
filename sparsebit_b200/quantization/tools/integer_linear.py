"""Turn a calibrated model into an integer-inference model: every eligible ``QLinear`` becomes a ``QLinearInt8``."""
from ..modules import QLinear, QLinearInt8, int8_ineligibility


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
