"""Turn a calibrated model into an integer-inference model: every eligible ``QLinear`` becomes a ``QLinearInt8``
(``to_integer_linears``), every eligible ``QConv2d`` a ``QConv2dInt8`` (``to_integer_convs``), every eligible ``QMatMul``
a ``QMatMulInt8`` (``to_integer_matmuls``), every eligible grouped or depthwise ``QConv2d`` a ``QConv2dGroupInt8``
(``to_integer_group_convs``), every eligible ``QAttention`` a ``QAttentionInt8`` (``to_integer_attentions``), and,
opt-in, every ``QLinear`` whose weight is 2:4 sparse on the grid a ``QLinearSparse24Int8``
(``to_sparse24_integer_linears``) and every such ``QConv2d`` a ``QConv2dSparse24Int8`` (``to_sparse24_integer_convs``),
and every ``QLinear`` / ``QConv2d`` with a DoReFa or AdaRound quantizer its integer-grid layer
(``to_integer_dorefa_adaround``)."""
from ..modules import (QAttention, QAttentionInt8, QConv2d, QConv2dGroupInt8, QConv2dInt8, QConv2dSparse24Int8,
                       QLinear, QLinearInt8, QLinearSparse24Int8, QMatMul, QMatMulInt8, dorefa_adaround_ineligibility,
                       from_dorefa_adaround, int8_attention_ineligibility, int8_conv_ineligibility,
                       int8_group_conv_ineligibility, int8_ineligibility, int8_matmul_ineligibility,
                       int8_sparse24_conv_ineligibility, int8_sparse24_ineligibility)


def _swap(model, kind, ineligibility, convert):
    """Replace, in place, every ``kind`` submodule of ``model`` that has no ineligibility reason by ``convert`` of it;
    returns the qualified names of the replaced modules, in ``named_modules`` order."""
    targets = [(name, m) for name, m in model.named_modules() if isinstance(m, kind) and name]
    converted = []
    for name, m in targets:
        if ineligibility(m) is not None:
            continue
        parent_name, _, attr = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        setattr(parent, attr, convert(m))
        converted.append(name)
    return converted


def to_integer_linears(model):
    """Swap, in place, every ``QLinear`` of ``model`` that ``QLinearInt8.from_qlinear`` accepts; the others stay
    ``QLinear``.  Returns the qualified names of the converted modules, in ``named_modules`` order."""
    return _swap(model, QLinear, int8_ineligibility, QLinearInt8.from_qlinear)


def to_integer_convs(model):
    """Swap, in place, every ``QConv2d`` of ``model`` that ``QConv2dInt8.from_qconv2d`` accepts; the others stay
    ``QConv2d``.  Returns the qualified names of the converted modules, in ``named_modules`` order."""
    return _swap(model, QConv2d, int8_conv_ineligibility, QConv2dInt8.from_qconv2d)


def to_integer_matmuls(model):
    """Swap, in place, every ``QMatMul`` of ``model`` that ``QMatMulInt8.from_qmatmul`` accepts; the others stay
    ``QMatMul``.  Returns the qualified names of the converted modules, in ``named_modules`` order."""
    return _swap(model, QMatMul, int8_matmul_ineligibility, QMatMulInt8.from_qmatmul)


def to_integer_group_convs(model):
    """Swap, in place, every grouped or depthwise ``QConv2d`` of ``model`` that ``QConv2dGroupInt8.from_qconv2d``
    accepts; dense convs (groups = 1, see ``to_integer_convs``) and ineligible ones stay ``QConv2d``.  Returns the
    qualified names of the converted modules, in ``named_modules`` order."""
    return _swap(model, QConv2d, int8_group_conv_ineligibility, QConv2dGroupInt8.from_qconv2d)


def to_integer_attentions(model):
    """Swap, in place, every ``QAttention`` of ``model`` that ``QAttentionInt8.from_qattention`` accepts; the others
    stay ``QAttention``.  Run it before ``to_integer_matmuls``, which would otherwise convert the two matmuls of each
    attention separately.  Returns the qualified names of the converted modules, in ``named_modules`` order."""
    return _swap(model, QAttention, int8_attention_ineligibility, QAttentionInt8.from_qattention)


def to_sparse24_integer_linears(model):
    """Swap, in place, every ``QLinear`` of ``model`` that ``QLinearSparse24Int8.from_qlinear`` accepts (its weight 2:4
    sparse on the grid, e.g. pruned by the 2:4 sparser with the mask folded into the weight); the others stay
    ``QLinear``, and ``int8_sparse24_ineligibility`` says why.  Opt-in: the weight format differs from ``QLinearInt8``'s,
    and where the sparse layer beats the dense one depends on the shape.  Run it before ``to_integer_linears``, which
    would otherwise convert the sparse layers to dense ``QLinearInt8``.  Returns the qualified names of the converted
    modules, in ``named_modules`` order."""
    return _swap(model, QLinear, int8_sparse24_ineligibility, QLinearSparse24Int8.from_qlinear)


def to_sparse24_integer_convs(model):
    """Swap, in place, every ``QConv2d`` of ``model`` that ``QConv2dSparse24Int8.from_qconv2d`` accepts (groups = 1, its
    weight 2:4 sparse on the grid along the rows of ``weight.reshape(C_out, -1)``, e.g. pruned by the 2:4 sparser with
    the mask folded into the weight); the others stay ``QConv2d``, and ``int8_sparse24_conv_ineligibility`` says why.
    Opt-in, as ``to_sparse24_integer_linears``: where the sparse conv beats the dense one depends on the layer.  Run it
    before ``to_integer_convs``, which would otherwise convert the sparse convs to dense ``QConv2dInt8``.  Returns the
    qualified names of the converted modules, in ``named_modules`` order."""
    return _swap(model, QConv2d, int8_sparse24_conv_ineligibility, QConv2dSparse24Int8.from_qconv2d)


def to_integer_dorefa_adaround(model):
    """Swap, in place, every ``QLinear`` / ``QConv2d`` of ``model`` that ``from_dorefa_adaround`` accepts: its input
    quantizer is DoReFa, or its weight quantizer DoReFa or AdaRound (the DoReFa and PACT QAT recipes, AdaRound PTQ).
    The others stay, and ``dorefa_adaround_ineligibility`` says why.  Opt-in: the plain converters keep refusing these
    layers, and this one refuses every layer they convert, so the converters can run in any order.  Returns the
    qualified names of the converted modules, in ``named_modules`` order."""
    return _swap(model, (QLinear, QConv2d), dorefa_adaround_ineligibility, from_dorefa_adaround)
