"""``QuantLinear`` for 2 / 3 / 4-bit GPTQ checkpoints (large_language_models/llama/quantization/utils/
quant.py:147-420): same buffers (``qweight`` int32 [rows, N], ``scales`` / ``zeros`` [N, G, 1] with
zeros = zero * scale, ``bias``), same packed layouts, same forward contract -- the 4-bit matmul runs in
``sb200_gptq4_matmul`` (wgmma tensor cores for prefill-sized M, HBM-bound SIMT for decode), 3 / 2-bit in
``sb200_gptq_matmul`` (SIMT)."""
import torch
import torch.nn as nn

from . import cuda_kernel


def find_params(weight, bit=4, groupsize=-1):
    """Asymmetric per-(row, group) grid: GPTQ ``Quantizer.configure(bit, perchannel=True, sym=False,
    mse=False)`` + ``find_params(weight=True)`` (utils/quant.py:43-89,117-124).
    Returns (scale, zero) shaped [N, G, 1] (or [N, 1] when groupsize == -1)."""
    n, k = weight.shape
    groups = 1 if groupsize == -1 else k // groupsize
    x = weight.reshape(n * groups, -1).float()
    lo = torch.clamp(x.min(dim=1).values, max=0)
    hi = torch.clamp(x.max(dim=1).values, min=0)
    dead = (lo == 0) & (hi == 0)
    lo = torch.where(dead, torch.full_like(lo, -1), lo)
    hi = torch.where(dead, torch.full_like(hi, 1), hi)
    scale = (hi - lo) / (2**bit - 1)
    zero = torch.round(-lo / scale)
    shape = (n, groups, 1) if groups > 1 else (n, 1)
    return scale.reshape(shape), zero.reshape(shape)


def _bit_positions(bit, k_padded):
    """(word row, shift) of the LSB of every input channel, plus the straddle spill, for
    QuantLinear.pack (utils/quant.py:210-258).  2/4-bit: 32/bit values per word.  3-bit: 32 values per
    3 words, value 10 at bits 30-31 of word 0 + bit 0 of word 1, value 21 at bit 31 of word 1 + bits
    0-1 of word 2."""
    k = torch.arange(k_padded, dtype=torch.int64)
    if bit in (2, 4):
        per = 32 // bit
        return k // per, (k % per) * bit
    unit, j = k // 32, k % 32
    word = torch.where(j <= 10, 0, torch.where(j <= 21, 1, 2))
    shift = torch.where(j <= 10, 3 * j, torch.where(j <= 21, 3 * (j - 11) + 1, 3 * (j - 22) + 2))
    return unit * 3 + word, shift


def pack_rows(infeatures, bit):
    """Rows of ``qweight``: ceil(K*bit / (32*p)) * p with p = 3 for 3-bit (utils/quant.py:172-184)."""
    p = 3 if bit == 3 else 1
    return -(-infeatures * bit // (32 * p)) * p


def pack_intweight(q, bit):
    """q: int64 [K, N] values in [0, 2^bit) -> int32 [rows, N] in the reference's packed layout.  Runs on
    q's device (the full-size reference test shapes, 12288 x 49152, are packed on the GPU)."""
    k, n = q.shape
    rows = pack_rows(k, bit)
    per_unit = {2: 16, 3: 32, 4: 8}[bit]
    k_padded = -(-k // per_unit) * per_unit
    if k_padded != k:
        padded = torch.zeros(k_padded, n, dtype=torch.int64, device=q.device)
        padded[:k] = q
    else:
        padded = q
    if bit in (2, 4):  # no straddling values: word r = sum_j q[per*r + j] << (bit*j)
        words = torch.zeros(rows, n, dtype=torch.int64, device=q.device)
        v = padded.view(rows, per_unit, n)
        for j in range(per_unit):
            words |= v[:, j, :] << (bit * j)
    else:
        row, shift = _bit_positions(bit, k_padded)
        row, shift = row.to(q.device), shift.to(q.device)
        words = torch.zeros(rows + 1, n, dtype=torch.int64, device=q.device)  # +1: spill row of a straddler in the last unit
        shifted = padded << shift.view(-1, 1)
        words.index_add_(0, row, shifted & 0xFFFFFFFF)
        words.index_add_(0, row + 1, shifted >> 32)  # the straddling high bits
        words = words[:rows] & 0xFFFFFFFF
    words = torch.where(words >= 2**31, words - 2**32, words)
    return words.to(torch.int32)


def find_params_int4(weight, groupsize=-1):
    return find_params(weight, 4, groupsize)


def _input_grad(ctx, grad):
    """dL/dinput = grad @ dequant(qweight) through sb200_gptq_matmul_dgrad; None (and no launch) when the input does not
    need it.  qweight / scales / zeros are frozen buffers: they never get a gradient."""
    if not ctx.needs_input_grad[0]:
        return None
    from .. import ops

    qweight, scales, zeros = ctx.saved_tensors
    dev = ctx.dev
    g = grad.to(device=dev, dtype=torch.float32).contiguous()
    gi = torch.zeros(ctx.in_shape, dtype=torch.float32, device=dev)
    ops.gptq_matmul_dgrad(g, qweight.to(dev), gi, scales.to(dev).contiguous(), zeros.to(dev).contiguous(), ctx.bit,
                          0 if ctx.groupsize == -1 else int(ctx.groupsize))
    return gi.to(device=ctx.in_device, dtype=ctx.in_dtype)


class QuantMatmul(torch.autograd.Function):
    """Quant{2,3,4}Matmul (utils/quant.py:281-420): y = bias broadcast, then the kernel accumulates
    x @ W^T in place.  The backward returns the input gradient (sb200_gptq_matmul_dgrad); the weights are frozen."""

    @staticmethod
    def forward(ctx, input, qweight, scales, zeros, bias, groupsize=-1, bit=4):
        lead = list(input.shape[:-1])
        was_cuda = input.is_cuda
        dev = input.device if was_cuda else torch.device("cuda")
        # references, not copies: a weight overwritten in place before backward raises autograd's version-counter error
        ctx.save_for_backward(qweight, scales, zeros)
        ctx.dev, ctx.in_shape, ctx.in_device, ctx.in_dtype = dev, input.shape, input.device, input.dtype
        ctx.groupsize, ctx.bit = groupsize, bit
        x = input.to(dev).contiguous()
        # a private copy (the reference uses .repeat): expand(...).contiguous() of a [1, N] view would alias the
        # bias buffer itself and the in-place accumulation below would corrupt it
        y = bias.to(device=dev, dtype=x.dtype).expand(lead + [bias.numel()]).clone(memory_format=torch.contiguous_format)
        plain = {2: cuda_kernel.vecquant2matmul, 3: cuda_kernel.vecquant3matmul, 4: cuda_kernel.vecquant4matmul}[bit]
        grouped = {2: cuda_kernel.vecgroupquant2matmul, 3: cuda_kernel.vecgroupquant3matmul,
                   4: cuda_kernel.vecgroupquant4matmul}[bit]
        args = (x, qweight.to(dev), y, scales.to(dev).contiguous(), zeros.to(dev).contiguous())
        if groupsize == -1:
            plain(*args)
        else:
            grouped(*args, groupsize)
        return y if was_cuda else y.cpu()

    @staticmethod
    def backward(ctx, grad):
        return (_input_grad(ctx, grad),) + (None,) * 6


class Quant4Matmul(QuantMatmul):
    @staticmethod
    def forward(ctx, input, qweight, scales, zeros, bias, groupsize=-1):
        return QuantMatmul.forward(ctx, input, qweight, scales, zeros, bias, groupsize, 4)

    @staticmethod
    def backward(ctx, grad):
        return (_input_grad(ctx, grad),) + (None,) * 5


class QuantLinear(nn.Module):
    def __init__(self, infeatures, outfeatures, bit=4, groupsize=-1):
        super().__init__()
        assert bit in [2, 3, 4], "only support 2/3/4 bit now"
        if groupsize != -1:
            assert groupsize % {4: 128, 3: 128, 2: 64}[bit] == 0
            assert infeatures % groupsize == 0
        self.infeatures, self.outfeatures = infeatures, outfeatures
        self.bit, self.groupsize = bit, groupsize
        self.groups = 1 if groupsize == -1 else infeatures // groupsize
        qshape = (outfeatures, self.groups, 1) if self.groups > 1 else (outfeatures, 1)
        self.register_buffer("zeros", torch.zeros(qshape))
        self.register_buffer("scales", torch.zeros(qshape))
        self.register_buffer("bias", torch.zeros(outfeatures))
        self.register_buffer("qweight", torch.zeros((pack_rows(infeatures, bit), outfeatures), dtype=torch.int32))

    @torch.no_grad()
    def pack(self, linear, scales, zeros):
        """utils/quant.py:187-260: intweight = round((w + zero*scale) / scale), packed LSB first along K
        (see ``_bit_positions``)."""
        self.zeros = (zeros * scales).to(self.zeros.dtype)
        self.scales = scales.clone()
        self.bias = linear.bias.clone() if linear.bias is not None else torch.zeros(self.outfeatures)
        w = linear.weight.data.float()  # packs on the weight's device (CPU like the reference, or the GPU)
        z, s = self.zeros.float().to(w.device), self.scales.float().to(w.device)
        if self.groups > 1:
            q = torch.round((w.view(self.outfeatures, self.groups, -1) + z) / s).view(self.outfeatures, self.infeatures)
        else:
            q = torch.round((w + z) / s)
        self.qweight = pack_intweight(q.to(torch.int64).t().contiguous(), self.bit)

    def forward(self, x):
        if self.bit == 4 and x.is_cuda and x.dtype == torch.float16 and self.qweight.is_cuda and not torch.is_grad_enabled():
            # the model path (fp16 activations): one library call, no per-call casts of x / scales / zeros / bias and no
            # fp32 copy of the result (the reference casts all of them every forward, utils/quant.py:262-278)
            from .. import ops

            fresh = getattr(self, "_f32_tables", None) is None or self._f32_tables[0].device != x.device
            if fresh:
                self._f32_tables = (self.scales.float().contiguous().to(x.device), self.zeros.float().contiguous().to(x.device),
                                    self.bias.float().contiguous().to(x.device))
            sc, zr, bs = self._f32_tables
            # the buffers of a loaded model are constants (SB200_GPTQ4_STATIC_WEIGHTS) -- except in the call that has
            # just produced the fp32 tables with the kernels immediately in front of this one
            return ops.gptq4_linear_f16(x.contiguous(), self.qweight, sc, zr, bs, 0 if self.groupsize == -1 else self.groupsize,
                                        static_weights=not fresh)
        # fp32 math like the reference (utils/quant.py:262-278), result cast back to x.dtype
        y = QuantMatmul.apply(x.float(), self.qweight, self.scales.float(), self.zeros.float(), self.bias.float(),
                              self.groupsize, self.bit)
        return y.to(x.dtype)


def make_quant(module, layers_bit, name="", groupsize=-1):
    """Swap ``nn.Linear`` children named in ``layers_bit`` for ``QuantLinear`` (utils/quant.py:422-445)."""
    if isinstance(module, QuantLinear):
        return
    for attr, child in list(module.named_children()):
        full = f"{name}.{attr}" if name else attr
        if full in layers_bit and isinstance(child, nn.Linear):
            setattr(module, attr, QuantLinear(child.in_features, child.out_features, bit=layers_bit[full], groupsize=groupsize))
        else:
            make_quant(child, layers_bit, full, groupsize)
