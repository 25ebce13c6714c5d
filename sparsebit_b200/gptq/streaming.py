"""Layer-streaming execution of a stack of GPTQ decoder layers -- the ``single_device_mode`` of the reference's LLaMA
wrapper (large_language_models/llama/quantization/utils/llama_wrapper.py:848-924): the packed ``qweight`` of every
``QuantLinear`` lives in (pinned) host memory and is copied to the GPU only for the layer that is about to run, on a
side stream, while the previous layer computes.

What differs from the reference:
* two fixed device slots per weight shape are reused round-robin (the reference allocates fresh device tensors with
  ``.to(cuda)`` for every layer of every forward and relies on the caching allocator);
* the host copies are pinned once, so the H2D copies are truly asynchronous (``.to(cuda)`` from pageable memory, as
  the reference does it, serialises with the host);
* readiness / reuse is tracked with CUDA events per slot instead of three new streams per layer.
scales / zeros / bias stay resident like in the reference (they are 1/8 of the packed weights).  On an 80 GB H100 a
7B ... 65B int4 model fits entirely (65B: 33 GB of packed weights), so this is for models beyond HBM or for sharing the GPU; it is part of the
reference's inference path (SURVEY 8f #3) and kept behaviour-compatible: same outputs as the resident execution."""
import torch

from .quant_linear import QuantLinear


class LayerStreamer:
    def __init__(self, layers, device=None, slots=2):
        self.layers = list(layers)
        self.device = torch.device(device or "cuda")
        self.slots = max(2, int(slots))
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self._linears = [[m for m in layer.modules() if isinstance(m, QuantLinear)] for layer in self.layers]
        # host side: pinned copies of every packed weight; the modules keep their small tables resident
        self._host = []
        for layer, linears in zip(self.layers, self._linears):
            host = []
            for m in linears:
                h = m.qweight.detach().to("cpu").contiguous()
                host.append(h.pin_memory() if torch.cuda.is_available() else h)
                m.qweight = torch.empty(0, dtype=torch.int32, device=self.device)  # nothing resident until the layer runs
            self._host.append(host)
            for m in layer.modules():
                if not isinstance(m, QuantLinear):
                    m.to(self.device)
                else:
                    m.scales, m.zeros, m.bias = m.scales.to(self.device), m.zeros.to(self.device), m.bias.to(self.device)
                    m._f32_tables = None
        # device side: `slots` buffers per linear position, sized for the largest weight at that position
        npos = max((len(h) for h in self._host), default=0)
        self._dev = []
        for s in range(self.slots):
            bufs = []
            for p in range(npos):
                numel = max(h[p].numel() for h in self._host if len(h) > p)
                bufs.append(torch.empty(numel, dtype=torch.int32, device=self.device))
            self._dev.append(bufs)
        self._ready = [torch.cuda.Event() for _ in range(self.slots)]  # H2D of the slot's current layer finished
        self._free = [torch.cuda.Event() for _ in range(self.slots)]   # compute that read the slot finished
        for e in self._free:
            e.record(torch.cuda.current_stream(self.device))

    def resident_bytes(self):
        return sum(b.numel() * 4 for bufs in self._dev for b in bufs)

    def _prefetch(self, idx):
        slot = idx % self.slots
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self._free[slot])  # the layer that last used this slot has finished computing
            for p, h in enumerate(self._host[idx]):
                self._dev[slot][p][: h.numel()].view(h.shape).copy_(h, non_blocking=True)
            self._ready[slot].record(self.copy_stream)

    def _bind(self, idx):
        slot = idx % self.slots
        for p, (m, h) in enumerate(zip(self._linears[idx], self._host[idx])):
            m.qweight = self._dev[slot][p][: h.numel()].view(h.shape)

    def _unbind(self, idx):
        for m in self._linears[idx]:
            m.qweight = torch.empty(0, dtype=torch.int32, device=self.device)

    def forward(self, hidden, layer_fn=None):
        """Run ``hidden`` through all layers (``layer_fn(layer, hidden)`` defaults to ``layer(hidden)``)."""
        call = layer_fn or (lambda layer, h: layer(h))
        compute = torch.cuda.current_stream(self.device)
        n = len(self.layers)
        for i in range(min(self.slots - 1, n)):
            self._prefetch(i)
        for idx in range(n):
            if idx + self.slots - 1 < n:
                self._prefetch(idx + self.slots - 1)  # next layer's copy overlaps this layer's compute
            compute.wait_event(self._ready[idx % self.slots])
            self._bind(idx)
            hidden = call(self.layers[idx], hidden)
            self._free[idx % self.slots].record(compute)
            self._unbind(idx)
        return hidden

    __call__ = forward
