"""Sparsifiers (GRACE ``compressor`` key): topk / threshold / randomk / none.

Contracts per SURVEY §2.5: wire tensors are ``(values fp32, indices int64)``,
ctx is the ``torch.Size`` (the reference calls ``ctx.numel()``,
pytorch/deepreduce.py:64-68), decompress = zeros + scatter.
On CUDA tensors the selection runs through the hand-written radix-select
kernel (``ops.topk_select``); on CPU it is plain torch.
"""
from __future__ import annotations

import torch

from .. import spec
from .base import Compressor


def _desparsify(tensors, shape: torch.Size) -> torch.Tensor:
    values, indices = tensors
    out = torch.zeros(shape.numel(), dtype=values.dtype, device=values.device)
    # index_add_, not scatter_: a sparsifier that found fewer than K non-zeros pads with (index 0, value 0.0); adding
    # zeros is exact and order-independent, while scatter_ with duplicate indices is nondeterministic
    out.index_add_(0, indices.long(), values)
    return out.view(shape)


class NoneCompressor(Compressor):
    """``'compressor': 'none'`` — dense baseline (reference run_deepreduce.sh:51)."""

    def compress(self, tensor, name):
        return [tensor], None

    def decompress(self, tensors, ctx):
        return tensors[0]


class _Scheduled:
    """The sparsity warm-up of a ratio sparsifier (``spec.Warmup``, or None: ``compress_ratio`` throughout).  A bare
    ``grc.step(grad, name)`` has no other step counter, so the exchanges are counted per tensor name: a tensor that
    gets no gradient on some step falls behind in its count by that step."""

    def _init_warmup(self, compress_ratio, warmup):
        self.compress_ratio = compress_ratio
        self.warmup = warmup
        self.exchanges: dict = {}

    def _ratio(self, name) -> float:
        if self.warmup is None:
            return self.compress_ratio
        e = self.exchanges.get(name, 0)
        self.exchanges[name] = e + 1
        return self.warmup.ratio_at(e)

    def state_dict(self) -> dict:
        return {"exchanges": dict(self.exchanges)}

    def load_state_dict(self, state: dict) -> None:
        self.exchanges = {k: int(v) for k, v in state.get("exchanges", {}).items()}


class TopKCompressor(_Scheduled, Compressor):
    def __init__(self, compress_ratio: float = 0.01, average: bool = True, warmup: spec.Warmup | None = None):
        super().__init__(average=average, tensors_size_are_same=True)
        self._init_warmup(compress_ratio, warmup)

    def compress(self, tensor, name):
        flat = tensor.flatten()
        k = spec.topk_k(flat.numel(), self._ratio(name))
        if flat.is_cuda:
            from .. import ops
            values, indices = ops.topk_select(flat, k)
        else:
            _, indices = torch.topk(flat.abs(), k, sorted=False)
            values = flat[indices]
        return (values, indices), tensor.size()

    def decompress(self, tensors, ctx):
        return _desparsify(tensors, ctx)


class ThresholdCompressor(Compressor):
    """All entries with |x| > threshold (``threshold: 0.0`` ⇒ all non-zeros;
    used for inherently sparse NCF gradients, reference run_deepreduce.sh:66)."""

    def __init__(self, threshold: float = 0.0, average: bool = True):
        super().__init__(average=average, tensors_size_are_same=False)
        self.threshold = threshold

    def compress(self, tensor, name):
        flat = tensor.flatten()
        indices = torch.nonzero(flat.abs() > self.threshold, as_tuple=False).flatten()
        values = flat[indices]
        return (values, indices), tensor.size()

    def decompress(self, tensors, ctx):
        return _desparsify(tensors, ctx)


class RandomKCompressor(_Scheduled, Compressor):
    """Uniform random K coordinates, the same on every rank for a given
    (step, name) — TF twin: tensorflow/deepreduce.py:290-298."""

    def __init__(self, compress_ratio: float = 0.01, average: bool = True, seed: int = 1,
                 warmup: spec.Warmup | None = None):
        super().__init__(average=average, tensors_size_are_same=True)
        self._init_warmup(compress_ratio, warmup)
        self.seed = seed
        self.global_step = 0

    def compress(self, tensor, name):
        flat = tensor.flatten()
        d = flat.numel()
        k = spec.topk_k(d, self._ratio(name))
        tid = sum(name.encode()) if isinstance(name, str) else int(name)
        seed = spec.policy_seed(self.global_step + self.seed, tid)
        self.global_step += 1
        keys = spec.policy_hash(torch.arange(d, device=flat.device), seed)
        # K smallest keys, ties broken by index: sort on (key << 32 | idx)
        comp = (keys << 31) | torch.arange(d, device=flat.device)
        indices = torch.sort(comp).values[:k] & 0x7FFFFFFF
        indices = torch.sort(indices).values
        return (flat[indices], indices), tensor.size()

    def decompress(self, tensors, ctx):
        return _desparsify(tensors, ctx)
