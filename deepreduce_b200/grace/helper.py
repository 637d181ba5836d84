"""``grace_from_params`` / ``tensor_bits`` (GRACE helper contract, SURVEY §2.5;
used by the reference at pytorch/deepreduce.py:8,29,94-95)."""
from __future__ import annotations

from typing import Iterable

import torch

from .communicators import Allgather, Allreduce
from .memory import DgcMemory, NoneMemory, ResidualMemory
from .sparsifiers import NoneCompressor, RandomKCompressor, ThresholdCompressor, TopKCompressor

_BITS = {torch.float64: 64, torch.int64: 64, torch.float32: 32, torch.int32: 32,
         torch.float16: 16, torch.bfloat16: 16, torch.int16: 16, torch.uint8: 8,
         torch.int8: 8, torch.bool: 8}


def tensor_bits(tensors: Iterable) -> int:
    """Σ numel · bit-width over a list of wire tensors (tuples are flattened —
    ``polyfit_cpu`` ships a tuple, reference pytorch/deepreduce.py:672-675)."""
    total = 0
    for t in tensors:
        if isinstance(t, (tuple, list)):
            total += tensor_bits(t)
        elif torch.is_tensor(t):
            total += t.numel() * _BITS.get(t.dtype, t.element_size() * 8)
    return total


def sparsifier_of(grc):
    """The sparsifier of a GRACE communicator, under the DeepReduce codec wrapper if there is one."""
    return getattr(grc.compressor, "sparsifier", grc.compressor)


def grace_from_params(params: dict):
    """Build ``Communicator(compressor, memory)`` from the GRACE params dict
    (reference README.md:36-38)."""
    comp = params.get('compressor', 'none')
    mem = params.get('memory', 'none')
    comm = params.get('communicator', 'allreduce')
    world_size = params.get('world_size', None)
    average = params.get('average', True)

    from ..config import warmup_from_params
    warmup = warmup_from_params(params)
    if comp == 'topk':
        compressor = TopKCompressor(params.get('compress_ratio', 0.01), average=average, warmup=warmup)
    elif comp == 'threshold':
        compressor = ThresholdCompressor(params.get('threshold', 0.0), average=average)
    elif comp == 'randomk':
        compressor = RandomKCompressor(params.get('compress_ratio', 0.01), average=average, warmup=warmup)
    elif comp in ('none', None):
        compressor = NoneCompressor(average=average)
    elif comp in ('SKCompressCPU', 'SKCompressGPU', 'sketch'):
        raise NotImplementedError(
            f"compressor '{comp}' is a comparison baseline from a GRACE fork and is out of scope (SURVEY §2.5)")
    else:
        raise ValueError(f"unknown compressor '{comp}'")

    if mem == 'residual':
        memory = ResidualMemory(params.get('beta', 1.0), params.get('gamma', 1.0))
    elif mem == 'dgc':
        import torch.distributed as dist
        memory = DgcMemory(params.get('momentum', 0.9), params.get('weight_decay', 0.0), params.get('clip_norm'),
                           dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1,
                           nesterov=params.get('nesterov', False),
                           weight_decay_exclude=params.get('weight_decay_exclude', ()))
    elif mem in ('none', None):
        memory = NoneMemory()
    else:
        raise ValueError(f"unknown memory '{mem}'")

    if comm == 'allgather':
        return Allgather(compressor, memory, world_size)
    if comm == 'allreduce':
        return Allreduce(compressor, memory, world_size)
    raise ValueError(f"unknown communicator '{comm}'")
