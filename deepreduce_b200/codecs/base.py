"""Sparse-codec plug-in interface + registry.

Mirrors reference pytorch/deepreduce.py:14-25 (``SparseCompressor``) and the
registry dict ``compressor`` at :913-922.  A codec works on the triple
``(vals, idxs, shape)`` and returns a triple of the same form with one
component replaced by its compressed wire tensor.
"""
from __future__ import annotations

from typing import Dict, Type


class SparseCompressor(object):
    """Interface for compressing and decompressing a given sparse tensor."""

    order_preserving = True   # does decompress return entries in the order compress received them?
    kind = "value"            # "value" | "index"

    @staticmethod
    def compress(sparse_tensor, params):
        """Compress ``(vals, idxs, shape)``; returns a triple of the same form."""
        raise NotImplementedError("compress was not implemented.")

    @staticmethod
    def decompress(sparse_tensor, params):
        """Inverse of compress."""
        raise NotImplementedError("decompress was not implemented.")


compressor: Dict[str, Type[SparseCompressor]] = {}


def register(name: str, *aliases: str):
    """Decorator: ``@register('bloom')`` adds a custom codec to the registry
    (reference README.md:31-34: "...(other custom methods)")."""

    def deco(cls):
        for n in (name,) + aliases:
            compressor[n] = cls
        return cls

    return deco


def use_cuda(t) -> bool:
    """True when the hand-written sm_90a kernels should handle ``t``."""
    if not getattr(t, "is_cuda", False):
        return False
    from .. import ops
    return ops.require()  # raises loudly on a GPU box with a missing extension
