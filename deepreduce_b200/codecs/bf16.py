"""bf16 value codec (``'value': 'bf16'``).

Every shipped value is rounded to bfloat16 (round to nearest, ties to even) and travels as 16 bits; decompress
widens it back to fp32, which is exact.  bf16 keeps fp32's exponent range, so a value never overflows unless it is
within half a bf16 ulp of fp32's largest finite value, and the relative error of a normal value is at most 2^-8
(8 significant bits).  With a residual or 'dgc' memory the rounding error is not lost: ``v - widen(bf16(v))`` is
exact in fp32, and the memories already keep ``v - decompress(compress(v))``.

Wire: ``bfloat16[K]``.  The fused engine ships the same 16-bit words (``parallel/plan.py``, ``VMODE_BF16``); its kernel
rounds a NaN to the quiet NaN 0x7FC0 (``bf16_bits_oracle``), where torch's own cast may give another NaN pattern.
"""
from __future__ import annotations

import torch

from .base import SparseCompressor, register


def bf16_bits_oracle(vals: torch.Tensor) -> torch.Tensor:
    """bf16 bit patterns (int32 in [0, 0xFFFF]) of the fp32 ``vals``, as the fused engine writes them: round to
    nearest, ties to even, in integer arithmetic on the fp32 pattern (a finite value that rounds past the largest
    bf16 becomes +-inf), and every NaN becomes 0x7FC0.  Equal to torch's ``.to(torch.bfloat16)`` bits on every
    non-NaN value."""
    u = vals.detach().float().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    q = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    return torch.where(nan, torch.full_like(q, 0x7FC0), q).to(torch.int32)


def bf16_widen_oracle(bits: torch.Tensor) -> torch.Tensor:
    """fp32 values of bf16 bit patterns (the low 16 bits of ``bits``): exact."""
    w = (bits.to(torch.int64) & 0xFFFF) << 16
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32).view(torch.float32)


@register("bf16")
class BF16(SparseCompressor):
    order_preserving = True
    kind = "value"

    @staticmethod
    def compress(sparse_tensor, params):
        vals, idxs, shape = sparse_tensor
        return vals.float().to(torch.bfloat16), idxs, shape

    @staticmethod
    def decompress(sparse_tensor, params):
        wire, idxs, shape = sparse_tensor
        return wire.float(), idxs, shape
