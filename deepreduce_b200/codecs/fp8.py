"""FP8 value codec (``'value': 'fp8'``): E4M3 values with a power-of-two scale byte per block of 32 (the OCP MXFP8
layout, with the scale rounded up instead of down).

The shipped values, in ascending index order, are cut into blocks of 32; the last block may be short.  For each block:

* A is the largest ``bits(v) & 0x7FFFFFFF`` over the block (an integer max).
* A >= 0x7F800000 (an inf or a NaN in the block): the scale byte is 0xFF, every element byte 0x00, and every value of
  the block decodes to NaN.  The other blocks are unaffected.
* Otherwise the block exponent e is the smallest integer with float(A) * 2^-e <= 448 (E4M3's largest finite value),
  clamped below at -127.  For a normal a = m * 2^E with m in [1, 2) that is E - 8 if m <= 1.75, else E - 7; for 0 and
  fp32 subnormals it is -127.  The scale byte is e + 127 (at most 247).  OCP's floor(log2 a) - 8 can clip the block
  maximum by up to 12.5 %; rounding the scale up means no element saturates, so the bytes differ from OCP's on blocks
  whose maximum has m > 1.75.
* Element byte: q = RNE_E4M3(v * 2^-e), the E4M3 "fn" code (no inf, largest 448; -0.0 ships 0x80).  v * 2^-e is exact in
  fp32 wherever it can round to a non-zero code, and |v * 2^-e| <= 448, so nothing saturates.
* Decode: d = widen(q) * 2^e in fp32, exact (at most 4 significant bits, the lowest at 2^-136 or above), except that
  a block maximum of at least 1.9375 * 2^127 can round up to 2^128 and decode to inf.

Where ``|v| * 2^-e >= 2^-6`` (E4M3's normal range), ``|v - d| <= 2^-4 |v|``; elsewhere ``|v - d| <= 2^(e - 10)``.
The residual and 'dgc' memories keep ``v - d`` where d is finite (0 where it is not); 'dgc' clears the momentum where
``d != 0``, so a value that rounds to zero keeps both.

Wire: ``int32[1 + ceil(K/128) + ceil(K/4)]``: K, the scale bytes, then the element bytes, each packed four per word
(byte p in bits 8 (p % 4) of word p // 4, zero-padded).  K travels because 'both' decodes without the index list.  In
'value' mode compress first puts the pairs in ascending index order, so its blocks are the fused engine's
(``parallel/plan.py`` ``VMODE_FP8``); in 'both' they already arrive in the index codec's ascending order.  CUDA tensors
are coded by the sm_90a kernels (``ops.fp8_encode`` / ``ops.fp8_decode``), CPU tensors by the torch reference below;
both give the same words.
"""
from __future__ import annotations

import torch

from .base import SparseCompressor, register, use_cuda

FP8_BLOCK = 32
FP8_NONFINITE = 0xFF          # scale byte of a block holding an inf or a NaN


def fp8_scale_bytes(vals: torch.Tensor) -> torch.Tensor:
    """int64[ceil(K/32)]: the scale byte of every block of the fp32 ``vals``, from the integer exponent rule."""
    v = vals.detach().float().reshape(-1)
    K = v.numel()
    nb = (K + FP8_BLOCK - 1) // FP8_BLOCK
    x = torch.zeros(nb * FP8_BLOCK, dtype=torch.float32, device=v.device)
    x[:K] = v
    A = (x.view(torch.int32).to(torch.int64) & 0x7FFFFFFF).view(nb, FP8_BLOCK).amax(dim=1) if nb else \
        torch.zeros(0, dtype=torch.int64, device=v.device)
    E8, m = A >> 23, A & 0x7FFFFF
    s = torch.where(m <= 0x600000, E8 - 8, E8 - 7).clamp(min=0)
    s = torch.where(E8 == 0, torch.zeros_like(s), s)
    return torch.where(A >= 0x7F800000, torch.full_like(s, FP8_NONFINITE), s)


def _pack_bytes(b: torch.Tensor) -> torch.Tensor:
    """int32[ceil(n/4)] of the bytes ``b`` (values 0..255), byte p in bits 8 (p % 4) of word p // 4, zero-padded."""
    n = b.numel()
    nw = (n + 3) // 4
    w = torch.zeros(nw * 4, dtype=torch.int64, device=b.device)
    w[:n] = b.to(torch.int64)
    w = (w.view(nw, 4) << torch.tensor([0, 8, 16, 24], device=b.device)).sum(dim=1)
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32)


def _unpack_bytes(words: torch.Tensor, n: int) -> torch.Tensor:
    p = torch.arange(int(n), device=words.device)
    return ((words.to(torch.int64) & 0xFFFFFFFF)[p // 4] >> (8 * (p % 4))) & 0xFF


def _pow2(k: torch.Tensor) -> torch.Tensor:
    """fp32 2^k for integer k in [-149, 127], built from its bit pattern (2^-127 and below are subnormal)."""
    bits = torch.where(k >= -126, (k + 127) << 23, torch.full_like(k, 1 << 22) >> (-127 - k).clamp(min=0, max=31))
    return bits.to(torch.int32).view(torch.float32)


def fp8_encode_oracle(vals: torch.Tensor):
    """(scale words int32[ceil(K/128)], element words int32[ceil(K/4)]) of the fp32 ``vals`` under the rule above."""
    v = vals.detach().float().reshape(-1)
    K = v.numel()
    s = fp8_scale_bytes(v)
    sp = torch.where(s == FP8_NONFINITE, torch.full_like(s, 127), s)[torch.arange(K, device=v.device) // FP8_BLOCK]
    x = v * _pow2(127 - sp)                          # v * 2^-e, one fp32 multiply by a normal power of two
    q = x.to(torch.float8_e4m3fn).view(torch.uint8).to(torch.int64)
    q = torch.where(s[torch.arange(K, device=v.device) // FP8_BLOCK] == FP8_NONFINITE, torch.zeros_like(q), q)
    return _pack_bytes(s), _pack_bytes(q)


def fp8_decode_oracle(scales: torch.Tensor, elems: torch.Tensor, K: int) -> torch.Tensor:
    """fp32[K]: value p decodes to widen(q_p) * 2^e of its block, NaN in a block of scale byte 0xFF."""
    K = int(K)
    nb = (K + FP8_BLOCK - 1) // FP8_BLOCK
    s = _unpack_bytes(scales, nb)[torch.arange(K, device=elems.device) // FP8_BLOCK]
    q = _unpack_bytes(elems, K)
    w = q.to(torch.uint8).view(torch.float8_e4m3fn).float()        # exact widening
    d = w * _pow2(s - 127)
    return torch.where(s == FP8_NONFINITE, torch.full_like(d, float("nan")), d)


def _split(wire: torch.Tensor):
    K = int(wire[0].item())
    ns, ne = (K + 127) // 128, (K + 3) // 4
    if K < 0 or wire.numel() != 1 + ns + ne:
        raise ValueError(f"fp8 wire of {wire.numel()} words does not hold K = {K} values")
    return K, wire[1:1 + ns], wire[1 + ns:]


@register("fp8")
class FP8(SparseCompressor):
    order_preserving = True
    kind = "value"

    @staticmethod
    def compress(sparse_tensor, params):
        vals, idxs, shape = sparse_tensor
        vals = vals.float().reshape(-1)
        if idxs is not None and idxs.numel() > 1:
            order = torch.argsort(idxs.reshape(-1), stable=True)
            vals, idxs = vals[order], idxs.reshape(-1)[order]
        if use_cuda(vals):
            from .. import ops
            scales, elems = ops.fp8_encode(vals)
        else:
            scales, elems = fp8_encode_oracle(vals)
        head = torch.tensor([vals.numel()], dtype=torch.int32, device=vals.device)
        return torch.cat([head, scales, elems]), idxs, shape

    @staticmethod
    def decompress(sparse_tensor, params):
        wire, idxs, shape = sparse_tensor
        K, scales, elems = _split(wire)
        if use_cuda(wire):
            from .. import ops
            vals = ops.fp8_decode(scales, elems, K)
        else:
            vals = fp8_decode_oracle(scales, elems, K)
        return vals, idxs, shape
