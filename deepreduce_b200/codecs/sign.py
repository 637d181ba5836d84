"""Scaled-sign value codec (``'value': 'sign'``): EF-signSGD's compressor (Karimireddy et al., 2019), and after top-k
the value half of Sparse Ternary Compression (Sattler et al., 2019).

The shipped values, in ascending index order, are cut into buckets of 512.  Bucket b ships one fp32 scale
mu_b = fl32(S_b / n_b), where S_b is the fp64 sum of |v| over the bucket zero-padded to 512 in a fixed adjacent-pair
tree (nine levels) and n_b its number of values, and one bit per value, set iff v < 0 (so -0.0, +0.0 and NaN give 0).
A value decodes to bit ? -mu_b : +mu_b.  mu_b <= max |v|, so a finite bucket has a finite scale; a NaN in a bucket
makes its scale NaN and an inf makes it inf, and the whole bucket decodes to that.  The residual and 'dgc' memories
keep ``v - d``, which is where the code's bias goes.

Wire: ``int32[1 + ceil(K/32) + ceil(K/512)]``: K, the sign bits (value p is bit p % 32 of word p // 32, LSB first),
then the scales' fp32 bits.  K travels because 'both' decodes without the index list, and the two lengths do not
determine it.  In 'value' mode compress first puts the pairs in ascending index order, so its buckets are the fused
engine's (``parallel/plan.py`` ``VMODE_SIGN``); in 'both' they already arrive in the index codec's ascending order.
CUDA tensors are coded by the sm_90a kernels (``ops.sign_encode`` / ``ops.sign_decode``), CPU tensors by the torch
reference below; both give the same words.
"""
from __future__ import annotations

import torch

from .base import SparseCompressor, register, use_cuda

SIGN_BUCKET = 512


def sign_encode_oracle(vals: torch.Tensor):
    """(bits int32[ceil(K/32)], scales fp32[ceil(K/512)]) of the fp32 ``vals`` under the rule above."""
    v = vals.detach().float().reshape(-1)
    K = v.numel()
    nb = (K + SIGN_BUCKET - 1) // SIGN_BUCKET
    x = torch.zeros(nb * SIGN_BUCKET, dtype=torch.float64, device=v.device)
    x[:K] = v.abs().double()
    x = x.view(nb, SIGN_BUCKET)
    while x.shape[1] > 1:                       # the adjacent-pair tree: (0,1), (2,3), ..., nine levels
        x = x[:, 0::2] + x[:, 1::2]
    n = torch.full((nb,), SIGN_BUCKET, dtype=torch.float64, device=v.device)
    if nb:
        n[-1] = K - (nb - 1) * SIGN_BUCKET
    scales = (x[:, 0] / n).float()
    nw = (K + 31) // 32
    neg = torch.zeros(nw * 32, dtype=torch.int64, device=v.device)
    neg[:K] = (v < 0).long()
    words = (neg.view(nw, 32) << torch.arange(32, device=v.device)).sum(dim=1)
    bits = torch.where(words >= 1 << 31, words - (1 << 32), words).to(torch.int32)
    return bits, scales


def sign_decode_oracle(bits: torch.Tensor, scales: torch.Tensor, K: int) -> torch.Tensor:
    """fp32[K]: value p decodes to -mu if its bit is set, else +mu, mu the scale of its bucket."""
    p = torch.arange(int(K), device=bits.device)
    b = ((bits.to(torch.int64) & 0xFFFFFFFF)[p // 32] >> (p % 32)) & 1
    mu = scales.float()[p // SIGN_BUCKET]
    return torch.where(b.bool(), -mu, mu)


def _split(wire: torch.Tensor):
    K = int(wire[0].item())
    nw, nb = (K + 31) // 32, (K + SIGN_BUCKET - 1) // SIGN_BUCKET
    if K < 0 or wire.numel() != 1 + nw + nb:
        raise ValueError(f"sign wire of {wire.numel()} words does not hold K = {K} values")
    return K, wire[1:1 + nw], wire[1 + nw:].contiguous().view(torch.float32)


@register("sign")
class Sign(SparseCompressor):
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
            bits, scales = ops.sign_encode(vals)
        else:
            bits, scales = sign_encode_oracle(vals)
        head = torch.tensor([vals.numel()], dtype=torch.int32, device=vals.device)
        return torch.cat([head, bits, scales.contiguous().view(torch.int32)]), idxs, shape

    @staticmethod
    def decompress(sparse_tensor, params):
        wire, idxs, shape = sparse_tensor
        K, bits, scales = _split(wire)
        if use_cuda(wire):
            from .. import ops
            vals = ops.sign_decode(bits, scales, K)
        else:
            vals = sign_decode_oracle(bits, scales, K)
        return vals, idxs, shape
