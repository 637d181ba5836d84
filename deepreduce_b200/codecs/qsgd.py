"""Bucketed QSGD value codec (``'value': 'qsgd'``).

Parity with reference pytorch/deepreduce.py:849-907: per ``bucket_size`` (512)
bucket, ``level = quantum_num*|v|/||v||_2`` stochastically rounded, signed,
stored as int8 (quantum_num < 128) or int16; the bucket's fp32 L2 norm travels
as 4 raw bytes.  The reference does a host sync + ``struct.pack`` per bucket
(:876-880); here all buckets are processed in one kernel and the stochastic
rounding uses a counter-based hash RNG (``spec.policy_hash(idx, seed)/2^32``)
so encode is reproducible and does not touch the global torch RNG.

Wire: ``int8[K + 4*nb]`` (or ``int16[K + 2*nb]``): all levels, then the norms'
IEEE-754 bytes.
"""
from __future__ import annotations

import torch

from .. import spec
from .base import SparseCompressor, register, use_cuda


def _nb(K: int, bucket: int) -> int:
    return (K + bucket - 1) // bucket


def qsgd_encode_oracle(vals: torch.Tensor, q: int, bucket: int, seed: int):
    K = vals.numel()
    nb = _nb(K, bucket)
    v = vals.float()
    pad = nb * bucket - K
    vp = torch.cat([v, v.new_zeros(pad)]).view(nb, bucket)
    norm = vp.norm(dim=1)
    safe = torch.where(norm > 0, norm, torch.ones_like(norm))
    level_f = q / safe[:, None] * vp.abs()
    prev = level_f.floor()
    idx = torch.arange(nb * bucket, device=v.device)
    u = (spec.policy_hash(idx, seed).double() / 4294967296.0).float().view(nb, bucket)
    # level_f rounds above q when the norm is |v| itself (a bucket dominated by one value): clamp, so that level
    # q + 1 never wraps the int8 / int16 wire type
    lvl = (prev + (u < (level_f - prev)).float()).clamp(max=q)
    lvl = (lvl * vp.sign()).flatten()[:K]
    return lvl, norm


def qsgd_decode_oracle(levels: torch.Tensor, norms: torch.Tensor, q: int, bucket: int):
    K = levels.numel()
    b = torch.arange(K, device=levels.device) // bucket
    return norms[b] / q * levels.float()


@register("qsgd")
class QSGD(SparseCompressor):
    order_preserving = True
    kind = "value"

    @staticmethod
    def compress(sparse_tensor, params):
        vals, idxs, shape = sparse_tensor
        q = int(params.get('quantum_num', 127))
        bucket = int(params.get('bucket_size', 512))
        seed = int(params.get('qsgd_seed', 0x51ED))
        dt = torch.int8 if q < 128 else torch.int16
        if use_cuda(vals):
            from .. import ops
            lvl, norm = ops.qsgd_encode(vals, q, bucket, seed)
        else:
            lvl, norm = qsgd_encode_oracle(vals, q, bucket, seed)
        wire = torch.cat([lvl.to(dt), norm.float().contiguous().view(dt)])
        return wire, idxs, shape

    @staticmethod
    def decompress(sparse_tensor, params):
        wire, idxs, shape = sparse_tensor
        q = int(params.get('quantum_num', 127))
        bucket = int(params.get('bucket_size', 512))
        per = 4 // wire.element_size()
        # K + per*ceil(K/bucket) = n  -> solve for K
        n = wire.numel()
        K = idxs.numel() if idxs is not None and idxs.numel() + per * _nb(idxs.numel(), bucket) == n else None
        if K is None:                                   # no index list given ('both' ships none): n = K + per*ceil(K/bucket)
            K, nb_try = 0, max(1, -(-n // (bucket + per)))
            while n > 0:
                K = n - per * nb_try
                if K >= 0 and _nb(K, bucket) == nb_try:
                    break
                if K < 0:
                    raise ValueError(f"QSGD wire of {n} elements is not K + {per}*ceil(K/{bucket}) for any K")
                nb_try += 1
        nb = _nb(K, bucket)
        lvl = wire[:K]
        norm = wire[K:K + per * nb].clone().view(torch.float32)
        if use_cuda(wire):
            from .. import ops
            vals = ops.qsgd_decode(lvl, norm, q, bucket)
        else:
            vals = qsgd_decode_oracle(lvl, norm, q, bucket)
        return vals, idxs, shape
