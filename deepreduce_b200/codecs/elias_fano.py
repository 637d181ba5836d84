"""Tile-local Elias-Fano index codec (``'index': 'elias_fano'``).

Lossless, like the run-length index, and of a size fixed by the entry count: about 2 + log2(4096 / n) bits per index
for n entries per 4096-element tile.  The format is ``spec.ef_layout``, the one the fused engine ships (its slot holds
the same three parts, each 4-word aligned): ``enc`` is the uint32 words (as int32) ``[u16 count per tile | low stream
| high stream]`` with the capacity K taken from the values' count, and the values are reordered to ascending index.
The streams are built with torch ops over the ``bitpack`` kernels, so CPU and CUDA give the same words.
"""
from __future__ import annotations

import torch

from .. import spec
from . import bitpack
from .base import SparseCompressor, register


def _words(b: torch.Tensor, n_words: int) -> torch.Tensor:
    """uint8 bytes zero-padded (or cut) to ``n_words`` little-endian words."""
    out = torch.zeros(4 * n_words, dtype=torch.uint8, device=b.device)
    n = min(int(b.numel()), 4 * n_words)
    out[:n] = b[:n]
    return out


@register("elias_fano")
class EliasFano(SparseCompressor):
    order_preserving = False
    kind = "index"

    @staticmethod
    def compress(sparse_tensor, params):
        vals, idxs, shape = sparse_tensor
        idxs, mapping = idxs.long().sort(descending=False)
        vals = vals[mapping]
        d, K = shape.numel(), int(idxs.numel())
        n_tiles = (d + spec.TILE - 1) // spec.TILE
        L, lo_words, hi_words = spec.ef_layout(K, n_tiles)
        tile, e = idxs // spec.TILE, idxs % spec.TILE
        cnt = torch.bincount(tile, minlength=n_tiles)
        cnt_b = torch.stack([cnt & 0xFF, cnt >> 8], dim=1).flatten().to(torch.uint8)
        lo_b = bitpack.pack_bits(e & ((1 << L) - 1), L) if L and K else cnt_b[:0]
        hb = torch.arange(K, device=idxs.device) + tile * (spec.TILE >> L) + (e >> L)
        bits = torch.zeros(32 * hi_words, dtype=torch.int64, device=idxs.device)
        bits[hb] = 1
        enc = torch.cat([_words(cnt_b, (n_tiles + 1) // 2), _words(lo_b, lo_words),
                         _words(bitpack.pack_bits(bits, 1), hi_words)])
        return vals, enc.view(torch.int32), shape

    @staticmethod
    def decompress(ef_sparse_tensor, params):
        vals, enc, shape = ef_sparse_tensor
        d, K = shape.numel(), int(vals.numel())
        n_tiles = (d + spec.TILE - 1) // spec.TILE
        L, lo_words, hi_words = spec.ef_layout(K, n_tiles)
        b = enc.contiguous().view(torch.uint8)
        c0 = 4 * ((n_tiles + 1) // 2)
        cnt = b[0:2 * n_tiles:2].long() | (b[1:2 * n_tiles:2].long() << 8)
        lo = (bitpack.unpack_bits(b[c0:c0 + 4 * lo_words], K, L) if L and K
              else torch.zeros(K, dtype=torch.int64, device=b.device))
        q = torch.nonzero(bitpack.unpack_bits(b[c0 + 4 * lo_words:], 32 * hi_words, 1)).flatten()
        if int(q.numel()) != K or int(cnt.sum()) != K:
            raise ValueError(f"elias_fano: {int(q.numel())} high bits and {int(cnt.sum())} counted entries for {K} values")
        tile = torch.repeat_interleave(torch.arange(n_tiles, device=b.device), cnt)
        h = q - torch.arange(K, device=b.device) - tile * (spec.TILE >> L)
        return vals, tile * spec.TILE + ((h << L) | lo), shape
