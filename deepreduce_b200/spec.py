"""Wire / hashing specification shared by the torch oracle, the C++ CPU ops and
the sm_90a kernels.

The reference keeps a precomputed ``hash_table[d_max, k_max]`` of MurmurHash3
values on every GPU (reference pytorch/deepreduce.py:42-44, 461, 471) and
re-reduces it ``% size`` on every call.  That table is O(d*k) memory and the
file is not even shipped, so the new framework hashes on the fly.  Everything
in this file is *normative*: the CUDA kernels in ``ops/csrc`` implement exactly
these formulas and the tests compare them bit-for-bit.

Hash family (Kirsch–Mitzenmacher double hashing over two murmur3 finalisers)::

    a      = fmix32(x ^ seed)
    b      = fmix32((x ^ seed) * 0x9E3779B1 + 0x7F4A7C15) | 1
    h_j    = (a + j*b) mod 2^32                 j = 0 .. k-1
    pos_j  = (h_j * m_bits) >> 32               Lemire range reduction, no '%'
    word   = pos_j >> 5 ; bit = pos_j & 31      LSB-first inside a uint32 word

Filters are bit-packed uint32 words from birth (the reference keeps 1 byte per
bit and packs with cupy just before the collective, reference :446-455).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Tuple

import torch

MASK32 = 0xFFFFFFFF
DEFAULT_SEED = 0x9747B28C
GOLDEN = 0x9E3779B1
B_ADD = 0x7F4A7C15
FMIX_C1 = 0x85EBCA6B
FMIX_C2 = 0xC2B2AE35

# Codec is bypassed for tensors with <= this many elements (reference :68,115,259).
SMALL_TENSOR_NUMEL = 1000

# Elements per tile in the bucket engine (one CTA pass).  Part of the wire
# format because the per-tile selected-prefix table is shipped.
TILE = 4096

LN2 = 0.693147180  # the reference's literal (pytorch/deepreduce.py:499)


# ----------------------------------------------------------------------------
# scalar (python int) versions — used by tests and by the C++ parity checks
# ----------------------------------------------------------------------------
def fmix32_int(h: int) -> int:
    h &= MASK32
    h ^= h >> 16
    h = (h * FMIX_C1) & MASK32
    h ^= h >> 13
    h = (h * FMIX_C2) & MASK32
    h ^= h >> 16
    return h


def hash_ab_int(x: int, seed: int = DEFAULT_SEED) -> Tuple[int, int]:
    y = (x ^ seed) & MASK32
    a = fmix32_int(y)
    b = fmix32_int((y * GOLDEN + B_ADD) & MASK32) | 1
    return a, b


def bloom_positions_int(x: int, k: int, m_bits: int, seed: int = DEFAULT_SEED):
    a, b = hash_ab_int(x, seed)
    return [(((a + j * b) & MASK32) * m_bits) >> 32 for j in range(k)]


# ----------------------------------------------------------------------------
# tensor versions (int64 arithmetic emulating uint32) — the oracle
# ----------------------------------------------------------------------------
def fmix32(h: torch.Tensor) -> torch.Tensor:
    h = h & MASK32
    h = h ^ (h >> 16)
    h = (h * FMIX_C1) & MASK32
    h = h ^ (h >> 13)
    h = (h * FMIX_C2) & MASK32
    h = h ^ (h >> 16)
    return h


def hash_ab(x: torch.Tensor, seed: int = DEFAULT_SEED):
    y = (x.to(torch.int64) ^ seed) & MASK32
    a = fmix32(y)
    b = fmix32((y * GOLDEN + B_ADD) & MASK32) | 1
    return a, b


def bloom_positions(x: torch.Tensor, k: int, m_bits: int, seed: int = DEFAULT_SEED) -> torch.Tensor:
    """[n] indices -> [n, k] bit positions in [0, m_bits)."""
    assert m_bits < (1 << 31)
    a, b = hash_ab(x, seed)
    j = torch.arange(k, device=x.device, dtype=torch.int64)
    h = (a[:, None] + j[None, :] * b[:, None]) & MASK32
    return (h * m_bits) >> 32


def policy_hash(x: torch.Tensor, seed: int) -> torch.Tensor:
    """Rank key for the seeded 'random' (P1) policy: K positives with the
    smallest key are selected.  Replaces ``torch.manual_seed(42); randperm``
    (reference :487-488) which clobbers the global RNG."""
    y = (x.to(torch.int64) * GOLDEN + (seed & MASK32)) & MASK32
    return fmix32(y ^ 0x5BD1E995)


def policy_hash_int(x: int, seed: int) -> int:
    y = (x * GOLDEN + (seed & MASK32)) & MASK32
    return fmix32_int(y ^ 0x5BD1E995)


def policy_seed(step: int, tensor_id: int) -> int:
    """Per-(step, tensor) seed so sender, residual update and receivers agree
    (the C++ reference seeds with the training step, policies.hpp:171)."""
    return fmix32_int(((step & MASK32) * 0x01000193) ^ ((tensor_id + 1) * GOLDEN & MASK32))


# ----------------------------------------------------------------------------
# bloom sizing
# ----------------------------------------------------------------------------
def get_BFconfig(capacity: int, fpr: float) -> Tuple[int, int]:
    """(num_hash, num_bits) exactly as reference pytorch/deepreduce.py:495-500."""
    num_hash = math.log(1 / fpr, 2)
    num_bits = num_hash * capacity / LN2
    return math.ceil(num_hash), math.ceil(num_bits)


def default_fpr(num_indices: int, grad_size: int) -> float:
    """reference :511 — fpr = 0.1 * K / d."""
    return 0.1 * num_indices / grad_size


def bloom_layout(capacity: int, grad_size: int, fpr: float | None = None, max_hash: int = 16) -> Tuple[int, int, int]:
    """(num_hash, m_bits, n_words).  m_bits is the reference's num_bits rounded
    up to whole 32-bit words (the filter is word-packed from birth); num_hash is
    clamped to [1, max_hash] like ``min(num_hash, hash_table.size(1))`` (:440)."""
    capacity = max(1, int(capacity))
    if fpr is None:
        fpr = default_fpr(capacity, grad_size)
    fpr = min(max(float(fpr), 1e-9), 0.999)
    k, bits = get_BFconfig(capacity, fpr)
    k = max(1, min(int(k), max_hash))
    n_words = max(1, (int(bits) + 31) // 32)
    return k, n_words * 32, n_words


def bloom_configuration(k: int, fpr: float) -> Tuple[int, int]:
    """TF-side sizing, (m_bytes, h) — reference tensorflow/deepreduce.py:260-271."""
    m = (k * abs(math.log(fpr))) / (math.pow(math.log(2), 2))
    m = int(m / 8)
    rem = m % 8
    if rem != 0 or m == 0:
        m += 1
    h = (m * 8 / k) * math.log(2)
    return m, int(math.ceil(h))


def ef_layout(cap: int, n_tiles: int) -> Tuple[int, int, int]:
    """Tile-local Elias-Fano index (``'index': 'elias_fano'``) of a tensor of ``n_tiles`` tiles holding up to ``cap``
    entries: (L, low-stream words, high-stream words).  L = argmin over 0..12 of cap * L + n_tiles * (TILE >> L), the
    smallest on ties.  Entry p (its rank in ascending index order), with in-tile offset e in tile-local tile t, puts
    e & (2^L - 1) at bit p * L of the low stream (cap * L bits) and sets bit p + t * (TILE >> L) + (e >> L) of the high
    stream (cap + n_tiles * (TILE >> L) bits), both LSB-first; a u16 entry count per tile (the run-length index's table)
    goes with them.  Tile t owns the high bits [pre_t + t * B, pre_t + c_t + (t + 1) * B), B = TILE >> L, where pre_t
    entries lie in the earlier tiles and c_t in t: its j-th set bit q gives e = ((q - pre_t - t * B - j) << L) | low."""
    L = min(range(13), key=lambda l: cap * l + n_tiles * (TILE >> l))
    return L, (cap * L + 31) // 32, (cap + n_tiles * (TILE >> L) + 31) // 32


def topk_k(numel: int, ratio: float) -> int:
    """GRACE top-k K (SURVEY §2.5)."""
    return max(1, int(numel * ratio))


@dataclass(frozen=True)
class Warmup:
    """DGC's sparsity warm-up (params keys ``'warmup_ratios'``, ``'warmup_steps'``): exchange ``e`` (0-based, counted
    in exchanges, not micro-steps) is in stage ``min(e // steps, len(ratios))``; stage ``s < len(ratios)`` selects with
    compress ratio ``ratios[s]``, the last stage with ``final`` (the dict's ``'compress_ratio'``).  Every route reads
    the ratio of an exchange from here."""
    ratios: Tuple[float, ...]
    steps: int
    final: float

    @property
    def n_stages(self) -> int:
        return len(self.ratios) + 1

    def stage(self, exchange: int) -> int:
        return min(int(exchange) // self.steps, len(self.ratios))

    def ratio(self, stage: int) -> float:
        return self.ratios[stage] if stage < len(self.ratios) else self.final

    def ratio_at(self, exchange: int) -> float:
        return self.ratio(self.stage(exchange))


def bits_for(n: int) -> int:
    """Bits needed to store values in [0, n)."""
    return max(1, int(n - 1).bit_length()) if n > 1 else 1
