"""Bloom-filter index codec (``'index': 'bloom'``).

Behavioural parity with reference pytorch/deepreduce.py:429-555 (``Bloomfilter``
+ ``Bloom``) and tensorflow/policies.hpp:148-194 (selection policies):

* sizing ``get_BFconfig`` (:495-500), default ``fpr = 0.1*K/d`` (:511);
* false-positive-aware value fill: when ``params['dense_tensor']`` is present the
  values shipped are ``dense[S~]`` for the policy-selected set S~ (:519-523);
* policies ``leftmost`` / ``random`` / ``p0`` (:479-492) plus ``conflict_sets``
  (P2, C++ only in the reference);
* ``p0`` prepends K to the values so the receiver can recompute (k, m) (:525-527).

Differences by design (SURVEY §3.7): hashing is on-the-fly (``spec``), the filter
is bit-packed ``int32`` words from birth, indices come back **ascending**, the
``random`` policy uses a seeded hash-rank (no global-RNG reseed), sizes are in
whole 32-bit words.  On CUDA tensors every step runs in hand-written sm_90a
kernels (``ops``); the functions named ``*_oracle`` are the plain-torch
reference of the same ops used on CPU and in the numerics tests.
"""
from __future__ import annotations

import torch

from .. import spec
from .base import SparseCompressor, register, use_cuda

POLICIES = ("leftmost", "random", "p0", "conflict_sets")
_POLICY_ALIASES = {"leftmostK": "leftmost", "randomK": "random", "policy_zero": "p0",
                   "P0": "p0", "P1": "random", "P2": "conflict_sets"}


def canonical_policy(p: str) -> str:
    p = _POLICY_ALIASES.get(p, p)
    if p not in POLICIES:
        raise ValueError(f"unknown bloom policy '{p}'")
    return p


# ----------------------------------------------------------------------------
# torch oracle
# ----------------------------------------------------------------------------
def words_from_bits(bits: torch.Tensor) -> torch.Tensor:
    """bool[m_bits] (m_bits % 32 == 0) -> int32[n_words], LSB-first."""
    w = bits.view(-1, 32).to(torch.int64)
    weights = (1 << torch.arange(32, device=bits.device, dtype=torch.int64))
    v = (w * weights).sum(dim=1)
    v = torch.where(v >= (1 << 31), v - (1 << 32), v)
    return v.to(torch.int32)


def bits_from_words(words: torch.Tensor) -> torch.Tensor:
    sh = torch.arange(32, device=words.device, dtype=torch.int64)
    return (((words.to(torch.int64)[:, None] >> sh[None, :]) & 1) != 0).flatten()


def bloom_insert_oracle(idxs: torch.Tensor, k: int, m_bits: int, seed: int = spec.DEFAULT_SEED) -> torch.Tensor:
    bits = torch.zeros(((m_bits + 31) // 32) * 32, dtype=torch.bool, device=idxs.device)
    if idxs.numel():
        pos = spec.bloom_positions(idxs.flatten(), k, m_bits, seed).flatten()
        bits[pos] = True
    return words_from_bits(bits)


def bloom_query_oracle(words: torch.Tensor, d: int, k: int, m_bits: int,
                       seed: int = spec.DEFAULT_SEED, chunk: int = 1 << 20) -> torch.Tensor:
    """All positives in [0, d), ascending (reference ``Bloomfilter.query`` :466-477)."""
    bits = bits_from_words(words)
    out = []
    for lo in range(0, d, chunk):
        x = torch.arange(lo, min(d, lo + chunk), device=words.device)
        pos = spec.bloom_positions(x, k, m_bits, seed)
        hit = bits[pos].all(dim=1)
        out.append(x[hit])
    return torch.cat(out) if out else torch.empty(0, dtype=torch.int64, device=words.device)


def conflict_sets_cuda(positives: torch.Tensor, K: int, k: int, m_bits: int, seed: int, pseed: int):
    """P2 on the device.  The conflict sets (positives grouped by filter bit) are built with a sort of the
    (bit position, rank) pairs and ordered by (size, bit position); the draw itself — sequential by definition —
    runs in the one-warp kernel ``conflict_sets_pick_kernel`` (ops/csrc/ops.cu).  Same result as the host routine
    (``native_cpu.cpp::conflict_sets_impl`` / the reference's policies.hpp:43-146), no device->host bounce of the
    positives.  Returns None when the positives do not fit the kernel's shared-memory bitmap (> 1.6 M)."""
    from .. import ops
    P = int(positives.numel())
    if P == 0 or P > 1_600_000:
        return None if P else positives
    dev = positives.device
    pos = spec.bloom_positions(positives, k, m_bits, seed)                    # [P, k] filter bits of every positive
    rank = torch.arange(P, device=dev, dtype=torch.int64)[:, None].expand(P, k)
    key = torch.unique((pos << 32 | rank).flatten())                          # sorted; a positive enters a set once
    bit, member = key >> 32, (key & 0xFFFFFFFF).to(torch.int32)
    start = torch.ones(key.numel(), dtype=torch.bool, device=dev)
    start[1:] = bit[1:] != bit[:-1]
    first = torch.nonzero(start).flatten()                                    # first entry of every set (sets in bit order)
    size = torch.diff(first, append=torch.tensor([key.numel()], device=dev))
    order = torch.argsort(size << 32 | bit[first])                            # visit order: (size, bit position)
    size_v = size[order]
    off_v = torch.zeros(order.numel() + 1, dtype=torch.int64, device=dev)
    off_v[1:] = torch.cumsum(size_v, 0)
    # gather the members set by set in visit order
    idx = torch.repeat_interleave(first[order] - off_v[:-1], size_v) + torch.arange(key.numel(), device=dev)
    members_v = member[idx].contiguous()
    chosen = ops.cuda_module().conflict_sets_pick(off_v.to(torch.int32).contiguous(), members_v,
                                                  size_v.to(torch.int32).contiguous(), P, int(K), int(pseed) & spec.MASK32)
    bits = ((chosen.to(torch.int64)[:, None] >> torch.arange(32, device=dev)) & 1).flatten()[:P].bool()
    return positives[bits]


def conflict_sets_oracle(positives: torch.Tensor, K: int, k: int, m_bits: int, seed: int, pseed: int):
    """P2 (reference policies.hpp:43-146, paper Alg. 1).  Sequential by nature;
    runs in the native C++ op when built, else in Python (small inputs only).
    Deterministic tie-breaks are part of the spec: conflict sets are ordered by
    (size, bit position); members are kept ascending; the random member is
    ``policy_hash(draw_counter, pseed) % len(set)``; a full pass without a pick
    falls back to leftmost among the unchosen (the reference spins forever,
    SURVEY §3.7)."""
    from .. import ops
    if positives.is_cuda and ops.has_cuda_native():
        sel = conflict_sets_cuda(positives, K, k, m_bits, seed, pseed)
        if sel is not None:
            return sel
    if ops.has_cpu_native():
        return ops.cpu.conflict_sets(positives.cpu().to(torch.int64), int(K), int(k), int(m_bits),
                                     int(seed), int(pseed)).to(positives.device)
    P = positives.cpu().tolist()
    sets: dict[int, list[int]] = {}
    for x in P:
        for pos in spec.bloom_positions_int(x, k, m_bits, seed):
            s = sets.setdefault(pos, [])
            if not s or s[-1] != x:
                s.append(x)
    ordered = sorted(sets.items(), key=lambda kv: (len(kv[1]), kv[0]))
    ordered = [list(v) for _, v in ordered]
    chosen: set[int] = set()
    left = min(K, len(P))
    draw = 0
    while left > 0:
        picked = False
        for cset in ordered:
            if left == 0:
                break
            before = len(cset)
            cset[:] = [x for x in cset if x not in chosen]
            if len(cset) == before and cset:
                r = spec.policy_hash_int(draw, pseed) % len(cset)
                draw += 1
                chosen.add(cset.pop(r))
                left -= 1
                picked = True
        if not picked:
            for x in P:
                if left == 0:
                    break
                if x not in chosen:
                    chosen.add(x)
                    left -= 1
    return torch.tensor(sorted(chosen), dtype=torch.int64, device=positives.device)


def apply_policy_oracle(positives: torch.Tensor, K: int, policy: str, pseed: int = 42,
                        k: int = 0, m_bits: int = 0, seed: int = spec.DEFAULT_SEED) -> torch.Tensor:
    """Choose S~ from the positives; result ascending."""
    policy = canonical_policy(policy)
    if policy == "p0" or positives.numel() <= K and policy != "conflict_sets":
        return positives
    if policy == "leftmost":
        return positives[:K]
    if policy == "random":
        keys = spec.policy_hash(positives, pseed)
        comp = (keys << 31) | positives          # key-major, index-minor; fits int64 (idx < 2^31)
        sel = torch.sort(comp).values[:K] & 0x7FFFFFFF
        return torch.sort(sel).values
    return conflict_sets_oracle(positives, K, k, m_bits, seed, pseed)


# ----------------------------------------------------------------------------
# dispatch (CUDA kernels vs oracle)
# ----------------------------------------------------------------------------
def bloom_insert(idxs, k, m_bits, seed=spec.DEFAULT_SEED):
    if use_cuda(idxs):
        from .. import ops
        return ops.bloom_insert(idxs, k, m_bits, seed)
    return bloom_insert_oracle(idxs, k, m_bits, seed)


def bloom_select(words, d, K, k, m_bits, policy, pseed=42, seed=spec.DEFAULT_SEED):
    """Universe query + policy -> ascending int64 indices."""
    policy = canonical_policy(policy)
    if use_cuda(words):
        from .. import ops
        if policy != "conflict_sets":
            return ops.bloom_select(words, d, K, k, m_bits, policy, pseed, seed)
        pos = ops.bloom_select(words, d, K, k, m_bits, "p0", pseed, seed)     # all positives (query kernel), then P2 on the device
        return conflict_sets_oracle(pos, K, k, m_bits, seed, pseed)
    pos = bloom_query_oracle(words, d, k, m_bits, seed)
    return apply_policy_oracle(pos, K, policy, pseed, k, m_bits, seed)


class Bloomfilter(object):
    """Object form of the primitive for API parity with reference :431-492."""

    def __init__(self, size, num_hash, params=None, bit_array=None, seed=spec.DEFAULT_SEED, device=None):
        self.n_words = (int(size) + 31) // 32
        self.size = self.n_words * 32
        self.num_hash = int(num_hash)
        self.params = params or {}
        self.seed = seed
        self.bit_array = bit_array if bit_array is not None else torch.zeros(
            self.n_words, dtype=torch.int32, device=device)

    def __len__(self):
        return self.size

    def add(self, items):
        new = bloom_insert(items, self.num_hash, self.size, self.seed)
        self.bit_array = self.bit_array.to(new.device) | new

    def query(self, query_range):
        return bloom_select(self.bit_array, int(query_range), 0, self.num_hash, self.size, "p0", 0, self.seed)

    def policy(self, positives, k, policy, pseed=42):
        return apply_policy_oracle(positives, k, policy, pseed, self.num_hash, self.size, self.seed)

    # the filter is packed from birth; kept as no-ops for source compatibility (:446-455)
    def pack_bitarray(self):
        return self.bit_array

    def unpack_bitarray(self):
        return self.bit_array


get_BFconfig = spec.get_BFconfig


@register("bloom")
class Bloom(SparseCompressor):
    order_preserving = False
    kind = "index"

    @staticmethod
    def _config(num_indices, grad_size, params):
        fpr = params.get('fpr', None)
        return spec.bloom_layout(num_indices, grad_size, fpr, params.get('max_hash', 16))

    @staticmethod
    def compress(sparse_tensor, params):
        vals, idxs, shape = sparse_tensor
        grad_size = shape.numel()
        num_indices = int(idxs.numel())
        policy = canonical_policy(params.get('policy', 'leftmost'))
        seed = params.get('hash_seed', spec.DEFAULT_SEED)
        k, m_bits, _ = Bloom._config(num_indices, grad_size, params)
        words = bloom_insert(idxs, k, m_bits, seed)

        dense_tensor = params.get('dense_tensor', None)
        if dense_tensor is not None:   # false-positive aware (reference :519-523)
            new_idxs = bloom_select(words, grad_size, num_indices, k, m_bits, policy,
                                    params.get('policy_seed', 42), seed)
            vals = dense_tensor.flatten()[new_idxs]
        if policy == 'p0':
            head = torch.as_tensor([num_indices], dtype=vals.dtype, device=vals.device)
            vals = torch.cat([head, vals], dim=0)
        return vals, words, shape

    @staticmethod
    def decompress(bf_sparse_tensor, params):
        vals, words, shape = bf_sparse_tensor
        policy = canonical_policy(params.get('policy', 'leftmost'))
        seed = params.get('hash_seed', spec.DEFAULT_SEED)
        if policy == 'p0':
            num_indices = int(vals[0].item())
            vals = vals[1:]
        else:
            num_indices = int(vals.numel())
        grad_size = shape.numel()
        k, m_bits, _ = Bloom._config(num_indices, grad_size, params)
        idxs = bloom_select(words, grad_size, num_indices, k, m_bits, policy,
                            params.get('policy_seed', 42), seed)
        if policy != 'p0' and idxs.numel() > vals.numel():
            idxs = idxs[: vals.numel()]
        if idxs.numel() < vals.numel():   # cannot happen for a well-formed payload; stay safe
            vals = vals[: idxs.numel()]
        return vals, idxs, shape
