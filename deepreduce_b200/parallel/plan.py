"""Bucket plan: static layout of a flat gradient bucket and of its compressed slot.

A bucket is a list of tensors flattened back to back (each start aligned to 32
floats) and cut into ``spec.TILE``-element tiles that never cross a tensor.  The
"per tensor" semantics of the reference (top-k ratio, bloom sizing ``fpr =
0.1*K/d``, the ≤1000-element bypass — reference pytorch/deepreduce.py:68,115,
495-500,511) are preserved per segment; only the launch granularity changes.
Field order of ``TensorDesc`` mirrors ``ops/csrc/plan.h``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np
import torch

from .. import spec
from ..codecs.dexp import MIN_NUMEL as DEXP_MIN_NUMEL

MODE_RAW, MODE_BLOOM, MODE_RLE, MODE_SHARED, MODE_EF = 0, 1, 2, 3, 4
# TensorDesc.vmode (plan.h ValueMode)
VMODE_FP32, VMODE_POLYFIT, VMODE_QSGD, VMODE_DEXP, VMODE_BF16, VMODE_SIGN, VMODE_FP8 = 0, 1, 2, 3, 4, 5, 6
KEY_SPAN = 1 << 31                    # select keys are 31-bit
POLICY_ID = {"leftmost": 0, "random": 1, "p0": 2, "conflict_sets": 3}
P2_MAX_POS_CAP = 1 << 20              # P2: the draw keeps one chosen bit per positive in shared memory (128 KB)
P2_ENTRY_WORDS = 10                   # P2 scratch table entry (ops/csrc/p2.cu P2Entry)
P2_MAX_HASH = 16                      # P2: filter bits per positive the sender stage holds (p2.cu kMaxHash)
P2_SIZE_CAP = 32                      # P2: sets of at least this many members are ordered by a separate pass (p2.cu kSizeCap)
SLOT_HEADER_WORDS = 8
DYN_WORDS = 4
ARENA_HDR_WORDS = 128
HIST_BINS = 2048
NUM_HIST = 3
ALIGN_ELEMS = 32
MAX_SEGMENTS = 22
# (segment start, one-tile tensor) cost in tiles' worth for the four phase classes of the kernel's tile -> CTA partition
# (accumulate, insert, query, emit): least-squares fit of the per-CTA phase durations of a ResNet-50 bucket taken with
# scripts/cta_timeline.py on the previous target GPU and not re-fitted on the H100; BucketEngine.calibrate_partition
# measures the per-CTA speeds of the GPU it runs on and re-cuts the partition from them
PART_WEIGHTS = ((5.0, 1.0), (2.0, 0.0), (5.5, 1.5), (3.0, 0.0))


def update_cta_speeds(speeds, dur, gain: float = 0.8):
    """One calibration step of the per-CTA relative speeds of a phase class: a CTA that took ``dur[b]`` for its current
    share when the median CTA took ``median(dur)`` gets its speed (= its share of the next cut) scaled by
    ``(median / dur[b]) ** gain``; clipped to [0.5, 2] and renormalised to mean 1.  ``gain`` < 1 damps the measurement
    noise of a single round (BucketEngine.calibrate_partition)."""
    speeds = np.asarray(speeds, dtype=np.float64)
    dur = np.asarray(dur, dtype=np.float64)
    rel = np.median(dur) / np.maximum(dur, 1e-3)
    out = np.clip(speeds * rel ** gain, 0.5, 2.0)
    return out / out.mean()
MAX_POLY_K = 1 << 17      # the all-pairs rank pass is O(K^2): larger tensors keep fp32 values
DEXP_COEF_WORDS = 8       # 'dexp': {a, b, p, q} of the positive run, then of the non-positive run (ops/csrc/plan.h)
DESC_WORDS = 32
RANK_BINS = 8192


def rle_stream_words(k: int) -> int:
    return (k * 12 + 31) // 32 + 1


def _align(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def randomk_capacity(d: int, k: int) -> int:
    """Slot capacity of a 'randomk' tensor: K plus room for the elements that share the threshold's 22-bit key prefix
    (about d / 2^22 expected; more than the slack are cut left-most, consistently on every rank)."""
    return min(d, k + 16 + (d >> 20))


def randomk_bound(d: int, k: int) -> int:
    """Static candidate bound of a 'randomk' tensor: the hash key above which K + 8 sqrt(K) + 16 of its d uniformly
    distributed keys are expected, rounded down to a 22-bit prefix boundary (so it never splits the threshold's bin).
    The K-th largest key falls below it only if the count above it is some 8 standard deviations short; then the
    kernel's fallback phase redoes the select over every key."""
    m = k + int(math.ceil(8.0 * math.sqrt(k))) + 16
    if m >= d:
        return 0
    return (KEY_SPAN * (d - m) // d) & ~511


def split_large(numels, names, shapes, split_numel: Optional[int]):
    """Opt-in chunking of huge tensors (params key ``'split_numel'``): a tensor with more than ``split_numel``
    elements enters the plan as consecutive chunks of ``split_numel`` (rounded down to whole 4096-element tiles), each
    with its own top-k, filter and header — so every bloom filter stays small enough to be staged in shared memory
    (the 31 M-element BERT embedding needs a 560 KB filter as one tensor, 70 KB as eight chunks) and the selection of a
    single giant tensor is spread over the bucket's tiles.  Chunks are tile multiples, hence contiguous in the flat
    buffer: the parameter's gradient view spans them.  Semantics: top-k per chunk instead of per tensor (the reference
    is per tensor) — which is why it is opt-in.  Returns (numels, names, shapes, owner): owner[j] = index of the
    original tensor chunk j belongs to."""
    if not split_numel:
        return list(numels), list(names), list(shapes), list(range(len(numels)))
    step = max(spec.TILE, (int(split_numel) // spec.TILE) * spec.TILE)
    out_n, out_names, out_shapes, owner = [], [], [], []
    for i, (d, nm, sh) in enumerate(zip(numels, names, shapes)):
        d = int(d)
        if d <= step:
            out_n.append(d); out_names.append(nm); out_shapes.append(tuple(sh)); owner.append(i)
            continue
        off, c = 0, 0
        while off < d:
            n = min(step, d - off)
            out_n.append(n); out_names.append(f"{nm}#{c}"); out_shapes.append((n,)); owner.append(i)
            off += n; c += 1
    return out_n, out_names, out_shapes, owner


def auto_split_numel(compress_ratio: float, fpr: Optional[float], filter_smem_bytes: int = 80 * 1024,
                     max_hash: int = 16) -> int:
    """Largest chunk size (whole tiles) whose bloom filter still fits the kernel's SMEM staging buffer.  A filter that
    does not fit is probed from global / L2 memory instead — an order of magnitude slower (BERT-large's 31 M-element
    word embedding needs 560 KB at 1 %).  Used as the default ``split_numel`` of the bucketed DDP wrapper."""
    words_cap = filter_smem_bytes // 4
    lo, hi = spec.TILE, 1 << 31
    while lo + spec.TILE < hi:                       # largest d with n_filter_words(d) <= words_cap
        mid = (lo + hi) // 2
        k = min(mid, spec.topk_k(mid, compress_ratio))
        if spec.bloom_layout(k, mid, fpr, max_hash)[2] <= words_cap:
            lo = mid
        else:
            hi = mid
    return max(spec.TILE, (lo // spec.TILE) * spec.TILE)


@dataclass
class TensorPlan:
    name: str
    numel: int
    shape: tuple
    elem_off: int
    k: int
    tile_begin: int
    n_tiles: int
    mode: int
    m_bits: int = 0
    n_hash: int = 0
    off_vals: int = 0
    off_filter: int = 0
    off_prefix: int = 0
    off_idx: int = 0
    val_cap: int = 0
    salt: int = 0
    n_filter_words: int = 0
    off_hint: int = 0
    vmode: int = 0
    off_coef: int = 0
    off_rankmap: int = 0
    off_selidx: int = 0
    off_sorted: int = 0
    poly_degree: int = 5
    rank_u32: int = 0
    poly_off: int = 0
    poly_ord: int = 0
    fixed_thr: int = 0        # 'threshold' sparsifier: select |x| bit pattern >= fixed_thr (0: top-k radix select)
    shared_lb: int = 0        # MODE_SHARED: static candidate bound on the hash key (randomk_bound)
    pos_cap: int = 0          # P2: the pick runs over the first min(n_pos, pos_cap) positives
    off_pos_prefix: int = 0   # P2: [n_tiles] positives before each tile, capped at pos_cap
    off_pick: int = 0         # P2: [ceil(pos_cap / 32)] pick bitmask over the positives
    ef_low_bits: int = 0      # MODE_EF: L of spec.ef_layout (the low stream is at off_idx)
    off_hi: int = 0           # MODE_EF: the high stream

    def words(self) -> List[int]:
        return [self.elem_off, self.numel, self.k, self.tile_begin, self.n_tiles, self.mode, self.m_bits,
                self.n_hash, self.off_vals, self.off_filter, self.off_prefix, self.off_idx, self.val_cap,
                self.salt, self.n_filter_words, self.off_hint, self.vmode, self.off_coef, self.off_rankmap,
                self.off_selidx, self.off_sorted, self.poly_degree, self.rank_u32, self.poly_off, self.poly_ord,
                self.fixed_thr, self.shared_lb, self.pos_cap, self.off_pos_prefix, self.off_pick, self.ef_low_bits,
                self.off_hi]

    @property
    def ranked(self) -> bool:
        """The values travel as a fitted curve + the rank map of the shipped values (polyfit, dexp)."""
        return self.vmode in (VMODE_POLYFIT, VMODE_DEXP)

    @property
    def coded(self) -> bool:
        """A fix phase writes the residual (polyfit, QSGD, dexp, sign, fp8); emit knows the other modes' decoded
        values."""
        return self.vmode in (VMODE_POLYFIT, VMODE_QSGD, VMODE_DEXP, VMODE_SIGN, VMODE_FP8)

    @property
    def coef_words(self) -> int:
        """Words of a ranked tensor's curve, before its {num_pos, n} tail."""
        return DEXP_COEF_WORDS if self.vmode == VMODE_DEXP else MAX_SEGMENTS * (self.poly_degree + 1)

    @property
    def value_bytes(self) -> int:
        """Shipped bytes of the values (unpadded)."""
        if self.ranked:
            return 4 * (self.coef_words + 2) + (4 if self.rank_u32 else 2) * self.val_cap
        if self.vmode == VMODE_QSGD:
            return 4 * ((self.val_cap + 511) // 512) + self.val_cap * (2 if self.rank_u32 else 1)
        if self.vmode == VMODE_SIGN:
            return 4 * ((self.val_cap + 511) // 512) + 4 * ((self.val_cap + 31) // 32)
        if self.vmode == VMODE_FP8:
            return (self.val_cap + 31) // 32 + self.val_cap
        return (2 if self.vmode == VMODE_BF16 else 4) * self.val_cap

    @property
    def index_bytes(self) -> int:
        """Shipped bytes of the index (unpadded); 'randomk' ships none, every rank draws the index set itself."""
        if self.mode == MODE_BLOOM:                    # filter, per-tile prefix, hint; P2: positives per tile + the pick
            return 4 * (self.n_filter_words + self.n_tiles + (4 * self.n_tiles if self.off_hint else 0) +
                        (self.n_tiles + (self.pos_cap + 31) // 32 if self.pos_cap else 0))
        if self.mode == MODE_RLE:
            return 4 * ((self.n_tiles + 1) // 2 + rle_stream_words(self.val_cap))
        if self.mode == MODE_EF:
            _, lo, hi = spec.ef_layout(self.val_cap, self.n_tiles)
            return 4 * ((self.n_tiles + 1) // 2 + lo + hi)
        return 0 if self.mode == MODE_SHARED else 4 * self.val_cap


@dataclass
class BucketPlan:
    numels: Sequence[int]
    names: Optional[Sequence[str]] = None
    shapes: Optional[Sequence[tuple]] = None
    compress_ratio: float = 0.01
    index: Optional[str] = "bloom"        # 'bloom', 'rle' (lossless tile-local run coding), 'elias_fano' (lossless
                                          # tile-local Elias-Fano, spec.ef_layout) or None (plain top-k pairs)
    fpr: Optional[float] = None
    policy: str = "leftmost"
    min_numel: int = spec.SMALL_TENSOR_NUMEL
    max_hash: int = 16
    ks: Optional[Sequence[int]] = None    # explicit per-tensor K (overrides compress_ratio)
    hint: bool = True                     # ship the 1-bit-per-32-elements occupancy hint next to each bloom filter
    value: Optional[str] = None           # None (fp32 values), 'polyfit', 'qsgd', 'dexp', 'bf16', 'sign' or 'fp8'
                                          # ('both': an index codec + value codec)
    quantum_num: int = 127                # QSGD levels (int8 on the wire)
    poly_degree: int = 5
    poly_min_k: int = 512                 # tensors shipping fewer values keep them as fp32 (the fit header would be larger)
    dexp_min_numel: int = DEXP_MIN_NUMEL  # 'dexp' fits tensors of more elements than this (the per-tensor codec's rule)
    sparsifier: str = "topk"              # 'topk' (radix select of the K largest) | 'threshold' (|x| > threshold, variable K)
                                          # | 'randomk' (seeded index draw every rank repeats: only values are shipped)
    threshold: float = 0.0
    capacity_ratio: Optional[float] = None   # 'threshold': slot capacity as a fraction of d (default 1.0 = lossless)
    raw_slack: int = 0                    # plain-pair tensors: room for this many coordinates beyond K (the select keeps
                                          # every element sharing the threshold's 22-bit prefix; ops.topk_select resolves them)
    tensors: List[TensorPlan] = field(default_factory=list, init=False)

    def __post_init__(self):
        if self.index not in (None, "bloom", "rle", "elias_fano"):
            raise ValueError(f"fused engine index codecs: None, 'bloom', 'rle', 'elias_fano'; got {self.index!r}")
        if self.value not in (None, "polyfit", "qsgd", "dexp", "bf16", "sign", "fp8"):
            raise ValueError(f"fused engine value codecs: None, 'polyfit', 'qsgd', 'dexp', 'bf16', 'sign', 'fp8'; "
                             f"got {self.value!r}")
        if self.sparsifier not in ("topk", "threshold", "randomk"):
            raise ValueError(f"fused engine sparsifiers: 'topk', 'threshold', 'randomk'; got {self.sparsifier!r}")
        shared = self.sparsifier == "randomk"
        if shared and self.index is not None:
            raise ValueError("'randomk' ships no index (every rank draws the same set): pass index=None")
        if shared and self.value in ("polyfit", "dexp"):
            # rank_bin centres the value bins on the selection threshold, which here is a hash, not a magnitude
            raise NotImplementedError(f"'randomk' is fused with fp32, QSGD, bf16, sign or fp8 values, not with "
                                      f"{self.value!r}")
        if self.value == "qsgd" and not (1 <= int(self.quantum_num) <= 32767):
            raise ValueError("quantum_num must be in [1, 32767]")
        fixed_thr = 0
        if self.sparsifier == "threshold":
            # GRACE threshold: |x| > threshold  <=>  key > bits(threshold)  <=>  key >= bits(threshold) + 1
            thr = max(0.0, float(self.threshold))
            fixed_thr = int(np.array([thr], dtype=np.float32).view(np.uint32)[0]) + 1
        if self.policy == "conflict_sets" and (self.index != "bloom" or self.sparsifier != "topk"):
            # under 'threshold' K is the slot capacity (default d): the draw would keep every positive, false ones too
            raise ValueError("the fused 'conflict_sets' policy needs the bloom index and the top-k sparsifier")
        if self.policy not in POLICY_ID:
            raise ValueError(f"fused engine supports policies {list(POLICY_ID)}; got {self.policy!r}")
        names = list(self.names) if self.names is not None else [f"t{i}" for i in range(len(self.numels))]
        shapes = list(self.shapes) if self.shapes is not None else [(int(n),) for n in self.numels]
        elem = 0
        tile = 0
        word = SLOT_HEADER_WORDS + DYN_WORDS * len(self.numels)
        word = _align(word, 4)
        scratch: List[tuple] = []           # (tensor, kind, words) placed after the shipped payload
        for i, d in enumerate(self.numels):
            d = int(d)
            assert d > 0
            if self.ks is not None:
                k = max(1, min(d, int(self.ks[i])))
            elif fixed_thr:                    # variable K: the slot is provisioned for capacity_ratio * d coordinates
                cr = 1.0 if self.capacity_ratio is None else float(self.capacity_ratio)
                k = max(1, min(d, int(math.ceil(d * cr))))
            else:
                k = min(d, spec.topk_k(d, self.compress_ratio))
            n_tiles = (d + spec.TILE - 1) // spec.TILE
            tp = TensorPlan(name=names[i], numel=d, shape=tuple(shapes[i]), elem_off=elem, k=k, tile_begin=tile,
                            n_tiles=n_tiles, mode=MODE_RAW, salt=i, poly_degree=int(self.poly_degree),
                            fixed_thr=fixed_thr)
            if shared:
                # values only (+ the dyn header); the per-tile prefix is sender-local scratch the decode reads back
                tp.mode = MODE_SHARED
                tp.val_cap = randomk_capacity(d, k)
                tp.shared_lb = randomk_bound(d, k)
                if d > self.min_numel:
                    word = self._value_region(tp, word, scratch)
                else:
                    tp.off_vals = word
                    word = _align(word + tp.val_cap, 4)
                scratch.append((tp, "off_prefix", n_tiles))
            elif self.index == "bloom" and d > self.min_numel:
                n_hash, m_bits, n_words = spec.bloom_layout(k, d, self.fpr, self.max_hash)
                tp.mode = MODE_BLOOM
                tp.m_bits, tp.n_hash, tp.n_filter_words = m_bits, n_hash, n_words
                fpr = self.fpr if self.fpr is not None else spec.default_fpr(k, d)
                if self.policy == "p0":
                    tp.val_cap = min(d, k + int(math.ceil(2.0 * fpr * d)) + 64)
                else:
                    tp.val_cap = k
                if self.policy == "conflict_sets":
                    tp.pos_cap = min(d, k + int(math.ceil(2.0 * fpr * d)) + 64)
                    if n_hash > P2_MAX_HASH:
                        raise ValueError(f"conflict_sets: tensor {names[i]!r} has {n_hash} hash functions, more than the "
                                         f"{P2_MAX_HASH} the fused draw holds per positive; lower 'max_hash' or raise 'fpr'")
                    if tp.pos_cap > P2_MAX_POS_CAP:
                        raise ValueError(f"conflict_sets: tensor {names[i]!r} would draw over up to {tp.pos_cap} positives, "
                                         f"more than the {P2_MAX_POS_CAP} the fused draw holds; split it ('split_numel')")
                word = self._value_region(tp, word, scratch)
                tp.off_filter = word
                word = _align(word + n_words, 4)
                tp.off_prefix = word
                word = _align(word + n_tiles, 4)
                if self.hint:
                    tp.off_hint = word
                    word = _align(word + 4 * n_tiles, 4)
                if tp.pos_cap:
                    tp.off_pos_prefix = word
                    word = _align(word + n_tiles, 4)
                    tp.off_pick = word
                    word = _align(word + (tp.pos_cap + 31) // 32, 4)
            elif self.index == "rle" and d > self.min_numel:
                # lossless run coding of the selection bitmap, tile-local: a u16 count per tile and, per selected
                # element, the zeros+ones run offset from the tile start (< 4096 -> 12 bits), bit-packed; the values
                # (fp32, or a value codec with its fp32 values in sender-local scratch) come first
                tp.mode = MODE_RLE
                tp.val_cap = k
                word = self._value_region(tp, word, scratch)
                tp.off_prefix = word
                word = _align(word + (n_tiles + 1) // 2, 4)
                tp.off_idx = word
                word = _align(word + rle_stream_words(k), 4)
            elif self.index == "elias_fano" and d > self.min_numel:
                # lossless tile-local Elias-Fano (spec.ef_layout): the values, rle's u16 count per tile, then the low
                # and the high stream; a static size for the capacity k, whatever is selected
                tp.mode = MODE_EF
                tp.val_cap = k
                word = self._value_region(tp, word, scratch)
                tp.off_prefix = word
                word = _align(word + (n_tiles + 1) // 2, 4)
                tp.ef_low_bits, lo_words, hi_words = spec.ef_layout(k, n_tiles)
                tp.off_idx = word
                tp.off_hi = word + lo_words                  # the two streams back to back
                word = _align(tp.off_hi + hi_words, 4)
            else:
                tp.val_cap = min(d, k + int(self.raw_slack))
                if d > self.min_numel:           # value-only mode ('deepreduce': 'value'): coded values + plain indices
                    word = self._value_region(tp, word, scratch)
                else:
                    tp.off_vals = word
                    word = _align(word + tp.val_cap, 4)
                tp.off_idx = word
                word = _align(word + tp.val_cap, 4)
            self.tensors.append(tp)
            elem = _align(elem + d, ALIGN_ELEMS)
            tile += n_tiles
        self.total_elems = _align(elem, ALIGN_ELEMS)
        self.n_tiles = tile
        self.payload_words = word
        for tp, attr, n in scratch:            # sender-local scratch lives in the slot but is never pushed
            setattr(tp, attr, word)
            word = _align(word + n, 4)
        self.slot_words = _align(word, 64)
        self.poly_tables()                     # assigns poly_off / poly_ord

    def _value_region(self, tp: TensorPlan, word: int, scratch: list) -> int:
        """Lay out the value side of a tensor's slot region (fp32 values, or a value codec + sender-local scratch)."""
        poly = self.value == "polyfit" and tp.k >= self.poly_min_k
        dexp = self.value == "dexp" and tp.numel > self.dexp_min_numel
        if (poly or dexp) and tp.val_cap <= MAX_POLY_K:
            # curve coefficients + {num_pos, n} | rank map of the shipped values in their descending order
            tp.vmode = VMODE_POLYFIT if poly else VMODE_DEXP
            tp.rank_u32 = int(tp.val_cap > 65536)
            tp.off_coef = word
            word = _align(word + tp.coef_words + 2, 4)
            tp.off_rankmap = word
            word = _align(word + (tp.val_cap if tp.rank_u32 else (tp.val_cap + 1) // 2), 4)
            scratch += [(tp, "off_vals", tp.val_cap), (tp, "off_selidx", tp.val_cap), (tp, "off_sorted", tp.val_cap)]
        elif self.value == "qsgd":
            # bucketed QSGD (512 values per bucket): int8 levels (int16 when quantum_num >= 128, reference
            # pytorch/deepreduce.py:873) + one fp32 norm per bucket
            tp.vmode = VMODE_QSGD
            tp.poly_degree = int(self.quantum_num)      # field re-used: quantum_num
            tp.rank_u32 = int(self.quantum_num >= 128)  # field re-used: 16-bit levels
            tp.off_coef = word                           # norms
            word = _align(word + (tp.val_cap + 511) // 512, 4)
            tp.off_rankmap = word                        # levels
            word = _align(word + ((tp.val_cap + 1) // 2 if tp.rank_u32 else (tp.val_cap + 3) // 4), 4)
            scratch += [(tp, "off_vals", tp.val_cap), (tp, "off_selidx", tp.val_cap)]
        elif self.value == "sign":
            # scaled sign (codecs/sign.py), 512-value buckets: one fp32 scale per bucket + one sign bit per value; the
            # fix phase codes them from the fp32 values in sender-local scratch, as QSGD's does
            tp.vmode = VMODE_SIGN
            tp.off_coef = word                           # scales
            word = _align(word + (tp.val_cap + 511) // 512, 4)
            tp.off_rankmap = word                        # sign bits, LSB first
            word = _align(word + (tp.val_cap + 31) // 32, 4)
            scratch += [(tp, "off_vals", tp.val_cap), (tp, "off_selidx", tp.val_cap)]
        elif self.value == "fp8":
            # E4M3 values (codecs/fp8.py), a scale byte per 32-value block: the scale bytes, then the element bytes,
            # each four per word; the fix phase codes them from the fp32 values in sender-local scratch, as sign's does
            tp.vmode = VMODE_FP8
            tp.off_coef = word                           # scale bytes
            word = _align(word + (tp.val_cap + 127) // 128, 4)
            tp.off_rankmap = word                        # element bytes
            word = _align(word + (tp.val_cap + 3) // 4, 4)
            scratch += [(tp, "off_vals", tp.val_cap), (tp, "off_selidx", tp.val_cap)]
        else:
            # fp32 values, or bf16 values two per word (the p-th value in the low half of word p // 2): emit rounds them
            # as it gathers and knows the decoded value, so there is no sender scratch and no later phase
            tp.vmode = VMODE_BF16 if self.value == "bf16" else VMODE_FP32
            tp.off_vals = word
            word = _align(word + (tp.value_bytes + 3) // 4, 4)
        return word

    def poly_tables(self):
        """(ranked tensor ids, largest K first ; per-value tasks of the coded tensors {tensor, first value of a
        512-chunk})."""
        ids = sorted([i for i, t in enumerate(self.tensors) if t.ranked], key=lambda i: -self.tensors[i].val_cap)
        off = 0
        for o, i in enumerate(ids):
            self.tensors[i].poly_off, self.tensors[i].poly_ord = off, o
            off += self.tensors[i].val_cap
        self.poly_total = off
        coded = sorted([i for i, t in enumerate(self.tensors) if t.coded], key=lambda i: -self.tensors[i].val_cap)
        tasks = [(i, c) for i in coded for c in range(0, self.tensors[i].val_cap, 512)]
        ids_t = torch.tensor(ids if ids else [0], dtype=torch.int32)
        tasks_t = torch.tensor(tasks if tasks else [(0, 0)], dtype=torch.int32).reshape(-1)
        return ids_t, len(ids), tasks_t, len(tasks)

    def p2_tables(self):
        """Scratch of the P2 sender stage (ops/csrc/p2.cu): (int32 table of P2_ENTRY_WORDS per P2 tensor, scratch words,
        largest pos_cap).  Entry: {tensor, pos_idx, set_off, cursor, members, ord, last, tmp, misc, pair_cap} — word
        offsets into one int32 buffer.  pos_idx[pos_cap]: element of the q-th positive; set_off[m_bits + 1] / cursor
        [m_bits]: the counting sort of the (filter bit, positive) pairs; members[pos_cap * n_hash]: set members in bit
        order; ord / last[min(m_bits, pairs)]: the sets' visit order and the draw's last-visit counts (one entry per
        non-empty filter bit); tmp: reorder scratch of the sets with >= P2_SIZE_CAP members; misc[4]."""
        rows, off, cap_max = [], 0, 0
        for i, t in enumerate(self.tensors):
            if not t.pos_cap:
                continue
            pair_cap = t.pos_cap * t.n_hash
            n_sets = min(t.m_bits, pair_cap)
            n_large = min(t.m_bits, pair_cap // P2_SIZE_CAP)
            row = [i]
            for n in (t.pos_cap, t.m_bits + 1, t.m_bits, pair_cap, n_sets, n_sets, n_large, 4):
                row.append(off)
                off = _align(off + n, 4)
            row.append(pair_cap)
            rows.append(row)
            cap_max = max(cap_max, t.pos_cap)
        table = torch.tensor(rows if rows else [[0] * P2_ENTRY_WORDS], dtype=torch.int32).reshape(-1)
        return table, len(rows), max(off, 4), cap_max

    # ---- device tables -----------------------------------------------------
    def tensor_table(self) -> torch.Tensor:
        arr = np.array([t.words() for t in self.tensors], dtype=np.int64).astype(np.uint32).view(np.int32)
        return torch.from_numpy(arr.reshape(-1).copy())

    def tile_table(self) -> torch.Tensor:
        """[n_tiles, 4] int32: {tensor id, element offset in the flat buffers, valid count, offset inside the tensor}."""
        out = np.empty((self.n_tiles, 4), dtype=np.int64)
        for i, t in enumerate(self.tensors):
            loc = np.arange(t.n_tiles, dtype=np.int64) * spec.TILE
            rows = out[t.tile_begin:t.tile_begin + t.n_tiles]
            rows[:, 0] = i
            rows[:, 1] = t.elem_off + loc
            rows[:, 2] = np.minimum(spec.TILE, t.numel - loc) | ((1 << 31) if t.n_tiles == 1 else 0)
            rows[:, 3] = loc
        return torch.from_numpy(out.astype(np.uint32).view(np.int32).copy())

    def cost_prefix(self, seg_cost: float = 6.0, single_cost: float = 2.0) -> torch.Tensor:
        """[n_tiles + 1] int32 cumulative tile costs for the kernel's equal-cost partition (``tile_range``): a tile costs
        its share of 4096 elements, plus ``seg_cost`` tiles' worth where a multi-tile tensor starts (histogram merge,
        ticket, resolve, filter staging) and ``single_cost`` for a one-tile tensor.  Units: 1/16 tile."""
        c = np.zeros(self.n_tiles, dtype=np.int64)
        for t in self.tensors:
            loc = np.arange(t.n_tiles, dtype=np.int64) * spec.TILE
            n = np.minimum(spec.TILE, t.numel - loc)
            c[t.tile_begin:t.tile_begin + t.n_tiles] = np.maximum(1, np.rint(16.0 * n / spec.TILE)).astype(np.int64)
            c[t.tile_begin] += int(round(16 * (single_cost if t.n_tiles == 1 else seg_cost)))
        pre = np.concatenate([[0], np.cumsum(c)])
        assert pre[-1] < 2 ** 31
        return torch.from_numpy(pre.astype(np.int32))

    def phase_cuts(self, grid: int, speeds=None, weights=None) -> torch.Tensor:
        """[4, grid + 1] int32: first tile of every CTA for the kernel's four phase classes (accumulate / insert / query /
        emit, ``Part`` in ops/csrc/plan.h).  Class c cuts the tiles where the cumulative cost (``cost_prefix`` with the
        class's own segment / one-tile weights, ``PART_WEIGHTS``) reaches the cumulative share of the CTAs' relative
        ``speeds[c]`` ([4, grid], default all ones): a CTA on a slower SM gets proportionally less work."""
        weights = PART_WEIGHTS if weights is None else weights
        out = np.zeros((len(weights), grid + 1), dtype=np.int64)
        for c, (seg_c, single_c) in enumerate(weights):
            pre = self.cost_prefix(seg_c, single_c).numpy().astype(np.float64)
            sp = np.ones(grid) if speeds is None else np.maximum(np.asarray(speeds[c], dtype=np.float64), 1e-3)
            share = np.concatenate([[0.0], np.cumsum(sp)]) / sp.sum()
            cuts = np.searchsorted(pre, pre[-1] * share[1:-1], side="left")
            out[c, 1:-1] = np.minimum(np.maximum.accumulate(cuts), self.n_tiles)
            out[c, -1] = self.n_tiles
        return torch.from_numpy(out.astype(np.int32))

    def cta_ranges(self, grid: int, balanced: bool = True):
        """(begin, end) tile range of every CTA of a `grid`-CTA launch — mirrors ``tile_range`` in engine.cu."""
        if not balanced:
            return [(self.n_tiles * b // grid, self.n_tiles * (b + 1) // grid) for b in range(grid)]
        pre = self.cost_prefix().numpy().astype(np.int64)
        total = int(pre[-1])
        cuts = [0] + [int(np.searchsorted(pre, total * b // grid, side="left")) for b in range(1, grid)] + [self.n_tiles]
        return [(cuts[b], cuts[b + 1]) for b in range(grid)]

    def stage2_layout(self, world: int):
        """(entries, words) of a stage-2 slot of the sharded decode.  A rank's slice receives what all W senders
        selected inside it: about sum(K) entries when selections are spread evenly, but up to W * sum(K) (or every
        element of the slice) when they cluster — e.g. hot embedding rows.  The default capacity is that worst case,
        so the exchange can never drop entries; the payload actually pushed is only the live count.  DR_S2_SLACK=<f>
        selects the compact sizing f * sum(K) + 8192 instead (overflow is then reported as engine status 6)."""
        import os
        k_total = sum(t.val_cap for t in self.tensors)
        slack = os.environ.get("DR_S2_SLACK", "")
        if slack:
            cap = int(float(slack) * k_total) + 8192
        else:
            slice_elems = (self.n_tiles + world - 1) // world * spec.TILE
            cap = min(world * k_total, slice_elems) + 64
        cap = _align(cap, 4)
        return cap, _align(4 + 2 * cap, 64)

    def arena_words(self, world: int, shard: bool = True) -> int:
        words = ARENA_HDR_WORDS + 2 * world * self.slot_words
        if shard and world > 1:
            words += 2 * world * self.stage2_layout(world)[1]
        return words

    def slot_offset(self, world: int, parity: int, src: int) -> int:
        """Word offset in an arena of sender `src`'s slot of the given step parity (plan.h ``slot_offset``)."""
        return ARENA_HDR_WORDS + (parity * world + src) * self.slot_words

    def stage2_offset(self, world: int, parity: int, src: int) -> int:
        """Word offset in an arena of sender `src`'s stage-2 slot of the given step parity (plan.h ``s2_offset``)."""
        return ARENA_HDR_WORDS + 2 * world * self.slot_words + (parity * world + src) * self.stage2_layout(world)[1]

    # ---- accounting --------------------------------------------------------
    def wire_bytes(self) -> int:
        """Bytes a rank ships per step (the pushed payload)."""
        return self.payload_words * 4

    def dense_bytes(self) -> int:
        return sum(t.numel for t in self.tensors) * 4

    def topk_pair_bytes(self) -> int:
        """What plain top-k (fp32 value + int64 index, GRACE) would ship."""
        return sum(t.k * 12 for t in self.tensors)

    def views(self, flat: torch.Tensor):
        """Per-tensor views into a flat bucket buffer."""
        return [flat[t.elem_off:t.elem_off + t.numel].view(t.shape) for t in self.tensors]
