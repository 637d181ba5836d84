"""Python driver + torch oracle for the fused bucket engine (``ops/csrc/engine.cu``).

``BucketEngine`` owns the flat gradient / residual buffers of one bucket, the
select state, the symmetric arena (CUDA IPC, or NVLS-capable symmetric memory
with ``DR_NVLS=1``, for W>1) and the C++ ``Engine`` context; ``step()`` launches
the single persistent kernel that does sparsify → encode → P2P push → sharded
decode → slice exchange for the whole bucket.

``engine_oracle`` is the plain-PyTorch specification of the same step,
including the wire format of the slot, used by the tests (GPU kernels vs
oracle: slots bit-exact, dense output allclose).

Parity with the reference (hangxu0304/DeepReduce), per tensor of the bucket:
  * residual compensate / update  — GRACE ResidualMemory, TF twin tensorflow/deepreduce.py:31-52;
  * top-k select                  — GRACE TopK (``torch.topk(abs(x), k)``), here a 22-bit-threshold radix select;
  * bloom insert / universe query / policy / FP-aware re-gather — pytorch/deepreduce.py:457-492,505-529;
  * 'both' (index first, value codec on the re-gathered values, mapping back) — :250-302;
    polyfit segments / fit / restore — :341-425; QSGD — :861-907;
  * per-rank decode + aggregate (+ average) — GRACE Allgather communicator, reference README.md:37;
  * lossless run-length index (``'index': 'rle'``) — :805-846, here tile-local (see ``ops/csrc/plan.h``);
  * lossless tile-local Elias-Fano index (``'index': 'elias_fano'``, ``spec.ef_layout``) — no reference counterpart.
"""
from __future__ import annotations

import math
import os

from collections import OrderedDict
from typing import Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist

from .. import spec
from ..codecs.bf16 import bf16_bits_oracle, bf16_widen_oracle
from ..codecs.bloom import bloom_insert_oracle, bloom_query_oracle, conflict_sets_oracle
from ..codecs.fp8 import fp8_decode_oracle, fp8_encode_oracle
from ..codecs.polyfit import get_segments, polyfit_eval_oracle, polyfit_fit_oracle
from ..codecs.qsgd import qsgd_decode_oracle, qsgd_encode_oracle
from ..codecs.sign import sign_decode_oracle, sign_encode_oracle
from ..grace.memory import clip_factor, is_dense, pairwise_sumsq
from .plan import update_cta_speeds
from .plan import (DYN_WORDS, HIST_BINS, MODE_BLOOM, MODE_EF, MODE_RLE, MODE_SHARED, NUM_HIST, POLICY_ID, SLOT_HEADER_WORDS,
                   VMODE_BF16, VMODE_DEXP, VMODE_FP8, VMODE_QSGD, VMODE_SIGN, BucketPlan, rle_stream_words)

(PH_ACCUM, PH_FALLBACK, PH_HIST2, PH_INSERT, PH_QUERY, PH_EMIT, PH_RANK_HIST, PH_RANK_SCAN, PH_RANK_SCATTER,
 PH_RANK_EXACT, PH_FIT, PH_FIX, PH_PUSH, PH_SIGNAL, PH_EXPAND, PH_DECODE, PH_COMPACT, PH_PUSH2, PH_SIGNAL2,
 PH_SCATTER, PH_END) = range(21)
MAGIC = 0xD33B2000
STATUS_NAMES = {0: "ok", 1: "(unused)", 2: "peer flag watchdog", 3: "select resolve failed", 4: "grid barrier watchdog", 5: "TMA mbarrier watchdog",
                6: "stage-2 slot overflow (sharded decode)",
                7: "ranks disagree on the 'randomk' draw (a sender's header differs from the receiver's)"}


def status_error(row) -> str:
    """The error text of an engine status word ``[code, aux, ...]`` with a non-zero code."""
    return f"deepreduce engine error: {STATUS_NAMES.get(int(row[0]), int(row[0]))} (aux={int(row[1])})"


class StatusPoller:
    """Failure detection without a host sync: each ``poll`` copies the engines' status words to pinned host memory on
    the current stream, and reads the copy the previous call enqueued once its event has completed (a step later)."""

    def __init__(self):
        self._host, self._event, self._labels = None, None, []

    def poll(self, engines) -> Optional[tuple]:
        """``engines``: ``(label, BucketEngine)`` pairs.  Returns ``(label, status_error text)`` of the first failed
        engine in the previous call's copy, and then enqueues nothing; else enqueues the copy and returns None."""
        if self._event is not None and self._event.query():
            for label, row in zip(self._labels, self._host.tolist()):
                if row[0] != 0:
                    return label, status_error(row)
        if not engines:
            return None
        if self._host is None or len(self._host) != len(engines):
            self._host = torch.zeros(len(engines), 8, dtype=torch.int32).pin_memory()
            self._event = torch.cuda.Event()
        for b, (_, e) in enumerate(engines):
            self._host[b].copy_(e.status, non_blocking=True)
        self._labels = [label for label, _ in engines]
        self._event.record()
        return None


# ---------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------
def rle_pack12(pos: np.ndarray, cap: int) -> np.ndarray:
    """12-bit fields, LSB-first, entry j at bit 12*j (the kModeRle index stream)."""
    out = np.zeros(rle_stream_words(cap), dtype=np.uint64)
    j = np.arange(pos.size, dtype=np.int64)
    bit = 12 * j
    w, sh = bit >> 5, (bit & 31).astype(np.uint64)
    v = pos.astype(np.uint64) << sh                       # up to 43 bits
    np.bitwise_or.at(out, w, v & np.uint64(0xFFFFFFFF))
    np.bitwise_or.at(out, w + 1, v >> np.uint64(32))
    return out.astype(np.uint32)


def rle_unpack12(stream: np.ndarray, n: int) -> np.ndarray:
    j = np.arange(n, dtype=np.int64)
    bit = 12 * j
    w, sh = bit >> 5, (bit & 31).astype(np.uint64)
    s64 = stream.astype(np.uint64)
    both = s64[w] | (s64[np.minimum(w + 1, s64.size - 1)] << np.uint64(32))
    return ((both >> sh) & np.uint64(0xFFF)).astype(np.int64)


def ef_pack(idx: np.ndarray, numel: int, cap: int):
    """The tile-local Elias-Fano index (``spec.ef_layout``) of the ascending in-tensor indices ``idx`` (at most ``cap``
    of them) of a ``numel``-element tensor: uint32 words (u16 count per tile, low stream, high stream)."""
    n_tiles = (int(numel) + spec.TILE - 1) // spec.TILE
    L, lo_words, hi_words = spec.ef_layout(int(cap), n_tiles)
    idx = np.asarray(idx, dtype=np.int64)
    assert idx.size <= cap and np.all(np.diff(idx) > 0) and (idx.size == 0 or (idx[0] >= 0 and idx[-1] < numel))
    tile, e = idx // spec.TILE, idx % spec.TILE
    p = np.arange(idx.size, dtype=np.int64)
    cnt = np.zeros(((n_tiles + 1) // 2) * 2, dtype=np.uint16)
    cnt[:n_tiles] = np.bincount(tile, minlength=n_tiles)
    lo = np.zeros(lo_words + 1, dtype=np.uint64)
    if L:
        bit = p * L
        v = (e & ((1 << L) - 1)).astype(np.uint64) << (bit & 31).astype(np.uint64)     # up to 43 bits
        np.bitwise_or.at(lo, bit >> 5, v & np.uint64(0xFFFFFFFF))
        np.bitwise_or.at(lo, (bit >> 5) + 1, v >> np.uint64(32))
    hb = p + tile * (spec.TILE >> L) + (e >> L)
    hi = np.zeros(hi_words, dtype=np.uint32)
    np.bitwise_or.at(hi, hb >> 5, np.left_shift(np.uint32(1), (hb & 31).astype(np.uint32)))
    return cnt.view(np.uint32), lo[:lo_words].astype(np.uint32), hi


def ef_unpack(cnt_words: np.ndarray, lo: np.ndarray, hi: np.ndarray, numel: int, cap: int, n: int) -> np.ndarray:
    """The receiver side of ``ef_pack``: the ``n`` ascending in-tensor indices, read tile by tile as the kernel does
    (the j-th set bit q of tile t's range gives e = ((q - pre_t - t * B - j) << L) | low(pre_t + j))."""
    n_tiles = (int(numel) + spec.TILE - 1) // spec.TILE
    L, lo_words, hi_words = spec.ef_layout(int(cap), n_tiles)
    B = spec.TILE >> L
    cnt = np.asarray(cnt_words, dtype=np.uint32).view(np.uint16)[:n_tiles].astype(np.int64)
    assert int(cnt.sum()) == n <= cap, (int(cnt.sum()), n, cap)
    bits = np.unpackbits(np.asarray(hi, dtype=np.uint32)[:hi_words].view(np.uint8), bitorder="little")
    lo64 = np.concatenate([np.asarray(lo, dtype=np.uint32)[:lo_words], [0]]).astype(np.uint64)
    out, pre = [], 0
    for t in range(n_tiles):
        c = int(cnt[t])
        rng = bits[pre + t * B:pre + c + (t + 1) * B]
        q = np.flatnonzero(rng)
        assert q.size == c, (t, q.size, c)           # the range holds exactly the tile's entries
        j = np.arange(c, dtype=np.int64)
        h = q - j
        assert np.all(h < B)
        p = pre + j
        if L:
            bit = p * L
            w, sh = bit >> 5, (bit & 31).astype(np.uint64)
            low = (((lo64[w] | (lo64[w + 1] << np.uint64(32))) >> sh) & np.uint64((1 << L) - 1)).astype(np.int64)
        else:
            low = np.zeros(c, dtype=np.int64)
        out.append(t * spec.TILE + ((h << L) | low))
        pre += c
    idx = np.concatenate(out) if out else np.zeros(0, dtype=np.int64)
    assert idx.size == 0 or idx[-1] < numel
    return idx


def _abs_keys(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int32).to(torch.int64) & 0x7FFFFFFF


def select_topk_oracle(acc: torch.Tensor, k: int):
    """The engine's selection rule (normative, see ops/csrc/plan.h): with key = |x| bit pattern and
    T22 = (K-th largest key) >> 9, select every element with (key >> 9) >= max(T22, 1).  At least K
    elements (when K non-zeros exist) plus the few sharing the threshold's 22-bit prefix; exact zeros
    never.  Returns (ascending indices, threshold key lower bound)."""
    keys = _abs_keys(acc)
    kth = int(torch.topk(keys, k, sorted=True).values[-1].item())
    T22 = max(kth >> 9, 1)
    sel = torch.nonzero((keys >> 9) >= T22).flatten()
    return sel, T22 << 9


def select_threshold_oracle(acc: torch.Tensor, fixed_thr: int):
    """'threshold' sparsifier (GRACE: |x| > threshold): every element whose |x| bit pattern is >= fixed_thr."""
    return torch.nonzero(_abs_keys(acc) >= fixed_thr).flatten(), int(fixed_thr)


def select_randomk_oracle(numel: int, k: int, epoch: int, salt: int):
    """'randomk' selection rule of the fused engine (normative, see ops/csrc/plan.h): with
    key(i) = (0xFFFFFFFF - policy_hash(i, policy_seed(epoch, salt))) >> 1, the top-k rule on the keys.  A superset of
    the K smallest hashes plus the few sharing the threshold's 22-bit prefix; it depends on (numel, K, epoch, salt)
    only, so every rank computes the same set.  Returns (ascending indices, threshold key lower bound)."""
    h = spec.policy_hash(torch.arange(int(numel), dtype=torch.int64), spec.policy_seed(int(epoch), int(salt)))
    keys = (0xFFFFFFFF - h) >> 1
    kth = int(torch.topk(keys, int(k), sorted=True).values[-1].item())
    T22 = max(kth >> 9, 1)
    return torch.nonzero((keys >> 9) >= T22).flatten(), T22 << 9


def random_policy_filter(pos: torch.Tensor, n_ins: int, limit: int, epoch: int, salt: int, T: Optional[int] = None):
    """'random' policy of the fused engine: keep the positives x with policy_hash(x, policy_seed(step, tensor)) <= T,
    T = floor(2^32 * min(n_ins, limit) / n_pos) (0xFFFFFFFF = keep all when nothing has to go).  Sender: T from the
    counts; receiver: T from the header (pass it in).  Returns (surviving positives, T)."""
    if T is None:
        n_pos, target = int(pos.numel()), min(int(n_ins), int(limit))
        T = 0xFFFFFFFF if n_pos <= target else (target << 32) // n_pos
    if T != 0xFFFFFFFF:
        pos = pos[spec.policy_hash(pos, spec.policy_seed(epoch, salt)) <= T]
    return pos, T


def conflict_sets_pick_oracle(tp, pos: torch.Tensor, seed: int, epoch: int):
    """P2 of the fused engine: the draw over the first ``tp.pos_cap`` positives (ascending), as a bitmask over their
    ranks.  Returns (picked positives ascending, pick words uint32[ceil(pos_cap / 32)])."""
    head = pos[:tp.pos_cap]
    if head.numel():
        sel = conflict_sets_oracle(head, tp.k, tp.n_hash, tp.m_bits, seed, spec.policy_seed(epoch, tp.salt))
        sel = sel.to(torch.int64).cpu()
    else:
        sel = head
    bits = np.zeros(((tp.pos_cap + 31) // 32) * 32, dtype=np.uint8)
    bits[torch.searchsorted(head, sel).numpy()] = 1
    words = np.packbits(bits.reshape(-1, 32)[:, ::-1], axis=1).view(">u4").astype(np.uint32).reshape(-1)
    return sel, words


def conflict_sets_keep_oracle(tp, pos: torch.Tensor, pick_words: np.ndarray) -> torch.Tensor:
    """Receiver side of P2: the positives whose rank q is below pos_cap and set in the shipped pick."""
    head = pos[:tp.pos_cap]
    q = np.arange(head.numel(), dtype=np.int64)
    keep = (pick_words.astype(np.int64)[q >> 5] >> (q & 31)) & 1
    return head[torch.from_numpy(keep.astype(bool))]


def dexp_runs_fit_oracle(desc: torch.Tensor, num_pos: int) -> torch.Tensor:
    """'dexp' of the fused engine (VMODE_DEXP): the values in descending order split at num_pos (the positives) into two
    runs, each fitted by ``codecs.dexp.double_exponential_fit`` (fp64) on its own abscissa (i + 1) / length: the
    positives by ascending value, the rest by ascending magnitude.  Returns the shipped fp32 words
    (a, b, p, q) of the positive run, then of the rest."""
    from ..codecs.dexp import double_exponential_fit
    desc = desc.detach().cpu().double()
    runs = (desc[:num_pos].flip(0), -desc[num_pos:])
    return torch.stack([c for y in runs for c in double_exponential_fit(y)]).float()


def dexp_runs_eval_oracle(coef: torch.Tensor, num_pos: int, n: int) -> torch.Tensor:
    """The fitted values of the n ranks (descending order) from the shipped fp32 words: fp64 evaluation
    (``codecs.dexp.double_exponential_eval``), rounded to fp32, negated on the non-positive run."""
    from ..codecs.dexp import double_exponential_eval
    return torch.cat([double_exponential_eval(coef[:4], num_pos).flip(0),
                      -double_exponential_eval(coef[4:], n - num_pos)])


def _ranked_curve(t, a: np.ndarray) -> torch.Tensor:
    """The fitted values of a ranked tensor's ranks (descending order), from the curve words and the {num_pos, n} tail
    in its slot region: the sender's residual and every receiver's decode go through this one evaluation."""
    nc = t.coef_words
    coef = torch.from_numpy(a[t.off_coef:t.off_coef + nc].view(np.float32).copy())
    num_pos, n = int(a[t.off_coef + nc]), int(a[t.off_coef + nc + 1])
    if t.vmode == VMODE_DEXP:
        return dexp_runs_eval_oracle(coef, num_pos, n)
    return polyfit_eval_oracle(coef, get_segments(n, num_pos), t.poly_degree)


def _write_rank_map(tp, slot: np.ndarray, rank: torch.Tensor):
    n = int(rank.numel())
    if tp.rank_u32:
        slot[tp.off_rankmap:tp.off_rankmap + n] = rank.numpy().astype(np.uint32)
    else:
        r16 = np.zeros(((n + 1) // 2) * 2, dtype=np.uint16)
        r16[:n] = rank.numpy().astype(np.uint16)
        slot[tp.off_rankmap:tp.off_rankmap + (n + 1) // 2] = r16.view(np.uint32)


def _read_rank_map(t, a: np.ndarray, n: int) -> torch.Tensor:
    if t.rank_u32:
        return torch.from_numpy(a[t.off_rankmap:t.off_rankmap + n].astype(np.int64))
    return torch.from_numpy(a[t.off_rankmap:t.off_rankmap + (n + 1) // 2].view(np.uint16)[:n].astype(np.int64))


def encode_tensor_oracle(tp, acc: torch.Tensor, slot: np.ndarray, t_index: int, policy: str, seed: int, epoch: int = 1):
    """Encode one tensor into `slot` (uint32 numpy view); returns new residual."""
    if tp.mode == MODE_SHARED:
        sel_topk, T = select_randomk_oracle(tp.numel, tp.k, epoch, tp.salt)
    elif getattr(tp, "fixed_thr", 0):
        sel_topk, T = select_threshold_oracle(acc, tp.fixed_thr)
    else:
        sel_topk, T = select_topk_oracle(acc, tp.k)
    dyn = SLOT_HEADER_WORDS + DYN_WORDS * t_index
    resid = acc.clone()
    if tp.mode == MODE_BLOOM:
        words = bloom_insert_oracle(sel_topk, tp.n_hash, tp.m_bits, seed)
        pos = bloom_query_oracle(words, tp.numel, tp.n_hash, tp.m_bits, seed)
        if tp.off_hint:
            # occupancy hint: bit g of the tile's 128-bit field <=> the 32-element group g holds a selected element;
            # positives outside occupied groups are dropped on both sides (they can only be false positives)
            groups = torch.unique(sel_topk // 32)
            occ = torch.zeros((tp.numel + 31) // 32, dtype=torch.bool)
            occ[groups] = True
            pos = pos[occ[pos // 32]]
            hint = np.zeros(4 * tp.n_tiles, dtype=np.uint32)
            g = groups.numpy().astype(np.int64)
            tile, gi = g // 128, g % 128            # group gi of a tile covers elements [32*gi, 32*gi+32) of that tile...
            # ...in the kernel's (slot c, warp w) order: element e = c*512 + w*32 + lane  ->  gi = e // 32 = c*16 + w
            np.bitwise_or.at(hint, tile * 4 + gi // 32, (np.uint32(1) << (gi % 32).astype(np.uint32)))
            slot[tp.off_hint:tp.off_hint + 4 * tp.n_tiles] = hint
        limit = tp.val_cap if policy == "p0" else min(tp.k, tp.val_cap)
        n_pos = int(pos.numel())
        if policy == "random":
            # P1: seeded Bernoulli draw of rate target/n_pos over the positives (ops/csrc/engine.cu::policy_filter); the
            # acceptance threshold travels in header word 2, the receiver repeats the test on its own positives
            # (T now names the acceptance threshold: that is what header word 2 carries for this policy)
            pos, T = random_policy_filter(pos, int(sel_topk.numel()), limit, epoch, tp.salt)
        if policy == "conflict_sets":
            # P2: the draw over the first pos_cap positives, shipped as a bitmask over their ranks plus the positives
            # before every tile (ops/csrc/p2.cu); the receiver keeps exactly the picked positives
            starts_p = torch.arange(tp.n_tiles, dtype=torch.int64) * spec.TILE
            slot[tp.off_pos_prefix:tp.off_pos_prefix + tp.n_tiles] = \
                torch.clamp(torch.searchsorted(pos.cpu(), starts_p), max=tp.pos_cap).numpy().astype(np.uint32)
            pos, pick = conflict_sets_pick_oracle(tp, pos.cpu(), seed, epoch)
            slot[tp.off_pick:tp.off_pick + pick.size] = pick
        sel = pos[:limit]
        slot[tp.off_filter:tp.off_filter + tp.n_filter_words] = words.cpu().numpy().view(np.uint32)
        starts = torch.arange(tp.n_tiles, dtype=torch.int64) * spec.TILE
        slot[tp.off_prefix:tp.off_prefix + tp.n_tiles] = torch.searchsorted(sel.cpu(), starts).numpy().astype(np.uint32)
        cutoff = int(sel[-1].item()) if int(pos.numel()) >= limit and limit > 0 else 0xFFFFFFFF
        if policy == "conflict_sets":
            cutoff = 0xFFFFFFFF                # the pick says which positives carry values
    elif tp.mode == MODE_RLE:
        n_pos = int(sel_topk.numel())
        limit = tp.val_cap
        sel = sel_topk[:limit]
        s_np = sel.cpu().numpy().astype(np.int64)
        cnt = np.zeros(((tp.n_tiles + 1) // 2) * 2, dtype=np.uint16)
        cnt[:tp.n_tiles] = np.bincount(s_np // spec.TILE, minlength=tp.n_tiles).astype(np.uint16)
        slot[tp.off_prefix:tp.off_prefix + (tp.n_tiles + 1) // 2] = cnt.view(np.uint32)
        slot[tp.off_idx:tp.off_idx + rle_stream_words(tp.val_cap)] = rle_pack12(s_np % spec.TILE, tp.val_cap)
        cutoff = int(sel[-1].item()) if n_pos >= limit else 0xFFFFFFFF
    elif tp.mode == MODE_EF:
        # the run-length index's shipped set, counts and cutoff; the in-tile offsets as the two Elias-Fano streams
        n_pos = int(sel_topk.numel())
        limit = tp.val_cap
        sel = sel_topk[:limit]
        cnt, lo, hi = ef_pack(sel.cpu().numpy(), tp.numel, tp.val_cap)
        slot[tp.off_prefix:tp.off_prefix + cnt.size] = cnt
        slot[tp.off_idx:tp.off_idx + lo.size] = lo
        slot[tp.off_hi:tp.off_hi + hi.size] = hi
        cutoff = int(sel[-1].item()) if n_pos >= limit else 0xFFFFFFFF
    elif tp.mode == MODE_SHARED:
        # no index on the wire: every receiver draws the same set (the per-tile prefix is sender-local scratch)
        n_pos = int(sel_topk.numel())
        limit = tp.val_cap
        sel = sel_topk[:limit]
        cutoff = int(sel[-1].item()) if n_pos >= limit else 0xFFFFFFFF
    else:
        n_pos = int(sel_topk.numel())
        limit = tp.val_cap
        sel = sel_topk[:limit]                 # capacity K: the left-most of the (>= K) selected
        slot[tp.off_idx:tp.off_idx + sel.numel()] = sel.cpu().numpy().astype(np.uint32)
        cutoff = int(sel[-1].item()) if n_pos >= limit else 0xFFFFFFFF
    vals = acc[sel].float()
    n = int(sel.numel())
    if tp.ranked:
        # 'both': stable descending sort -> rank map; the fitted curve is shipped, the residual keeps value - fitted
        order = torch.sort(vals, descending=True, stable=True).indices
        rank = torch.empty(n, dtype=torch.int64)
        rank[order] = torch.arange(n)
        num_pos = int((vals > 0).sum())
        if tp.vmode == VMODE_DEXP:
            coef = dexp_runs_fit_oracle(vals[order], num_pos)
        else:
            coef = polyfit_fit_oracle(vals[order], get_segments(n, num_pos), tp.poly_degree)
        nc = tp.coef_words
        slot[tp.off_coef:tp.off_coef + nc] = coef.numpy().view(np.uint32)
        slot[tp.off_coef + nc] = num_pos
        slot[tp.off_coef + nc + 1] = n
        _write_rank_map(tp, slot, rank)
        fitted = _ranked_curve(tp, slot)[rank]
        resid[sel] = vals - fitted
        vals = fitted
    elif tp.vmode == VMODE_QSGD:
        q = int(tp.poly_degree)
        lvl, norms = qsgd_encode_oracle(vals, q, 512, 0x51ED + epoch)
        dec = qsgd_decode_oracle(lvl, norms, q, 512) if n else vals
        nb = (n + 511) // 512
        slot[tp.off_coef:tp.off_coef + nb] = norms.float().numpy().view(np.uint32)
        if tp.rank_u32:                      # quantum_num >= 128: 16-bit levels
            l16 = np.zeros(((n + 1) // 2) * 2, dtype=np.int16)
            l16[:n] = lvl.numpy().astype(np.int16)
            slot[tp.off_rankmap:tp.off_rankmap + (n + 1) // 2] = l16.view(np.uint32)
        else:
            l8 = np.zeros(((n + 3) // 4) * 4, dtype=np.int8)
            l8[:n] = lvl.numpy().astype(np.int8)
            slot[tp.off_rankmap:tp.off_rankmap + (n + 3) // 4] = l8.view(np.uint32)
        resid[sel] = vals - dec
        vals = dec
    elif tp.vmode == VMODE_SIGN:
        # scaled sign: a scale per 512-value bucket and a bit per value; the residual keeps v - d where d is finite,
        # and is 0 where it is not (a NaN or inf in the bucket)
        bits, scales = sign_encode_oracle(vals)
        slot[tp.off_coef:tp.off_coef + scales.numel()] = scales.numpy().view(np.uint32)
        slot[tp.off_rankmap:tp.off_rankmap + bits.numel()] = bits.numpy().view(np.uint32)
        dec = sign_decode_oracle(bits, scales, n)
        resid[sel] = torch.where(torch.isfinite(dec), vals - dec, torch.zeros_like(dec))
        vals = dec
    elif tp.vmode == VMODE_FP8:
        # E4M3 values with a scale byte per 32-value block; the residual keeps v - d where d is finite, and is 0 where
        # it is not (an inf or a NaN in the block)
        scales, elems = fp8_encode_oracle(vals)
        slot[tp.off_coef:tp.off_coef + scales.numel()] = scales.numpy().view(np.uint32)
        slot[tp.off_rankmap:tp.off_rankmap + elems.numel()] = elems.numpy().view(np.uint32)
        dec = fp8_decode_oracle(scales, elems, n)
        resid[sel] = torch.where(torch.isfinite(dec), vals - dec, torch.zeros_like(dec))
        vals = dec
    elif tp.vmode == VMODE_BF16:
        # bf16 values (round to nearest even, NaN -> 0x7FC0), two per word; the residual keeps the exact rounding error
        # where the widened value is finite, and is 0 (as for fp32 values) where it is not
        q = np.zeros(((n + 1) // 2) * 2, dtype=np.uint16)
        bits = bf16_bits_oracle(vals)
        q[:n] = bits.numpy().astype(np.uint16)
        slot[tp.off_vals:tp.off_vals + (n + 1) // 2] = q.view(np.uint32)
        dec = bf16_widen_oracle(bits)
        resid[sel] = torch.where(torch.isfinite(dec), vals - dec, torch.zeros_like(dec))
        vals = dec
    else:
        slot[tp.off_vals:tp.off_vals + sel.numel()] = vals.cpu().numpy().view(np.uint32)
        resid[sel] = 0
    slot[dyn + 0] = sel.numel()
    slot[dyn + 1] = cutoff
    slot[dyn + 2] = T
    slot[dyn + 3] = n_pos
    return resid, sel, vals


def owner_spans(plan: BucketPlan, owner: Optional[Sequence[int]] = None) -> list:
    """Per plan tensor, (first tile, tile count) of the parameter it belongs to: ``owner[j]`` is the parameter of plan
    tensor j (``split_large``; default: one each).  A parameter's chunks must be consecutive plan tensors."""
    tensors = plan.tensors
    owner = list(range(len(tensors))) if owner is None else [int(o) for o in owner]
    if len(owner) != len(tensors):
        raise ValueError(f"owner has {len(owner)} entries for the plan's {len(tensors)} tensors")
    spans, j = [None] * len(tensors), 0
    while j < len(tensors):
        k = j
        while k + 1 < len(tensors) and owner[k + 1] == owner[j]:
            k += 1
        if owner[j] in owner[:j]:
            raise ValueError(f"owner {owner}: the chunks of parameter {owner[j]} are not consecutive")
        span = (tensors[j].tile_begin, sum(tensors[i].n_tiles for i in range(j, k + 1)))
        for i in range(j, k + 1):
            spans[i] = span
        j = k + 1
    return spans


def clip_oracle(plan: BucketPlan, g: torch.Tensor, thr: float, owner: Optional[Sequence[int]] = None) -> torch.Tensor:
    """'dgc' local gradient clipping of the flat fp32 gradient ``g`` (plan layout) at ``thr`` = c / sqrt(W): per
    parameter (the chunks of ``owner`` together), the squared norm by ``pairwise_sumsq`` over its elements in plan
    order, and g = fl32(g * f) where ``clip_factor`` gives a factor."""
    g = g.clone()
    spans = owner_spans(plan, owner)
    j = 0
    while j < len(plan.tensors):
        k = j
        while k + 1 < len(plan.tensors) and spans[k + 1] == spans[j]:
            k += 1
        chunks = [slice(t.elem_off, t.elem_off + t.numel) for t in plan.tensors[j:k + 1]]
        f = clip_factor(pairwise_sumsq(torch.cat([g[c] for c in chunks])), thr)
        if f is not None:
            for c in chunks:
                g[c] = g[c] * f
        j = k + 1
    return g


def tensor_decays(plan: BucketPlan, weight_decay: float = 0.0, weight_decays: Optional[Sequence[float]] = None,
                  owner: Optional[Sequence[int]] = None) -> list:
    """The weight decay factor of every plan tensor: ``weight_decays[owner[j]]`` for plan tensor j when one factor per
    parameter is given (``owner``: ``split_large``'s map, default one plan tensor each), else ``weight_decay``.  Every
    factor must be a finite number >= 0."""
    n = len(plan.tensors)
    if weight_decays is None:
        out = [weight_decay] * n
    else:
        owner = list(range(n)) if owner is None else [int(o) for o in owner]
        if len(owner) != n or len(weight_decays) != (max(owner) + 1 if owner else 0):
            raise ValueError(f"weight_decays: {len(weight_decays)} factors for owner {owner} of the plan's {n} tensors")
        out = [weight_decays[o] for o in owner]
    for wd in out:
        if isinstance(wd, bool) or not isinstance(wd, (int, float)) or not math.isfinite(wd) or wd < 0:
            raise ValueError(f"weight decay factors must be finite numbers >= 0 (got {wd!r})")
    return [float(wd) for wd in out]


def decay_oracle(plan: BucketPlan, g: torch.Tensor, w: torch.Tensor, decays: Sequence[float]) -> torch.Tensor:
    """d = g + (decays[j] * w), two roundings, over every plan tensor j whose factor is not 0, its padding included
    (where w is 0); the other tensors keep g as it is, and their w is never used (a NaN there changes nothing)."""
    lam = torch.zeros(plan.total_elems, dtype=torch.float32)
    ends = [t.elem_off for t in plan.tensors[1:]] + [plan.total_elems]
    for t, end, wd in zip(plan.tensors, ends, decays):
        lam[t.elem_off:end] = float(wd)
    return torch.where(lam != 0, g + (lam * w), g)


def engine_oracle(plan: BucketPlan, grads: Sequence[torch.Tensor], resids: Sequence[torch.Tensor], *, beta=1.0,
                  gamma=1.0, average=True, seed=spec.DEFAULT_SEED, epoch=1, momentum=None, moms=None,
                  weight_decay=0.0, weights=None, clip_norm=None, owner=None, nesterov=False, weight_decays=None):
    """One bucket step for W ranks on the CPU.  grads/resids: per-rank flat
    buffers (plan.total_elems).  Returns (dense_out, new_resids, slots).

    ``momentum`` set ('dgc' memory, beta = gamma = 1): ``moms`` are the per-rank momenta u, the step is
    u = momentum * u + g, r = r + u (each a separately rounded fp32 op) before the select, and u is cleared wherever
    the rank's own decoded value is non-zero; returns (dense_out, new_resids, slots, new_moms).

    ``weight_decay`` wd != 0 (with ``momentum``): ``weights`` are the per-rank parameters, flat in plan layout (zeros in
    the padding), and g is replaced by d = g + (wd * w), two roundings, before the momentum.

    ``clip_norm`` c (with ``momentum``): ahead of that, each rank's gradient is clipped per parameter at c / sqrt(W)
    (``clip_oracle``; ``owner`` maps the plan tensors to parameters as ``split_large`` returns it).

    ``weight_decays`` (with ``momentum``, instead of ``weight_decay``): one factor per parameter, mapped to the plan
    tensors through ``owner`` (``tensor_decays``); a tensor whose factor is 0 keeps g (``decay_oracle``).

    ``nesterov`` (with ``momentum`` > 0): Nesterov momentum, r = r + v with v = d + (momentum * u), the new u, instead
    of r = r + u; u itself is unchanged."""
    W = len(grads)
    dgc = momentum is not None
    if dgc and (beta != 1.0 or gamma != 1.0 or moms is None or len(moms) != W):
        raise ValueError("engine_oracle: momentum needs beta = gamma = 1 and one momentum buffer per rank")
    if weight_decay != 0.0 and (not dgc or weights is None or len(weights) != W):
        raise ValueError("engine_oracle: weight_decay needs momentum and one parameter buffer per rank")
    decays = None
    if weight_decays is not None:
        if weight_decay != 0.0:
            raise ValueError("engine_oracle: give weight_decay or weight_decays, not both")
        decays = tensor_decays(plan, 0.0, weight_decays, owner)
        if any(decays) and (not dgc or weights is None or len(weights) != W):
            raise ValueError("engine_oracle: weight_decays needs momentum and one parameter buffer per rank")
    if clip_norm is not None and not dgc:
        raise ValueError("engine_oracle: clip_norm needs momentum")
    if nesterov and not (dgc and float(momentum) > 0.0):
        raise ValueError("engine_oracle: nesterov needs a momentum > 0")
    out = torch.zeros(plan.total_elems, dtype=torch.float32)
    new_resids, slots, new_moms = [], [], []
    for r in range(W):
        g = grads[r].detach().cpu().float()
        res = resids[r].detach().cpu().float()
        if clip_norm is not None:
            g = clip_oracle(plan, g, float(clip_norm) / math.sqrt(W), owner)
        if weight_decay != 0.0:
            g = g + (float(weight_decay) * weights[r].detach().cpu().float())
        elif decays is not None and any(decays):
            g = decay_oracle(plan, g, weights[r].detach().cpu().float(), decays)
        if dgc:
            u = float(momentum) * moms[r].detach().cpu().float() + g
            acc_flat = res + (g + (float(momentum) * u) if nesterov else u)
        else:
            acc_flat = beta * res + gamma * g if beta != 0.0 else gamma * g
        slot = np.zeros(plan.payload_words, dtype=np.uint32)
        slot[0:5] = [MAGIC, epoch, len(plan.tensors), plan.payload_words, r]
        nres = acc_flat.clone()
        for ti, tp in enumerate(plan.tensors):
            seg = slice(tp.elem_off, tp.elem_off + tp.numel)
            resid_t, sel, vals = encode_tensor_oracle(tp, acc_flat[seg], slot, ti, plan.policy, seed, epoch)
            nres[seg] = resid_t
            out[seg].index_add_(0, sel, vals)
            if dgc:                                  # momentum factor masking on the own decoded contribution
                u[seg][sel[vals != 0]] = 0.0
        new_resids.append(nres)
        slots.append(slot)
        if dgc:
            new_moms.append(u)
    if average:
        out = out / W
    if dgc:
        return out, new_resids, slots, new_moms
    return out, new_resids, slots


def decode_slot_oracle(plan: BucketPlan, slot, *, seed=spec.DEFAULT_SEED) -> torch.Tensor:
    """Receiver-side specification: rebuild one sender's dense contribution (flat, ``plan.total_elems``, unscaled)
    from NOTHING but the plan and the words of its slot — what ``phase_decode`` does per (tile, sender).  Together
    with ``encode_tensor_oracle`` this pins the wire format from both ends: the tests check that the sum of the
    decoded slots equals the aggregate ``engine_oracle`` builds on the sender side."""
    a = slot.detach().cpu().numpy().view(np.uint32) if torch.is_tensor(slot) else np.asarray(slot, dtype=np.uint32)
    assert int(a[0]) == MAGIC and int(a[2]) == len(plan.tensors), "not a slot of this plan"
    out = torch.zeros(plan.total_elems, dtype=torch.float32)
    for ti, t in enumerate(plan.tensors):
        idx = shipped_index_oracle(plan, a, ti, seed=seed)
        n = int(idx.numel())
        if n == 0:
            continue
        if t.ranked:
            vals = _ranked_curve(t, a)[_read_rank_map(t, a, n)]
        elif t.vmode == VMODE_QSGD:
            norms = torch.from_numpy(a[t.off_coef:t.off_coef + (n + 511) // 512].view(np.float32).copy())
            if t.rank_u32:
                lvl = torch.from_numpy(a[t.off_rankmap:t.off_rankmap + (n + 1) // 2].view(np.int16)[:n].astype(np.int64))
            else:
                lvl = torch.from_numpy(a[t.off_rankmap:t.off_rankmap + (n + 3) // 4].view(np.int8)[:n].astype(np.int64))
            vals = qsgd_decode_oracle(lvl, norms, int(t.poly_degree), 512)
        elif t.vmode == VMODE_SIGN:
            scales = torch.from_numpy(a[t.off_coef:t.off_coef + (n + 511) // 512].view(np.float32).copy())
            bits = torch.from_numpy(a[t.off_rankmap:t.off_rankmap + (n + 31) // 32].view(np.int32).copy())
            vals = sign_decode_oracle(bits, scales, n)
        elif t.vmode == VMODE_FP8:
            scales = torch.from_numpy(a[t.off_coef:t.off_coef + (n + 127) // 128].view(np.int32).copy())
            elems = torch.from_numpy(a[t.off_rankmap:t.off_rankmap + (n + 3) // 4].view(np.int32).copy())
            vals = fp8_decode_oracle(scales, elems, n)
        elif t.vmode == VMODE_BF16:
            bits = a[t.off_vals:t.off_vals + (n + 1) // 2].view(np.uint16)[:n].astype(np.int64)
            vals = bf16_widen_oracle(torch.from_numpy(bits))
        else:
            vals = torch.from_numpy(a[t.off_vals:t.off_vals + n].view(np.float32).copy())
        out[t.elem_off:t.elem_off + t.numel].index_add_(0, idx, vals.float())
    return out


def shipped_index_oracle(plan: BucketPlan, slot, ti: int, *, seed=spec.DEFAULT_SEED) -> torch.Tensor:
    """The ascending element indices (within tensor ``ti``) whose values one sender's slot carries, rebuilt from the
    plan and the slot's words alone; the p-th shipped value belongs to the p-th index."""
    a = slot.detach().cpu().numpy().view(np.uint32) if torch.is_tensor(slot) else np.asarray(slot, dtype=np.uint32)
    t = plan.tensors[ti]
    d0 = SLOT_HEADER_WORDS + DYN_WORDS * ti
    n_sel, cutoff = int(a[d0]), int(a[d0 + 1])
    if n_sel == 0:
        return torch.empty(0, dtype=torch.int64)
    if t.mode == MODE_BLOOM:
        words = torch.from_numpy(a[t.off_filter:t.off_filter + t.n_filter_words].view(np.int32).copy())
        pos = bloom_query_oracle(words, t.numel, t.n_hash, t.m_bits, seed)          # ascending positives of the universe
        if t.off_hint:                                                               # only inside occupied 32-element groups
            hint = a[t.off_hint:t.off_hint + 4 * t.n_tiles]
            grp = pos // 32                                                          # group id: tile*128 + (e // 32)
            tile, gi = grp // 128, grp % 128
            bit = (torch.from_numpy(hint.astype(np.int64))[tile * 4 + gi // 32] >> (gi % 32)) & 1
            pos = pos[bit.bool()]
        if plan.policy == "random":
            pos, _ = random_policy_filter(pos, 0, 0, int(a[1]), t.salt, T=int(a[d0 + 2]))
        if plan.policy == "conflict_sets":
            starts = torch.arange(t.n_tiles, dtype=torch.int64) * spec.TILE
            pp = torch.from_numpy(a[t.off_pos_prefix:t.off_pos_prefix + t.n_tiles].astype(np.int64))
            assert torch.equal(torch.clamp(torch.searchsorted(pos, starts), max=t.pos_cap), pp), t.name
            pos = conflict_sets_keep_oracle(t, pos, a[t.off_pick:t.off_pick + (t.pos_cap + 31) // 32])
        if cutoff != 0xFFFFFFFF:
            pos = pos[pos <= cutoff]
        idx = pos[:n_sel]
        # the per-tile prefix table must agree with what the receiver recomputes (the kernel starts ranks from it)
        starts = torch.arange(t.n_tiles, dtype=torch.int64) * spec.TILE
        pre = torch.from_numpy(a[t.off_prefix:t.off_prefix + t.n_tiles].astype(np.int64))
        assert torch.equal(torch.minimum(torch.searchsorted(pos, starts), torch.tensor(n_sel)), pre), t.name
    elif t.mode == MODE_RLE:
        cnt = a[t.off_prefix:t.off_prefix + (t.n_tiles + 1) // 2].view(np.uint16)[:t.n_tiles].astype(np.int64)
        assert int(cnt.sum()) == n_sel, t.name
        local = rle_unpack12(a[t.off_idx:t.off_idx + rle_stream_words(t.val_cap)], n_sel)
        idx = torch.from_numpy(np.repeat(np.arange(t.n_tiles, dtype=np.int64), cnt) * spec.TILE + local)
    elif t.mode == MODE_EF:
        _, lo_words, hi_words = spec.ef_layout(t.val_cap, t.n_tiles)
        idx = torch.from_numpy(ef_unpack(a[t.off_prefix:t.off_prefix + (t.n_tiles + 1) // 2],
                                         a[t.off_idx:t.off_idx + lo_words], a[t.off_hi:t.off_hi + hi_words],
                                         t.numel, t.val_cap, n_sel))
    elif t.mode == MODE_SHARED:
        # the index set is drawn again from the plan and the epoch in slot word 1; the sender's threshold must match
        pos, thr = select_randomk_oracle(t.numel, t.k, int(a[1]), t.salt)
        assert thr == int(a[d0 + 2]), (t.name, thr, int(a[d0 + 2]))
        if cutoff != 0xFFFFFFFF:
            pos = pos[pos <= cutoff]
        idx = pos[:n_sel]
        assert int(idx.numel()) == n_sel, t.name
    else:
        idx = torch.from_numpy(a[t.off_idx:t.off_idx + n_sel].astype(np.int64))
    return idx


# ---------------------------------------------------------------------------
# engine
# ---------------------------------------------------------------------------
def stats_from_slot(plan: BucketPlan, slot) -> dict:
    """Per-step counters of one sender, read from the 4-word dynamic header every tensor carries in the slot
    (``{n_sel, cutoff, thr_bits, n_pos}``, written on the device by the emit phase — SURVEY §5 "per-step counters
    accumulated on device"): shipped coordinates, bloom positives / false positives among the universe, the magnitude
    threshold of the selection, and the wire bytes by component (static, from the plan)."""
    a = slot.detach().cpu().numpy().view(np.uint32) if torch.is_tensor(slot) else np.asarray(slot, dtype=np.uint32)
    per, tot = [], {"k": 0, "n_sel": 0, "n_pos": 0, "false_pos": 0, "value_bytes": 0, "index_bytes": 0}
    p2_tot = {"beyond_cap": 0, "tensors_beyond_cap": 0}
    for ti, t in enumerate(plan.tensors):
        d0 = SLOT_HEADER_WORDS + DYN_WORDS * ti
        n_sel, cutoff, thr_bits, n_pos = (int(x) for x in a[d0:d0 + 4])
        thr = float(np.array([thr_bits], dtype=np.uint32).view(np.float32)[0])
        # bloom: positives beyond the K inserted (upper bound under 22-bit ties)
        false_pos = max(0, n_pos - min(t.k, n_pos)) if t.mode == MODE_BLOOM else 0
        row = {"name": t.name, "numel": t.numel, "k": t.k, "n_sel": n_sel, "n_pos": n_pos, "false_pos": false_pos,
               "threshold": thr, "cutoff": None if cutoff == 0xFFFFFFFF else cutoff,
               "value_bytes": t.value_bytes, "index_bytes": t.index_bytes}
        if plan.policy == "random" and t.mode == MODE_BLOOM:   # header word 2 is the policy's acceptance threshold here
            row["threshold"] = None
            row["accept_rate"] = 1.0 if thr_bits == 0xFFFFFFFF else thr_bits / 2.0 ** 32
        if t.mode == MODE_SHARED:                            # header word 2 is a hash-key threshold, not a magnitude
            row["threshold"] = None
        if t.pos_cap:                                        # P2: positives past pos_cap that the draw never saw
            row["beyond_cap"] = max(0, n_pos - t.pos_cap)
            p2_tot["beyond_cap"] += row["beyond_cap"]
            p2_tot["tensors_beyond_cap"] += int(row["beyond_cap"] > 0)
        per.append(row)
        for key in tot:
            tot[key] += row[key]
    if plan.policy == "conflict_sets":
        tot.update(p2_tot)
    tot["header_bytes"] = 4 * (SLOT_HEADER_WORDS + DYN_WORDS * len(plan.tensors))
    tot["wire_bytes"] = plan.wire_bytes()
    tot["dense_bytes"] = plan.dense_bytes()
    tot["relative_volume"] = tot["wire_bytes"] / max(1, tot["dense_bytes"])
    return {"tensors": per, "total": tot}


def total_stats(engines) -> dict:
    """``stats()["total"]`` of the last exchanged step summed over ``engines``, with its relative volume; synchronises."""
    torch.cuda.synchronize(engines[0].device)
    tot: dict = {}
    for e in engines:
        for k, v in e.stats()["total"].items():
            tot[k] = tot.get(k, 0) + v
    tot["relative_volume"] = tot["wire_bytes"] / max(1, tot["dense_bytes"])
    return tot


class BucketEngine:
    """One flat bucket + its fused exchange kernel."""

    def __init__(self, plan: BucketPlan, device=None, group=None, *, beta: float = 1.0, gamma: float = 1.0,
                 average: bool = True, use_history: bool = True, blocks_per_sm: int = 2,
                 seed: int = spec.DEFAULT_SEED, spin_limit: int = 20_000_000, world: Optional[int] = None,
                 rank: Optional[int] = None, filter_smem_bytes: Optional[int] = None, use_tma: bool = True,
                 hist_shift: int = 22, shard: Optional[bool] = None, transport: Optional[str] = None,
                 peer_timeout_ms: Optional[int] = None, fault: int = 0, grad_dtype: torch.dtype = torch.float32,
                 momentum: Optional[float] = None, weight_decay: float = 0.0, clip_norm: Optional[float] = None,
                 owner: Optional[Sequence[int]] = None, grad: Optional[torch.Tensor] = None, nesterov: bool = False,
                 weight_decays: Optional[Sequence[float]] = None):
        # grad: adopt this flat gradient buffer (``plan.total_elems`` of ``grad_dtype`` on ``device``) instead of
        # allocating one, so that views into it (``p.grad``) stay valid across engines of the same layout (the sparsity
        # warm-up's stage switch); calibrate_partition scribbles on it like on an own buffer
        # grad_dtype=torch.bfloat16: the flat gradient (in: local, out: aggregate) is bf16.  The residual, the select,
        # the codecs and the wire stay fp32 (widening bf16 is exact), so the engine computes exactly what an fp32 engine
        # fed the widened gradient computes, and rounds the aggregate once (to nearest even) where it is final.  The
        # rounding error is not fed back into the residual, as torch's bf16 DDP does with its reduced sum.
        if grad_dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"grad_dtype must be torch.float32 or torch.bfloat16 (got {grad_dtype})")
        # momentum=m: the 'dgc' memory.  An fp32 momentum buffer ``mom`` next to the residual: u = m*u + g, r = r + u
        # before the select, u cleared wherever this rank's own decoded value is non-zero (engine_oracle)
        if momentum is not None and (float(beta) != 1.0 or float(gamma) != 1.0 or not 0.0 <= float(momentum) < 1.0):
            raise ValueError(f"momentum needs beta = gamma = 1 and a value in [0, 1) (got beta={beta}, gamma={gamma}, "
                             f"momentum={momentum})")
        self.momentum = None if momentum is None else float(momentum)
        # weight_decay=wd ('dgc' only): d = g + wd*w ahead of the momentum, w read from the parameters that
        # ``bind_parameters`` points the kernel at (engine_oracle(weight_decay=..., weights=...))
        wd = weight_decay
        if isinstance(wd, bool) or not isinstance(wd, (int, float)) or not math.isfinite(wd) or wd < 0:
            raise ValueError(f"weight_decay must be a finite number >= 0 (got {wd!r})")
        if wd != 0 and momentum is None:
            raise ValueError("weight_decay is added inside the 'dgc' memory: it needs momentum")
        self.weight_decay = float(wd)
        # weight_decays: one factor per original parameter (``owner``'s numbering) instead of weight_decay: one value
        # for all, or 0 for the parameters excluded from the decay ('weight_decay_exclude'); decays: the factor of
        # every plan tensor
        if weight_decays is not None and wd != 0:
            raise ValueError("give weight_decay or weight_decays, not both")
        self.decays = tensor_decays(plan, self.weight_decay, weight_decays, owner)
        if any(self.decays) and momentum is None:
            raise ValueError("weight_decays are added inside the 'dgc' memory: they need momentum")
        self.reads_parameters = any(self.decays)     # some tensor takes the decay: phase 0 reads its parameter
        if len(set(d for d in self.decays if d != 0.0)) > 1:
            raise ValueError(f"weight_decays: one factor for every parameter, or 0 to exclude one (got "
                             f"{sorted(set(self.decays))})")
        self._bound = None                       # (parameters, owner, data_ptrs, strides) of the last bind_parameters
        # nesterov=True ('dgc' only, momentum > 0): r = r + (d + m*u) with the new u (engine_oracle(nesterov=True))
        if not isinstance(nesterov, bool):
            raise ValueError(f"nesterov must be True or False (got {nesterov!r})")
        if nesterov and not (momentum is not None and float(momentum) > 0.0):
            raise ValueError("nesterov needs the 'dgc' momentum, with a momentum > 0")
        self.nesterov = nesterov
        # clip_norm=c ('dgc' only): DGC's local gradient clipping of every parameter at c / sqrt(W), ahead of the weight
        # decay; ``owner`` (split_large) makes the chunks of a split parameter one norm (engine_oracle(clip_norm=...))
        c = clip_norm
        if c is not None:
            if isinstance(c, bool) or not isinstance(c, (int, float)) or not math.isfinite(c) or c <= 0:
                raise ValueError(f"clip_norm must be a finite number > 0 (got {c!r})")
            if momentum is None:
                raise ValueError("clip_norm clips inside the 'dgc' memory: it needs momentum")
        self.clip_norm = None if c is None else float(c)
        self.owner = None if owner is None else [int(o) for o in owner]
        from .. import ops
        self.mod = ops.cuda_module()
        self.plan = plan
        self.grad_dtype = grad_dtype
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.group = group
        if world is None:
            world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
            rank = dist.get_rank(group) if dist.is_available() and dist.is_initialized() else 0
        self.world, self.rank = int(world), int(rank or 0)
        self.beta, self.gamma, self.average = float(beta), float(gamma), bool(average)
        self.epoch = 0
        # sharded decode (W > 1): each rank decodes 1/W of the tiles for all senders, then the exact slices are
        # exchanged by a second in-kernel push.  DR_SHARD=0 restores the every-rank-decodes-everything path.
        self.shard = (os.environ.get("DR_SHARD", "1") != "0") if shard is None else bool(shard)
        # transport of the compressed slots between ranks: 'p2p' = in-kernel stores into peer-mapped arenas (one
        # NVLink/NVSwitch domain, the default), 'nccl' = encode phases -> ONE in-place NCCL all_gather of the slots per
        # bucket -> decode phases (ranks on different hosts, or no peer access).  None: DR_TRANSPORT, else auto.
        self.transport = self._pick_transport(transport)
        if self.transport == "nccl":
            self.shard = False
        dev = self.device
        nT, nt = len(plan.tensors), plan.n_tiles
        with torch.cuda.device(dev):
            if grad is None:
                self.grad = torch.zeros(plan.total_elems, dtype=grad_dtype, device=dev)
            elif (grad.shape != (plan.total_elems,) or grad.dtype != grad_dtype or grad.device != dev
                  or not grad.is_contiguous()):
                raise ValueError(f"grad must be a flat {grad_dtype} buffer of {plan.total_elems} elements on {dev} (got "
                                 f"{grad.dtype} {tuple(grad.shape)} on {grad.device})")
            else:
                self.grad = grad
            self.resid = torch.zeros(plan.total_elems, dtype=torch.float32, device=dev)
            self.mom = (torch.zeros(plan.total_elems, dtype=torch.float32, device=dev) if self.momentum is not None
                        else None)
            self.tensor_table = plan.tensor_table().to(dev)
            self.tile_table = plan.tile_table().to(dev)
            self.hist = torch.zeros(NUM_HIST * nT * HIST_BINS, dtype=torch.int32, device=dev)
            self.hist_total = torch.zeros(NUM_HIST * nT, dtype=torch.int32, device=dev)
            self.sel = torch.zeros(nT * 8, dtype=torch.int32, device=dev)
            # per-tile positive counts + two per-tensor counters (positives, inserted) used by the random policy
            self.tile_count = torch.zeros(nt + 2 * len(plan.tensors), dtype=torch.int32, device=dev)
            # scratch of the candidate / bitmask pipeline (ops/csrc/engine.cu): one mask word per 32-element group
            # (own positives, decode scratch) and the candidate lists — (key, in-tile offset) of every element above
            # the history bound, 256 slots per (tile, warp) at a fixed place (8 B per element, touched sparsely)
            self.pos_mask = torch.zeros(nt * 128, dtype=torch.int32, device=dev)
            # decode scratch: one mask slot per (sender, tile of the slice this rank decodes)
            span_max = (nt // self.world + 1) if (self.shard and self.world > 1) else nt
            self.dec_mask = torch.zeros(self.world * span_max * 128, dtype=torch.int32, device=dev)
            self.cand = torch.empty(nt * 4096 * 2, dtype=torch.int32, device=dev)
            self.cand_cnt = torch.zeros(nt * 16, dtype=torch.int32, device=dev)
            self.barrier = torch.zeros(16, dtype=torch.int32, device=dev)
            self.status = torch.zeros(8, dtype=torch.int32, device=dev)
            self._setup_arena()
            self.ctx = self.mod.Engine(
                self.tensor_table.data_ptr(), self.tile_table.data_ptr(), nT, nt, plan.slot_words, plan.payload_words,
                self.grad.data_ptr() if grad_dtype == torch.float32 else 0, self.resid.data_ptr(), self.hist.data_ptr(),
                self.hist_total.data_ptr(),
                self.sel.data_ptr(), self.tile_count.data_ptr(),
                self.barrier.data_ptr(), self.status.data_ptr(), self.arena_ptrs, self.rank, self.world)
            # equal-COST tile ranges per CTA (DR_BALANCE=0: equal counts)
            self.balanced = os.environ.get("DR_BALANCE", "1") != "0"
            if self.balanced:
                seg_c, single_c = (float(x) for x in os.environ.get("DR_SEG_COST", "6.0,2.0").split(","))
                self.cost_prefix = plan.cost_prefix(seg_c, single_c).to(dev)
                self.ctx.set_cost_prefix(self.cost_prefix.data_ptr())
            self.cta_speeds = None          # [4, grid] relative CTA speeds per phase class (calibrate_partition)
            self.cuts = None
            self.ctx.set_scratch(self.pos_mask.data_ptr(), self.dec_mask.data_ptr(), self.cand.data_ptr(),
                                 self.cand_cnt.data_ptr())
            if self.mom is not None:
                self.ctx.set_momentum(self.mom.data_ptr(), self.momentum, self.nesterov)
            # one parameter address per plan tensor (bind_parameters); the kernel reads it only where the decay is on
            # and the tensor's flag in ``decayed`` is set
            self.wparams = torch.zeros(nT, dtype=torch.int64, device=dev)
            self.decayed = torch.tensor([d != 0.0 for d in self.decays], dtype=torch.uint8, device=dev)
            self.clip_thr = None
            if self.clip_norm is not None:
                self.clip_thr = self.clip_norm / math.sqrt(self.world)
                spans = owner_spans(plan, self.owner)
                self.clip_owner = torch.tensor([v for sp in spans for v in sp], dtype=torch.int32, device=dev)
                self.clip_part = torch.zeros(nt, dtype=torch.float64, device=dev)
                self.clip_f = torch.ones(nT, dtype=torch.float32, device=dev)
                self.ctx.set_clip(self.clip_part.data_ptr(), self.clip_f.data_ptr(), self.clip_owner.data_ptr(),
                                  self.clip_thr)
            if grad_dtype == torch.bfloat16:
                # fp32 sums of the bloom apply (every sender of a tile is added before the one rounding): one 4096-float
                # row per tile this rank decodes; not needed when every bloom tensor is scattered by emit (W = 1, fp32
                # or bf16 values on the wire: emit knows the decoded value)
                applied = any(t.mode == MODE_BLOOM and (self.world > 1 or t.coded) for t in plan.tensors)
                acc_tiles = span_max if applied else 0
                self.acc32 = torch.zeros(max(acc_tiles, 1) * 4096, dtype=torch.float32, device=dev)
                self.ctx.set_bf16(self.grad.data_ptr(), self.acc32.data_ptr(), acc_tiles)
            # a peer that does not signal within this wall time is fatal (status 2, output poisoned, see wait_flags)
            if peer_timeout_ms is None:
                peer_timeout_ms = int(os.environ.get("DR_PEER_TIMEOUT_MS", "120000"))
            self.ctx.set_peer_timeout_ms(int(peer_timeout_ms))
            self.ctx.set_fault(int(fault))
            # DR_DETERMINISTIC=1: rank-ordered decode sums (bit-reproducible run to run); default: independent
            # (sender, tile) work items with RED.ADD.F32.  Sharded, every rank still ends with identical bits: the owner
            # of a slice computes it and the others receive its bits.  Unsharded (DR_SHARD=0, and always with the NCCL
            # transport) every rank sums every tile itself, and at W > 2 the RED.ADD order would let the ranks' bits
            # drift apart, so those engines always take the rank-ordered sums (at W = 2, 0 + a + b is order-free).
            self.deterministic = os.environ.get("DR_DETERMINISTIC", "0") == "1"
            self.rank_ordered = self.deterministic or (not self.shard and self.world > 2)
            self.ctx.set_deterministic(int(self.rank_ordered))
            scale = (1.0 / self.world) if average else 1.0
            if filter_smem_bytes is None:      # <1>: 128 regs, 1 CTA/SM; <2>: 64 regs, 2 CTAs/SM
                filter_smem_bytes = 160 * 1024 if blocks_per_sm < 2 else 80 * 1024
            if self.shard and self.world > 1:
                cap, s2w = plan.stage2_layout(self.world)
                self.ctx.set_shard(1, s2w, cap)
            if getattr(self, "multicast_ptr", 0):
                self.ctx.set_multicast(self.multicast_ptr)
            self.ctx.set_has_rle(int(any(t.mode in (MODE_RLE, MODE_EF) for t in plan.tensors)))
            # P2 ('conflict_sets'): scratch of the sender stage the C++ engine launches before emit (ops/csrc/p2.cu)
            p2_table, n_p2, p2_words, p2_cap = plan.p2_tables()
            self.p2_table = p2_table.to(dev)
            self.p2_scratch = torch.zeros(p2_words, dtype=torch.int32, device=dev)
            if n_p2:
                self.ctx.set_p2(self.p2_table.data_ptr(), n_p2, self.p2_scratch.data_ptr(), p2_cap)
            self.ctx.set_has_shared(int(any(t.mode == MODE_SHARED for t in plan.tensors)))
            self.ctx.set_has_bf16_values(int(any(t.vmode == VMODE_BF16 for t in plan.tensors)))
            ids, n_poly, tasks, n_tasks = plan.poly_tables()
            self.poly_ids, self.poly_tasks = ids.to(dev), tasks.to(dev)
            from .plan import RANK_BINS
            tot = max(int(plan.poly_total), 1)
            self.poly_bins = torch.zeros(max(n_poly, 1) * 2 * RANK_BINS, dtype=torch.int32, device=dev)
            self.bucket_val = torch.zeros(tot, dtype=torch.float32, device=dev)
            self.bucket_pos = torch.zeros(tot, dtype=torch.int32, device=dev)
            self.expand_buf = torch.zeros(self.world * tot, dtype=torch.float32, device=dev)
            self.ctx.set_poly(self.poly_ids.data_ptr(), n_poly, self.poly_tasks.data_ptr(), n_tasks,
                              self.poly_bins.data_ptr(), self.bucket_val.data_ptr(), self.bucket_pos.data_ptr(),
                              self.expand_buf.data_ptr(), int(plan.poly_total))
            self.ctx.configure(self.beta, self.gamma, scale, int(seed), POLICY_ID[plan.policy], int(use_history),
                               int(spin_limit), int(blocks_per_sm), int(filter_smem_bytes), int(use_tma), int(hist_shift))
            # per-phase-class partitions (own cost weights per class; per-CTA speeds once calibrated); DR_CUTS=0: the
            # single cost prefix above for every phase
            if self.balanced and os.environ.get("DR_CUTS", "1") != "0":
                self._set_cuts()
        self.grad_views = plan.views(self.grad)

    def _set_cuts(self):
        g = self.grid()
        self.cuts = self.plan.phase_cuts(g, self.cta_speeds).contiguous().to(self.device)
        self.ctx.set_cuts(self.cuts.data_ptr(), g)

    @torch.no_grad()
    def calibrate_partition(self, steps: int = 3, rounds: int = 2, gain: float = 0.8, verbose: bool = False):
        """Measure how fast every CTA of the persistent kernel gets through its share of the accumulate / insert / query /
        emit phases (``%globaltimer`` stamps, ``set_debug_times``) on synthetic gradients and re-cut the four tile
        partitions so that slow CTAs get less work.  Why: the two co-resident CTAs of an SM do not run the issue-bound
        phases at the same speed (per-CTA timelines from scripts/cta_timeline.py show the second-launched CTA of an SM
        slower in accumulate and query), and every phase ends at a grid barrier, i.e. lasts
        as long as its slowest CTA.  Collective at W > 1 (runs ``(rounds + 1) * (steps + 1)`` exchange steps).  Resets
        residual / select history / gradient afterwards; the step counter keeps running (flags are epoch-valued).
        Resets the momentum of a 'dgc' engine too.  Returns the per-round phase maxima / medians."""
        G = self.grid()
        dbg = torch.zeros((PH_END + 1) * G * 2, dtype=torch.int64, device=self.device)
        self.ctx.set_debug_times(dbg.data_ptr())
        gen = torch.Generator(device=self.device).manual_seed(977 + self.rank)
        speeds = np.ones((4, G)) if self.cta_speeds is None else np.asarray(self.cta_speeds, dtype=np.float64).copy()
        phases = (PH_ACCUM, PH_INSERT, PH_QUERY, PH_EMIT)
        log = []
        try:
            for rnd in range(rounds + 1):                  # the last round only measures the result
                dur = np.zeros((4, G))
                for i in range(steps + 1):
                    self.grad.normal_(generator=gen).mul_(1e-2)
                    dbg.zero_()
                    self.step()
                    torch.cuda.synchronize(self.device)
                    self.check_status()
                    if i == 0:
                        continue                           # first step of a round: no select history for the new cut
                    t = dbg.cpu().numpy().reshape(PH_END + 1, G, 2)
                    for c, ph in enumerate(phases):
                        dur[c] += (t[ph, :, 1] - t[ph, :, 0]) / 1e3 / steps
                log.append({"max_us": dur.max(axis=1).round(1).tolist(), "median_us": np.median(dur, axis=1).round(1).tolist()})
                if verbose and self.rank == 0:
                    print(f"[calibrate] round {rnd}: max {log[-1]['max_us']} median {log[-1]['median_us']}", flush=True)
                if rnd == rounds:
                    break
                for c in range(4):
                    speeds[c] = update_cta_speeds(speeds[c], dur[c], gain)   # finished early -> more work next cut
                self.cta_speeds = speeds
                self._set_cuts()
        finally:
            self.ctx.set_debug_times(0)
        self.reset_state()
        return log

    def memory_buffers(self) -> dict:
        """The engine's per-element memory by name: the residual ``resid``, and with a momentum ('dgc') ``mom``."""
        return {"resid": self.resid} if self.mom is None else {"resid": self.resid, "mom": self.mom}

    def reset_state(self):
        """Zero the memory buffers, the select history and the gradient buffer."""
        for t in (*self.memory_buffers().values(), self.sel, self.grad):
            t.zero_()

    # ---- arena -------------------------------------------------------------
    def _setup_arena(self):
        words = self.plan.arena_words(self.world, self.shard)
        self._ipc = self.world > 1
        if not self._ipc:
            self.arena = torch.zeros(words, dtype=torch.int32, device=self.device)
            self.arena_ptrs = [self.arena.data_ptr()]
            return
        self.multicast_ptr = 0
        if self.transport == "nccl":          # peers' slots arrive by all_gather into MY arena: nothing to map
            self._ipc = False
            self.arena = torch.zeros(words, dtype=torch.int32, device=self.device)
            self.arena_ptrs = [self.arena.data_ptr()] * self.world      # peer entries are never dereferenced
            return
        if os.environ.get("DR_NVLS", "0") == "1" and self._setup_arena_nvls(words):
            return
        # peer-map only the GPUs of this group's ranks (never every device of the box)
        devs = [None] * self.world
        dist.all_gather_object(devs, int(self.device.index or 0), group=self.group)
        self.mod.enable_peer_access([int(d) for d in devs])
        self._arena_ptr = self.mod.arena_alloc(words * 4)
        self.arena = self.mod.arena_as_tensor(self._arena_ptr, words, self.device.index or 0)
        handle = self.mod.arena_export(self._arena_ptr)
        handles = [None] * self.world
        dist.all_gather_object(handles, handle, group=self.group)
        self.arena_ptrs = []
        self._imported = []
        for r in range(self.world):
            if r == self.rank:
                self.arena_ptrs.append(self._arena_ptr)
            else:
                p = self.mod.arena_import(handles[r])
                self._imported.append(p)
                self.arena_ptrs.append(p)
        dist.barrier(group=self.group)

    def _pick_transport(self, transport: Optional[str]) -> str:
        t = transport or os.environ.get("DR_TRANSPORT", "") or "auto"
        if t not in ("auto", "p2p", "nccl"):
            raise ValueError(f"transport must be 'p2p', 'nccl' or None/'auto' (got {t!r})")
        if self.world == 1:
            return "p2p"
        if t != "auto":
            return t
        # auto: peer-mapped arenas need every rank on the same host.  torchrun exports LOCAL_WORLD_SIZE: when it equals
        # the size of the (default) group the answer is known without a collective
        lws = os.environ.get("LOCAL_WORLD_SIZE", "")
        if self.group is None and lws.isdigit() and int(lws) == self.world:
            return "p2p"
        import socket
        hosts = [None] * self.world
        dist.all_gather_object(hosts, socket.gethostname(), group=self.group)
        return "p2p" if len(set(hosts)) == 1 else "nccl"

    def _setup_arena_nvls(self, words: int) -> bool:
        """Arena in NVLS-capable symmetric memory (cuMem + multicast object, torch's symmetric-memory rendezvous does the
        handle exchange): peers' arenas are mapped like the IPC path and a multicast VA lets ONE store reach all of
        them through the NVSwitch.  Every rank must agree, so the outcome is all-reduced; False -> IPC path."""
        ok, hdl, t = 1, None, None
        try:
            import torch.distributed._symmetric_memory as symm
            t = symm.empty(words, dtype=torch.int32, device=self.device)
            grp = self.group if self.group is not None else dist.group.WORLD
            hdl = symm.rendezvous(t, group=grp)
            if int(hdl.multicast_ptr) == 0 or hdl.world_size != self.world:
                ok = 0
        except Exception as e:  # noqa: BLE001
            self._nvls_error = repr(e)
            ok = 0
        flag = torch.tensor([ok], device=self.device, dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            return False
        t.zero_()
        torch.cuda.synchronize(self.device)
        self._symm_tensor, self._symm_handle = t, hdl
        self.arena = t
        self.arena_ptrs = [int(p) for p in hdl.buffer_ptrs]
        self.multicast_ptr = int(hdl.multicast_ptr)
        self._ipc = False
        self._imported = []
        dist.barrier(group=self.group)
        return True

    def close(self):
        if getattr(self, "_ipc", False):
            torch.cuda.synchronize(self.device)
            if dist.is_initialized():
                dist.barrier(group=self.group)
            for p in self._imported:
                self.mod.arena_close(p)
            self._imported = []
            self.mod.arena_free(self._arena_ptr)
            self._ipc = False

    # ---- parameters ('dgc' weight decay) --------------------------------------
    def bind_parameters(self, parameters: Sequence[torch.Tensor], owner: Optional[Sequence[int]] = None):
        """Point the kernel at the parameters whose values the weight decay reads: ``parameters`` in plan order, one per
        original tensor, and ``owner[j]`` the parameter plan tensor j belongs to (``split_large``; default: one plan
        tensor each).  A chunk reads its parameter from the chunk's offset on.  Every parameter must be on this
        engine's device, of the bucket's dtype, and dense, so that its storage order is the order of its gradient in
        the bucket.  The table is uploaded on the current stream; call it again (or ``refresh_parameters``) when a
        parameter's storage moves."""
        params = list(parameters)
        owner = list(range(len(params))) if owner is None else [int(o) for o in owner]
        tensors = self.plan.tensors
        if len(owner) != len(tensors) or sorted(set(owner)) != list(range(len(params))):
            raise ValueError(f"bind_parameters: {len(params)} parameters and owner {owner} do not cover the plan's "
                             f"{len(tensors)} tensors")
        done = [0] * len(params)                 # elements of each parameter covered by its earlier chunks
        ptrs = []
        for j, t in enumerate(tensors):
            i = owner[j]
            p = params[i]
            if p.device != self.device or p.dtype != self.grad_dtype:
                raise ValueError(f"bind_parameters: parameter {i} ({t.name}) is {p.dtype} on {p.device}; the engine's "
                                 f"bucket is {self.grad_dtype} on {self.device}")
            if not is_dense(p):
                raise ValueError(f"bind_parameters: parameter {i} ({t.name}) is not dense in memory: its storage order "
                                 f"is not the order of its gradient in the bucket")
            ptrs.append(p.data_ptr() + done[i] * p.element_size())
            done[i] += t.numel
        for i, p in enumerate(params):
            if done[i] != p.numel():
                raise ValueError(f"bind_parameters: parameter {i} has {p.numel()} elements, the plan {done[i]}")
        self.wparams.copy_(torch.tensor(ptrs, dtype=torch.int64))
        self._bound = (params, owner, [p.data_ptr() for p in params], [tuple(p.stride()) for p in params])
        self.ctx.set_weight_decay(self.wparams.data_ptr(), max(self.decays), self.decayed.data_ptr())

    def refresh_parameters(self):
        """Before a launch: rebuild the parameter table if a bound parameter's storage moved (``p.data = ...``).  The
        check is a host-side comparison of data pointers; it raises if weight decay is on and nothing is bound.  A moved
        parameter must keep the strides it was bound with: the bucket holds its gradient in that storage order (e.g.
        ``model.to(memory_format=...)`` after the buckets were built raises here)."""
        if not self.reads_parameters:
            return
        if self._bound is None:
            raise RuntimeError("weight decay > 0 reads the parameters: call bind_parameters() before the first step")
        params, owner, ptrs, layouts = self._bound
        if any(p.data_ptr() != q for p, q in zip(params, ptrs)):
            changed = [i for i, (p, l) in enumerate(zip(params, layouts)) if tuple(p.stride()) != l]
            if changed:
                raise ValueError(f"weight decay: parameters {changed} of the bucket changed their layout since they "
                                 f"were bound; the bucket keeps their gradients in the old storage order")
            self.bind_parameters(params, owner)

    def parameter_buffer(self) -> torch.Tensor:
        """The bound parameters as one flat fp32 buffer in plan layout (zeros in the padding), what the kernel reads:
        the ``weights`` of ``engine_oracle``."""
        if self._bound is None:
            raise RuntimeError("no parameters are bound (bind_parameters)")
        params, owner, _, _ = self._bound
        out = torch.zeros(self.plan.total_elems, dtype=torch.float32, device=self.device)
        done = [0] * len(params)
        for j, t in enumerate(self.plan.tensors):
            p = params[owner[j]].detach()
            flat = p.as_strided((p.numel(),), (1,))                  # storage order
            out[t.elem_off:t.elem_off + t.numel] = flat[done[owner[j]]:done[owner[j]] + t.numel].float()
            done[owner[j]] += t.numel
        return out

    # ---- run ---------------------------------------------------------------
    def step(self, epoch: Optional[int] = None):
        """Launch the fused kernel on the current stream.  In: ``self.grad``
        (local dense grads).  Out: ``self.grad`` (aggregated), ``self.resid``."""
        self.refresh_parameters()
        self.epoch = self.epoch + 1 if epoch is None else int(epoch)
        if self.transport == "nccl" and self.world > 1:
            self._step_nccl()
        else:
            self.ctx.run(self.epoch, PH_ACCUM, PH_END)

    def _step_nccl(self):
        """Multi-host form of the step: the same kernel runs its encode phases, the slots travel by ONE in-place
        NCCL all_gather per bucket (the slot of rank r sits at index r of the parity's slot array in every arena, so
        the output buffer is the arena itself), then the kernel runs expand + decode.  Still no per-tensor
        collectives and no size exchange (static offsets), cf. the reference's 2-3 all_gathers per tensor."""
        W, sw = self.world, self.plan.slot_words
        self.ctx.run(self.epoch, PH_ACCUM, PH_PUSH)
        base = self.plan.slot_offset(W, self.epoch & 1, 0)
        out = self.arena[base:base + W * sw]
        dist.all_gather_into_tensor(out, out[self.rank * sw:(self.rank + 1) * sw], group=self.group)
        self.ctx.run(self.epoch, PH_EXPAND, PH_PUSH2)      # expand, probe pass, apply pass (unsharded: no stage 2)

    def run_phases(self, begin: int, end: int, epoch: Optional[int] = None):
        """Debug / unfused chain: run a sub-range of phases (one launch)."""
        if epoch is not None:
            self.epoch = int(epoch)
        self.ctx.run(self.epoch, begin, end)

    def run_unfused(self, epoch: Optional[int] = None):
        self.epoch = self.epoch + 1 if epoch is None else int(epoch)
        for ph in range(PH_ACCUM, PH_END):
            self.ctx.run(self.epoch, ph, ph + 1)

    def slot(self, src_rank: Optional[int] = None, epoch: Optional[int] = None) -> torch.Tensor:
        """int32 view of the local copy of `src_rank`'s slot for `epoch`."""
        e = self.epoch if epoch is None else epoch
        r = self.rank if src_rank is None else src_rank
        off = self.plan.slot_offset(self.world, e & 1, r)
        return self.arena[off:off + self.plan.payload_words]

    def stats(self, src_rank: Optional[int] = None, epoch: Optional[int] = None) -> dict:
        """Counters of the last step for one sender (default: this rank): see :func:`stats_from_slot`.  One small
        device-to-host copy of the slot's header region; call it off the critical path (e.g. every N steps)."""
        n_hdr = SLOT_HEADER_WORDS + DYN_WORDS * len(self.plan.tensors)
        return stats_from_slot(self.plan, self.slot(src_rank, epoch)[:n_hdr])

    def stage2_bytes(self) -> int:
        """Bytes this rank pushed in the stage-2 exchange of the last step (8 B per entry, to W-1 peers)."""
        if not (self.shard and self.world > 1):
            return 0
        cap = self.plan.stage2_layout(self.world)[0]
        n = min(int(self.arena[self.plan.stage2_offset(self.world, self.epoch & 1, self.rank)].item()), cap)
        return 8 * n * (self.world - 1)

    def check_status(self):
        st = self.status.cpu().tolist()
        if st[0] != 0:
            raise RuntimeError(status_error(st))

    def grid(self) -> int:
        return int(self.ctx.grid())

    # ---- state (checkpoint / resume; SURVEY §5) ----------------------------
    def state_dict(self):
        out = {k: t.detach().cpu().clone() for k, t in self.memory_buffers().items()}
        out.update(epoch=self.epoch, sel=self.sel.detach().cpu().clone())
        return out

    def load_state_dict(self, state):
        buffers = self.memory_buffers()
        if ("mom" in state) != ("mom" in buffers):
            raise ValueError("engine state of another memory: a 'dgc' engine loads only 'dgc' states (with 'mom'), "
                             "any other engine only states without it")
        for k, t in buffers.items():
            t.copy_(state[k].to(self.device))
        self.sel.copy_(state["sel"].to(self.device))
        # never move the step counter backwards inside a live process group: the peers' flags in the arena carry
        # epochs this engine has already used (e.g. during calibrate_partition)
        self.epoch = max(self.epoch, int(state["epoch"]))


# ---------------------------------------------------------------------------
# exact top-k via the engine's radix select (used by TopKCompressor on CUDA)
# ---------------------------------------------------------------------------
_TOPK_CACHE: "OrderedDict[tuple, BucketEngine]" = OrderedDict()
_TOPK_CACHE_MAX = 64


def topk_select_cuda(flat: torch.Tensor, k: int):
    """(values[k], indices int64[k] ascending) of the k largest |x| — exact, ties broken towards the smaller index
    (what ``torch.topk`` on a stable sort would give).

    The engine's radix select resolves the threshold to 22 bits and ships EVERY element sharing that prefix (>= k of
    them, plan.h "Selection rule"); the slot is provisioned with slack for those extra coordinates and the final k are
    picked here from that short list by (|x| descending, index ascending).  If the prefix class is larger than the
    slack (massive ties) the call falls back to ``torch.topk``.  With fewer than k non-zeros the result is padded with
    (index 0, value 0.0) — harmless for ``index_add_``-style desparsification."""
    d = flat.numel()
    k = max(1, min(int(k), d))
    key = (d, k, flat.device.index)
    eng = _TOPK_CACHE.get(key)
    if eng is None:
        plan = BucketPlan([d], index=None, ks=[k], raw_slack=max(64, k // 8), min_numel=d)   # min_numel=d: never value-coded
        eng = BucketEngine(plan, device=flat.device, beta=0.0, gamma=1.0, average=False, use_history=False,
                           world=1, rank=0)
        _TOPK_CACHE[key] = eng
        if len(_TOPK_CACHE) > _TOPK_CACHE_MAX:
            _TOPK_CACHE.popitem(last=False)
    else:
        _TOPK_CACHE.move_to_end(key)
    tp = eng.plan.tensors[0]
    x = flat.detach().float().flatten()
    with torch.cuda.device(flat.device):
        eng.grad[:d].copy_(x)
        eng.hist.zero_()
        eng.tile_count.zero_()
        eng.hist_total.zero_()
        eng.epoch += 1
        eng.ctx.run(eng.epoch, PH_ACCUM, PH_EMIT + 1)
        slot = eng.slot()
        n_sel, _, _, n_pos = (int(v) for v in slot[SLOT_HEADER_WORDS:SLOT_HEADER_WORDS + 4].tolist())
        n_sel, n_pos = n_sel & 0xFFFFFFFF, n_pos & 0xFFFFFFFF
        # the select never takes |x| < 2^-140 (a 22-bit key prefix of 0), so fewer than k selected may still leave
        # non-zeros out
        n_nz = int(torch.count_nonzero(x)) if n_sel < k else k
        if n_pos > tp.val_cap or n_nz > n_sel:    # more ties at the 22-bit prefix than the slack, or tiny non-zeros
            m = min(k, n_nz)                      # exact fallback: stable sort, so ties still go to the smaller index
            idxs = torch.sort(x.abs(), descending=True, stable=True).indices[:m].sort().values
            vals = x[idxs]
            if m < k:
                vals = torch.cat([vals, vals.new_zeros(k - m)])
                idxs = torch.cat([idxs, idxs.new_zeros(k - m)])
            return vals.to(flat.dtype), idxs
        vals = slot[tp.off_vals:tp.off_vals + n_sel].view(torch.float32).clone()
        idxs = slot[tp.off_idx:tp.off_idx + n_sel].to(torch.int64)
        if n_sel > k:                             # drop the smallest of the prefix class; stable => smaller index wins ties
            order = torch.sort(vals.abs(), descending=True, stable=True).indices[:k]
            keep = torch.sort(order).values
            vals, idxs = vals[keep], idxs[keep]
        elif n_sel < k:                           # fewer than k non-zeros
            pad = k - n_sel
            vals = torch.cat([vals, vals.new_zeros(pad)])
            idxs = torch.cat([idxs, idxs.new_zeros(pad)])
    return vals.to(flat.dtype), idxs
