"""The conflict-sets (P2) bloom policy of the fused engine, on the CPU: slot layout, the oracle's pick against
``conflict_sets_oracle``, the receiver-side decode of the shipped pick, and the opt-in routing."""
import math
import warnings

import numpy as np
import pytest
import torch

from deepreduce_b200 import spec
from deepreduce_b200.codecs.bloom import bloom_insert_oracle, bloom_query_oracle, conflict_sets_oracle
from deepreduce_b200.config import ConfigError, validate_params
from deepreduce_b200.parallel.engine import (conflict_sets_keep_oracle, conflict_sets_pick_oracle, decode_slot_oracle,
                                             engine_oracle, select_topk_oracle, stats_from_slot)
from deepreduce_b200.parallel.plan import MODE_BLOOM, POLICY_ID, BucketPlan, TensorPlan

SHAPES = [50_000, 3000, 20_000, 800, 9000]


def _grads(plan, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(plan.total_elems, generator=g) * (1 + torch.rand(plan.total_elems, generator=g)) for _ in range(W)]


def test_plan_layout_and_wire_bytes():
    base = BucketPlan(SHAPES, compress_ratio=0.01, policy="leftmost")
    p2 = BucketPlan(SHAPES, compress_ratio=0.01, policy="conflict_sets")
    assert POLICY_ID["conflict_sets"] == 3
    extra = 0
    for a, t in zip(base.tensors, p2.tensors):
        assert (t.mode, t.k, t.val_cap, t.m_bits, t.n_hash) == (a.mode, a.k, a.val_cap, a.m_bits, a.n_hash)
        if t.mode != MODE_BLOOM:
            assert t.pos_cap == t.off_pos_prefix == t.off_pick == 0
            continue
        fpr = spec.default_fpr(t.k, t.numel)
        assert t.pos_cap == min(t.numel, t.k + int(math.ceil(2.0 * fpr * t.numel)) + 64)
        # vals | filter | tile prefix | hint | positives per tile | pick, each 4-word aligned
        assert t.off_pos_prefix == t.off_hint + ((4 * t.n_tiles + 3) // 4) * 4
        assert t.off_pick == t.off_pos_prefix + ((t.n_tiles + 3) // 4) * 4
        n_pick = (t.pos_cap + 31) // 32
        extra += ((t.n_tiles + 3) // 4) * 4 + ((n_pick + 3) // 4) * 4
        w = t.words()
        assert w[27:30] == [t.pos_cap, t.off_pos_prefix, t.off_pick]
    assert p2.payload_words >= base.payload_words + extra - 8        # the header alignment can absorb a few words
    assert p2.wire_bytes() == 4 * p2.payload_words
    table, n, words, cap = p2.p2_tables()
    assert n == sum(t.mode == MODE_BLOOM for t in p2.tensors) and cap == max(t.pos_cap for t in p2.tensors)
    assert table.numel() == 10 * n and words > 0


def test_plan_rejects():
    """Host-side limits of the fused P2: index and sparsifier, hash count, positives per tensor."""
    with pytest.raises(ValueError):
        BucketPlan([50_000], policy="conflict_sets", index="rle")
    with pytest.raises(ValueError, match="top-k"):
        BucketPlan([50_000], policy="conflict_sets", sparsifier="threshold", threshold=0.5)
    with pytest.raises(ValueError, match="hash"):
        BucketPlan([50_000], policy="conflict_sets", fpr=1e-6, max_hash=20)
    assert max(t.n_hash for t in BucketPlan([50_000], policy="conflict_sets", fpr=1e-6, max_hash=16).tensors) == 16
    with pytest.raises(ValueError):
        BucketPlan([50_000], policy="conflict_sets", index=None, sparsifier="randomk")
    with pytest.raises(ValueError, match="split"):
        BucketPlan([40_000_000], compress_ratio=0.1, policy="conflict_sets")


def _pick_words_to_ranks(words, n):
    q = np.arange(n)
    return q[((words.astype(np.int64)[q >> 5] >> (q & 31)) & 1).astype(bool)]


@pytest.mark.parametrize("hint", [True, False])
@pytest.mark.parametrize("d,ratio,fpr", [(60_000, 0.01, None), (30_000, 0.05, 0.02), (9000, 0.1, 0.3), (5000, 0.5, None)])
def test_oracle_pick_is_conflict_sets_oracle(hint, d, ratio, fpr):
    """What the oracle puts around the draw: the positives the receiver's probe sees (hint filtering), the pos_cap cut,
    the bitmask packing and the header.  The draw itself is conflict_sets_oracle in both places; the device draw is
    checked independently against the host routine in test_gpu_p2_fused.py::test_device_pick_equals_host_conflict_sets."""
    plan = BucketPlan([d], compress_ratio=ratio, fpr=fpr, policy="conflict_sets", hint=hint)
    tp = plan.tensors[0]
    full = _grads(plan, 1, seed=d)[0]
    full[d:] = 0
    acc = full[:d]
    for epoch in (1, 4):
        out, _, slots = engine_oracle(plan, [full], [torch.zeros(plan.total_elems)], epoch=epoch, average=False)
        slot = slots[0]
        sel, _ = select_topk_oracle(acc, tp.k)
        words = bloom_insert_oracle(sel, tp.n_hash, tp.m_bits)
        pos = bloom_query_oracle(words, d, tp.n_hash, tp.m_bits)
        if hint:
            occ = torch.zeros((d + 31) // 32, dtype=torch.bool)
            occ[sel // 32] = True
            pos = pos[occ[pos // 32]]
        want = conflict_sets_oracle(pos[:tp.pos_cap], tp.k, tp.n_hash, tp.m_bits, spec.DEFAULT_SEED,
                                    spec.policy_seed(epoch, tp.salt))
        assert want.numel() == min(tp.k, min(pos.numel(), tp.pos_cap))
        ranks = _pick_words_to_ranks(slot[tp.off_pick:tp.off_pick + (tp.pos_cap + 31) // 32], tp.pos_cap)
        assert torch.equal(pos[torch.from_numpy(ranks)], want)
        assert torch.equal(torch.nonzero(out[:d]).flatten(), want[acc[want] != 0])
        n_sel, cutoff, _, n_pos = (int(x) for x in slot[8:12])
        assert (n_sel, cutoff, n_pos) == (want.numel(), 0xFFFFFFFF, pos.numel())


def test_more_positives_than_pos_cap():
    plan = BucketPlan([40_000], compress_ratio=0.02, fpr=0.2, policy="conflict_sets", hint=False)
    tp = plan.tensors[0]
    tp.pos_cap = tp.k + 40                         # the slot region is larger than needed; the draw sees fewer positives
    acc = _grads(plan, 1, seed=3)[0]
    out, _, slots = engine_oracle(plan, [acc], [torch.zeros(plan.total_elems)], epoch=2, average=False)
    st = stats_from_slot(plan, slots[0])
    assert st["tensors"][0]["beyond_cap"] > 0 and st["total"]["tensors_beyond_cap"] == 1
    assert torch.equal(decode_slot_oracle(plan, torch.from_numpy(slots[0].view(np.int32))), out)
    pp = slots[0][tp.off_pos_prefix:tp.off_pos_prefix + tp.n_tiles]
    assert int(pp.max()) <= tp.pos_cap and int(pp[-1]) == tp.pos_cap


def test_pick_helpers_termination_fallback_and_edges():
    # inputs whose draw reaches the termination fallback (a pass with no pick), with a 3-bit filter
    few = torch.tensor([34, 728, 1304, 1992, 2718, 2816, 2867, 3495, 3588, 3872, 4082, 4212, 4214, 4389, 4489, 4502])
    tp = TensorPlan(name="t", numel=5000, shape=(5000,), elem_off=0, k=16, tile_begin=0, n_tiles=2, mode=MODE_BLOOM,
                    m_bits=3, n_hash=2, salt=0, pos_cap=len(few) + 5)
    for epoch in range(1, 40):
        sel, words = conflict_sets_pick_oracle(tp, few, spec.DEFAULT_SEED, epoch)
        want = conflict_sets_oracle(few, 16, 2, 3, spec.DEFAULT_SEED, spec.policy_seed(epoch, 0))
        assert torch.equal(sel, want) and sel.numel() == 16
        assert torch.equal(conflict_sets_keep_oracle(tp, few, words), want)
    tp.k = 100                                     # K >= n_pos: everything is picked
    sel, words = conflict_sets_pick_oracle(tp, few, spec.DEFAULT_SEED, 1)
    assert torch.equal(sel, few)
    sel, words = conflict_sets_pick_oracle(tp, few[:0], spec.DEFAULT_SEED, 1)   # nothing selected
    assert sel.numel() == 0 and not words.any()


def test_nothing_selected():
    plan = BucketPlan([20_000, 5000], compress_ratio=0.01, policy="conflict_sets")
    g = torch.zeros(plan.total_elems)
    g[plan.tensors[1].elem_off + 7] = 1.0
    out, _, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)], average=False)
    assert int(slots[0][8]) == 0 and int(slots[0][11]) == 0
    assert torch.equal(decode_slot_oracle(plan, torch.from_numpy(slots[0].view(np.int32))), out)


@pytest.mark.parametrize("value,qn", [(None, 127), ("polyfit", 127), ("qsgd", 127), ("qsgd", 1000)])
@pytest.mark.parametrize("W", [1, 2, 3, 4])
def test_decode_sum_equals_oracle_aggregate(W, value, qn):
    plan = BucketPlan(SHAPES, compress_ratio=0.02, policy="conflict_sets", value=value, quantum_num=qn, poly_min_k=64)
    grads = _grads(plan, W, seed=W)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in (1, 2):
        out, res, slots = engine_oracle(plan, grads, res, epoch=epoch, average=False)
        dec = sum(decode_slot_oracle(plan, torch.from_numpy(s.view(np.int32))) for s in slots)
        assert torch.allclose(dec, out, rtol=0, atol=1e-6 * float(out.abs().max())), (W, value, epoch)


def test_routing_and_config():
    """The key opts in (top-k only); without it, or with any value but True, routing is what it was."""
    from deepreduce_b200.parallel.ddp import _fused_supported, fused_path, plan_kwargs_from_params
    base = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
    for dr in ('index', 'both'):
        p = {**base, 'deepreduce': dr, 'index': 'bloom', 'policy': 'conflict_sets'}
        assert not fused_path(p) and not _fused_supported(p)
        assert not fused_path({**p, 'p2_pick_mask': False})
        assert fused_path({**p, 'p2_pick_mask': True})
        assert fused_path({**p, 'policy': 'P2', 'p2_pick_mask': True})
        assert plan_kwargs_from_params({**p, 'p2_pick_mask': True})['policy'] == 'conflict_sets'
        assert not fused_path({**p, 'p2_pick_mask': 1})
        assert not fused_path({**p, 'compressor': 'threshold', 'threshold': 0.1, 'p2_pick_mask': True})
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        validate_params({**base, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'conflict_sets', 'p2_pick_mask': True},
                        strict=True)
    for bad in ({**base, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'leftmost', 'p2_pick_mask': True},
                {**base, 'deepreduce': 'index', 'index': 'rle', 'policy': 'conflict_sets', 'p2_pick_mask': True},
                {**base, 'deepreduce': 'value', 'policy': 'conflict_sets', 'p2_pick_mask': True},
                {**base, 'policy': 'conflict_sets', 'p2_pick_mask': True},
                {**base, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'conflict_sets', 'p2_pick_mask': 1},
                {**base, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'conflict_sets', 'p2_pick_mask': 'yes'},
                {**base, 'compressor': 'threshold', 'threshold': 0.1, 'deepreduce': 'index', 'index': 'bloom',
                 'policy': 'conflict_sets', 'p2_pick_mask': True}):
        with pytest.raises(ConfigError):
            validate_params(bad)
