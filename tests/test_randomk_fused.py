"""The fused engine's 'randomk' mode on the CPU: the selection rule, the plan's slot layout, the wire format from both
ends (sender oracle vs receiver oracle) and the routing of ``params`` dicts to the fused engine."""
import math

import numpy as np
import pytest
import torch

from deepreduce_b200 import spec
from deepreduce_b200.parallel import BucketPlan, decode_slot_oracle, engine_oracle
from deepreduce_b200.parallel.engine import select_randomk_oracle, stats_from_slot
from deepreduce_b200.parallel.plan import (DYN_WORDS, KEY_SPAN, MODE_SHARED, SLOT_HEADER_WORDS, randomk_bound,
                                           randomk_capacity)

SIZES = [10, 64, 1000, 1001, 4096, 4097, 36864, 147456]


def _hashes(d, epoch, salt):
    return spec.policy_hash(torch.arange(d, dtype=torch.int64), spec.policy_seed(epoch, salt))


@pytest.mark.parametrize("d,ratio", [(1, 0.01), (10, 0.5), (1000, 0.01), (4097, 0.01), (147456, 0.01), (200000, 0.1)])
def test_randomk_set_holds_the_k_smallest_hashes(d, ratio):
    k = min(d, spec.topk_k(d, ratio))
    for epoch in (1, 2, 7):
        for salt in (0, 3):
            sel, thr = select_randomk_oracle(d, k, epoch, salt)
            smallest = torch.topk(_hashes(d, epoch, salt), k, largest=False).indices
            assert set(smallest.tolist()) <= set(sel.tolist()), (d, k, epoch, salt)
            assert sel.numel() <= randomk_capacity(d, k)
            assert torch.equal(sel, torch.sort(sel).values) and thr % 512 == 0 and thr >= 512
            # the static bound lies below the threshold (the kernel's candidate lists hold every selected key)
            assert randomk_bound(d, k) <= thr


def test_randomk_set_depends_on_the_draw_arguments_only():
    d, k = 36864, 368
    a, ta = select_randomk_oracle(d, k, 5, 2)
    b, tb = select_randomk_oracle(d, k, 5, 2)
    assert torch.equal(a, b) and ta == tb
    assert not torch.equal(a[:k], select_randomk_oracle(d, k, 6, 2)[0][:k])      # another step, another draw
    assert not torch.equal(a[:k], select_randomk_oracle(d, k, 5, 3)[0][:k])      # another tensor, another draw
    # the gradient plays no part: two very different buckets ship the same coordinates
    plan = BucketPlan([d], compress_ratio=0.01, index=None, sparsifier="randomk")
    g1 = torch.randn(plan.total_elems, generator=torch.Generator().manual_seed(0))
    g2 = torch.zeros(plan.total_elems)
    g2[:d] = torch.arange(d, dtype=torch.float32)
    o1, _, _ = engine_oracle(plan, [g1], [torch.zeros_like(g1)], epoch=5)
    o2, _, _ = engine_oracle(plan, [g2], [torch.zeros_like(g2)], epoch=5)
    sel = select_randomk_oracle(d, plan.tensors[0].k, 5, 0)[0]
    assert torch.equal(torch.nonzero(o1[:d]).flatten(), sel)
    assert torch.equal(torch.nonzero(o2[:d]).flatten(), sel[sel > 0])          # element 0 of g2 is an exact zero


def test_randomk_bound_is_a_key_quantile():
    for d, k in ((4096, 40), (147456, 1474), (2359296, 23592)):
        lb = randomk_bound(d, k)
        m = k + int(math.ceil(8 * math.sqrt(k))) + 16
        assert lb % 512 == 0 and abs(d * (KEY_SPAN - lb) / KEY_SPAN - m) < 1 + d * 512 / KEY_SPAN
        keys = (0xFFFFFFFF - _hashes(d, 1, 0)) >> 1
        n_above = int((keys >= lb).sum())
        assert k < n_above < m + 8 * math.sqrt(m) + 16, (d, k, n_above)
    assert randomk_bound(100, 90) == 0                                          # m >= d: every element is a candidate


@pytest.mark.parametrize("value", [None, "qsgd"])
def test_randomk_plan_ships_headers_and_values_only(value):
    plan = BucketPlan(SIZES, compress_ratio=0.01, index=None, value=value, sparsifier="randomk")
    word = SLOT_HEADER_WORDS + DYN_WORDS * len(SIZES)
    word = (word + 3) // 4 * 4
    for t in plan.tensors:
        assert t.mode == MODE_SHARED and t.off_idx == 0 and t.off_filter == 0 and t.n_filter_words == 0
        assert t.val_cap == randomk_capacity(t.numel, t.k) and t.shared_lb == randomk_bound(t.numel, t.k)
        assert t.words()[26] == t.shared_lb
        coded = value == "qsgd" and t.numel > plan.min_numel
        assert t.vmode == (2 if coded else 0)
        if coded:
            assert t.off_coef == word
            word += (t.val_cap + 511) // 512
            word = (word + 3) // 4 * 4
            assert t.off_rankmap == word
            word += (t.val_cap + 3) // 4
        else:
            assert t.off_vals == word
            word += t.val_cap
        word = (word + 3) // 4 * 4
        assert t.off_prefix >= plan.payload_words                               # the per-tile prefix is never shipped
    assert plan.payload_words == word and plan.wire_bytes() == 4 * word
    st = stats_from_slot(plan, np.zeros(plan.payload_words, dtype=np.uint32))["total"]
    assert st["index_bytes"] == 0


def test_randomk_plan_rejects_what_it_does_not_fuse():
    with pytest.raises(ValueError):
        BucketPlan([4096], index="bloom", sparsifier="randomk")
    with pytest.raises(NotImplementedError):
        BucketPlan([4096], index=None, value="polyfit", sparsifier="randomk")


@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("value", [None, "qsgd"])
def test_randomk_decode_of_the_slots_is_the_aggregate(W, value):
    """Sender spec (``engine_oracle``) against the receiver (``decode_slot_oracle``, plan + slot words only)."""
    plan = BucketPlan(SIZES, compress_ratio=0.01, index=None, value=value, sparsifier="randomk")
    gen = torch.Generator().manual_seed(W)
    resids = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in (1, 2, 3):
        grads = [torch.randn(plan.total_elems, generator=gen) for _ in range(W)]
        for g in grads:                                                         # padding stays zero
            mask = torch.zeros(plan.total_elems, dtype=torch.bool)
            for t in plan.tensors:
                mask[t.elem_off:t.elem_off + t.numel] = True
            g[~mask] = 0
        out, resids, slots = engine_oracle(plan, grads, resids, average=False, epoch=epoch)
        dec = [decode_slot_oracle(plan, s) for s in slots]
        rec = torch.zeros(plan.total_elems)
        for d in dec:
            rec = rec + d
        if value is None:
            assert torch.equal(rec, out), (W, epoch)
        else:
            assert torch.allclose(rec, out, atol=1e-6 * float(out.abs().max()), rtol=1e-6), (W, epoch)
        for r, s in enumerate(slots):
            assert int(s[1]) == epoch
            for ti, t in enumerate(plan.tensors):
                n_sel = int(s[SLOT_HEADER_WORDS + DYN_WORDS * ti])
                assert t.k <= n_sel <= t.val_cap
                # every rank ships the same header words for the tensor
                assert np.array_equal(s[SLOT_HEADER_WORDS + DYN_WORDS * ti:][:3],
                                      slots[0][SLOT_HEADER_WORDS + DYN_WORDS * ti:][:3])


def test_randomk_selfcheck_decoder_covers_the_mode():
    from deepreduce_b200.utils.selfcheck import decode_slot_torch
    plan = BucketPlan(SIZES, compress_ratio=0.01, index=None, sparsifier="randomk")
    g = torch.randn(plan.total_elems, generator=torch.Generator().manual_seed(1))
    out, _, slots = engine_oracle(plan, [g], [torch.zeros_like(g)], epoch=4)
    dec = decode_slot_torch(plan, torch.from_numpy(slots[0].view("int32").copy()))
    assert dec is not None and torch.equal(dec, out)


def test_randomk_routing():
    """Which 'randomk' params dicts ``DeepReduceDDP`` runs through the fused engine (``fused_path``), and that the
    top-k / threshold routing (``_fused_supported``) keeps its answers."""
    from deepreduce_b200.parallel.ddp import _fused_randomk_supported, _fused_supported, fused_path, plan_kwargs_from_params
    rk = {'compressor': 'randomk', 'memory': 'residual', 'compress_ratio': 0.01}
    qsgd = {'deepreduce': 'value', 'value': 'qsgd'}
    for comm in ('allgather', 'allreduce'):
        assert fused_path({**rk, 'communicator': comm})
        assert fused_path({**rk, 'communicator': comm, **qsgd})
        assert fused_path({**rk, 'communicator': comm, **qsgd, 'quantum_num': 1000, 'bucket_size': 512})
        assert not fused_path({**rk, 'communicator': comm, **qsgd, 'bucket_size': 256})
        assert not fused_path({**rk, 'communicator': comm, 'deepreduce': 'value', 'value': 'polyfit'})
        assert not fused_path({**rk, 'communicator': comm, 'deepreduce': 'index', 'index': 'bloom'})
        assert not fused_path({**rk, 'communicator': comm, 'deepreduce': 'index', 'index': 'rle'})
        assert not fused_path({**rk, 'communicator': comm, 'deepreduce': 'both', 'index': 'bloom', 'value': 'qsgd'})
    assert fused_path(rk)                                                       # allgather is the default
    assert not fused_path({**rk, 'communicator': 'broadcast'})
    # the shared-index mode is its own predicate: the per-rank-index routing is unchanged
    assert not _fused_supported(rk) and _fused_randomk_supported(rk)
    kw = plan_kwargs_from_params({**rk, **qsgd})
    assert kw['sparsifier'] == 'randomk' and kw['index'] is None and kw['value'] == 'qsgd'
    plan = BucketPlan([4096, 100], **plan_kwargs_from_params(rk))
    assert all(t.mode == MODE_SHARED for t in plan.tensors)
    # the top-k / threshold rows keep their answers through fused_path as well
    tk = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
    for p in (tk, {**tk, 'deepreduce': 'index', 'index': 'bloom'}, {**tk, 'deepreduce': 'both', 'value': 'polyfit'},
              {'compressor': 'threshold', 'communicator': 'allgather', 'threshold': 0.0}):
        assert fused_path(p) and _fused_supported(p) and not _fused_randomk_supported(p), p
    for p in ({**tk, 'communicator': 'allreduce'}, {'compressor': 'threshold', 'communicator': 'allreduce'},
              {**tk, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'conflict_sets'},
              {'compressor': 'none', 'memory': 'none', 'communicator': 'allreduce'}):
        assert not fused_path(p), p
    assert 'sparsifier' not in plan_kwargs_from_params(tk)

