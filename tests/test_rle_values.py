"""QSGD and polyfit values over the fused run-length index ('fused_rle_values'), on the CPU: the slot layout, the wire
bytes, the oracle's encode against its receiver-side decode, mixed plans, the threshold sparsifier, and the opt-in
routing and config checks."""
import os
import tempfile
import warnings

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.nn as nn

from deepreduce_b200.config import ConfigError, validate_params
from deepreduce_b200.parallel.engine import decode_slot_oracle, engine_oracle, stats_from_slot
from deepreduce_b200.parallel.plan import (DYN_WORDS, MAX_POLY_K, MAX_SEGMENTS, MODE_RAW, MODE_RLE, SLOT_HEADER_WORDS,
                                           BucketPlan, rle_stream_words)

SHAPES = [50_000, 3000, 20_000, 800, 9000, 70_000]
VALUES = [("qsgd", 127), ("qsgd", 1000), ("polyfit", 127)]


def _al(x):
    return (x + 3) // 4 * 4


def _grads(plan, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(plan.total_elems, generator=g) * (1 + torch.rand(plan.total_elems, generator=g)) for _ in range(W)]


def _resnet50_numels():
    from deepreduce_b200.models import resnet50
    return [p.numel() for p in reversed(list(resnet50().parameters()))]


def _index_words(plan, slot, t):
    """The words of tensor t's run-length index: its per-tile counts and its 12-bit position stream."""
    nc = (t.n_tiles + 1) // 2
    return np.concatenate([slot[t.off_prefix:t.off_prefix + nc], slot[t.off_idx:t.off_idx + rle_stream_words(t.val_cap)]])


# ---------------------------------------------------------------------------
# layout
# ---------------------------------------------------------------------------
def test_layout_without_values_is_unchanged():
    """rle plans without a value codec keep the layout they always had: fp32 values | tile counts | 12-bit stream."""
    for sizes, ratio in ((SHAPES, 0.01), (_resnet50_numels(), 0.001)):
        plan = BucketPlan(sizes, compress_ratio=ratio, index="rle")
        word = _al(SLOT_HEADER_WORDS + DYN_WORDS * len(sizes))
        for t in plan.tensors:
            assert t.vmode == 0 and t.off_coef == t.off_rankmap == t.off_selidx == t.off_sorted == 0
            assert t.off_vals == word
            if t.mode == MODE_RLE:
                assert t.off_prefix == _al(word + t.k)
                assert t.off_idx == _al(t.off_prefix + (t.n_tiles + 1) // 2)
                word = _al(t.off_idx + rle_stream_words(t.k))
            else:
                assert t.mode == MODE_RAW and t.off_idx == _al(word + t.val_cap)
                word = _al(t.off_idx + t.val_cap)
        assert plan.payload_words == word and plan.slot_words == (word + 63) // 64 * 64


@pytest.mark.parametrize("value,qn", VALUES)
def test_layout_shipped_region_and_scratch(value, qn):
    base = BucketPlan(SHAPES, compress_ratio=0.02, index="rle")
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index="rle", value=value, quantum_num=qn, poly_min_k=64)
    P = plan.payload_words
    assert P < base.payload_words
    coded = 0
    for a, t in zip(base.tensors, plan.tensors):
        assert (t.mode, t.k, t.val_cap, t.n_tiles) == (a.mode, a.k, a.val_cap, a.n_tiles)
        if t.mode != MODE_RLE:
            assert t.vmode == 0 and t.off_vals < P
            continue
        if t.vmode == 0:                 # polyfit under poly_min_k: fp32 values, shipped
            assert value == "polyfit" and t.k < 64 and t.off_vals + t.val_cap <= t.off_prefix
            continue
        coded += 1
        # shipped: codec header | codec body | tile counts | 12-bit stream, each 4-word aligned
        assert t.off_coef < t.off_rankmap < t.off_prefix < t.off_idx < P
        if value == "qsgd":
            assert t.vmode == 2 and t.poly_degree == qn and t.rank_u32 == int(qn >= 128)
            assert t.off_rankmap == t.off_coef + _al((t.val_cap + 511) // 512)
            body = (t.val_cap + 1) // 2 if t.rank_u32 else (t.val_cap + 3) // 4
            scratch = [t.off_vals, t.off_selidx]
        else:
            assert t.vmode == 1 and t.rank_u32 == 0
            assert t.off_rankmap == t.off_coef + _al(MAX_SEGMENTS * (t.poly_degree + 1) + 2)
            body = (t.val_cap + 1) // 2
            scratch = [t.off_vals, t.off_selidx, t.off_sorted]
        assert t.off_prefix == t.off_rankmap + _al(body)
        assert t.off_idx == t.off_prefix + _al((t.n_tiles + 1) // 2)
        # sender-local scratch (the fp32 values, the selected element of each, the sorted values) is never pushed
        assert all(P <= s and s + t.val_cap <= plan.slot_words for s in scratch)
        w = t.words()
        assert w[16:20] == [t.vmode, t.off_coef, t.off_rankmap, t.off_selidx]
    assert coded >= 4
    assert plan.wire_bytes() == 4 * P


@pytest.mark.parametrize("value,qn", VALUES)
def test_stats_split_value_and_index_bytes(value, qn):
    base = BucketPlan(SHAPES, compress_ratio=0.02, index="rle")
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index="rle", value=value, quantum_num=qn, poly_min_k=64)
    _, _, slots = engine_oracle(plan, _grads(plan, 1), [torch.zeros(plan.total_elems)], average=False)
    _, _, bslots = engine_oracle(base, _grads(base, 1), [torch.zeros(base.total_elems)], average=False)
    st, bst = stats_from_slot(plan, slots[0]), stats_from_slot(base, bslots[0])
    for t, row, brow in zip(plan.tensors, st["tensors"], bst["tensors"]):
        assert row["index_bytes"] == brow["index_bytes"]
        assert row["n_sel"] == brow["n_sel"] and row["false_pos"] == 0
        if t.vmode == 2:
            assert row["value_bytes"] == 4 * ((t.val_cap + 511) // 512) + t.val_cap * (2 if t.rank_u32 else 1)
        elif t.vmode == 1:
            assert row["value_bytes"] == 4 * (MAX_SEGMENTS * (t.poly_degree + 1) + 2) + 2 * t.val_cap
        else:
            assert row["value_bytes"] == 4 * t.val_cap
    tot = st["total"]
    assert tot["value_bytes"] < bst["total"]["value_bytes"]
    assert tot["value_bytes"] + tot["index_bytes"] + tot["header_bytes"] <= tot["wire_bytes"] == plan.wire_bytes()


@pytest.mark.parametrize("ratio", [0.001, 0.01, 0.03])
def test_wire_bytes_resnet50(ratio):
    """On ResNet-50's tensors rle + QSGD ships less than rle alone and less than bloom (+ hint) + QSGD."""
    numels = _resnet50_numels()
    rle = BucketPlan(numels, compress_ratio=ratio, index="rle").wire_bytes()
    rle_q = BucketPlan(numels, compress_ratio=ratio, index="rle", value="qsgd").wire_bytes()
    rle_p = BucketPlan(numels, compress_ratio=ratio, index="rle", value="polyfit").wire_bytes()
    bloom_q = BucketPlan(numels, compress_ratio=ratio, index="bloom", value="qsgd").wire_bytes()
    bloom_p = BucketPlan(numels, compress_ratio=ratio, index="bloom", value="polyfit").wire_bytes()
    assert rle_q < rle and rle_q < bloom_q
    assert rle_p < rle and rle_p < bloom_p


# ---------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("value,qn", VALUES)
def test_index_side_equals_plan_without_values(value, qn):
    """At step 0 (no residual) the value codec leaves the index alone: the dyn headers, the tile counts and the 12-bit
    stream are word for word those of the plan without values."""
    base = BucketPlan(SHAPES, compress_ratio=0.02, index="rle")
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index="rle", value=value, quantum_num=qn, poly_min_k=64)
    grads = _grads(plan, 2, seed=5)
    _, _, bslots = engine_oracle(base, grads, [torch.zeros(base.total_elems)] * 2, epoch=1)
    _, _, slots = engine_oracle(plan, grads, [torch.zeros(plan.total_elems)] * 2, epoch=1)
    for a, b in zip(slots, bslots):
        h = SLOT_HEADER_WORDS + DYN_WORDS * len(SHAPES)
        assert np.array_equal(a[SLOT_HEADER_WORDS:h], b[SLOT_HEADER_WORDS:h])
        for t, u in zip(plan.tensors, base.tensors):
            if t.mode == MODE_RLE:
                assert np.array_equal(_index_words(plan, a, t), _index_words(base, b, u)), t.name


@pytest.mark.parametrize("value,qn", VALUES)
@pytest.mark.parametrize("W", [1, 2, 3])
def test_decode_sum_equals_oracle_aggregate(W, value, qn):
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index="rle", value=value, quantum_num=qn, poly_min_k=64)
    grads = _grads(plan, W, seed=W)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in (1, 2, 3):
        out, res, slots = engine_oracle(plan, grads, res, epoch=epoch, average=False)
        dec = sum(decode_slot_oracle(plan, torch.from_numpy(s.view(np.int32))) for s in slots)
        assert torch.allclose(dec, out, rtol=0, atol=1e-6 * float(out.abs().max())), (W, value, epoch)


@pytest.mark.parametrize("value,qn", VALUES)
def test_residual_is_accumulated_minus_decoded(value, qn):
    """Error feedback sees the codec's error: on the shipped set the new residual is the accumulated gradient minus what
    the receivers decode; elsewhere it is the accumulated gradient."""
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index="rle", value=value, quantum_num=qn, poly_min_k=64)
    g = _grads(plan, 1, seed=11)[0]
    res = torch.zeros(plan.total_elems)
    for epoch in (1, 2):
        acc = res + g
        out, new_res, slots = engine_oracle(plan, [g], [res], epoch=epoch, average=False)
        a = slots[0]
        dec = decode_slot_oracle(plan, torch.from_numpy(a.view(np.int32)))
        shipped = torch.zeros(plan.total_elems, dtype=torch.bool)
        for ti, t in enumerate(plan.tensors):
            n_sel = int(a[SLOT_HEADER_WORDS + DYN_WORDS * ti])
            if t.mode == MODE_RLE:
                from deepreduce_b200.parallel.engine import rle_unpack12
                cnt = a[t.off_prefix:t.off_prefix + (t.n_tiles + 1) // 2].view(np.uint16)[:t.n_tiles].astype(np.int64)
                local = rle_unpack12(a[t.off_idx:t.off_idx + rle_stream_words(t.val_cap)], n_sel)
                idx = np.repeat(np.arange(t.n_tiles, dtype=np.int64), cnt) * 4096 + local
            else:
                idx = a[t.off_idx:t.off_idx + n_sel].astype(np.int64)
            assert len(idx) == n_sel
            shipped[t.elem_off + torch.from_numpy(idx)] = True
        assert int(shipped.sum()) > 0 and not bool(shipped.all())
        assert torch.equal(new_res[0][~shipped], acc[~shipped])
        sc = float(acc.abs().max())
        assert torch.allclose(new_res[0][shipped], acc[shipped] - dec[shipped], rtol=0, atol=1e-6 * sc)
        assert torch.allclose(dec, out, rtol=0, atol=1e-6 * sc)
        res = new_res[0]


def test_mixed_plan_keeps_fp32_values_where_the_codec_does_not_apply():
    """In one bucket: the <= min_numel bypass tensors (plain pairs), rle tensors under poly_min_k and over MAX_POLY_K keep
    fp32 values; the others ship polyfit values."""
    sizes = [600, 30_000, 400_000, 1_400_000, 10]
    plan = BucketPlan(sizes, compress_ratio=0.1, index="rle", value="polyfit", poly_min_k=4000)
    modes = [(t.mode, t.vmode) for t in plan.tensors]
    assert modes == [(MODE_RAW, 0), (MODE_RLE, 0), (MODE_RLE, 1), (MODE_RLE, 0), (MODE_RAW, 0)]
    assert plan.tensors[1].k < 4000 and plan.tensors[3].val_cap > MAX_POLY_K
    for t in plan.tensors:
        if t.vmode == 0:
            assert t.off_vals + t.val_cap <= plan.payload_words       # fp32 values are shipped
        else:
            assert t.off_vals >= plan.payload_words                   # fp32 values stay in scratch
    grads = _grads(plan, 2, seed=3)
    res = [torch.zeros(plan.total_elems) for _ in range(2)]
    for epoch in (1, 2):
        out, new_res, slots = engine_oracle(plan, grads, res, epoch=epoch, average=False)
        decs = [decode_slot_oracle(plan, torch.from_numpy(s.view(np.int32))) for s in slots]
        assert torch.allclose(sum(decs), out, rtol=0, atol=1e-6 * float(out.abs().max()))
        for r in range(2):
            acc = res[r] + grads[r]
            for t in plan.tensors:
                seg = slice(t.elem_off, t.elem_off + t.numel)
                if t.vmode == 0:         # lossless values: the shipped set is exact and its residual exactly zero
                    sent = decs[r][seg] != 0
                    assert torch.equal(decs[r][seg][sent], acc[seg][sent])
                    assert bool((new_res[r][seg][sent] == 0).all())
        res = new_res
    qs = BucketPlan(sizes, compress_ratio=0.1, index="rle", value="qsgd")
    assert [(t.mode, t.vmode) for t in qs.tensors] == [(MODE_RAW, 0), (MODE_RLE, 2), (MODE_RLE, 2), (MODE_RLE, 2),
                                                       (MODE_RAW, 0)]


@pytest.mark.parametrize("value,qn", VALUES)
def test_threshold_sparsifier(value, qn):
    plan = BucketPlan(SHAPES, index="rle", value=value, quantum_num=qn, poly_min_k=64, sparsifier="threshold",
                      threshold=1.0, capacity_ratio=0.5)
    assert all(t.val_cap == t.k for t in plan.tensors)
    grads = _grads(plan, 2, seed=8)
    res = [torch.zeros(plan.total_elems) for _ in range(2)]
    for epoch in (1, 2):
        out, res, slots = engine_oracle(plan, grads, res, epoch=epoch, average=False)
        dec = sum(decode_slot_oracle(plan, torch.from_numpy(s.view(np.int32))) for s in slots)
        assert torch.allclose(dec, out, rtol=0, atol=1e-6 * float(out.abs().max()))
        for s in slots:
            for ti, t in enumerate(plan.tensors):
                assert 0 < int(s[SLOT_HEADER_WORDS + DYN_WORDS * ti]) <= t.val_cap


# ---------------------------------------------------------------------------
# routing and config
# ---------------------------------------------------------------------------
BASE = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
RLE_Q = {**BASE, 'deepreduce': 'both', 'index': 'rle', 'value': 'qsgd'}
RLE_P = {**BASE, 'deepreduce': 'both', 'index': 'rle', 'value': 'polyfit'}
THR = {'compressor': 'threshold', 'threshold': 0.01, 'memory': 'residual', 'communicator': 'allgather'}


def test_routing():
    from deepreduce_b200.parallel.ddp import _fused_supported, fused_path, plan_kwargs_from_params
    for p in (RLE_Q, RLE_P, {**RLE_Q, 'quantum_num': 1000, 'bucket_size': 512}, {**THR, **RLE_P, 'compressor': 'threshold'},
              {**RLE_P, 'policy': 'p0'}):
        assert not fused_path(p) and not _fused_supported(p), p              # without the key: the per-tensor route
        assert not fused_path({**p, 'fused_rle_values': False}), p
        assert not fused_path({**p, 'fused_rle_values': 1}), p
        assert fused_path({**p, 'fused_rle_values': True}) and _fused_supported({**p, 'fused_rle_values': True}), p
        kw = plan_kwargs_from_params({**p, 'fused_rle_values': True})
        assert kw['index'] == 'rle' and kw['value'] == p['value']
        plan = BucketPlan([80_000, 700], **kw)
        assert plan.tensors[0].mode == MODE_RLE and plan.tensors[0].vmode == (2 if p['value'] == 'qsgd' else 1)
    for p in ({**RLE_Q, 'bucket_size': 256}, {**RLE_Q, 'value': 'gzip'}, {**RLE_Q, 'communicator': 'allreduce'},
              {**RLE_Q, 'compressor': 'randomk'}, {**RLE_Q, 'index': 'huffman'},
              {**RLE_P, 'policy': 'conflict_sets'}):
        assert not fused_path({**p, 'fused_rle_values': True}), p
    # the key changes no other route
    for p in (BASE, {**BASE, 'deepreduce': 'index', 'index': 'rle'}, {**BASE, 'deepreduce': 'both', 'index': 'bloom'}):
        assert fused_path({**p, 'fused_rle_values': True}) == fused_path(p)


def test_config():
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        for p in (RLE_Q, RLE_P, {**RLE_Q, 'quantum_num': 32767, 'bucket_size': 512}, {**THR, **RLE_P, **THR}):
            validate_params({**p, 'fused_rle_values': True}, strict=True)
            validate_params({**p, 'fused_rle_values': False}, strict=True)
    bad = [
        {**RLE_Q, 'fused_rle_values': 1}, {**RLE_Q, 'fused_rle_values': 'yes'}, {**RLE_Q, 'fused_rle_values': None},
        {**RLE_Q, 'bucket_size': 256, 'fused_rle_values': True},
        {**RLE_Q, 'quantum_num': 0, 'fused_rle_values': True}, {**RLE_Q, 'quantum_num': 32768, 'fused_rle_values': True},
        {**RLE_Q, 'value': 'dexp', 'fused_rle_values': True},
        {**RLE_Q, 'index': 'bloom', 'fused_rle_values': True},
        {**RLE_Q, 'deepreduce': 'index', 'fused_rle_values': True},
        {**RLE_Q, 'deepreduce': 'value', 'fused_rle_values': True},
        {**BASE, 'fused_rle_values': True},
        {**RLE_Q, 'compressor': 'randomk', 'fused_rle_values': True},
        {**RLE_Q, 'communicator': 'allreduce', 'fused_rle_values': True},
    ]
    for p in bad:
        with pytest.raises(ConfigError):
            validate_params(p)


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.a, self.b = nn.Linear(60, 90), nn.Linear(90, 4)

    def forward(self, x):
        return self.b(torch.relu(self.a(x)))


@pytest.fixture
def gloo_world1():
    f = tempfile.NamedTemporaryFile(delete=False)
    f.close()
    os.unlink(f.name)
    dist.init_process_group("gloo", init_method=f"file://{f.name}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


def test_cpu_runs_the_per_tensor_path_unchanged(gloo_world1):
    """On the CPU the key changes nothing: DeepReduceDDP and the DDP hook state take the per-tensor path, with the same
    gradients bit for bit as the dict without the key."""
    from deepreduce_b200.parallel import DeepReduceDDP
    from deepreduce_b200.parallel.comm_hook import DeepReduceHookState
    for p in (RLE_Q, RLE_P):
        outs = []
        for params in (p, {**p, 'fused_rle_values': True}):
            net = _Net()
            ddp = DeepReduceDDP(net, params)
            assert not ddp.fused and ddp.grc is not None
            st = DeepReduceHookState(params, _Net())
            assert st.path(torch.zeros(4)) == "grace"
            grads = []
            for step in range(3):
                x = torch.randn(16, 60, generator=torch.Generator().manual_seed(step))
                net.zero_grad()
                net(x).pow(2).sum().backward()
                ddp.finish()
                grads.append([q.grad.clone() for q in net.parameters()])
            outs.append(grads)
        for ga, gb in zip(*outs):
            assert all(torch.equal(a, b) for a, b in zip(ga, gb))
