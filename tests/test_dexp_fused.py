"""Double-exponential values in the fused engine ('fused_dexp'), on the CPU: the config and routing rules, the slot
layout and wire bytes, the oracle's two curves per tensor against the per-tensor codec, and a training run of the
oracle engine against dense SGD."""
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn

from deepreduce_b200.codecs import dexp
from deepreduce_b200.config import ConfigError, validate_params
from deepreduce_b200.parallel.engine import (decode_slot_oracle, dexp_runs_eval_oracle, dexp_runs_fit_oracle,
                                             engine_oracle, shipped_index_oracle, stats_from_slot)
from deepreduce_b200.parallel.plan import (DEXP_COEF_WORDS, DYN_WORDS, MAX_POLY_K, MODE_BLOOM, MODE_RAW, MODE_RLE,
                                           SLOT_HEADER_WORDS, BucketPlan)

BASE = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
RLE_D = {**BASE, 'deepreduce': 'both', 'index': 'rle', 'value': 'dexp'}
BLOOM_D = {**BASE, 'deepreduce': 'both', 'index': 'bloom', 'value': 'dexp'}
VALUE_D = {**BASE, 'deepreduce': 'value', 'value': 'dexp'}
THR = {'compressor': 'threshold', 'threshold': 0.01}
SHAPES = [50_000, 3000, 20_000, 800, 9000, 9001, 70_000]


def _al(x):
    return (x + 3) // 4 * 4


def _resnet50_numels():
    from deepreduce_b200.models import resnet50
    return [p.numel() for p in reversed(list(resnet50().parameters()))]


# ---------------------------------------------------------------------------
# config and routing
# ---------------------------------------------------------------------------
GOOD = [RLE_D, BLOOM_D, VALUE_D, {**RLE_D, **THR}, {**BLOOM_D, **THR}, {**VALUE_D, 'index': 'rle'},
        {**RLE_D, 'value': 'double_exp'}, {**BLOOM_D, 'policy': 'random'}, {**BLOOM_D, 'policy': 'p0'},
        {**BLOOM_D, 'policy': 'conflict_sets', 'p2_pick_mask': True},
        {**RLE_D, 'dexp_min_numel': 20_000}]


def test_config_accepts():
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        for p in GOOD:
            validate_params({**p, 'fused_dexp': True}, strict=True)
            validate_params({**p, 'fused_dexp': False}, strict=True)


def test_config_rejects():
    bad = [
        {**RLE_D, 'fused_dexp': 1}, {**RLE_D, 'fused_dexp': 'yes'}, {**RLE_D, 'fused_dexp': None},
        {**RLE_D, 'compressor': 'randomk', 'fused_dexp': True},
        {**RLE_D, 'communicator': 'allreduce', 'fused_dexp': True},
        {**BASE, 'fused_dexp': True},                                             # deepreduce None
        {**RLE_D, 'deepreduce': 'index', 'fused_dexp': True},
        {**RLE_D, 'value': 'polyfit', 'fused_dexp': True}, {**RLE_D, 'value': 'qsgd', 'fused_dexp': True},
        {**RLE_D, 'value': 'gzip', 'fused_dexp': True},
        {**RLE_D, 'index': 'huffman', 'fused_dexp': True}, {**RLE_D, 'index': 'integer', 'fused_dexp': True},
        {**VALUE_D, 'index': 'huffman', 'fused_dexp': True},
        {**BLOOM_D, 'policy': 'conflict_sets', 'fused_dexp': True},                # P2 without the pick mask
        {**RLE_D, 'fused_rle_values': True},                                       # 'fused_rle_values' still rejects dexp
        {**RLE_D, 'fused_rle_values': True, 'fused_dexp': True},
    ]
    for p in bad:
        with pytest.raises(ConfigError):
            validate_params(p)


def test_routing():
    from deepreduce_b200.parallel.ddp import _fused_supported, fused_path, plan_kwargs_from_params
    for p in GOOD:
        assert not fused_path(p) and not _fused_supported(p), p             # without the key: the per-tensor route
        assert not fused_path({**p, 'fused_dexp': False}), p
        assert not fused_path({**p, 'fused_dexp': 1}), p
        assert fused_path({**p, 'fused_dexp': True}), p
        kw = plan_kwargs_from_params({**p, 'fused_dexp': True})
        assert kw['value'] == 'dexp' and kw['dexp_min_numel'] == p.get('dexp_min_numel', 9000)
        assert kw['index'] == (None if p['deepreduce'] == 'value' else p['index'])
        plan = BucketPlan([80_000, 700], **kw)
        assert [t.vmode for t in plan.tensors] == [3, 0]
    for p in ({**RLE_D, 'compressor': 'randomk'}, {**RLE_D, 'communicator': 'allreduce'}, {**RLE_D, 'index': 'huffman'},
              {**RLE_D, 'value': 'gzip'}, {**BLOOM_D, 'policy': 'conflict_sets'},
              {**RLE_D, 'policy': 'conflict_sets'}, {**BLOOM_D, 'policy': 'conflict_sets', 'p2_pick_mask': True,
                                                     **THR}):
        assert not fused_path({**p, 'fused_dexp': True}), p


UNKEYED = [BASE, {**BASE, **THR}, {'compressor': 'randomk', 'memory': 'residual'}, {**BASE, 'compressor': 'none'},
           {**BASE, 'deepreduce': 'index', 'index': 'bloom'}, {**BASE, 'deepreduce': 'index', 'index': 'rle'},
           {**BASE, 'deepreduce': 'index', 'index': 'huffman'}, {**BASE, 'deepreduce': 'both', 'value': 'polyfit'},
           {**BASE, 'deepreduce': 'both', 'value': 'qsgd'}, {**BASE, 'deepreduce': 'value', 'value': 'polyfit'},
           {**BASE, 'deepreduce': 'both', 'index': 'rle', 'value': 'qsgd'},
           {**BASE, 'deepreduce': 'both', 'index': 'rle', 'value': 'polyfit', 'fused_rle_values': True},
           {**BASE, 'deepreduce': 'index', 'policy': 'conflict_sets', 'p2_pick_mask': True},
           {**BASE, 'deepreduce': 'both', 'value': 'gzip'}, RLE_D, BLOOM_D, VALUE_D, {**RLE_D, 'value': 'double_exp'}]


def test_routing_without_the_key_is_unchanged():
    """The key is the only way in: every dict without it routes as the per-tensor rules and the other opt-in keys
    say, and the dexp dicts take the per-tensor path."""
    from deepreduce_b200.parallel.ddp import _fused_randomk_supported, _fused_supported, fused_path
    for p in UNKEYED:
        want = _fused_supported(p) or _fused_randomk_supported(p)
        assert fused_path(p) == want, p
        assert fused_path({**p, 'fused_dexp': False}) == want, p
        if p.get('value') in ('dexp', 'double_exp'):
            assert not want, p


# ---------------------------------------------------------------------------
# plan layout and wire bytes
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("index", ["rle", "bloom", None])
def test_layout(index):
    base = BucketPlan(SHAPES, compress_ratio=0.02, index=index)
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index=index, value="dexp")
    P = plan.payload_words
    assert P < base.payload_words
    for a, t in zip(base.tensors, plan.tensors):
        assert (t.mode, t.k, t.val_cap, t.n_tiles) == (a.mode, a.k, a.val_cap, a.n_tiles)
        assert t.vmode == (3 if t.numel > 9000 else 0), t.name
        if t.vmode == 0:
            assert t.off_vals + t.val_cap <= P                       # fp32 values, shipped
            continue
        # coef[8] | num_pos, n | rank map (u16), each 4-word aligned, in front of the index
        assert t.off_rankmap == t.off_coef + _al(DEXP_COEF_WORDS + 2)
        end = t.off_rankmap + _al((t.val_cap + 1) // 2)
        assert t.rank_u32 == 0
        nxt = {MODE_RLE: t.off_prefix, MODE_BLOOM: t.off_filter, MODE_RAW: t.off_idx}[t.mode]
        assert nxt == end
        # sender-local scratch: the fp32 values, their element indices and the sorted copy
        for s in (t.off_vals, t.off_selidx, t.off_sorted):
            assert P <= s and s + t.val_cap <= plan.slot_words
    ids, n_poly, tasks, n_tasks = plan.poly_tables()
    coded = [i for i, t in enumerate(plan.tensors) if t.vmode == 3]
    assert sorted(ids.tolist()) == coded and n_poly == len(coded)
    assert n_tasks == sum((plan.tensors[i].val_cap + 511) // 512 for i in coded)
    assert plan.poly_total == sum(plan.tensors[i].val_cap for i in coded)
    assert plan.wire_bytes() == 4 * P


def test_eligibility_rules():
    """d > dexp_min_numel and val_cap <= MAX_POLY_K, like polyfit's rule; the tensors under the bypass keep plain
    pairs; a u32 rank map past 65 536 values."""
    sizes = [600, 9000, 9001, 400_000, 7_000_000, 10]
    plan = BucketPlan(sizes, compress_ratio=0.1, index="rle", value="dexp")
    assert [(t.mode, t.vmode) for t in plan.tensors] == [(MODE_RAW, 0), (MODE_RLE, 0), (MODE_RLE, 3), (MODE_RLE, 3),
                                                         (MODE_RLE, 0), (MODE_RAW, 0)]
    assert plan.tensors[3].rank_u32 == 0 and plan.tensors[4].val_cap > MAX_POLY_K
    big = BucketPlan([1_000_000], compress_ratio=0.1, index="rle", value="dexp")
    assert big.tensors[0].vmode == 3 and big.tensors[0].rank_u32 == 1
    assert big.tensors[0].off_prefix == big.tensors[0].off_rankmap + _al(big.tensors[0].val_cap)
    raised = BucketPlan(sizes, compress_ratio=0.1, index="rle", value="dexp", dexp_min_numel=500_000)
    assert [t.vmode for t in raised.tensors] == [0, 0, 0, 0, 0, 0]
    with pytest.raises(NotImplementedError):
        BucketPlan(sizes, value="dexp", index=None, sparsifier="randomk")


@pytest.mark.parametrize("ratio", [0.001, 0.01])
def test_wire_bytes_resnet50(ratio):
    """On ResNet-50: rle + dexp ships less than rle + polyfit, and bloom (+ hint) + dexp less than bloom + polyfit."""
    numels = _resnet50_numels()
    w = {(i, v): BucketPlan(numels, compress_ratio=ratio, index=i, value=v).wire_bytes()
         for i in ("rle", "bloom") for v in (None, "polyfit", "dexp")}
    assert w["rle", "dexp"] < w["rle", "polyfit"] < w["rle", None]
    assert w["bloom", "dexp"] < w["bloom", "polyfit"] < w["bloom", None]


# ---------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------
def _grads(plan, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(plan.total_elems, generator=g) * (1 + torch.rand(plan.total_elems, generator=g))
            for _ in range(W)]


@pytest.mark.parametrize("index", ["rle", "bloom", None])
def test_oracle_curves_match_the_codec(index):
    """Each shipped curve is ``DoubleExp`` (the per-tensor codec) fitted on that run alone: the positives by ascending
    value, the rest by ascending magnitude, both to the last bit of the fp32 words.  The rank map is the stable
    descending sort and the header tail holds {num_pos, n}."""
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index=index, value="dexp")
    acc = _grads(plan, 1, seed=4)[0]
    _, _, slots = engine_oracle(plan, [acc], [torch.zeros(plan.total_elems)], beta=0.0, average=False)
    a = slots[0]
    n_coded = 0
    for ti, t in enumerate(plan.tensors):
        if t.vmode != 3:
            continue
        n_coded += 1
        idx = shipped_index_oracle(plan, a, ti)
        v = acc[t.elem_off + idx]
        n, num_pos = int(idx.numel()), int((v > 0).sum())
        assert 0 < num_pos < n
        assert [int(a[t.off_coef + DEXP_COEF_WORDS]), int(a[t.off_coef + DEXP_COEF_WORDS + 1])] == [num_pos, n]
        order = torch.sort(v, descending=True, stable=True).indices
        rank = a[t.off_rankmap:t.off_rankmap + (n + 1) // 2].view(np.uint16)[:n].astype(np.int64)
        assert np.array_equal(rank[order.numpy()], np.arange(n))
        coef = a[t.off_coef:t.off_coef + DEXP_COEF_WORDS].view(np.float32)
        for run, cw in ((v[v > 0], coef[:4]), (v[v <= 0], coef[4:])):
            # the codec sorts |v| ascending and fits one curve: here one run, so its magnitudes are the whole tensor
            shape = torch.Size([t.numel])
            got, _, _ = dexp.DoubleExp.compress((run, torch.arange(run.numel()), shape), {})
            assert np.array_equal(got.numpy().view(np.uint32), cw.view(np.uint32)), (t.name, got, cw)
    assert n_coded == 4


def test_eval_is_the_codec_decode_with_the_run_sign():
    """The receiver's values are the codec's fp64 evaluation rounded to fp32, negated on the non-positive run, in
    descending rank order."""
    g = torch.Generator().manual_seed(1)
    v = torch.randn(3000, generator=g)
    desc = torch.sort(v, descending=True).values
    num_pos = int((v > 0).sum())
    coef = dexp_runs_fit_oracle(desc, num_pos)
    got = dexp_runs_eval_oracle(coef, num_pos, v.numel())
    pos = dexp.double_exponential_eval(coef[:4], num_pos)
    neg = dexp.double_exponential_eval(coef[4:], v.numel() - num_pos)
    assert torch.equal(got[:num_pos], pos.flip(0)) and torch.equal(got[num_pos:], -neg)
    # the curves follow the data
    assert float(torch.linalg.norm(got - desc)) <= 0.15 * float(torch.linalg.norm(desc))


@pytest.mark.parametrize("run", [[], [0.5], [0.5, 0.25], [0.37] * 40, [0.0] * 40, [-0.0, 0.0] * 20])
def test_degenerate_runs_give_finite_curves(run):
    """Runs of length 0, 1 and 2, all equal, all zeros and mixed signed zeros, as the non-positive run next to a
    one-value positive run."""
    desc = torch.tensor([3.0] + [-x for x in run], dtype=torch.float32)
    coef = dexp_runs_fit_oracle(desc, 1)
    assert bool(torch.isfinite(coef).all()), coef
    vals = dexp_runs_eval_oracle(coef, 1, desc.numel())
    assert bool(torch.isfinite(vals).all())
    assert float(vals[0]) == 3.0
    if len(run) != 2:                 # two points, four unknowns: the fit is underdetermined
        assert torch.allclose(vals[1:], desc[1:], atol=1e-6)


@pytest.mark.parametrize("index", ["rle", "bloom", None])
@pytest.mark.parametrize("W", [1, 2, 3])
def test_decode_sum_and_residual(W, index):
    """The sum of the receivers' decodes is the sender-side aggregate, and each sender's residual on its shipped set
    is the accumulated value minus what the receivers decode."""
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index=index, value="dexp")
    grads = _grads(plan, W, seed=W)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in (1, 2):
        accs = [r + g for r, g in zip(res, grads)]
        out, res, slots = engine_oracle(plan, grads, res, epoch=epoch, average=False)
        decs = [decode_slot_oracle(plan, torch.from_numpy(s.view(np.int32))) for s in slots]
        assert torch.equal(sum(decs, torch.zeros(plan.total_elems)), out) if W == 1 else \
            torch.allclose(sum(decs), out, rtol=0, atol=1e-6 * float(out.abs().max()))
        for r in range(W):
            for ti, t in enumerate(plan.tensors):
                idx = t.elem_off + shipped_index_oracle(plan, slots[r], ti)
                assert torch.equal(res[r][idx], accs[r][idx] - decs[r][idx]), (r, t.name)


def test_stats_value_bytes():
    plan = BucketPlan(SHAPES, compress_ratio=0.02, index="rle", value="dexp")
    _, _, slots = engine_oracle(plan, _grads(plan, 1), [torch.zeros(plan.total_elems)])
    st = stats_from_slot(plan, slots[0])
    for t, row in zip(plan.tensors, st["tensors"]):
        assert row["value_bytes"] == (4 * (DEXP_COEF_WORDS + 2) + 2 * t.val_cap if t.vmode == 3 else 4 * t.val_cap)
    tot = st["total"]
    assert tot["value_bytes"] + tot["index_bytes"] + tot["header_bytes"] <= tot["wire_bytes"] == plan.wire_bytes()


# ---------------------------------------------------------------------------
# training: the oracle engine on a small model against dense SGD
# ---------------------------------------------------------------------------
class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(0)
        self.a, self.b = nn.Linear(32, 400), nn.Linear(400, 32)

    def forward(self, x):
        return self.b(torch.tanh(self.a(x)))


def _train(exchange, steps=150, W=2, lr=0.05):
    net = _Net()
    teacher = _Net()
    with torch.no_grad():
        for p in teacher.parameters():
            p.add_(torch.randn(p.shape, generator=torch.Generator().manual_seed(p.numel())) * 0.3)
    params = list(net.parameters())
    gen = torch.Generator().manual_seed(7)
    xs = torch.randn(W * 64, 32, generator=gen)
    ys = teacher(xs).detach()
    losses = []
    for step in range(steps):
        flat = []
        for r in range(W):
            net.zero_grad()
            sl = slice(64 * r, 64 * (r + 1))
            loss = (net(xs[sl]) - ys[sl]).pow(2).mean()
            loss.backward()
            flat.append(torch.cat([p.grad.reshape(-1) for p in params]))
        upd = exchange(flat, step)
        with torch.no_grad():
            off = 0
            for p in params:
                p -= lr * upd[off:off + p.numel()].view(p.shape)
                off += p.numel()
            losses.append(float((net(xs) - ys).pow(2).mean()))
    return losses


def test_oracle_engine_training_tracks_dense_sgd():
    """Top-k 5 % + rle index + dexp values, residual memory, W = 2, through engine_oracle: the loss falls to within
    a small factor of what dense SGD (the exact mean gradient) reaches on the same data."""
    numels = [p.numel() for p in _Net().parameters()]
    plan = BucketPlan(numels, compress_ratio=0.05, index="rle", value="dexp")
    assert sum(t.vmode == 3 for t in plan.tensors) == 2
    state = {"res": None}

    def to_plan(v):
        out = torch.zeros(plan.total_elems)
        off = 0
        for t in plan.tensors:
            out[t.elem_off:t.elem_off + t.numel] = v[off:off + t.numel]
            off += t.numel
        return out

    def from_plan(v):
        return torch.cat([v[t.elem_off:t.elem_off + t.numel] for t in plan.tensors])

    def fused(flat, step):
        g = [to_plan(f) for f in flat]
        if state["res"] is None:
            state["res"] = [torch.zeros(plan.total_elems) for _ in g]
        out, state["res"], _ = engine_oracle(plan, g, state["res"], epoch=step + 1)
        return from_plan(out)

    dense = _train(lambda flat, step: sum(flat) / len(flat))
    coded = _train(fused)
    assert all(np.isfinite(coded))
    assert coded[-1] < 0.5 * coded[0], (coded[0], coded[-1])
    assert coded[-1] < 2.0 * dense[-1] + 0.05 * dense[0], (coded[-1], dense[-1], dense[0])
