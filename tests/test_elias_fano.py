"""The tile-local Elias-Fano index ('index': 'elias_fano') on the CPU: the pack helpers and the per-tensor codec
round-trip and agree word for word, the fused oracle ships the codec's words and aggregates exactly what the run-length
index aggregates, the routing, and the wire volume against the run-length and bloom indices."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from hypothesis import given, settings, strategies as st

from deepreduce_b200 import spec
from deepreduce_b200.codecs.elias_fano import EliasFano
from deepreduce_b200.config import ConfigError, validate_params
from deepreduce_b200.parallel import BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import decode_slot_oracle, ef_pack, ef_unpack
from deepreduce_b200.parallel.plan import DYN_WORDS, MODE_EF, MODE_RAW, SLOT_HEADER_WORDS


def _layout_words(numel, cap):
    n_tiles = (numel + spec.TILE - 1) // spec.TILE
    L, lo, hi = spec.ef_layout(cap, n_tiles)
    return n_tiles, L, (n_tiles + 1) // 2, lo, hi


def _check_round_trip(idx, numel, cap):
    n_tiles, L, nc, lo_w, hi_w = _layout_words(numel, cap)
    assert lo_w == (cap * L + 31) // 32 and hi_w == (cap + n_tiles * (spec.TILE >> L) + 31) // 32
    cnt, lo, hi = ef_pack(idx, numel, cap)
    assert (cnt.size, lo.size, hi.size) == (nc, lo_w, hi_w)
    assert np.array_equal(ef_unpack(cnt, lo, hi, numel, cap, idx.size), idx)
    if idx.size == cap:                            # the codec's capacity is its value count
        vals = torch.randn(idx.size, generator=torch.Generator().manual_seed(idx.size))
        perm = torch.randperm(idx.size, generator=torch.Generator().manual_seed(1))
        v, enc, shape = EliasFano.compress((vals[perm], torch.from_numpy(idx)[perm], torch.Size([numel])), {})
        assert enc.dtype == torch.int32
        assert np.array_equal(enc.numpy().view(np.uint32), np.concatenate([cnt, lo, hi]))
        assert torch.equal(v, vals)                # reordered to ascending index
        v2, i2, _ = EliasFano.decompress((v, enc, shape), {})
        assert torch.equal(i2, torch.from_numpy(idx)) and torch.equal(v2, vals)
    return L


@settings(max_examples=60, deadline=None)
@given(numel=st.sampled_from([1001, 4096, 4097, 3 * 4096 + 17, 9 * 4096]), frac=st.floats(0.0, 1.0),
       seed=st.integers(0, 2 ** 31 - 1), slack=st.sampled_from([0, 0, 5]))
def test_round_trip_hypothesis(numel, frac, seed, slack):
    rng = np.random.default_rng(seed)
    n = max(1, int(round(frac * numel)))
    idx = np.sort(rng.choice(numel, n, replace=False)).astype(np.int64)
    _check_round_trip(idx, numel, min(numel, n + slack))


def test_round_trip_edges():
    """One element; a full tensor; tiles with 0 and with all 4096 entries; both ends of L."""
    Ls = set()
    for numel in (1001, 4096, 4097, 5 * 4096 + 3):
        Ls.add(_check_round_trip(np.array([numel - 1]), numel, 1))
        Ls.add(_check_round_trip(np.arange(numel, dtype=np.int64), numel, numel))
    # tile 0 full, tile 1 empty, tile 2 a few, tile 3 full up to the tensor's end
    idx = np.concatenate([np.arange(4096), 2 * 4096 + np.array([0, 7, 4095]), np.arange(3 * 4096, 4 * 4096 - 5)])
    Ls.add(_check_round_trip(idx.astype(np.int64), 4 * 4096 - 5, idx.size))
    assert 0 in Ls and 12 in Ls
    assert spec.ef_layout(1, 1)[0] == 11 and spec.ef_layout(1, 2)[0] == 12 and spec.ef_layout(4096, 1)[0] == 0


def test_layout_rule_is_the_smallest_argmin():
    for cap in (1, 2, 3, 40, 41, 1000, 4096, 10 ** 5):
        for n_tiles in (1, 2, 25, 577):
            L = spec.ef_layout(cap, n_tiles)[0]
            cost = [cap * l + n_tiles * (spec.TILE >> l) for l in range(13)]
            assert cost[L] == min(cost) and cost.index(min(cost)) == L


def test_codec_registered_and_empty_selection():
    from deepreduce_b200.codecs import compressor
    assert compressor["elias_fano"] is EliasFano
    v, enc, shape = EliasFano.compress((torch.zeros(0), torch.zeros(0, dtype=torch.int64), torch.Size([5000])), {})
    v2, i2, _ = EliasFano.decompress((v, enc, shape), {})
    assert i2.numel() == 0


# ---------------------------------------------------------------------------
# the fused oracle
# ---------------------------------------------------------------------------
SIZES = [500, 1001, 4096, 4097, 36864, 147456, 10, 300000]
VALUES = {"fp32": dict(), "bf16": dict(value="bf16"), "qsgd8": dict(value="qsgd"),
          "qsgd16": dict(value="qsgd", quantum_num=1000), "polyfit": dict(value="polyfit", poly_min_k=300),
          "dexp": dict(value="dexp")}


def _grads(plan, W, seed):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(W):
        g = torch.zeros(plan.total_elems)
        for v in plan.views(g):
            v.copy_(torch.randn(v.shape, generator=gen))
        out.append(g)
    return out


def test_plan_layout():
    plan = BucketPlan(SIZES, compress_ratio=0.01, index="elias_fano")
    rle = BucketPlan(SIZES, compress_ratio=0.01, index="rle")
    assert [t.mode for t in plan.tensors] == [MODE_RAW, MODE_EF, MODE_EF, MODE_EF, MODE_EF, MODE_EF, MODE_RAW, MODE_EF]
    for t, r in zip(plan.tensors, rle.tensors):
        assert t.val_cap == r.val_cap == t.k
        if t.mode != MODE_EF:
            continue
        L, lo, hi = spec.ef_layout(t.k, t.n_tiles)
        assert (t.ef_low_bits, t.off_hi) == (L, t.off_idx + lo)
        assert t.off_idx == t.off_prefix + -(-((t.n_tiles + 1) // 2) // 4) * 4
        assert t.index_bytes == 4 * ((t.n_tiles + 1) // 2 + lo + hi)
        assert t.words()[30:32] == [L, t.off_hi]
    # threshold at full capacity: L = 0, 2 bits per element
    thr = BucketPlan([4096 * 7], index="elias_fano", sparsifier="threshold", threshold=0.0)
    t = thr.tensors[0]
    assert t.val_cap == 4096 * 7 and t.ef_low_bits == 0 and t.index_bytes == 4 * (4 + 2 * 4096 * 7 // 32)
    assert BucketPlan([4096 * 7], index="elias_fano", sparsifier="threshold", capacity_ratio=0.01).tensors[0].ef_low_bits > 0
    with pytest.raises(ValueError):
        BucketPlan(SIZES, index="elias_fano", policy="conflict_sets")
    with pytest.raises(ValueError):
        BucketPlan(SIZES, index="elias_fano", sparsifier="randomk")


def test_oracle_slot_is_the_codec_words():
    plan = BucketPlan(SIZES, compress_ratio=0.02, index="elias_fano")
    (g,) = _grads(plan, 1, 3)
    _, _, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)])
    s = slots[0]
    for ti, t in enumerate(plan.tensors):
        if t.mode != MODE_EF:
            continue
        n_sel = int(s[SLOT_HEADER_WORDS + DYN_WORDS * ti])
        assert n_sel == t.val_cap                           # top-k ships its capacity
        acc = g[t.elem_off:t.elem_off + t.numel]
        from deepreduce_b200.parallel.engine import select_topk_oracle
        sel = select_topk_oracle(acc, t.k)[0][:t.val_cap]
        _, enc, _ = EliasFano.compress((acc[sel], sel, torch.Size([t.numel])), {})
        w = enc.numpy().view(np.uint32)
        _, _, nc, lo, hi = _layout_words(t.numel, t.val_cap)
        assert np.array_equal(s[t.off_prefix:t.off_prefix + nc], w[:nc]), t.name
        assert np.array_equal(s[t.off_idx:t.off_idx + lo + hi], w[nc:]), t.name


@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("sparsifier", ["topk", "threshold"])
def test_oracle_equals_rle_bit_for_bit(value, sparsifier):
    """Three steps at W = 3: output and residuals equal the run-length index's, bit for bit, and the receiver-side
    decode of the Elias-Fano slots gives the aggregate."""
    kw = dict(VALUES[value], compress_ratio=0.02)
    if sparsifier == "threshold":
        kw.update(sparsifier="threshold", threshold=1.0, capacity_ratio=0.5)
    ef, rle = BucketPlan(SIZES, index="elias_fano", **kw), BucketPlan(SIZES, index="rle", **kw)
    assert any(t.mode == MODE_EF and t.vmode == rle.tensors[i].vmode for i, t in enumerate(ef.tensors))
    W = 3
    ra = rb = [torch.zeros(ef.total_elems) for _ in range(W)]
    for epoch in (1, 2, 3):
        grads = _grads(ef, W, 10 + epoch)
        oa, ra, sa = engine_oracle(ef, grads, ra, epoch=epoch)
        ob, rb, _ = engine_oracle(rle, grads, rb, epoch=epoch)
        assert torch.equal(oa.view(torch.int32), ob.view(torch.int32)), epoch
        assert all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(ra, rb)), epoch
        dec = sum(decode_slot_oracle(ef, torch.from_numpy(s.view(np.int32))) for s in sa) / W
        assert torch.allclose(dec, oa, rtol=0, atol=1e-6 * float(oa.abs().max())), epoch


def test_wire_table():
    """DESIGN.md §7: ResNet-50's 161 tensors, bytes per rank per step.  The Elias-Fano index is at most the run-length
    index's from 1 % up (within one part in a thousand at 0.1 %), below bloom + hint everywhere, with every value mode."""
    from deepreduce_b200.models.resnet import resnet50
    numels = [p.numel() for p in resnet50().parameters()]
    assert len(numels) == 161
    want = {0.01: 1.315, 0.03: 3.761, 0.1: 11.926, 0.25: 28.789}     # MB, fp32 values
    for r in (0.001, 0.01, 0.03, 0.1, 0.25):
        for value in (None, "bf16", "qsgd"):
            ef = BucketPlan(numels, compress_ratio=r, index="elias_fano", value=value).wire_bytes()
            rle = BucketPlan(numels, compress_ratio=r, index="rle", value=value).wire_bytes()
            bloom = BucketPlan(numels, compress_ratio=r, index="bloom", value=value).wire_bytes()
            assert ef < bloom, (r, value)
            assert ef <= rle if r >= 0.01 else ef <= 1.001 * rle, (r, value)
            if value is None and r in want:
                assert abs(ef / 1e6 - want[r]) < 5e-4, (r, ef)


# ---------------------------------------------------------------------------
# routing and config
# ---------------------------------------------------------------------------
BASE = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
EF = {**BASE, 'deepreduce': 'index', 'index': 'elias_fano'}
EF_BOTH = {**BASE, 'deepreduce': 'both', 'index': 'elias_fano'}


def test_routing():
    from deepreduce_b200.parallel.ddp import _fused_supported, fused_path, plan_kwargs_from_params
    fused = [EF, {**EF, 'compressor': 'threshold', 'threshold': 0.01}, {**EF, 'memory': 'dgc', 'momentum': 0.9},
             {**EF, 'memory': 'none'}, {**EF, 'policy': 'p0'}]
    for v in ({'value': 'bf16'}, {'value': 'qsgd'}, {'value': 'qsgd', 'quantum_num': 1000, 'bucket_size': 512},
              {'value': 'polyfit'}, {'value': 'dexp'}, {'value': 'double_exp'}):
        fused += [{**EF_BOTH, **v}, {**EF_BOTH, **v, 'compressor': 'threshold', 'threshold': 0.01},
                  {**EF_BOTH, **v, 'memory': 'dgc', 'momentum': 0.9}]
    for p in fused:
        assert _fused_supported(p) and fused_path(p), p
        kw = plan_kwargs_from_params(p)
        assert kw['index'] == 'elias_fano'
        assert BucketPlan([80_000, 700], **kw).tensors[0].mode == MODE_EF
    for p in ({**EF, 'compressor': 'randomk'}, {**EF_BOTH, 'value': 'qsgd', 'compressor': 'randomk'},
              {**EF, 'policy': 'conflict_sets'}, {**EF, 'policy': 'conflict_sets', 'p2_pick_mask': True},
              {**EF_BOTH, 'value': 'qsgd', 'bucket_size': 256}, {**EF_BOTH, 'value': 'gzip'},
              {**EF, 'communicator': 'allreduce'}):
        assert not _fused_supported(p) and not fused_path(p), p


def test_config():
    for p in (EF, {**EF_BOTH, 'value': 'qsgd'}, {**EF_BOTH, 'value': 'bf16'}):
        validate_params(p, strict=True)
    for p in ({**EF_BOTH, 'value': 'qsgd', 'fused_rle_values': True},
              {**EF_BOTH, 'value': 'polyfit', 'fused_rle_values': True}):
        with pytest.raises(ConfigError):
            validate_params(p)


# ---------------------------------------------------------------------------
# the per-tensor path: gloo, W = 2
# ---------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, cfgs, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.trainer import Trainer
    for name, cfg in cfgs.items():
        torch.manual_seed(0)
        model = resnet20()
        tr = Trainer(model, cfg, lr=0.05, amp_dtype=None)
        assert not tr.ddp.fused
        gen = torch.Generator().manual_seed(100 + rank)
        for _ in range(3):
            tr.step(torch.randn(8, 3, 32, 32, generator=gen), target=torch.randint(0, 10, (8,), generator=gen))
        if rank == 0:
            ret[name] = torch.cat([p.detach().flatten() for p in model.parameters()])
    dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("extra", [{'deepreduce': 'index'}, {'deepreduce': 'both', 'value': 'qsgd'}])
def test_gloo_world2_per_tensor_equals_rle(extra):
    cfgs = {ix: {**BASE, **extra, 'index': ix} for ix in ('elias_fano', 'rle')}
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), cfgs, ret), nprocs=2, join=True)
    a, b = ret['elias_fano'], ret['rle']
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
