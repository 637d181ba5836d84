"""Scaled-sign values on the wire ('value': 'sign'), on the CPU: config and routing, the slot layout and wire bytes,
the bucket rule of the oracle at its branch points, the per-tensor codec against the fused oracle, decode against the
aggregate, error feedback, and training."""
import hashlib
import math
import os
import socket
import warnings

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from deepreduce_b200 import deepreduce_from_params, spec
from deepreduce_b200.codecs import Sign, compressor
from deepreduce_b200.codecs.sign import sign_decode_oracle, sign_encode_oracle
from deepreduce_b200.config import ConfigError, validate_params
from deepreduce_b200.parallel.engine import decode_slot_oracle, engine_oracle, stats_from_slot
from deepreduce_b200.parallel.plan import (MODE_BLOOM, MODE_EF, MODE_RAW, MODE_RLE, MODE_SHARED, VMODE_SIGN,
                                           BucketPlan)

BASE = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
THR = {'compressor': 'threshold', 'threshold': 0.01}
RANDK = {'compressor': 'randomk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
VALUE = {'deepreduce': 'value', 'value': 'sign'}
BOTH = {'deepreduce': 'both', 'value': 'sign'}
SHAPES = [30000, 5000, 300, 4097, 70000]


def _al(x):
    return (x + 3) // 4 * 4


def _resnet50_numels():
    from deepreduce_b200.models import resnet50
    return [p.numel() for p in reversed(list(resnet50().parameters()))]


# ---------------------------------------------------------------------------
# config and routing
# ---------------------------------------------------------------------------
FUSED = ([{**BASE, **VALUE}, {**BASE, **THR, **VALUE}, {**RANDK, **VALUE}, {**BASE, **VALUE, 'bucket_size': 512}]
         + [{**s, **BOTH, 'index': 'bloom', 'policy': p} for s in (BASE, {**BASE, **THR})
            for p in ('leftmost', 'random', 'p0')]
         + [{**BASE, **BOTH, 'index': 'bloom', 'policy': 'conflict_sets', 'p2_pick_mask': True},
            {**BASE, **BOTH, 'index': 'rle'}, {**BASE, **THR, **BOTH, 'index': 'rle'},
            {**BASE, **BOTH, 'index': 'elias_fano'}, {**BASE, **THR, **BOTH, 'index': 'elias_fano'}])


def test_config_accepts():
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        for p in FUSED:
            validate_params(p, strict=True)


def test_routing_fused():
    from deepreduce_b200.parallel.ddp import _fused_randomk_supported, _fused_supported, fused_path
    from deepreduce_b200.parallel.ddp import plan_kwargs_from_params
    for p in FUSED:
        assert fused_path(p), p
        assert _fused_randomk_supported(p) == (p['compressor'] == 'randomk'), p
        assert _fused_supported(p) == (p['compressor'] != 'randomk'), p
        kw = plan_kwargs_from_params(p)
        assert kw['value'] == 'sign', p
        BucketPlan(SHAPES, **{k: v for k, v in kw.items() if k != 'capacity_ratio'})
    # the shared-seed index gives the same aggregate under either communicator
    assert _fused_randomk_supported({**RANDK, **VALUE, 'communicator': 'allreduce'})


def test_routing_refused():
    from deepreduce_b200.parallel.ddp import fused_path
    # 'fused_rle_values' keeps its meaning and refuses sign values, and so does 'fused_dexp'
    p = {**BASE, **BOTH, 'index': 'rle', 'fused_rle_values': True}
    with pytest.raises(ConfigError):
        validate_params(p)
    assert not fused_path(p)
    for p in ({**BASE, **BOTH, 'index': 'rle', 'fused_dexp': True}, {**BASE, **VALUE, 'fused_dexp': True}):
        with pytest.raises(ConfigError):
            validate_params(p)
    for bs in (256, 1024, 1):
        for p in ({**BASE, **VALUE, 'bucket_size': bs}, {**BASE, **BOTH, 'index': 'rle', 'bucket_size': bs},
                  {**RANDK, **VALUE, 'bucket_size': bs}):
            with pytest.raises(ConfigError, match="512"):
                validate_params(p)
    # the per-tensor route: conflict_sets without the pick mask, 'both' under randomk, a host index codec
    for p in ({**BASE, **BOTH, 'index': 'bloom', 'policy': 'conflict_sets'}, {**RANDK, **BOTH, 'index': 'bloom'},
              {**BASE, **BOTH, 'index': 'huffman'}, {**BASE, **BOTH, 'index': 'integer'}):
        validate_params(p)
        assert not fused_path(p), p


def test_routing_of_existing_dicts_unchanged():
    from deepreduce_b200.parallel.ddp import fused_path
    fused = [BASE, {**BASE, 'deepreduce': 'index', 'index': 'bloom'}, {**BASE, 'deepreduce': 'index', 'index': 'rle'},
             {**BASE, 'deepreduce': 'index', 'index': 'elias_fano'},
             {**BASE, 'deepreduce': 'value', 'value': 'qsgd'}, {**BASE, 'deepreduce': 'both', 'value': 'polyfit'},
             {**BASE, 'deepreduce': 'value', 'value': 'bf16'}, {**BASE, 'deepreduce': 'both', 'value': 'bf16',
                                                               'index': 'rle'},
             {**BASE, 'deepreduce': 'both', 'value': 'qsgd', 'index': 'rle', 'fused_rle_values': True},
             {**BASE, 'deepreduce': 'both', 'value': 'dexp', 'index': 'rle', 'fused_dexp': True},
             {**RANDK, 'communicator': 'allreduce'}, {**RANDK, 'deepreduce': 'value', 'value': 'qsgd'},
             {**RANDK, 'deepreduce': 'value', 'value': 'bf16'}]
    per_tensor = [{**BASE, 'deepreduce': 'both', 'value': 'qsgd', 'index': 'rle'},
                  {**BASE, 'deepreduce': 'both', 'value': 'polyfit', 'index': 'rle'},
                  {**BASE, 'deepreduce': 'value', 'value': 'dexp'},
                  {**BASE, 'deepreduce': 'both', 'value': 'qsgd', 'bucket_size': 256},
                  {**RANDK, 'deepreduce': 'value', 'value': 'qsgd', 'bucket_size': 256},
                  {**RANDK, 'deepreduce': 'value', 'value': 'polyfit'},
                  {**BASE, 'deepreduce': 'both', 'index': 'bloom', 'policy': 'conflict_sets'},
                  {**BASE, 'communicator': 'allgather', 'deepreduce': 'value', 'value': 'gzip'}]
    assert all(fused_path(p) for p in fused)
    assert not any(fused_path(p) for p in per_tensor)


# ---------------------------------------------------------------------------
# layout
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(index=None), dict(index="bloom"), dict(index="bloom", policy="p0"),
                                dict(index="rle"), dict(index="elias_fano"), dict(index=None, sparsifier="randomk")],
                         ids=str)
def test_layout(kw):
    plan = BucketPlan(SHAPES, compress_ratio=0.05, value="sign", **kw)
    ref = BucketPlan(SHAPES, compress_ratio=0.05, **kw)
    P = plan.payload_words
    _, _, tasks, n_tasks = plan.poly_tables()
    want = sorted((i, c) for i, t in enumerate(plan.tensors) if t.vmode == VMODE_SIGN for c in range(0, t.val_cap, 512))
    assert sorted(map(tuple, tasks.view(-1, 2).tolist()[:n_tasks])) == want and n_tasks > 0
    saved = 0
    for t, r in zip(plan.tensors, ref.tensors):
        assert (t.mode, t.k, t.val_cap) == (r.mode, r.k, r.val_cap)
        if t.numel <= plan.min_numel:
            assert t.vmode == 0 and not t.coded
            continue
        assert t.vmode == VMODE_SIGN and t.coded and not t.ranked
        nb, nw = (t.val_cap + 511) // 512, (t.val_cap + 31) // 32
        assert t.value_bytes == 4 * nb + 4 * nw
        assert t.off_coef % 4 == 0 and t.off_rankmap == t.off_coef + _al(nb)
        nxt = {MODE_RAW: t.off_idx, MODE_BLOOM: t.off_filter, MODE_RLE: t.off_prefix, MODE_EF: t.off_prefix}.get(t.mode)
        if nxt is not None:
            assert nxt == t.off_rankmap + _al(nw)
        assert t.off_rankmap + nw <= P and t.off_vals >= P and t.off_selidx >= P        # fp32 values: scratch
        saved += _al(t.val_cap) - _al(nb) - _al(nw)
    assert ref.payload_words - P == saved
    stats = stats_from_slot(plan, engine_oracle(plan, [torch.randn(plan.total_elems)],
                                                [torch.zeros(plan.total_elems)])[2][0])
    assert stats["total"]["value_bytes"] == sum(t.value_bytes for t in plan.tensors)


# ResNet-50 wire bytes per rank per step with sign values, in KB, and the issue's layout estimates beside them
WIRE = {0.001: {"elias_fano": 62.7, "rle": 62.9, "bloom": 198.0, "plain": 113.4, "randomk": 14.9},
        0.01: {"elias_fano": 328.5, "rle": 438.5, "bloom": 626.5, "plain": 1063.4, "randomk": 45.5},
        0.1: {"elias_fano": 2052.3, "rle": 4206.2, "bloom": 3547.6, "plain": 10576.4, "randomk": 358.2}}
ESTIMATE = {(0.01, "elias_fano"): 328, (0.01, "rle"): 438, (0.01, "bloom"): 626, (0.01, "plain"): 1062,
            (0.01, "randomk"): 45, (0.001, "elias_fano"): 61, (0.1, "elias_fano"): 2052}
WIRE_KW = {"elias_fano": dict(index="elias_fano"), "rle": dict(index="rle"), "bloom": dict(index="bloom"),
           "plain": dict(index=None), "randomk": dict(index=None, sparsifier="randomk")}


@pytest.mark.parametrize("ratio", sorted(WIRE))
def test_wire_bytes_resnet50(ratio):
    numels = _resnet50_numels()
    for name, kw in WIRE_KW.items():
        sign = BucketPlan(numels, compress_ratio=ratio, value="sign", **kw).wire_bytes()
        qsgd = BucketPlan(numels, compress_ratio=ratio, value="qsgd", **kw).wire_bytes()
        assert sign < qsgd, name
        assert round(sign / 1000, 1) == WIRE[ratio][name], name
        if (ratio, name) in ESTIMATE:
            assert abs(sign / 1000 - ESTIMATE[(ratio, name)]) < 3.0, name


# digests of the device tensor table of plans without sign values, as the parent commit builds them
TABLES = {"plain": "ecc1a39e00fdfa11", "bloom": "81a7ee9891cb4392", "p0": "c737d44fcf2abfe0", "rle": "a9618ff29cda0ae3",
          "randomk": "40117f54f4dbd0f1", "rle_qsgd": "4e56737a1ab40339", "bloom_polyfit": "b900e5ce9a328cc1",
          "value_dexp": "9c7e4f6ecb8cf43b"}
TABLE_PLANS = {"plain": dict(index=None), "bloom": dict(index="bloom"), "p0": dict(index="bloom", policy="p0"),
               "rle": dict(index="rle"), "randomk": dict(index=None, sparsifier="randomk"),
               "rle_qsgd": dict(index="rle", value="qsgd"), "bloom_polyfit": dict(index="bloom", value="polyfit"),
               "value_dexp": dict(index=None, value="dexp")}


def _table_digest(plan):
    h = hashlib.sha256(plan.tensor_table().numpy().tobytes())
    h.update(np.array([plan.payload_words, plan.slot_words], dtype=np.int64).tobytes())
    for t in plan.poly_tables():
        h.update(t.numpy().tobytes() if torch.is_tensor(t) else np.int64(t).tobytes())
    return h.hexdigest()[:16]


@pytest.mark.parametrize("name", sorted(TABLE_PLANS))
def test_plans_without_sign_unchanged(name):
    plan = BucketPlan(_resnet50_numels(), compress_ratio=0.01, **TABLE_PLANS[name])
    assert _table_digest(plan) == TABLES[name]


# ---------------------------------------------------------------------------
# the bucket rule
# ---------------------------------------------------------------------------
def _f(bits):
    return torch.from_numpy(np.asarray(bits, dtype=np.uint32).view(np.float32).copy())


def _scale_ref(v):
    """fl32(fsum(|v|) / n): the exact mean, rounded once to fp64 and then to fp32."""
    return float(np.float32(math.fsum(abs(float(x)) for x in v) / len(v)))


def _check_rule(v):
    """The oracle's words against a plain-Python statement of the rule, bucket by bucket."""
    bits, scales = sign_encode_oracle(v)
    K = v.numel()
    assert bits.dtype == torch.int32 and bits.numel() == (K + 31) // 32
    assert scales.dtype == torch.float32 and scales.numel() == (K + 511) // 512
    b = bits.numpy().view(np.uint32)
    for p in range(K):
        assert ((int(b[p // 32]) >> (p % 32)) & 1) == int(bool(v[p] < 0)), p
    if K % 32:
        assert int(b[-1]) >> (K % 32) == 0                 # bits past K are 0
    for j in range(scales.numel()):
        seg = v[512 * j:512 * j + 512]
        if bool(torch.isfinite(seg).all()):
            mu, ref = float(scales[j]), _scale_ref(seg)
            assert abs(mu - ref) <= abs(float(np.spacing(np.float32(ref)))), (j, mu, ref)
    d = sign_decode_oracle(bits, scales, K)
    mu = scales[torch.arange(K) // 512]
    assert torch.equal(d.view(torch.int32), torch.where(v < 0, -mu, mu).view(torch.int32))
    return bits, scales, d


@pytest.mark.parametrize("n", [1, 31, 32, 33, 511, 512, 513, 1025])
def test_rule_at_the_bucket_edges(n):
    v = torch.randn(n, generator=torch.Generator().manual_seed(n)) * torch.exp(
        torch.randn(n, generator=torch.Generator().manual_seed(n + 1)) * 3)
    _check_rule(v)


def test_rule_same_exponent_is_exact():
    # values of one binade: the pair-tree sum is exact in fp64, so mu equals fl32(fsum / n)
    g = torch.Generator().manual_seed(3)
    for n in (1, 7, 512, 1000, 1537):
        v = (1.0 + torch.rand(n, generator=g)) * torch.sign(torch.randn(n, generator=g))
        _, scales, _ = _check_rule(v)
        for j in range(scales.numel()):
            assert float(scales[j]) == _scale_ref(v[512 * j:512 * j + 512])


def test_rule_special_values():
    zeros = _f([0x00000000, 0x80000000] * 8)                        # +0 and -0: bit 0
    sub = _f([0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF])        # subnormals keep their sign bit
    big = _f([0x7F7FFFFF, 0xFF7FFFFF, 0x7F7FFFFE, 0xFF7FFFFF])       # near FLT_MAX: mu stays finite
    v = torch.cat([zeros, sub, big, torch.randn(100)])
    bits, scales, d = _check_rule(v)
    b = bits.numpy().view(np.uint32)
    assert [(int(b[0]) >> p) & 1 for p in range(16)] == [0] * 16
    assert [(int(b[0]) >> p) & 1 for p in range(16, 20)] == [0, 1, 0, 1]
    assert bool(torch.isfinite(scales).all()) and float(scales[0]) > 0
    # a zero value decodes to +mu
    assert bool((d[:16] == scales[0]).all())
    # a bucket of subnormals only: mu is a subnormal too, exact to fp32 rounding
    s = _f([0x00000003, 0x80000005])
    assert float(sign_encode_oracle(s)[1][0]) == float(np.float32((3 + 5) * 2.0 ** -149 / 2))


def test_rule_nonfinite_buckets_stay_local():
    g = torch.Generator().manual_seed(5)
    v = torch.randn(4 * 512 + 100, generator=g)
    v[700] = float("nan")
    v[1100] = float("inf")
    v[1600] = -float("inf")
    bits, scales, d = _check_rule(v)
    assert math.isnan(float(scales[1])) and float(scales[2]) == math.inf and float(scales[3]) == math.inf
    assert bool(torch.isnan(d[512:1024]).all())
    assert bool(torch.isinf(d[1024:2048]).all())
    assert bool(torch.isfinite(d[:512]).all()) and bool(torch.isfinite(d[2048:]).all())
    assert ((int(bits[700 // 32]) >> (700 % 32)) & 1) == 0                # NaN ships bit 0


def _plant(plan, values):
    """One tensor of the plan holding exactly the planted values (all shipped) and zeros."""
    g = torch.zeros(plan.total_elems)
    g[:values.numel()] = values
    return g


@pytest.mark.parametrize("index", [None, "bloom", "rle", "elias_fano"])
@pytest.mark.parametrize("n", [1, 33, 512, 513, 1025])
def test_oracle_slot_words(index, n):
    vals = torch.randn(n, generator=torch.Generator().manual_seed(n)) * 4.0
    vals[vals.abs() < 1e-3] = 1.0                            # every planted value is selected
    plan = BucketPlan([4096], ks=[n], index=index, value="sign", min_numel=0)
    t = plan.tensors[0]
    g = _plant(plan, vals)
    out, res, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)])
    bits, scales = sign_encode_oracle(vals)
    a = slots[0]
    assert np.array_equal(a[t.off_coef:t.off_coef + scales.numel()], scales.numpy().view(np.uint32))
    assert np.array_equal(a[t.off_rankmap:t.off_rankmap + bits.numel()], bits.numpy().view(np.uint32))
    d = sign_decode_oracle(bits, scales, n)
    assert torch.equal(out[:n], d)
    assert torch.equal(res[0][:n], vals - d)
    assert torch.equal(decode_slot_oracle(plan, a)[:n], d)


def test_oracle_nonfinite_residual_and_dgc_momentum():
    n = 3 * 512
    vals = torch.randn(n, generator=torch.Generator().manual_seed(1)) + 3.0
    vals[600] = float("nan")                                 # bucket 1 decodes to NaN: residual 0
    plan = BucketPlan([4096], ks=[n], index=None, value="sign", min_numel=0)
    g = _plant(plan, vals)
    out, res, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)])
    assert bool(torch.isnan(out[512:1024]).all()) and bool((res[0][512:1024] == 0).all())
    assert torch.equal(res[0][:512], vals[:512] - out[:512]) and torch.equal(res[0][1024:n], vals[1024:] - out[1024:n])


def test_oracle_dgc_zero_bucket_keeps_momentum():
    """'randomk' ships values whatever they are.  A tensor whose every value is 0 has mu = 0 in every bucket: its
    values decode to 0 and keep their momentum.  In the other tensor mu != 0 and the shipped momentum is cleared."""
    plan = BucketPlan([20000, 20000], compress_ratio=0.1, index=None, sparsifier="randomk", value="sign", min_numel=0)
    a, b = plan.tensors
    g = torch.zeros(plan.total_elems)
    g[b.elem_off:b.elem_off + b.numel] = torch.randn(b.numel) + 5.0
    u0 = torch.randn(plan.total_elems)
    r0 = -(0.5 * u0 + g)                       # r + u = 0 wherever g = 0, so tensor a's values are all 0
    r0[b.elem_off:] = 0.0
    out, res, slots, mom = engine_oracle(plan, [g], [r0], momentum=0.5, moms=[u0])
    u = 0.5 * u0 + g
    nb_a = (int(slots[0][8]) + 511) // 512
    assert nb_a > 1 and not slots[0][a.off_coef:a.off_coef + nb_a].any()          # every scale of tensor a is 0
    assert bool((out[:a.numel] == 0).all()) and torch.equal(mom[0][:a.numel], u[:a.numel])
    shipped_b = out[b.elem_off:b.elem_off + b.numel] != 0
    assert int(shipped_b.sum()) >= b.k
    assert bool((mom[0][b.elem_off:b.elem_off + b.numel][shipped_b] == 0).all())
    assert torch.equal(mom[0][b.elem_off:b.elem_off + b.numel][~shipped_b], u[b.elem_off:b.elem_off + b.numel][~shipped_b])


# ---------------------------------------------------------------------------
# decode and aggregate
# ---------------------------------------------------------------------------
MODES = {"plain": dict(index=None), "threshold": dict(index=None, sparsifier="threshold", threshold=1.5),
         "bloom": dict(index="bloom"), "bloom_random": dict(index="bloom", policy="random", fpr=0.02),
         "bloom_p0": dict(index="bloom", policy="p0"), "bloom_p2": dict(index="bloom", policy="conflict_sets"),
         "rle": dict(index="rle"), "rle_threshold": dict(index="rle", sparsifier="threshold", threshold=1.5),
         "elias_fano": dict(index="elias_fano"), "randomk": dict(index=None, sparsifier="randomk")}


@pytest.mark.parametrize("W", [1, 2, 3])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_decode_sums_to_the_aggregate(mode, W):
    plan = BucketPlan(SHAPES, compress_ratio=0.02, value="sign", min_numel=1000, **MODES[mode])
    gen = torch.Generator().manual_seed(W)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    for e in (1, 2):
        grads = [torch.randn(plan.total_elems, generator=gen) for _ in range(W)]
        out, res, slots = engine_oracle(plan, grads, res, epoch=e, average=False)
        dec = torch.zeros(plan.total_elems)
        for s in slots:
            dec += decode_slot_oracle(plan, s)
        assert torch.equal(dec, out), (mode, W, e)
        assert any(t.vmode == VMODE_SIGN for t in plan.tensors)


@pytest.mark.parametrize("mode", ["plain", "bloom", "rle", "elias_fano", "randomk"])
def test_error_feedback(mode):
    """W = 1: per step, out + new residual equals r + g up to the rounding of v - d."""
    plan = BucketPlan(SHAPES, compress_ratio=0.01, value="sign", **MODES[mode])
    gen = torch.Generator().manual_seed(7)
    res = [torch.zeros(plan.total_elems)]
    for e in range(1, 9):
        g = torch.randn(plan.total_elems, generator=gen)
        acc = res[0] + g
        out, res, _ = engine_oracle(plan, [g], res, epoch=e)
        err = (out.double() + res[0].double() - acc.double()).abs()
        assert bool((err <= (acc.double() - out.double()).abs() * 2.0 ** -24).all()), e


# ---------------------------------------------------------------------------
# the per-tensor codec
# ---------------------------------------------------------------------------
def test_codec_round_trip():
    assert compressor["sign"] is Sign and Sign.kind == "value" and Sign.order_preserving
    g = torch.Generator().manual_seed(0)
    for K in (0, 1, 33, 512, 5000):
        v = torch.randn(K, generator=g)
        idx = torch.randperm(100_000, generator=g)[:K]                     # not in index order
        wire, i2, shape = Sign.compress((v, idx, torch.Size([100_000])), {})
        order = torch.argsort(idx)
        assert torch.equal(i2, idx[order])
        bits, scales = sign_encode_oracle(v[order])
        assert wire.dtype == torch.int32 and int(wire[0]) == K
        assert torch.equal(wire[1:], torch.cat([bits, scales.view(torch.int32)]))
        back, i3, _ = Sign.decompress((wire, i2, shape), {})
        assert i3 is i2 and torch.equal(back, sign_decode_oracle(bits, scales, K))
        back, _, _ = Sign.decompress((wire, None, shape), {})                 # 'both': no index list
        assert back.numel() == K
    with pytest.raises(ValueError):
        Sign.decompress((wire[:-1], None, shape), {})


@pytest.mark.parametrize("extra", [VALUE, {**BOTH, 'index': 'rle'}, {**BOTH, 'index': 'elias_fano'}], ids=str)
def test_grace_step_matches_the_fused_oracle(extra):
    """At W = 1 the per-tensor path and the fused oracle ship the same sign values and keep the same residuals, on a
    gradient whose top-k both select the same way (K values well above the rest)."""
    torch.manual_seed(0)
    n = 60000
    k = spec.topk_k(n, 0.01)
    grc = deepreduce_from_params({**BASE, **extra})
    plan = BucketPlan([n], compress_ratio=0.01, value="sign", index=extra.get('index') if extra is not VALUE else None)
    assert plan.tensors[0].val_cap > 512                                  # more than one bucket
    res = [torch.zeros(plan.total_elems)]
    for step in range(3):
        g = torch.randn(n) * 1e-3
        hot = torch.randperm(n)[:k]
        g[hot] = (torch.rand(k) + 1.0) * torch.sign(torch.randn(k)) * 10.0
        out = grc.step(g.clone(), "w")
        out_o, res, _ = engine_oracle(plan, [g], res, epoch=step + 1)
        assert torch.equal(out.flatten(), out_o[:n]), step
        assert torch.equal(grc.memory.residuals["w"].flatten(), res[0][:n]), step


# ---------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------
@pytest.mark.timeout(300)
def test_mlp_learns_with_sign_values():
    """The small MLP of test_convergence.py, trained through the per-tensor path with sign values, passes the same
    "learns about as well as dense" bounds."""
    from test_convergence import BASE as CBASE, _train
    dense = _train({'compressor': 'none', 'memory': 'none', 'communicator': 'allreduce'})
    d_end = sum(dense[-10:]) / 10
    for cfg in (dict(CBASE, **VALUE), dict(CBASE, **BOTH, index='rle'), dict(CBASE, **BOTH, index='elias_fano'),
                dict(RANDK, **VALUE, compress_ratio=0.05)):
        comp = _train(dict(cfg, min_numel=100))
        c_end = sum(comp[-10:]) / 10
        assert c_end < 0.35 * comp[0], (cfg, comp[0], c_end)
        assert c_end < 2.0 * d_end + 0.15, (cfg, d_end, c_end)


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
        losses = [float(tr.step(torch.randn(8, 3, 32, 32, generator=gen), target=torch.randint(0, 10, (8,), generator=gen)))
                  for _ in range(3)]
        ret[(name, rank)] = (torch.cat([p.detach().flatten() for p in model.parameters()]), losses)
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_gloo_world2_per_tensor_training():
    cfgs = {"value": {**BASE, **VALUE}, "rle": {**BASE, **BOTH, 'index': 'rle'},
            "elias_fano": {**BASE, **BOTH, 'index': 'elias_fano'}}
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), cfgs, ret), nprocs=2, join=True)
    for name in cfgs:
        (p0, l0), (p1, l1) = ret[(name, 0)], ret[(name, 1)]
        assert torch.equal(p0, p1), name                           # both ranks applied the same aggregate
        assert all(math.isfinite(x) for x in l0 + l1) and bool(torch.isfinite(p0).all()), name
    # 'both' over the two lossless indices ships the same values and indices: the same training run
    assert torch.equal(ret[("rle", 0)][0], ret[("elias_fano", 0)][0])
