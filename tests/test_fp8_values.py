"""FP8 values on the wire ('value': 'fp8'), on the CPU: config and routing, the slot layout and wire bytes, the block
rule of the oracle against an independent fp64 / brute-force statement of it, the per-tensor codec against the fused
oracle, decode against the aggregate, error feedback, and training."""
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
from deepreduce_b200.codecs import FP8, compressor
from deepreduce_b200.codecs.fp8 import fp8_decode_oracle, fp8_encode_oracle, fp8_scale_bytes
from deepreduce_b200.config import ConfigError, validate_params
from deepreduce_b200.parallel.engine import decode_slot_oracle, engine_oracle, stats_from_slot
from deepreduce_b200.parallel.plan import (MODE_BLOOM, MODE_EF, MODE_RAW, MODE_RLE, VMODE_FP8, BucketPlan)

BASE = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
THR = {'compressor': 'threshold', 'threshold': 0.01}
RANDK = {'compressor': 'randomk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
DGC = {'memory': 'dgc', 'momentum': 0.9, 'weight_decay': 1e-4, 'clip_norm': 10.0}
VALUE = {'deepreduce': 'value', 'value': 'fp8'}
BOTH = {'deepreduce': 'both', 'value': 'fp8'}
SHAPES = [30000, 5000, 300, 4097, 70000]


def _al(x):
    return (x + 3) // 4 * 4


def _resnet50_numels():
    from deepreduce_b200.models import resnet50
    return [p.numel() for p in reversed(list(resnet50().parameters()))]


# ---------------------------------------------------------------------------
# config and routing
# ---------------------------------------------------------------------------
FUSED = ([{**BASE, **VALUE}, {**BASE, **THR, **VALUE}, {**RANDK, **VALUE}, {**BASE, **VALUE, 'bucket_size': 32},
          {**BASE, **DGC, **VALUE}, {**BASE, **DGC, **BOTH, 'index': 'rle'},
          {**BASE, **VALUE, 'warmup_ratios': [0.25, 0.05], 'warmup_steps': 2}]
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
        assert kw['value'] == 'fp8', p
        plan = BucketPlan(SHAPES, **{k: v for k, v in kw.items() if k != 'capacity_ratio'})
        assert any(t.vmode == VMODE_FP8 for t in plan.tensors), p
    # the shared-seed index gives the same aggregate under either communicator
    assert _fused_randomk_supported({**RANDK, **VALUE, 'communicator': 'allreduce'})


def test_routing_refused():
    from deepreduce_b200.parallel.ddp import fused_path
    # 'fused_rle_values' keeps its meaning and refuses fp8 values, and so does 'fused_dexp'
    p = {**BASE, **BOTH, 'index': 'rle', 'fused_rle_values': True}
    with pytest.raises(ConfigError):
        validate_params(p)
    assert not fused_path(p)
    for p in ({**BASE, **BOTH, 'index': 'rle', 'fused_dexp': True}, {**BASE, **VALUE, 'fused_dexp': True}):
        with pytest.raises(ConfigError):
            validate_params(p)
    for bs in (512, 256, 64, 16, 1):
        for p in ({**BASE, **VALUE, 'bucket_size': bs}, {**BASE, **BOTH, 'index': 'rle', 'bucket_size': bs},
                  {**RANDK, **VALUE, 'bucket_size': bs}):
            with pytest.raises(ConfigError, match="32"):
                validate_params(p)
    # the per-tensor route: conflict_sets without the pick mask, 'both' under randomk, a host index codec
    for p in ({**BASE, **BOTH, 'index': 'bloom', 'policy': 'conflict_sets'}, {**RANDK, **BOTH, 'index': 'bloom'},
              {**BASE, **BOTH, 'index': 'huffman'}, {**BASE, **BOTH, 'index': 'integer'}):
        validate_params(p)
        assert not fused_path(p), p


def test_routing_of_existing_dicts_unchanged():
    from deepreduce_b200.parallel.ddp import fused_path, plan_kwargs_from_params
    fused = [BASE, {**BASE, 'deepreduce': 'index', 'index': 'bloom'}, {**BASE, 'deepreduce': 'index', 'index': 'rle'},
             {**BASE, 'deepreduce': 'index', 'index': 'elias_fano'},
             {**BASE, 'deepreduce': 'value', 'value': 'qsgd'}, {**BASE, 'deepreduce': 'both', 'value': 'polyfit'},
             {**BASE, 'deepreduce': 'value', 'value': 'bf16'}, {**BASE, 'deepreduce': 'both', 'value': 'bf16',
                                                               'index': 'rle'},
             {**BASE, 'deepreduce': 'value', 'value': 'sign'}, {**BASE, 'deepreduce': 'both', 'value': 'sign',
                                                               'index': 'elias_fano'},
             {**BASE, 'deepreduce': 'both', 'value': 'qsgd', 'index': 'rle', 'fused_rle_values': True},
             {**BASE, 'deepreduce': 'both', 'value': 'dexp', 'index': 'rle', 'fused_dexp': True},
             {**RANDK, 'communicator': 'allreduce'}, {**RANDK, 'deepreduce': 'value', 'value': 'qsgd'},
             {**RANDK, 'deepreduce': 'value', 'value': 'bf16'}, {**RANDK, 'deepreduce': 'value', 'value': 'sign'}]
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
    assert all(plan_kwargs_from_params(p)['value'] != 'fp8' for p in fused)
    # an existing dict with a 'bucket_size' other than 32 keeps its meaning: only 'fp8' values read it as a block size
    validate_params({**BASE, 'deepreduce': 'value', 'value': 'qsgd', 'bucket_size': 512})


# ---------------------------------------------------------------------------
# layout
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(index=None), dict(index="bloom"), dict(index="bloom", policy="p0"),
                                dict(index="rle"), dict(index="elias_fano"), dict(index=None, sparsifier="randomk")],
                         ids=str)
def test_layout(kw):
    plan = BucketPlan(SHAPES, compress_ratio=0.05, value="fp8", **kw)
    ref = BucketPlan(SHAPES, compress_ratio=0.05, **kw)
    P = plan.payload_words
    _, _, tasks, n_tasks = plan.poly_tables()
    want = sorted((i, c) for i, t in enumerate(plan.tensors) if t.vmode == VMODE_FP8 for c in range(0, t.val_cap, 512))
    assert sorted(map(tuple, tasks.view(-1, 2).tolist()[:n_tasks])) == want and n_tasks > 0
    saved = 0
    for t, r in zip(plan.tensors, ref.tensors):
        assert (t.mode, t.k, t.val_cap) == (r.mode, r.k, r.val_cap)
        if t.numel <= plan.min_numel:
            assert t.vmode == 0 and not t.coded
            continue
        assert t.vmode == VMODE_FP8 and t.coded and not t.ranked
        ns, ne = (t.val_cap + 127) // 128, (t.val_cap + 3) // 4
        assert t.value_bytes == (t.val_cap + 31) // 32 + t.val_cap
        assert t.off_coef % 4 == 0 and t.off_rankmap == t.off_coef + _al(ns)
        nxt = {MODE_RAW: t.off_idx, MODE_BLOOM: t.off_filter, MODE_RLE: t.off_prefix, MODE_EF: t.off_prefix}.get(t.mode)
        if nxt is not None:
            assert nxt == t.off_rankmap + _al(ne)
        assert t.off_rankmap + ne <= P and t.off_vals >= P and t.off_selidx >= P        # fp32 values: scratch
        saved += _al(t.val_cap) - _al(ns) - _al(ne)
    assert ref.payload_words - P == saved
    stats = stats_from_slot(plan, engine_oracle(plan, [torch.randn(plan.total_elems)],
                                                [torch.zeros(plan.total_elems)])[2][0])
    assert stats["total"]["value_bytes"] == sum(t.value_bytes for t in plan.tensors)


# ResNet-50 wire bytes per rank per step with fp8 values, in KB, and the estimates of the design (QSGD int8 plans with
# the value region swapped for the fp8 layout) beside them
WIRE = {0.001: {"elias_fano": 85.3, "rle": 85.6, "bloom": 220.6, "plain": 136.0, "randomk": 38.8},
        0.01: {"elias_fano": 557.6, "rle": 667.6, "bloom": 855.6, "plain": 1292.4, "randomk": 275.7},
        0.1: {"elias_fano": 4346.4, "rle": 6500.3, "bloom": 5841.7, "plain": 12870.5, "randomk": 2653.5}}
ESTIMATE = {"elias_fano": 557.6, "rle": 667.6, "bloom": 855.6, "plain": 1292.0, "randomk": 275.7}
WIRE_KW = {"elias_fano": dict(index="elias_fano"), "rle": dict(index="rle"), "bloom": dict(index="bloom"),
           "plain": dict(index=None), "randomk": dict(index=None, sparsifier="randomk")}


@pytest.mark.parametrize("ratio", sorted(WIRE))
def test_wire_bytes_resnet50(ratio):
    numels = _resnet50_numels()
    for name, kw in WIRE_KW.items():
        fp8 = BucketPlan(numels, compress_ratio=ratio, value="fp8", **kw).wire_bytes()
        qsgd = BucketPlan(numels, compress_ratio=ratio, value="qsgd", **kw).wire_bytes()
        bf16 = BucketPlan(numels, compress_ratio=ratio, value="bf16", **kw).wire_bytes()
        assert qsgd < fp8 < bf16, name
        assert round(fp8 / 1000, 1) == WIRE[ratio][name], name
        if ratio == 0.01:
            assert abs(fp8 / 1000 - ESTIMATE[name]) <= 1.0, name


# digests of the device tensor table of plans without fp8 values, as the parent commit builds them
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
def test_plans_without_fp8_unchanged(name):
    plan = BucketPlan(_resnet50_numels(), compress_ratio=0.01, **TABLE_PLANS[name])
    assert _table_digest(plan) == TABLES[name]


# ---------------------------------------------------------------------------
# the block rule, against an independent statement of it: fp64 arithmetic and a brute-force nearest-even search over
# the 127 non-negative finite E4M3 values
# ---------------------------------------------------------------------------
def _e4m3_value(c):
    E, m = (c >> 3) & 0xF, c & 7
    a = m * 2.0 ** -9 if E == 0 else (1 + m / 8) * 2.0 ** (E - 7)
    return -a if c & 0x80 else a


E4M3_POS = np.array([_e4m3_value(c) for c in range(0x7F)])         # codes 0x00 .. 0x7E: 0 .. 448, ascending


def _rne_ref(x):
    """The E4M3 code nearest to the fp64 x (|x| <= 448), ties to the even code; the sign bit follows x (-0.0: 0x80)."""
    a = abs(x)
    assert a <= 448.0
    dist = np.abs(E4M3_POS - a)
    best = np.nonzero(dist == dist.min())[0]
    c = int(best[0]) if len(best) == 1 else int(best[best % 2 == 0][0])
    return c | (0x80 if math.copysign(1.0, x) < 0 else 0)


def _exp_ref(a):
    """The smallest integer e with a * 2^-e <= 448, clamped below at -127, by fp64 search (a >= 0 finite)."""
    e = -127
    while math.ldexp(a, -e) > 448.0:
        e += 1
    return e


def _f(bits):
    return torch.from_numpy(np.asarray(bits, dtype=np.uint32).view(np.float32).copy())


def _bytes(words, n):
    return np.frombuffer(words.numpy().astype(np.int32).tobytes(), dtype=np.uint8)[:n].astype(np.int64)


def _check_rule(v):
    """The oracle's words and decode against the reference, block by block and value by value.  Returns the scale bytes,
    the element bytes and the decode."""
    K = v.numel()
    scales, elems = fp8_encode_oracle(v)
    nb = (K + 31) // 32
    assert scales.dtype == torch.int32 and scales.numel() == (K + 127) // 128
    assert elems.dtype == torch.int32 and elems.numel() == (K + 3) // 4
    s, q = _bytes(scales, 4 * scales.numel()), _bytes(elems, 4 * elems.numel())
    assert not s[nb:].any() and not q[K:].any()                          # zero padding
    d = fp8_decode_oracle(scales, elems, K)
    vd = v.double().numpy()
    for b in range(nb):
        blk = vd[32 * b:32 * b + 32]
        if not np.isfinite(blk).all():
            assert s[b] == 0xFF and not q[32 * b:32 * b + len(blk)].any(), b
            assert bool(torch.isnan(d[32 * b:32 * b + len(blk)]).all()), b
            continue
        e = _exp_ref(float(np.abs(blk).max()))
        assert s[b] == e + 127, (b, s[b], e)
        for j, x in enumerate(blk):
            p = 32 * b + j
            assert q[p] == _rne_ref(math.ldexp(x, -e)), (p, x, e, q[p])
            want = math.ldexp(_e4m3_value(int(q[p])), e)                  # fp64 product, exact
            if abs(want) <= float(np.finfo(np.float32).max):
                assert float(d[p]) == want, (p, float(d[p]), want)       # the fp32 decode is exact
    return s[:nb], q[:K], d


def test_rule_exponent_branch_points():
    cases = {0x3FE00000: 0 - 8,              # 1.75: a * 2^-e = 448 exactly
             0x3FE00001: 0 - 7,              # 1.75 + 1 ulp: the scale rounds up
             0x3F800000: 0 - 8, 0x40000000: 1 - 8,   # powers of two
             0x43E00000: 8 - 8, 0x43E00001: 8 - 7, 0x00800000: -127, 0x01000000: -127,
             0x04000000: -127, 0x04800000: -126,   # 2^-119 and 2^-118: the clamp and the first exponent above it
             0x007FFFFF: -127, 0x00000001: -127, 0x00000000: -127,   # subnormal maxima and 0
             0x7F7FFFFF: 127 - 7,            # FLT_MAX: scale byte 247
             0x7F600000: 127 - 8}
    for bits, e in cases.items():
        a = float(_f([bits])[0])
        assert _exp_ref(a) == e, hex(bits)
        v = torch.cat([_f([bits]), torch.zeros(31)])
        assert int(fp8_scale_bytes(v)[0]) == e + 127, hex(bits)
        assert int(fp8_scale_bytes(-v)[0]) == e + 127, hex(bits)
        _check_rule(v)
    assert int(fp8_scale_bytes(_f([0x7F7FFFFF]))[0]) == 247
    # a power of two for every exponent of the fp32 range
    for E in range(-149, 128):
        v = torch.tensor([2.0 ** E], dtype=torch.float32)
        assert int(fp8_scale_bytes(v)[0]) == _exp_ref(2.0 ** E) + 127, E


def test_rule_every_element_at_ties_subnormal_codes_and_zeros():
    """Every E4M3 value, every midpoint between neighbours (the ties), and points a quarter step either side, in
    blocks whose maximum fixes e; subnormal codes and +-0 included."""
    mids = (E4M3_POS[1:] + E4M3_POS[:-1]) / 2
    quarter = (E4M3_POS[1:] - E4M3_POS[:-1]) / 4
    pts = np.concatenate([E4M3_POS, mids, mids - quarter, mids + quarter])
    pts = np.concatenate([pts, -pts])
    for e in (-127, -60, 0, 7, 119):                   # 448 * 2^119 = 1.75 * 2^127 is the largest such maximum
        x = np.ldexp(pts, e).astype(np.float32)
        assert np.array_equal(x.astype(np.float64), np.ldexp(pts, e))     # exact in fp32
        n = len(x)
        blocks = np.zeros(((n + 30) // 31, 32), dtype=np.float32)
        blocks[:, 0] = np.float32(np.ldexp(448.0, e))                      # the block maximum: e exactly
        flat = blocks.reshape(-1)
        pos = (np.arange(n) // 31) * 32 + 1 + np.arange(n) % 31
        flat[pos] = x
        s, q, _ = _check_rule(torch.from_numpy(flat.copy()))
        assert (s == e + 127).all()
    z = _f([0x80000000] * 3 + [0x00000000] * 3)
    s, q, d = _check_rule(z)
    assert q.tolist() == [0x80] * 3 + [0x00] * 3 and s[0] == 0
    assert bool((d == 0).all())


def test_rule_error_bound():
    g = torch.Generator().manual_seed(9)
    for spread in (0.5, 3.0, 12.0):
        v = torch.randn(20000, generator=g) * torch.exp(torch.randn(20000, generator=g) * spread)
        v[torch.rand(20000, generator=g) < 0.02] = 0.0
        s, d = fp8_scale_bytes(v).numpy(), fp8_decode_oracle(*fp8_encode_oracle(v), v.numel())
        e = (s - 127)[np.arange(v.numel()) // 32]
        vd, dd = v.double().numpy(), d.double().numpy()
        err = np.abs(vd - dd)
        normal = np.abs(vd) * np.ldexp(1.0, -e) >= 2.0 ** -6
        assert (err[normal] <= 2.0 ** -4 * np.abs(vd[normal])).all(), spread
        assert (err[~normal] <= np.ldexp(1.0, e[~normal] - 10)).all(), spread


def test_rule_subnormal_values():
    v = _f([0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00400000, 0x00000200, 0x00123456])
    s, q, d = _check_rule(v)
    assert s[0] == 0                                            # e = -127
    # the largest subnormal, (2^23 - 1) * 2^-149, scales to just under 2 and decodes to 2^-126; 2^-149 scales to 2^-22
    # and rounds to 0
    assert float(d[2]) == 2.0 ** -126 and float(d[3]) == -2.0 ** -126 and float(d[0]) == 0.0


@pytest.mark.parametrize("n", [1, 31, 32, 33, 511, 512, 513, 1025])
def test_rule_at_the_block_edges(n):
    v = torch.randn(n, generator=torch.Generator().manual_seed(n)) * torch.exp(
        torch.randn(n, generator=torch.Generator().manual_seed(n + 1)) * 3)
    _check_rule(v)


def test_rule_nonfinite_blocks_stay_local():
    g = torch.Generator().manual_seed(5)
    v = torch.randn(8 * 32 + 10, generator=g)
    v[40] = float("nan")
    v[100] = float("inf")
    v[170] = -float("inf")
    v[250] = float("nan")
    v[251] = float("inf")
    s, q, d = _check_rule(v)
    bad = {1, 3, 5, 7}
    for b in range(9):
        blk = d[32 * b:32 * b + 32]
        assert (s[b] == 0xFF) == (b in bad), b
        assert bool(torch.isnan(blk).all()) if b in bad else bool(torch.isfinite(blk).all()), b


def test_rule_flt_max_block_decodes_to_inf():
    """A block maximum of at least 1.9375 * 2^127 rounds to 256 * 2^120 = 2^128: the decode is inf (and the residual
    keeps 0 there); just below it stays finite."""
    v = _f([0x7F780000, 0x7F77FFFF, 0x3F800000])
    s, q, d = _check_rule(v)
    assert s[0] == 247 and float(d[0]) == math.inf and math.isfinite(float(d[1])) and float(d[2]) == 0.0


# ---------------------------------------------------------------------------
# the fused oracle
# ---------------------------------------------------------------------------
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
    plan = BucketPlan([4096], ks=[n], index=index, value="fp8", min_numel=0)
    t = plan.tensors[0]
    g = _plant(plan, vals)
    out, res, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)])
    scales, elems = fp8_encode_oracle(vals)
    a = slots[0]
    assert np.array_equal(a[t.off_coef:t.off_coef + scales.numel()], scales.numpy().view(np.uint32))
    assert np.array_equal(a[t.off_rankmap:t.off_rankmap + elems.numel()], elems.numpy().view(np.uint32))
    d = fp8_decode_oracle(scales, elems, n)
    assert torch.equal(out[:n], d)
    assert torch.equal(res[0][:n], vals - d)
    assert torch.equal(decode_slot_oracle(plan, a)[:n], d)


def test_oracle_randomk_slot_words():
    plan = BucketPlan([20000, 9000], compress_ratio=0.05, index=None, sparsifier="randomk", value="fp8", min_numel=0)
    g = torch.randn(plan.total_elems, generator=torch.Generator().manual_seed(2))
    out, res, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)])
    assert torch.equal(decode_slot_oracle(plan, slots[0]), out)
    for t in plan.tensors:
        assert t.vmode == VMODE_FP8
        seg = slice(t.elem_off, t.elem_off + t.numel)
        sel = torch.nonzero(out[seg] != 0).flatten()
        assert torch.equal(res[0][seg][sel], (g[seg] - out[seg])[sel])


def test_oracle_residual_and_dgc_momentum():
    """Per block: finite blocks keep v - d; a block with an inf or a NaN decodes to NaN and keeps residual 0.  'dgc'
    clears the momentum where d != 0, so a value that rounds to 0 next to a large one keeps its residual and momentum."""
    n = 6 * 32
    vals = torch.randn(n, generator=torch.Generator().manual_seed(1)) + 3.0
    vals[0] = 1000.0
    vals[1:5] = torch.tensor([1e-4, -1e-4, 2.0 ** -20, -2.0 ** -30])       # round to +-0 under e = 2 (2^-8 is too small)
    vals[40] = float("nan")                                  # block 1 decodes to NaN
    vals[100] = float("inf")                                 # block 3 too
    plan = BucketPlan([4096], ks=[n], index=None, value="fp8", min_numel=0)
    g = _plant(plan, vals)
    z = torch.zeros(plan.total_elems)
    out, res, slots, mom = engine_oracle(plan, [g], [z], momentum=0.5, moms=[z.clone()])
    d = fp8_decode_oracle(*fp8_encode_oracle(vals), n)
    assert bool((d[1:5] == 0).all())
    for b in range(6):
        blk = slice(32 * b, 32 * b + 32)
        if b in (1, 3):
            assert bool(torch.isnan(out[blk]).all()) and bool((res[0][blk] == 0).all()) and bool((mom[0][blk] == 0).all())
        else:
            assert torch.equal(out[blk], d[blk])
            assert torch.equal(res[0][blk], vals[blk] - d[blk])
            nz = d[blk] != 0
            assert bool((mom[0][blk][nz] == 0).all()) and torch.equal(mom[0][blk][~nz], vals[blk][~nz])
    assert torch.equal(res[0][1:5], vals[1:5]) and torch.equal(mom[0][1:5], vals[1:5])


MODES = {"plain": dict(index=None), "threshold": dict(index=None, sparsifier="threshold", threshold=1.5),
         "bloom": dict(index="bloom"), "bloom_random": dict(index="bloom", policy="random", fpr=0.02),
         "bloom_p0": dict(index="bloom", policy="p0"), "bloom_p2": dict(index="bloom", policy="conflict_sets"),
         "rle": dict(index="rle"), "rle_threshold": dict(index="rle", sparsifier="threshold", threshold=1.5),
         "elias_fano": dict(index="elias_fano"), "randomk": dict(index=None, sparsifier="randomk")}


@pytest.mark.parametrize("W", [1, 2, 3])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_decode_sums_to_the_aggregate(mode, W):
    plan = BucketPlan(SHAPES, compress_ratio=0.02, value="fp8", min_numel=1000, **MODES[mode])
    gen = torch.Generator().manual_seed(W)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    for e in (1, 2):
        grads = [torch.randn(plan.total_elems, generator=gen) for _ in range(W)]
        out, res, slots = engine_oracle(plan, grads, res, epoch=e, average=False)
        dec = torch.zeros(plan.total_elems)
        for s in slots:
            dec += decode_slot_oracle(plan, s)
        assert torch.equal(dec, out), (mode, W, e)
        assert any(t.vmode == VMODE_FP8 for t in plan.tensors)


@pytest.mark.parametrize("mode", ["plain", "bloom", "rle", "elias_fano", "randomk"])
def test_error_feedback(mode):
    """W = 1: per step, out + new residual equals r + g up to the rounding of v - d."""
    plan = BucketPlan(SHAPES, compress_ratio=0.01, value="fp8", **MODES[mode])
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
    assert compressor["fp8"] is FP8 and FP8.kind == "value" and FP8.order_preserving
    g = torch.Generator().manual_seed(0)
    for K in (0, 1, 33, 128, 129, 512, 5000):
        v = torch.randn(K, generator=g)
        idx = torch.randperm(100_000, generator=g)[:K]                     # not in index order
        wire, i2, shape = FP8.compress((v, idx, torch.Size([100_000])), {})
        order = torch.argsort(idx)
        assert torch.equal(i2, idx[order])
        scales, elems = fp8_encode_oracle(v[order])
        assert wire.dtype == torch.int32 and int(wire[0]) == K
        assert wire.numel() == 1 + (K + 127) // 128 + (K + 3) // 4
        assert torch.equal(wire[1:], torch.cat([scales, elems]))
        back, i3, _ = FP8.decompress((wire, i2, shape), {})
        assert i3 is i2 and torch.equal(back, fp8_decode_oracle(scales, elems, K))
        back, _, _ = FP8.decompress((wire, None, shape), {})                  # 'both': no index list
        assert back.numel() == K
    with pytest.raises(ValueError):
        FP8.decompress((wire[:-1], None, shape), {})


@pytest.mark.parametrize("extra", [VALUE, {**BOTH, 'index': 'rle'}, {**BOTH, 'index': 'elias_fano'}], ids=str)
def test_grace_step_matches_the_fused_oracle(extra):
    """At W = 1 the per-tensor path and the fused oracle ship the same fp8 values and keep the same residuals, on a
    gradient whose top-k both select the same way (K values well above the rest)."""
    torch.manual_seed(0)
    n = 60000
    k = spec.topk_k(n, 0.01)
    grc = deepreduce_from_params({**BASE, **extra})
    plan = BucketPlan([n], compress_ratio=0.01, value="fp8", index=extra.get('index') if extra is not VALUE else None)
    assert plan.tensors[0].val_cap > 512                                  # more than one fix task
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
def test_mlp_learns_with_fp8_values():
    """The small MLP of test_convergence.py, trained through the per-tensor path with fp8 values, passes the same
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
