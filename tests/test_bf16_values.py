"""bf16 values on the wire ('value': 'bf16'), on the CPU: routing, the slot layout and wire bytes, the rounding rule
of the oracle at its branch points, decode against the aggregate, the per-tensor codec against the fused oracle, and
error feedback's conservation of mass."""
import hashlib
import warnings

import numpy as np
import pytest
import torch

from deepreduce_b200 import deepreduce_from_params, spec
from deepreduce_b200.codecs import BF16, compressor
from deepreduce_b200.codecs.bf16 import bf16_bits_oracle, bf16_widen_oracle
from deepreduce_b200.config import ConfigError, validate_params
from deepreduce_b200.parallel.engine import decode_slot_oracle, engine_oracle, stats_from_slot
from deepreduce_b200.parallel.plan import MODE_BLOOM, MODE_RAW, MODE_RLE, MODE_SHARED, BucketPlan

BASE = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
THR = {'compressor': 'threshold', 'threshold': 0.01}
RANDK = {'compressor': 'randomk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
VALUE = {'deepreduce': 'value', 'value': 'bf16'}
BOTH = {'deepreduce': 'both', 'value': 'bf16'}
SHAPES = [30000, 5000, 300, 4097, 70000]


def _al(x):
    return (x + 3) // 4 * 4


def _resnet50_numels():
    from deepreduce_b200.models import resnet50
    return [p.numel() for p in reversed(list(resnet50().parameters()))]


# ---------------------------------------------------------------------------
# config and routing
# ---------------------------------------------------------------------------
FUSED = ([{**BASE, **VALUE}, {**BASE, **THR, **VALUE}, {**RANDK, **VALUE}, {**BASE, **VALUE, 'index': 'rle'}]
         + [{**s, **BOTH, 'index': 'bloom', 'policy': p} for s in (BASE, {**BASE, **THR})
            for p in ('leftmost', 'random', 'p0')]
         + [{**BASE, **BOTH, 'index': 'bloom', 'policy': 'conflict_sets', 'p2_pick_mask': True},
            {**BASE, **BOTH, 'index': 'rle'}, {**BASE, **THR, **BOTH, 'index': 'rle'}])


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
        assert kw['value'] == 'bf16', p
        BucketPlan(SHAPES, **{k: v for k, v in kw.items() if k != 'capacity_ratio'})


def test_routing_refused():
    from deepreduce_b200.parallel.ddp import fused_path
    # 'fused_rle_values' keeps its meaning and still refuses bf16
    p = {**BASE, **BOTH, 'index': 'rle', 'fused_rle_values': True}
    with pytest.raises(ConfigError):
        validate_params(p)
    assert not fused_path(p)
    with pytest.raises(ConfigError):
        validate_params({**BASE, **BOTH, 'index': 'rle', 'fused_dexp': True})
    # the per-tensor route: conflict_sets without the pick mask, 'both' under randomk, a host index codec
    for p in ({**BASE, **BOTH, 'index': 'bloom', 'policy': 'conflict_sets'},
              {**RANDK, **BOTH, 'index': 'bloom'},
              {**BASE, **BOTH, 'index': 'huffman'}, {**BASE, **BOTH, 'index': 'integer'}):
        validate_params(p)
        assert not fused_path(p), p


def test_routing_of_existing_dicts_unchanged():
    from deepreduce_b200.parallel.ddp import fused_path
    fused = [BASE, {**BASE, 'deepreduce': 'index', 'index': 'bloom'}, {**BASE, 'deepreduce': 'index', 'index': 'rle'},
             {**BASE, 'deepreduce': 'value', 'value': 'qsgd'}, {**BASE, 'deepreduce': 'both', 'value': 'polyfit'},
             {**BASE, 'deepreduce': 'both', 'value': 'qsgd', 'index': 'rle', 'fused_rle_values': True},
             {**BASE, 'deepreduce': 'both', 'value': 'dexp', 'index': 'rle', 'fused_dexp': True},
             {**RANDK, 'communicator': 'allreduce'}, {**RANDK, 'deepreduce': 'value', 'value': 'qsgd'}]
    per_tensor = [{**BASE, 'deepreduce': 'both', 'value': 'qsgd', 'index': 'rle'},
                  {**BASE, 'deepreduce': 'both', 'value': 'polyfit', 'index': 'rle'},
                  {**BASE, 'deepreduce': 'value', 'value': 'dexp'},
                  {**BASE, 'deepreduce': 'both', 'value': 'qsgd', 'bucket_size': 256},
                  {**RANDK, 'deepreduce': 'value', 'value': 'polyfit'},
                  {**BASE, 'deepreduce': 'both', 'index': 'bloom', 'policy': 'conflict_sets'},
                  {**BASE, 'communicator': 'allgather', 'deepreduce': 'value', 'value': 'gzip'}]
    assert all(fused_path(p) for p in fused)
    assert not any(fused_path(p) for p in per_tensor)


# ---------------------------------------------------------------------------
# layout
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(index=None), dict(index="bloom"), dict(index="bloom", policy="p0"),
                                dict(index="rle"), dict(index=None, sparsifier="randomk")], ids=str)
def test_layout(kw):
    plan = BucketPlan(SHAPES, compress_ratio=0.05, value="bf16", **kw)
    ref = BucketPlan(SHAPES, compress_ratio=0.05, **kw)
    P = plan.payload_words
    assert plan.poly_tables()[1] == 0 and plan.poly_tables()[3] == 0          # no rank, fit or fix phase
    saved = 0
    for t, r in zip(plan.tensors, ref.tensors):
        assert (t.mode, t.k, t.val_cap) == (r.mode, r.k, r.val_cap)
        assert t.off_coef == t.off_rankmap == t.off_selidx == t.off_sorted == 0   # no sender scratch
        if t.numel <= plan.min_numel:
            assert t.vmode == 0
            continue
        assert t.vmode == 4 and t.off_vals < P and t.off_vals % 4 == 0
        nxt = {MODE_RAW: t.off_idx, MODE_BLOOM: t.off_filter, MODE_RLE: t.off_prefix}.get(t.mode)
        if nxt is not None:
            assert nxt == t.off_vals + _al((t.val_cap + 1) // 2)
        saved += _al(t.val_cap) - _al((t.val_cap + 1) // 2)
    assert ref.payload_words - P == saved
    # the shared mode's per-tile prefix stays sender-local scratch; nothing else follows the payload
    scratch = sum(_al(t.n_tiles) for t in plan.tensors if t.mode == MODE_SHARED)
    assert plan.slot_words == (P + scratch + 63) // 64 * 64


# expected wire bytes per rank per step on ResNet-50 (fp32 values -> bf16 values), in units of 100 bytes
WIRE = {0.001: {"plain": (2105, 1595), "rle": (1601, 1091), "bloom": (2951, 2442), "randomk": (1170, 636)},
        0.01: {"plain": (20495, 15389), "rle": (14246, 9141), "bloom": (16126, 11021), "randomk": (10364, 5235)},
        0.03: {"plain": (61375, 46054), "rle": (42359, 27039), "bloom": (43564, 28244), "randomk": (30804, 15459)}}


@pytest.mark.parametrize("ratio", sorted(WIRE))
def test_wire_bytes_resnet50(ratio):
    numels = _resnet50_numels()
    kws = {"plain": dict(index=None), "rle": dict(index="rle"), "bloom": dict(index="bloom"),
           "randomk": dict(index=None, sparsifier="randomk")}
    for name, kw in kws.items():
        fp32 = BucketPlan(numels, compress_ratio=ratio, **kw).wire_bytes()
        bf16 = BucketPlan(numels, compress_ratio=ratio, value="bf16", **kw).wire_bytes()
        assert (round(fp32 / 100), round(bf16 / 100)) == WIRE[ratio][name], name
    if ratio == 0.01:                 # rle + bf16 ships less than rle + polyfit
        assert (BucketPlan(numels, compress_ratio=ratio, index="rle", value="bf16").wire_bytes()
                < BucketPlan(numels, compress_ratio=ratio, index="rle", value="polyfit").wire_bytes())


# digests of the device tensor table of plans without bf16 values, as the parent commit builds them
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
def test_plans_without_bf16_unchanged(name):
    plan = BucketPlan(_resnet50_numels(), compress_ratio=0.01, **TABLE_PLANS[name])
    assert _table_digest(plan) == TABLES[name]


# ---------------------------------------------------------------------------
# the rounding rule
# ---------------------------------------------------------------------------
SPECIAL = np.array([0x00000000, 0x80000000, 0x00004000, 0x00007FFF, 0x00008000, 0x00008001, 0x00018000, 0x00010000,
                    0x80008001, 0x807FFFFF, 0x3F808000, 0x3F818000, 0x3F80FFFF, 0xBF808000, 0x7F7F7FFF, 0x7F7F8000,
                    0x7F7FFFFF, 0xFF7F8000, 0x7F800000, 0xFF800000, 0x00800000, 0x3F800000], dtype=np.uint32)
NAN = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF, 0xFF800001], dtype=np.uint32)


def _f(bits):
    return torch.from_numpy(bits.view(np.float32).copy())


def test_bits_match_torch_cast():
    x = torch.cat([_f(SPECIAL), torch.randn(100_000) * torch.exp(torch.randn(100_000) * 20)])
    want = x.to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0xFFFF
    assert torch.equal(bf16_bits_oracle(x), want)
    # ties to even, the subnormals, the overflow point
    b = bf16_bits_oracle(_f(SPECIAL)).tolist()
    assert b[2:8] == [0x0000, 0x0000, 0x0000, 0x0001, 0x0002, 0x0001]
    assert b[10:12] == [0x3F80, 0x3F82] and b[14:17] == [0x7F7F, 0x7F80, 0x7F80] and b[17] == 0xFF80
    assert bf16_bits_oracle(_f(NAN)).tolist() == [0x7FC0] * NAN.size
    w = bf16_widen_oracle(bf16_bits_oracle(x))
    assert torch.equal(w, x.to(torch.bfloat16).float())


def _plant(plan, values, seed=0):
    """One tensor of the plan filled with small noise and the planted values at its front (all of them shipped)."""
    g = torch.randn(plan.total_elems, generator=torch.Generator().manual_seed(seed)) * 1e-30
    t = plan.tensors[0]
    g[t.elem_off:t.elem_off + values.numel()] = values
    return g


@pytest.mark.parametrize("index", [None, "bloom", "rle"])
def test_oracle_branch_points(index):
    # no zeros, and no key below 2^9 (the select never ships those): every planted value is selected
    vals = torch.cat([_f(SPECIAL[2:]), torch.randn(200) * 1e3])
    K = int(vals.numel())
    plan = BucketPlan([4096], ks=[K], index=index, value="bf16", min_numel=100)
    g = _plant(plan, vals)
    g[K:4096] = 0.0
    out, res, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)])
    t = plan.tensors[0]
    q = slots[0][t.off_vals:t.off_vals + (K + 1) // 2].view(np.uint16)[:K].astype(np.int64)
    assert np.array_equal(q, bf16_bits_oracle(vals).numpy())
    w = bf16_widen_oracle(torch.from_numpy(q))
    assert torch.equal(out[:K], w)
    fin = torch.isfinite(w)
    # v == widen(q) + r, exactly (in fp64), wherever widen(q) is finite; r = 0 elsewhere
    assert torch.equal(vals.double()[fin], w.double()[fin] + res[0][:K].double()[fin])
    assert bool((res[0][:K][~fin] == 0).all()) and int((~fin).sum()) == 5
    assert torch.equal(decode_slot_oracle(plan, slots[0])[:K], w)
    row = stats_from_slot(plan, slots[0])["tensors"][0]
    assert row["value_bytes"] == 2 * t.val_cap and row["n_sel"] == K


def test_oracle_nan_rides_as_quiet_nan():
    vals = torch.cat([_f(NAN), torch.randn(100)])
    K = int(vals.numel())
    plan = BucketPlan([4096], ks=[K], index=None, value="bf16", min_numel=100)
    g = _plant(plan, vals)
    g[K:4096] = 0.0
    out, res, slots = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)])
    t = plan.tensors[0]
    q = slots[0][t.off_vals:t.off_vals + (K + 1) // 2].view(np.uint16)[:K]
    assert q[:NAN.size].tolist() == [0x7FC0] * NAN.size
    assert bool(torch.isnan(out[:NAN.size]).all()) and bool((res[0][:NAN.size] == 0).all())


def test_oracle_dgc_keeps_momentum_of_underflowed_values():
    # fp32 subnormals below half the smallest bf16 subnormal round to +-0: the coordinate is shipped, decodes to 0,
    # and keeps its momentum and its whole residual; one that rounds to the smallest subnormal loses its momentum
    tiny = _f(np.array([0x00004000, 0x80007FFF, 0x00007FFF, 0x00008001], dtype=np.uint32))
    vals = torch.cat([tiny, torch.randn(60)])
    K = int(vals.numel())
    plan = BucketPlan([4096], ks=[K], index=None, value="bf16", min_numel=100)
    g = torch.zeros(plan.total_elems)
    g[:K] = vals
    u0 = torch.zeros(plan.total_elems)
    out, res, slots, mom = engine_oracle(plan, [g], [torch.zeros(plan.total_elems)], momentum=0.5, moms=[u0])
    assert out[:3].abs().sum() == 0 and float(out[3]) == float(_f(np.array([0x00010000], dtype=np.uint32))[0])
    assert torch.equal(mom[0][:3], vals[:3]) and torch.equal(res[0][:3], vals[:3])
    assert float(mom[0][3]) == 0.0 and bool((mom[0][4:K] == 0).all())
    assert torch.equal(res[0][:K].double() + out[:K].double(), vals.double())


# ---------------------------------------------------------------------------
# decode and aggregate
# ---------------------------------------------------------------------------
MODES = {"plain": dict(index=None), "threshold": dict(index=None, sparsifier="threshold", threshold=1.5),
         "bloom": dict(index="bloom"), "bloom_random": dict(index="bloom", policy="random", fpr=0.02),
         "bloom_p0": dict(index="bloom", policy="p0"), "bloom_p2": dict(index="bloom", policy="conflict_sets"),
         "rle": dict(index="rle"), "rle_threshold": dict(index="rle", sparsifier="threshold", threshold=1.5),
         "randomk": dict(index=None, sparsifier="randomk")}


@pytest.mark.parametrize("W", [1, 2, 3])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_decode_sums_to_the_aggregate(mode, W):
    plan = BucketPlan(SHAPES, compress_ratio=0.02, value="bf16", min_numel=1000, **MODES[mode])
    gen = torch.Generator().manual_seed(W)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    for e in (1, 2):
        grads = [torch.randn(plan.total_elems, generator=gen) for _ in range(W)]
        out, res, slots = engine_oracle(plan, grads, res, epoch=e, average=False)
        dec = torch.zeros(plan.total_elems)
        for s in slots:
            dec += decode_slot_oracle(plan, s)
        assert torch.equal(dec, out), (mode, W, e)
        assert any(t.vmode == 4 for t in plan.tensors)


# ---------------------------------------------------------------------------
# the per-tensor codec
# ---------------------------------------------------------------------------
def test_codec_round_trip():
    assert compressor["bf16"] is BF16 and BF16.kind == "value" and BF16.order_preserving
    v = torch.randn(5000) * torch.exp(torch.randn(5000) * 10)
    idx = torch.arange(5000)
    wire, i2, shape = BF16.compress((v, idx, torch.Size([5000])), {})
    assert wire.dtype == torch.bfloat16 and i2 is idx and wire.numel() == 5000
    back, _, _ = BF16.decompress((wire, i2, shape), {})
    assert back.dtype == torch.float32 and torch.equal(back, v.to(torch.bfloat16).float())
    assert float(((back - v).abs() / v.abs()).max()) <= 2.0 ** -8      # 8 significant bits, round to nearest


@pytest.mark.parametrize("extra", [VALUE, {**BOTH, 'index': 'rle'}], ids=str)
def test_grace_step_matches_the_fused_oracle(extra):
    """At W = 1 the per-tensor path and the fused oracle ship the same bf16 values and keep the same residuals, on a
    gradient whose top-k both select the same way (K values well above the rest)."""
    torch.manual_seed(0)
    n = 20000
    k = spec.topk_k(n, 0.01)
    grc = deepreduce_from_params({**BASE, **extra})
    plan = BucketPlan([n], compress_ratio=0.01, value="bf16", index=extra.get('index') if extra is not VALUE else None)
    res = [torch.zeros(plan.total_elems)]
    for step in range(3):
        g = torch.randn(n) * 1e-3
        hot = torch.randperm(n)[:k]
        g[hot] = (torch.rand(k) + 1.0) * torch.sign(torch.randn(k)) * 10.0
        out = grc.step(g.clone(), "w")
        out_o, res, _ = engine_oracle(plan, [g], res, epoch=step + 1)
        assert torch.equal(out.flatten(), out_o[:n]), step
        assert torch.equal(grc.memory.residuals["w"].flatten(), res[0][:n]), step


@pytest.mark.parametrize("mode", ["plain", "bloom", "rle", "randomk"])
def test_error_feedback_conserves_mass(mode):
    """W = 1: per step, out + new residual == r + g exactly; over T steps the outputs plus the final residual equal
    the summed gradients up to the roundings of r + g."""
    plan = BucketPlan(SHAPES, compress_ratio=0.01, value="bf16", **MODES[mode])
    gen = torch.Generator().manual_seed(7)
    res = [torch.zeros(plan.total_elems)]
    sum_g = torch.zeros(plan.total_elems, dtype=torch.float64)
    sum_out = torch.zeros(plan.total_elems, dtype=torch.float64)
    bound = torch.zeros(plan.total_elems, dtype=torch.float64)
    for e in range(1, 9):
        g = torch.randn(plan.total_elems, generator=gen)
        acc = res[0] + g
        out, res, _ = engine_oracle(plan, [g], res, epoch=e)
        assert torch.equal(out.double() + res[0].double(), acc.double()), e
        sum_g += g.double()
        sum_out += out.double()
        bound += acc.double().abs() * 2.0 ** -24
    assert bool(((sum_out + res[0].double() - sum_g).abs() <= bound).all())
