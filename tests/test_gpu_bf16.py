"""bf16 gradient buckets on the GPU.  Contract: for the same plan, settings and epochs, a bf16 engine stepped on ``g``
matches an fp32 engine stepped on ``g.float()`` — residual, select state and every slot word bit for bit, and the
output equals the fp32 output rounded once to bf16 (bit for bit wherever the fp32 sums have a fixed order; within one
bf16 ulp of the oracle, and identical on all ranks, in the default RED.ADD apply at W >= 3)."""
import pytest
import torch
import torch.nn as nn

import test_engine_multirank as multirank
from deepreduce_b200.parallel import BucketEngine, BucketPlan, DeepReduceDDP, engine_oracle
from deepreduce_b200.parallel.plan import ARENA_HDR_WORDS, MODE_BLOOM
from test_gpu_engine import SIZES, _fill
from test_train_step_reference import ref_flat, unflatten

pytestmark = pytest.mark.gpu

# SIZES + a size that is not a multiple of 8 (or of 4096) + one large enough for many tiles per tensor
BF_SIZES = SIZES + [12345, 2359296]


def _bits(x):
    return x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32)


def _ordered_bf16(x):
    """bf16 values as integers that are consecutive for neighbouring bf16 values (+0 and -0 both 0)."""
    b = x.view(torch.int16).to(torch.int32)
    return torch.where(b < 0, -(b & 0x7FFF), b)


def _check_pair(e16, e32, tag, exact_out=True):
    e16.check_status()
    e32.check_status()
    assert torch.equal(_bits(e16.resid), _bits(e32.resid)), tag
    assert torch.equal(e16.sel, e32.sel), tag
    assert torch.equal(e16.slot(), e32.slot()), (tag, int((e16.slot() != e32.slot()).sum()))
    assert torch.equal(e16.status, e32.status), tag
    if exact_out:
        want = e32.grad.to(torch.bfloat16)
        assert torch.equal(_bits(e16.grad), _bits(want)), (tag, int((_bits(e16.grad) != _bits(want)).sum()))


def _pair(plan, **kw):
    e16 = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000, grad_dtype=torch.bfloat16, **kw)
    e32 = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000, **kw)
    return e16, e32


W1 = pytest.param
W1_CASES = [
    W1(dict(index="bloom"), True, 2, 1.0, id="bloom-leftmost-hint-tma-bps2"),
    W1(dict(index="bloom", hint=False), False, 1, 1.0, id="bloom-leftmost-nohint-cpasync-bps1"),
    W1(dict(index="bloom", policy="random", fpr=0.02), True, 1, 1.0, id="bloom-random-tma-bps1"),
    W1(dict(index="bloom", policy="p0"), False, 2, 0.0, id="bloom-p0-cpasync-noresid"),
    W1(dict(index="rle"), True, 2, 1.0, id="rle-tma"),
    W1(dict(index="rle"), False, 1, 0.0, id="rle-cpasync-bps1-noresid"),
    W1(dict(index=None), True, 2, 1.0, id="raw-tma"),
    W1(dict(index=None, value="polyfit", poly_min_k=300), True, 2, 1.0, id="value-polyfit"),
    W1(dict(index=None, value="qsgd"), False, 2, 1.0, id="value-qsgd8-cpasync"),
    W1(dict(index="bloom", value="qsgd", quantum_num=1000), True, 1, 1.0, id="bloom-qsgd16-bps1"),
    W1(dict(index="bloom", value="polyfit", poly_min_k=300), True, 2, 1.0, id="both-polyfit"),
    W1(dict(index="bloom", sparsifier="threshold", threshold=1.0, capacity_ratio=0.5), True, 2, 1.0, id="threshold-bloom"),
    W1(dict(index=None, sparsifier="threshold", threshold=1.5), False, 2, 0.0, id="threshold-raw-noresid"),
    W1(dict(index=None, sparsifier="randomk"), True, 2, 1.0, id="randomk"),
    W1(dict(index=None, sparsifier="randomk"), False, 1, 0.0, id="randomk-cpasync-noresid"),
    W1(dict(index=None, sparsifier="randomk", value="qsgd"), True, 2, 1.0, id="randomk-qsgd"),
]


@pytest.mark.parametrize("kw,tma,bps,beta", W1_CASES)
def test_bf16_engine_matches_fp32_on_widened_input_w1(kw, tma, bps, beta):
    plan = BucketPlan(BF_SIZES, compress_ratio=0.01, **kw)
    e16, e32 = _pair(plan, use_tma=tma, blocks_per_sm=bps, beta=beta)
    gen = torch.Generator().manual_seed(7)
    for step in range(5):               # history, the speculative digit 2, and (step 4, shrunk input) the fallback
        g = (_fill(plan, gen) * (0.2 if step == 4 else 1.0)).to(torch.bfloat16)
        e16.grad.copy_(g.cuda())
        e32.grad.copy_(g.float().cuda())
        if step == 2:
            e16.run_unfused()
            e32.run_unfused()
        else:
            e16.step()
            e32.step()
        torch.cuda.synchronize()
        _check_pair(e16, e32, f"w1 {kw} step {step}")
        assert e16.stats() == e32.stats()
    e16.close()
    e32.close()


def _edge_residual(plan):
    """fp32 values whose bf16 rounding is a tie (both parities), rounds to +-0, or to the largest finite bf16."""
    # half a bf16 ulp above a bf16 value with an even and with an odd last mantissa bit (ulp 2^-7 on [1, 2), 2^-6 on [2, 4))
    ties = torch.tensor([1 + 2.0 ** -8, 1 + 2.0 ** -7 + 2.0 ** -8, -(1 + 2.0 ** -8), -(2 + 2.0 ** -7),
                         2 + 2.0 ** -6 + 2.0 ** -7])
    tiny = torch.tensor([2.0 ** -135, -(2.0 ** -135), 2.0 ** -136, -(2.0 ** -137)])   # below half the smallest bf16 subnormal
    big = torch.tensor([0x7F7F7FFF, 0xFF7F7000 - (1 << 32)], dtype=torch.int32).view(torch.float32)  # -> +-largest finite
    edge = torch.cat([ties, tiny, big])
    r = torch.zeros(plan.total_elems)
    gen = torch.Generator().manual_seed(3)
    for v in plan.views(r):
        x = torch.randn(v.numel(), generator=gen)
        pick = torch.randint(0, edge.numel(), (v.numel(),), generator=gen)
        on = torch.rand(v.numel(), generator=gen) < 0.5
        x[on] = edge[pick[on]]
        v.copy_(x.view(v.shape))
    return r


@pytest.mark.parametrize("kw", [dict(index=None), dict(index="bloom"), dict(index="rle")], ids=["raw", "bloom", "rle"])
def test_bf16_rounding_edges_w1(kw):
    """All of a pre-loaded residual is shipped (threshold 0, capacity = the tensor): the output is the fp32 residual
    rounded once, ties to even, tiny values to signed zeros, huge values to the largest finite bf16."""
    plan = BucketPlan([4096, 5000, 1001], compress_ratio=0.01, sparsifier="threshold", threshold=0.0,
                      capacity_ratio=1.0, min_numel=0, **kw)
    e16, e32 = _pair(plan)
    r = _edge_residual(plan)
    for e in (e16, e32):
        e.resid.copy_(r.cuda())
        e.grad.zero_()
        e.step()
    torch.cuda.synchronize()
    _check_pair(e16, e32, f"edges {kw}")
    want = r.to(torch.bfloat16)
    live = torch.zeros(plan.total_elems, dtype=torch.bool)
    for t in plan.tensors:
        live[t.elem_off:t.elem_off + t.numel] = True
    assert torch.equal(_bits(e16.grad.cpu())[live], _bits(want)[live])
    w = _bits(want)[live]
    assert bool((w == 0x7F7F).any()) and bool((w == -0x8000).any()) and bool((w == 0).any())
    e16.close()
    e32.close()


@pytest.mark.parametrize("kw", [dict(index=None), dict(index="bloom")], ids=["raw", "bloom"])
def test_bf16_rounding_edges_stage2_drops_rounded_plus_zeros(kw):
    """W = 2 sharded: the stage-2 lists carry the rounded values and leave out exactly the entries that round to +0; an
    entry that rounds to -0 is shipped, so the receivers hold the owner's bits."""
    plan = BucketPlan([4096, 5000, 1001, 8192], compress_ratio=0.01, sparsifier="threshold", threshold=0.0,
                      capacity_ratio=1.0, min_numel=0, **kw)
    W = 2
    groups = {}
    for dt in (torch.bfloat16, torch.float32):
        arenas = [torch.zeros(plan.arena_words(W, True), dtype=torch.int32, device="cuda:0") for _ in range(W)]
        groups[dt] = [multirank._RankEngine(plan, arenas, r, shard=True, average=False, spin_limit=4_000_000,
                                            peer_timeout_ms=5000, grad_dtype=dt) for r in range(W)]
    r = _edge_residual(plan)
    for dt, engs in groups.items():
        for e in engs:
            e.resid.copy_((r * 0.5).cuda())      # every rank ships the same half: the sum is r, exactly
            e.grad.zero_()
        multirank._run_step(engs, "shard", 1)
    e16s, e32s = groups[torch.bfloat16], groups[torch.float32]
    for a, b in zip(e16s, e32s):
        _check_pair(a, b, f"edges-s2 {kw}")
    # the fp32 group's aggregate, rounded (the bloom apply's RED.ADD.F32 flushes subnormal addends, on both groups)
    want = e32s[0].grad.cpu().to(torch.bfloat16)
    _, tbase, tn = multirank._tiles(plan)
    s2w = plan.stage2_layout(W)[1]
    s2_base = ARENA_HDR_WORDS + 2 * W * plan.slot_words + W * s2w
    out = e16s[0].grad.cpu()
    for o, (sb, se) in enumerate(multirank._spans(plan.n_tiles, W)):
        mine = torch.zeros(plan.total_elems, dtype=torch.bool)
        for tile in range(sb, se):
            mine[tbase[tile]:tbase[tile] + tn[tile]] = True
        nz = torch.nonzero(mine & (_bits(out) != 0)).flatten()
        zero_rounded = mine & (r != 0) & (_bits(want) == 0)
        minus_zero = mine & (_bits(want) == -0x8000)
        assert bool(zero_rounded.any()) and (bool(minus_zero.any()) or kw["index"] is not None)
        s2 = e16s[1 - o].arena[s2_base + o * s2w:s2_base + (o + 1) * s2w].cpu()
        n = int(s2[0])
        pairs = s2[4:4 + 2 * n].view(n, 2)
        idx = pairs[:, 0].to(torch.int64)
        assert torch.equal(torch.sort(idx).values, nz)
        assert not bool(zero_rounded[idx].any())
        assert int(minus_zero[idx].sum()) == int(minus_zero.sum())          # every -0 entry is shipped
        assert torch.equal(pairs[:, 1], out.float().view(torch.int32)[idx])
    for r_ in range(1, W):
        assert torch.equal(_bits(e16s[r_].grad), _bits(e16s[0].grad))
    for e in e16s + e32s:
        e.close()


MR = pytest.param
MR_CASES = [
    MR("shard", 2, dict(index="bloom"), False, id="shard-bloom-W2-fast"),
    MR("shard", 4, dict(index="bloom"), True, id="shard-bloom-W4-det"),
    MR("shard", 4, dict(index="bloom", hint=False), False, id="shard-bloom-W4-fast"),
    MR("shard", 8, dict(index="bloom", policy="random", fpr=0.02), False, id="shard-random-W8-fast"),
    MR("shard", 3, dict(index="rle"), False, id="shard-rle-W3-fast"),
    MR("shard", 8, dict(index=None), False, id="shard-raw-W8-fast"),
    MR("shard", 4, dict(index=None, sparsifier="randomk"), False, id="shard-randomk-W4-fast"),
    MR("shard", 3, dict(index="bloom", value="qsgd"), True, id="shard-qsgd-W3-det"),
    MR("noshard", 3, dict(index="bloom"), False, id="noshard-bloom-W3"),
    MR("noshard", 4, dict(index="rle"), False, id="noshard-rle-W4"),
    MR("nccl", 4, dict(index="bloom"), False, id="nccl-bloom-W4"),
    MR("nccl", 3, dict(index=None, sparsifier="randomk"), True, id="nccl-randomk-W3-det"),
]


def _group(plan, W, config, dtype):
    kw = dict(average=True, spin_limit=4_000_000, peer_timeout_ms=5000, grad_dtype=dtype)
    if config == "nccl":
        return [BucketEngine(plan, device="cuda:0", world=W, rank=r, transport="nccl", **kw) for r in range(W)]
    shard = config == "shard"
    arenas = [torch.zeros(plan.arena_words(W, shard), dtype=torch.int32, device="cuda:0") for _ in range(W)]
    return [multirank._RankEngine(plan, arenas, r, shard=shard, **kw) for r in range(W)]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("config,W,kw,deterministic", MR_CASES)
def test_bf16_multirank_matches_fp32(monkeypatch, config, W, kw, deterministic):
    monkeypatch.setenv("DR_DETERMINISTIC", "1" if deterministic else "0")
    plan = BucketPlan(multirank.SIZES, compress_ratio=0.01, **kw)
    g16, g32 = _group(plan, W, config, torch.bfloat16), _group(plan, W, config, torch.float32)
    ordered = deterministic or (config != "shard" and W > 2)
    # order-dependent fp32 sums: bloom tensors in the RED.ADD apply at W >= 3 (every other decode is rank-ordered)
    loose = torch.zeros(plan.total_elems, dtype=torch.bool)
    if not ordered and W >= 3:
        for t in plan.tensors:
            if t.mode == MODE_BLOOM:
                loose[t.elem_off:t.elem_off + t.numel] = True
    resid_refs = [torch.zeros(plan.total_elems) for _ in range(W)]
    for step in range(3):
        epoch = step + 1
        grads = [(_fill(plan, torch.Generator().manual_seed(1000 * step + r)) * (0.2 if step == 2 else 1.0))
                 .to(torch.bfloat16) for r in range(W)]
        for e16, e32, g in zip(g16, g32, grads):
            e16.grad.copy_(g.cuda())
            e32.grad.copy_(g.float().cuda())
        multirank._run_step(g16, config, epoch)
        multirank._run_step(g32, config, epoch)
        tag = f"{config} W{W} {kw} step {step}"
        outs = [e.grad.cpu() for e in g16]
        for e16, e32 in zip(g16, g32):
            _check_pair(e16, e32, tag, exact_out=False)
            for s in range(W):                                  # every arena holds the same sender slots
                assert torch.equal(e16.slot(s), e32.slot(s)), (tag, e16.rank, s)
            want = e32.grad.cpu().to(torch.bfloat16)
            out = e16.grad.cpu()
            assert torch.equal(_bits(out)[~loose], _bits(want)[~loose]), (tag, e16.rank)
        for r in range(1, W):
            assert torch.equal(_bits(outs[r]), _bits(outs[0])), (tag, r)
        if bool(loose.any()):
            ref, resid_refs, _ = engine_oracle(plan, [g.float() for g in grads], resid_refs, average=True, epoch=epoch)
            d = (_ordered_bf16(outs[0]) - _ordered_bf16(ref.to(torch.bfloat16)))[loose].abs()
            assert int(d.max()) <= 1, (tag, int(d.max()))
    for e in g16 + g32:
        e.close()


# ---------------------------------------------------------------------------
# DeepReduceDDP: bf16 models, W = 1
# ---------------------------------------------------------------------------
class _Mixed(nn.Module):
    """bf16 MLP with one fp32 layer in the middle (explicit casts): two buckets, one per dtype."""

    def __init__(self):
        super().__init__()
        self.a = nn.Linear(64, 512).to(torch.bfloat16)
        self.b = nn.Linear(512, 256)
        self.c = nn.Linear(256, 10).to(torch.bfloat16)

    def forward(self, x):
        h = torch.relu(self.a(x)).float()
        h = torch.relu(self.b(h)).to(torch.bfloat16)
        return self.c(h)


def _mlp():
    return nn.Sequential(nn.Linear(64, 512), nn.ReLU(), nn.Linear(512, 512), nn.ReLU(), nn.Linear(512, 10)).to(torch.bfloat16)


def _loss(model, x, y):
    return nn.functional.cross_entropy(model(x).float(), y)


@pytest.mark.parametrize("model_fn,n_buckets", [(_mlp, 1), (_Mixed, 2)], ids=["bf16-mlp", "mixed"])
@pytest.mark.parametrize("cfg", [
    {'compressor': 'topk', 'compress_ratio': 0.01, 'deepreduce': 'index', 'index': 'bloom'},
    {'compressor': 'randomk', 'compress_ratio': 0.01},
], ids=["topk-bloom", "randomk"])
def test_ddp_bf16_training_step_bit_exact(model_fn, n_buckets, cfg):
    cfg = dict(cfg, memory='residual', communicator='allgather', calibrate_partition=False)
    torch.manual_seed(0)
    model = model_fn().cuda()
    ref = model_fn().cuda()
    ref.load_state_dict(model.state_dict())
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    assert len(ddp.engines) == n_buckets
    dts = sorted(str(e.grad.dtype) for e in ddp.engines)
    assert dts == sorted(str(items[0][1].dtype) for items in ddp.buckets)
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    ref_opt = torch.optim.SGD(ref.parameters(), lr=0.1)
    resid = [torch.zeros(e.plan.total_elems) for e in ddp.engines]
    gen = torch.Generator(device="cuda").manual_seed(1)
    for step in range(3):
        x = torch.randn(32, 64, device="cuda", generator=gen).to(torch.bfloat16)
        y = torch.randint(0, 10, (32,), device="cuda", generator=gen)
        ddp.zero_grad()
        loss = _loss(model, x, y)
        loss.backward()
        ddp.finish()
        ref_opt.zero_grad()
        ref_loss = _loss(ref, x, y)
        ref_loss.backward()
        assert torch.equal(loss, ref_loss), step
        grads = {}
        for b, (eng, items) in enumerate(zip(ddp.engines, ddp.buckets)):
            names = dict(ref.named_parameters())
            params = {n: names[n] for n, _ in items}
            flat = ref_flat(eng.plan, params, {n: q.grad for n, q in params.items()})
            out, new_res, _ = engine_oracle(eng.plan, [flat], [resid[b]], average=True, epoch=eng.epoch)
            resid[b] = new_res[0]
            out = out.to(eng.grad.dtype)
            assert torch.equal(eng.grad.cpu(), out), (step, b)
            assert torch.equal(_bits(eng.resid.cpu()), _bits(resid[b])), (step, b)
            grads.update(unflatten(eng.plan, params, out.float()))
        for n, q in ref.named_parameters():
            q.grad = grads[n]
        opt.step()
        ref_opt.step()
        for (n, p), q in zip(model.named_parameters(), ref.parameters()):
            assert torch.equal(p, q), (step, n)
    ddp.close()


@pytest.mark.parametrize("model_fn", [_mlp, _Mixed], ids=["bf16-mlp", "mixed"])
def test_ddp_dense_baseline_bf16_buckets(model_fn):
    torch.manual_seed(0)
    model = model_fn().cuda()
    ref = model_fn().cuda()
    ref.load_state_dict(model.state_dict())
    ddp = DeepReduceDDP(model, {'compressor': 'none', 'communicator': 'allreduce'}, overlap=False)
    assert {f.dtype for f in ddp.flat} == {p.dtype for p in model.parameters()}
    x = torch.randn(32, 64, device="cuda").to(torch.bfloat16)
    y = torch.randint(0, 10, (32,), device="cuda")
    ddp.zero_grad()
    _loss(model, x, y).backward()
    ddp.finish()
    _loss(ref, x, y).backward()
    for (n, p), q in zip(model.named_parameters(), ref.parameters()):
        assert p.grad.dtype == q.dtype and torch.equal(p.grad, q.grad), n
    assert ddp.dense_bytes() == sum(p.numel() * p.element_size() for p in model.parameters())
    ddp.close()
