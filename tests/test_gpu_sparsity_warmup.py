"""Sparsity warm-up on the GPU: the fused engine at the warm-up's dense ratios (25 %, 6.25 %) against
``engine_oracle`` in every fused mode, a bloom filter too large for the shared-memory stage probed from L2; the stage
switch's state carry (a fresh select history selects what a stale one does); ``DeepReduceDDP`` across two stage
boundaries against the oracle and the per-tensor GRACE route, with ``p.grad`` still viewing the bucket and the optimizer
step reading the switching exchange's aggregate; checkpoints mid-stage and at a boundary; the DDP hook across
boundaries with ``no_sync()`` steps; W = 2-4 ranks in one process across a switch; ``Trainer(accum_steps=2)``."""
import copy

import pytest
import torch
import torch.nn as nn

import deepreduce_b200 as dr
from deepreduce_b200 import spec
from deepreduce_b200.config import warmup_from_params
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.ddp import switch_engine
from deepreduce_b200.parallel.engine import decode_slot_oracle
from deepreduce_b200.parallel.plan import MODE_BLOOM
from test_engine_multirank import _RankEngine, _run_step
from test_fused_params import _prefix_tie
from test_gpu_dexp_fused import compare_dexp_slot
from test_gpu_dgc_weight_decay import MODES, _ConvNet, nccl_world1  # noqa: F401
from test_gpu_engine import _compare_slot, _fill

pytestmark = pytest.mark.gpu

# 700 000 elements at 25 %: a 168 KB bloom filter, larger than the shared-memory stage of either launch variant
SIZES = [64, 1000, 1001, 4097, 36864, 147456, 10, 589824, 700000]
EXACT = ("topk", "randomk", "bloom_leftmost", "bloom_random", "bloom_p0", "bloom_p2", "rle", "bloom_bf16",
         "randomk_bf16")
EXACT_RESID = tuple(m for m in EXACT if m != "bloom_p2")    # P2's residual agrees to ulps (test_gpu_p2_fused)
LAUNCH = {"fp32-tma-2cta": (torch.float32, dict(use_tma=True, blocks_per_sm=2)),
          "bf16-cpasync-1cta": (torch.bfloat16, dict(use_tma=False, blocks_per_sm=1)),
          "bf16-tma-2cta": (torch.bfloat16, dict(use_tma=True, blocks_per_sm=2))}


def _bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


def _plan(mode, ratio, sizes=SIZES):
    kw = dict(MODES[mode])
    if mode == "bloom_polyfit":
        kw["poly_min_k"] = 300
    return BucketPlan(list(sizes), compress_ratio=ratio, **kw)


@pytest.mark.parametrize("launch", list(LAUNCH))
@pytest.mark.parametrize("ratio", [0.25, 0.0625])
@pytest.mark.parametrize("mode", [m for m in MODES if m != "threshold"])
def test_engine_at_warmup_ratios_vs_oracle(mode, ratio, launch):
    dtype, kw = LAUNCH[launch]
    plan = _plan(mode, ratio)
    smem = (160 if kw["blocks_per_sm"] < 2 else 80) * 1024
    if ratio == 0.25 and plan.tensors[-1].mode == MODE_BLOOM:
        assert plan.tensors[-1].n_filter_words * 4 > smem          # probed from L2
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=4_000_000, grad_dtype=dtype, **kw)
    gen = torch.Generator().manual_seed(11)
    resid = torch.zeros(plan.total_elems)
    compare = compare_dexp_slot if "dexp" in mode else _compare_slot
    for step in range(2):
        g = (_fill(plan, gen) * (1.0 if step == 0 else 0.3)).to(dtype).float()   # step 1 shrinks: history fallback
        eng.grad.copy_(g.to(dtype).cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, new_res, slots = engine_oracle(plan, [g], [resid], epoch=eng.epoch)
        tag = f"{mode} ratio={ratio} {launch} step {step}"
        bad = compare(plan, eng.slot(), slots[0], tag)
        assert not bad, bad[:4]
        got = eng.grad.float().cpu()
        if mode in EXACT:
            want = out.to(torch.bfloat16).float() if dtype == torch.bfloat16 else out
            assert torch.equal(_bits(got), _bits(want)), tag
            if mode in EXACT_RESID:
                assert torch.equal(_bits(eng.resid), _bits(new_res[0])), tag
            else:
                assert torch.allclose(eng.resid.cpu(), new_res[0], rtol=1e-5, atol=1e-6), tag
            resid = new_res[0]
        else:                       # value codecs: fp32 fits on the GPU, fp64 in the oracle
            scale = float(out.abs().max())
            assert torch.allclose(got, out, atol=2e-3 * scale, rtol=1e-2), tag
            resid = eng.resid.cpu().clone()
    eng.close()


@pytest.mark.parametrize("mode", ["topk", "bloom_leftmost", "rle", "randomk", "bloom_p2"])
def test_switched_engine_history_does_not_matter(mode):
    """A stage switch's engine (residual and momentum carried, select history zero) gives the slots, residual, momentum
    and output of a fresh engine of that stage loaded with the same state and the OLD stage's select history, and both
    equal the oracle."""
    M = 0.9
    p0, p1 = _plan(mode, 0.25), _plan(mode, 0.0625)
    kw = dict(device="cuda:0", world=1, rank=0, momentum=M, beta=1.0, gamma=1.0, spin_limit=4_000_000)
    old = BucketEngine(p0, **kw)
    gen = torch.Generator().manual_seed(3)
    for _ in range(2):
        old.grad.copy_(_fill(p0, gen).cuda())
        old.step()
    torch.cuda.synchronize()
    old.check_status()
    assert int(old.sel.abs().sum()) != 0                          # there is a history to drop
    switched = BucketEngine(p1, grad=old.grad, **kw)
    assert switched.grad is old.grad
    switched.resid.copy_(old.resid)
    switched.mom.copy_(old.mom)
    switched.epoch = max(switched.epoch, old.epoch)
    stale = BucketEngine(p1, **kw)
    stale.load_state_dict(old.state_dict())
    res, mom = [old.resid.cpu()], [old.mom.cpu()]
    old.close()
    for step in range(2):
        g = _fill(p1, gen) * (1.0 if step == 0 else 0.2)
        for e in (switched, stale):
            e.grad.copy_(g.cuda())
            e.step()
        torch.cuda.synchronize()
        switched.check_status()
        stale.check_status()
        assert switched.epoch == stale.epoch
        out, res, slots, mom = engine_oracle(p1, [g], res, epoch=switched.epoch, momentum=M, moms=mom)
        tag = f"{mode} step {step}"
        assert torch.equal(switched.slot().cpu(), stale.slot().cpu()), tag
        assert not _compare_slot(p1, switched.slot(), slots[0], tag), tag
        for a, b, want in ((switched.resid, stale.resid, res[0]), (switched.mom, stale.mom, mom[0]),
                           (switched.grad, stale.grad, out)):
            assert torch.equal(_bits(a), _bits(b)), tag
            if mode in EXACT_RESID:
                assert torch.equal(_bits(a), _bits(want)), tag
            else:
                assert torch.allclose(a.cpu(), want, rtol=1e-5, atol=1e-6), tag
    switched.close()
    stale.close()


# ---- DeepReduceDDP ----------------------------------------------------------------------------------------------
WU = dict(warmup_ratios=[0.25, 0.0625], warmup_steps=2)
MEMS = {"residual": dict(memory='residual'),
        "dgc": dict(memory='dgc', momentum=0.9, weight_decay=1e-3, clip_norm=0.05)}


def _cfg(mem, **extra):
    return dict({'compressor': 'topk', 'communicator': 'allgather', 'compress_ratio': 0.01,
                 'calibrate_partition': False, 'min_numel': 100}, **MEMS[mem], **WU, **extra)


def _grads(model, gen):
    return {n: torch.randn(p.shape, generator=gen) * 1e-3 for n, p in model.named_parameters()}


@pytest.mark.parametrize("calibrate", [False, True], ids=["static", "calibrated"])
@pytest.mark.parametrize("mem", list(MEMS))
def test_ddp_fused_across_two_boundaries(mem, calibrate):
    """Six exchanges in stages of two: every p.grad equals engine_oracle on the stage's plan bit for bit, and the
    per-tensor GRACE route for the tensors without a 22-bit tie at K; p.grad stays the bucket's view; the optimizer
    step after each finish() (the switching ones included) applies that exchange's aggregate."""
    from deepreduce_b200.parallel import DeepReduceDDP
    cfg = _cfg(mem, calibrate_partition=calibrate)
    wu = warmup_from_params(cfg)
    torch.manual_seed(0)
    model = _ConvNet().cuda()
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    assert ddp.fused and len(ddp.engines) == 1
    opt = torch.optim.SGD(model.parameters(), lr=1.0)
    flat = ddp.flat[0]
    views = {n: p.grad for n, p in model.named_parameters()}
    grc = dr.deepreduce_from_params({k: v for k, v in cfg.items() if k != 'calibrate_partition'})
    if hasattr(grc.memory, "bind_parameters"):
        grc.memory.bind_parameters(model.named_parameters())
    plan0 = ddp.engines[0].plan
    res, mom = [torch.zeros(plan0.total_elems)], [torch.zeros(plan0.total_elems)]
    gen = torch.Generator().manual_seed(1)
    tied, epochs, compared = set(), [], 0
    for e in range(6):
        eng = ddp.engines[0]
        assert eng.plan.compress_ratio == wu.ratio_at(e) and ddp.stage == wu.stage(e)
        assert eng.grad is flat
        grads = _grads(model, gen)
        w = eng.parameter_buffer() if mem == "dgc" else None
        before = {n: p.detach().clone() for n, p in model.named_parameters()}
        with torch.no_grad():
            for n, p in model.named_parameters():
                assert p.grad is views[n]
                p.grad.copy_(grads[n])
        g_flat = eng.grad.float().cpu()
        ddp.finish()
        torch.cuda.synchronize()
        ddp.check()
        epochs.append(eng.epoch)
        if mem == "dgc":
            out, res, _, mom = engine_oracle(eng.plan, [g_flat], res, epoch=eng.epoch, momentum=0.9, moms=mom,
                                             weight_decay=1e-3, weights=[w], clip_norm=0.05, owner=eng.owner)
        else:
            out, res, _ = engine_oracle(eng.plan, [g_flat], res, epoch=eng.epoch)
        now = ddp.engines[0]
        assert (now is not eng) == (wu.stage(e + 1) != wu.stage(e))          # the switch happened in this finish()
        assert now.grad is flat
        assert torch.equal(_bits(flat), _bits(out)), e
        assert torch.equal(_bits(now.resid), _bits(res[0])), e
        if mem == "dgc":
            assert torch.equal(_bits(now.mom), _bits(mom[0])), e
        for n, p in model.named_parameters():
            assert p.grad is views[n]
            g = grads[n].cuda()
            acc = copy.deepcopy(grc.memory).compensate(g.clone(), n)
            if _prefix_tie(acc.flatten().cpu(), min(spec.topk_k(g.numel(), wu.ratio_at(e)), g.numel())):
                tied.add(n)                         # the routes part at a tie (the fused select ships both)
            want = grc.step(g.clone(), n).view_as(p)
            if n not in tied:
                assert torch.equal(p.grad, want), (e, n)
                compared += 1
        opt.step()
        for n, p in model.named_parameters():
            assert torch.equal(p.detach(), before[n] - views[n]), (e, n)
    assert all(a < b for a, b in zip(epochs, epochs[1:]))
    assert compared > 0
    ddp.close()


@pytest.mark.parametrize("cut", [2, 3])
def test_ddp_fused_checkpoint_resume(cut):
    from deepreduce_b200.parallel import DeepReduceDDP
    cfg = dict(_cfg("dgc"), deepreduce='index', index='bloom')
    cfg.pop("weight_decay")
    gen = torch.Generator().manual_seed(2)
    torch.manual_seed(0)
    steps = [_grads(_ConvNet(), gen) for _ in range(6)]

    def run(ddp, model, seq):
        out = []
        for grads in seq:
            with torch.no_grad():
                for n, p in model.named_parameters():
                    p.grad.copy_(grads[n])
            ddp.finish()
            out.append({n: p.grad.detach().cpu().clone() for n, p in model.named_parameters()})
        return out

    def fresh():
        torch.manual_seed(0)
        m = _ConvNet().cuda()
        return m, DeepReduceDDP(m, cfg, overlap=False)

    m, d = fresh()
    ref = run(d, m, steps)
    d.close()
    m, d = fresh()
    run(d, m, steps[:cut])
    st = d.state_dict()
    d.close()
    m, d = fresh()
    d.load_state_dict(st)
    assert d.stage == warmup_from_params(cfg).stage(cut)
    assert d.engines[0].plan.compress_ratio == warmup_from_params(cfg).ratio_at(cut)
    got = run(d, m, steps[cut:])
    for a, b in zip(ref[cut:], got):
        for n in a:
            assert torch.equal(_bits(a[n]), _bits(b[n])), (cut, n)
    d.close()


def test_ddp_stage_refused_at_construction():
    from deepreduce_b200.parallel import DeepReduceDDP
    cfg = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.001,
           'deepreduce': 'index', 'index': 'bloom', 'policy': 'conflict_sets', 'p2_pick_mask': True,
           'calibrate_partition': False, 'warmup_ratios': [0.25], 'warmup_steps': 1}
    model = nn.Linear(4096, 2048, bias=False).cuda()
    with pytest.raises(ValueError, match="positives"):
        DeepReduceDDP(model, cfg, overlap=False)
    d = DeepReduceDDP(model, {k: v for k, v in cfg.items() if not k.startswith("warmup")}, overlap=False)
    d.close()


def test_trainer_accumulation_switches_on_exchanges():
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.trainer import Trainer
    torch.manual_seed(0)
    cfg = dict(_cfg("residual"), warmup_steps=1, deepreduce='index', index='bloom')
    tr = Trainer(resnet20().cuda(), cfg, lr=0.01, amp_dtype=None, accum_steps=2)
    x = torch.randn(8, 3, 32, 32, device="cuda")
    y = torch.randint(0, 10, (8,), device="cuda")
    seen = []
    for _ in range(6):
        tr.step(x, target=y)
        seen.append((tr.ddp.step_count, tr.ddp.stage, tr.ddp.engines[0].plan.compress_ratio))
    torch.cuda.synchronize()
    tr.ddp.check()
    assert seen == [(0, 0, 0.25), (1, 1, 0.0625), (1, 1, 0.0625), (2, 2, 0.01), (2, 2, 0.01), (3, 2, 0.01)]
    assert tr.ddp.wire_bytes_per_step() == sum(e.plan.wire_bytes() for e in tr.ddp.engines)
    tr.close()


# ---- DDP hook ------------------------------------------------------------------------------------------------------
def test_ddp_hook_across_boundaries_with_no_sync(nccl_world1):
    """torch DDP + the DeepReduce hook on ResNet-20, stages of two exchanges, a no_sync() micro-step before every
    exchange: each bucket call equals engine_oracle on the plan of the exchange's stage, fed the packed bucket and the
    residual the engine holds; that residual is the one the previous exchange left, carried by parameter across the
    switches and DDP's bucket rebuild; epochs only grow."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import deepreduce_hook, pack_reference, unpack_reference
    torch.manual_seed(0)
    cfg = dict(_cfg("residual"), deepreduce='index', index='bloom')
    wu = warmup_from_params(cfg)
    model = resnet20().cuda()
    ddp = DDP(model, device_ids=[0], bucket_cap_mb=0.25)
    st = DeepReduceHookState(cfg, model)
    last_res, last_epoch, checked = {}, {}, []

    def spy_hook(state, bucket):
        buf = bucket.buffer()
        e = state.step_count
        lay = state._layout_for(bucket, buf)
        eng = lay.engine
        assert eng.plan.compress_ratio == wu.ratio_at(e)
        for p in lay.params:
            if id(p) in last_res:
                assert torch.equal(_bits(lay.resid_of(p)), last_res[id(p)]), e
        packed = pack_reference(buf.detach().float().cpu(), torch.zeros(eng.plan.total_elems), lay.table)
        resid = eng.resid.cpu().clone()
        fut = deepreduce_hook(state, bucket)
        torch.cuda.synchronize()
        eng.check_status()
        for p in lay.params:            # the engine that holds a parameter never reuses an epoch of the one before
            assert eng.epoch > last_epoch.get(id(p), 0), e
            last_epoch[id(p)] = eng.epoch
        out, new_res, _ = engine_oracle(eng.plan, [packed], [resid], epoch=eng.epoch)
        want = unpack_reference(out, buf.detach().float().cpu().clone(), lay.table)
        assert torch.equal(_bits(buf), _bits(want)), e
        assert torch.equal(_bits(eng.resid), _bits(new_res[0])), e
        for p in lay.params:
            last_res[id(p)] = _bits(lay.resid_of(p))
        checked.append(e)
        return fut
    ddp.register_comm_hook(st, spy_hook)
    gen = torch.Generator(device="cuda").manual_seed(5)
    try:
        for step in range(6):
            model.zero_grad(set_to_none=True)
            with ddp.no_sync():
                ddp(torch.randn(4, 3, 32, 32, device="cuda", generator=gen)).float().pow(2).mean().backward()
            ddp(torch.randn(4, 3, 32, 32, device="cuda", generator=gen)).float().pow(2).mean().backward()
            torch.cuda.synchronize()
            assert st.step_count == step + 1
        st.check()
        assert sorted(set(checked)) == list(range(6))
        assert st.state_dict()["step"] == 6
        assert all(l.plan.compress_ratio == 0.01 for l in st._layouts)
    finally:
        st.close()


@pytest.mark.parametrize("cfg_name", ["bloom_random", "randomk"])
def test_ddp_hook_without_keys_keeps_layout_epochs(nccl_world1, cfg_name):
    """Without the warm-up keys a layout met at DDP's bucket rebuild counts its epochs from its own start, as it always
    has: the epoch seeds the random policy and the randomk draw, so carrying the old engine's epoch would change the
    wire.  With 'calibrate_partition': False every engine's epoch is the number of exchanges it ran."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import deepreduce_hook
    from test_gpu_comm_hook import CONFIGS
    cfg = dict(CONFIGS[cfg_name], calibrate_partition=False)
    torch.manual_seed(0)
    model = resnet20().cuda()
    ddp = DDP(model, device_ids=[0], bucket_cap_mb=0.25)
    st = DeepReduceHookState(cfg, model)
    runs, made = {}, []

    def spy_hook(state, bucket):
        lay = state._layout_for(bucket, bucket.buffer())
        runs[id(lay)] = (lay, runs.get(id(lay), (lay, 0))[1] + 1)
        return deepreduce_hook(state, bucket)
    ddp.register_comm_hook(st, spy_hook)
    new_layout = st._new_layout

    def spy_layout(*a, **k):
        made.append(st.step_count)
        return new_layout(*a, **k)
    st._new_layout = spy_layout
    gen = torch.Generator(device="cuda").manual_seed(6)
    try:
        for _ in range(4):
            model.zero_grad(set_to_none=True)
            ddp(torch.randn(4, 3, 32, 32, device="cuda", generator=gen)).float().pow(2).mean().backward()
        torch.cuda.synchronize()
        st.check()
        assert any(e > 0 for e in made), "DDP's bucket rebuild was not met"
        for lay, n in runs.values():
            assert lay.engine.epoch == n, (lay.index, lay.engine.epoch, n)
    finally:
        st.close()


# ---- W ranks in one process ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("config", ["shard", "noshard"])
@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("mode", ["bloom_leftmost", "topk", "rle"])
def test_multirank_across_a_switch(monkeypatch, mode, W, config):
    """W ranks switch from 25 % to 6.25 % after two epochs through ``switch_engine`` (the per-bucket switch of
    ``DeepReduceDDP``): the ranks agree, epochs never repeat, each slot matches the oracle and the aggregate is the sum
    of the decoded shipped slots."""
    monkeypatch.setenv("DR_DETERMINISTIC", "1")
    M = 0.9
    shard = config == "shard"
    gen = torch.Generator().manual_seed(4)
    res = mom = None
    engs, used = [], []
    for ratio in (0.25, 0.0625):
        plan = _plan(mode, ratio, sizes=SIZES[:-2])
        arenas = [torch.zeros(plan.arena_words(W, shard), dtype=torch.int32, device="cuda:0") for _ in range(W)]
        kw = dict(momentum=M, average=False, spin_limit=4_000_000, peer_timeout_ms=5000, shard=shard)
        if engs:
            views = [e.grad for e in engs]
            engs = [switch_engine(o, lambda grad, r=r: _RankEngine(plan, arenas, r, grad=grad, **kw))
                    for r, o in enumerate(engs)]
            assert all(e.grad is v for e, v in zip(engs, views))
        else:
            engs = [_RankEngine(plan, arenas, r, **kw) for r in range(W)]
            res = [torch.zeros(plan.total_elems) for _ in range(W)]
            mom = [torch.zeros(plan.total_elems) for _ in range(W)]
        for _ in range(2):
            assert len({e.epoch for e in engs}) == 1                  # the ranks agree on the step counter
            epoch = engs[0].epoch + 1
            assert epoch not in used and all(epoch > u for u in used)
            used.append(epoch)
            grads = [_fill(plan, gen) * (0.5 + 0.5 * r) for r in range(W)]
            for r in range(W):
                engs[r].grad.copy_(grads[r].cuda())
            _run_step(engs, config, epoch)
            out, res, slots, mom = engine_oracle(plan, grads, res, epoch=epoch, average=False, momentum=M, moms=mom)
            dec = sum(decode_slot_oracle(plan, s) for s in slots)
            for r in range(W):
                tag = f"{mode} W={W} {config} ratio={ratio} epoch {epoch} rank {r}"
                assert not _compare_slot(plan, engs[r].slot(), slots[r], tag), tag
                assert torch.equal(_bits(engs[r].resid), _bits(res[r])), tag
                assert torch.equal(_bits(engs[r].mom), _bits(mom[r])), tag
                assert torch.equal(_bits(engs[r].grad), _bits(engs[0].grad)), tag
                assert torch.equal(_bits(engs[r].grad), _bits(out)), tag
            assert torch.allclose(out, dec, rtol=1e-6, atol=1e-6)
    for e in engs:
        e.close()
