"""The fused engine's 'dgc' memory with local gradient clipping ('clip_norm') on the GPU: phase 0 sums each
parameter's squares in fp64 by pairs (per tile, then over the parameter's tiles, across CTAs) and scales the gradient
by fl32(thr / nrm) ahead of the weight decay and the momentum.

Every fused mode is checked bit for bit against a 'dgc' engine without clipping fed ``clip_oracle``'s gradient, the
exact modes against ``engine_oracle(clip_norm=...)`` with weight decay on, W = 2-4 ranks in one process (where
thr = c / sqrt(W)), a parameter of more tiles than one shared-memory tree takes, and channels_last parameters through
``DeepReduceDDP`` (against the per-tensor GRACE route) and the DDP hook (against the oracle in bucket order)."""
import copy
import math

import pytest
import torch
import torch.nn as nn

import deepreduce_b200 as dr
from deepreduce_b200 import spec
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import clip_oracle
from deepreduce_b200.parallel.plan import split_large
from test_engine_multirank import _RankEngine, _run_step
from test_fused_params import _prefix_tie
from test_gpu_dgc_weight_decay import EXACT, MODES, _ConvNet, _setup, _storage, _weights, nccl_world1  # noqa: F401
from test_gpu_engine import _compare_slot, _fill

pytestmark = pytest.mark.gpu
M, WD, C = 0.9, 0.05, 60.0          # c = 60 clips the parameters past ~3600 elements of randn, not the small ones
LAUNCH = {"tma_2cta": dict(use_tma=True, blocks_per_sm=2), "cpasync_1cta": dict(use_tma=False, blocks_per_sm=1)}


def _bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


def _grad(plan, gen, dtype, step):
    return (_fill(plan, gen) * (0.5 + step)).to(dtype).float()      # the widened gradient the engine receives


@pytest.mark.parametrize("launch", list(LAUNCH))
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", list(MODES))
def test_clip_engine_vs_clipped_twin(mode, dtype, launch):
    plan, owner, _ = _setup(mode, dtype, split=True)
    kw = dict(device="cuda:0", world=1, rank=0, momentum=M, spin_limit=2_000_000, **LAUNCH[launch])
    eng = BucketEngine(plan, clip_norm=C, owner=owner, grad_dtype=dtype, **kw)
    twin = BucketEngine(plan, **kw)
    gen = torch.Generator().manual_seed(1)
    clipped = 0
    for step in range(3):
        g = _grad(plan, gen, dtype, step)
        gc = clip_oracle(plan, g, C, owner)
        clipped += int(not torch.equal(g, gc))
        eng.grad.copy_(g.to(dtype).cuda())
        twin.grad.copy_(gc.cuda())
        eng.step()
        twin.step()
        torch.cuda.synchronize()
        eng.check_status()
        twin.check_status()
        tag = f"{mode} {dtype} {launch} step {step}"
        assert torch.equal(eng.slot().cpu(), twin.slot().cpu()), tag
        assert torch.equal(_bits(eng.resid), _bits(twin.resid)), tag
        assert torch.equal(_bits(eng.mom), _bits(twin.mom)), tag
        if dtype == torch.float32:
            assert torch.equal(_bits(eng.grad), _bits(twin.grad)), tag
        else:
            assert torch.equal(eng.grad.cpu(), twin.grad.cpu().to(torch.bfloat16)), tag
    assert clipped == 3
    eng.close()
    twin.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", EXACT)
def test_clip_engine_vs_oracle_with_weight_decay(mode, dtype):
    plan, owner, params = _setup(mode, dtype, split=True)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, weight_decay=WD, clip_norm=C, owner=owner,
                       grad_dtype=dtype, spin_limit=2_000_000)
    eng.bind_parameters(params, owner)
    gen = torch.Generator().manual_seed(2)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    w = _weights(plan, owner, params)
    for step in range(3):
        g = _grad(plan, gen, dtype, step)
        eng.grad.copy_(g.to(dtype).cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom, weight_decay=WD,
                                             weights=[w], clip_norm=C, owner=owner)
        tag = f"{mode} {dtype} step {step}"
        assert not _compare_slot(plan, eng.slot(), slots[0], tag), tag
        if dtype == torch.float32:
            assert torch.equal(_bits(eng.grad), _bits(out)), tag
        else:
            assert torch.equal(eng.grad.cpu(), out.to(torch.bfloat16)), tag
        assert torch.equal(_bits(eng.resid), _bits(res[0])), tag
        assert torch.equal(_bits(eng.mom), _bits(mom[0])), tag
    eng.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_clip_many_tiles(dtype):
    """A parameter of 2 101 tiles (non-power-of-two, more than one 2048-leaf tree: the tile sums are reduced in blocks,
    then over the blocks), whole and as chunks, next to a tensor under min_numel; clipped, then not clipped."""
    n = 2100 * 4096 + 77
    for split in (None, 1 << 20):
        numels, names, shapes, owner = split_large([n, 500, 70000], ["big", "small", "mid"], [(n,), (500,), (70000,)],
                                                   split)
        plan = BucketPlan(numels, names, shapes, compress_ratio=0.01, index=None)
        eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, clip_norm=C, owner=owner,
                           grad_dtype=dtype, spin_limit=4_000_000)
        twin = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, spin_limit=4_000_000)
        gen = torch.Generator().manual_seed(3)
        for step, scale in enumerate((1.0, 1e-3)):
            g = (_fill(plan, gen) * scale).to(dtype).float()
            gc = clip_oracle(plan, g, C, owner)
            assert torch.equal(g, gc) == (scale < 1.0)
            eng.grad.copy_(g.to(dtype).cuda())
            twin.grad.copy_(gc.cuda())
            eng.step()
            twin.step()
            torch.cuda.synchronize()
            eng.check_status()
            tag = f"{dtype} split={split} step {step}"
            assert torch.equal(eng.slot().cpu(), twin.slot().cpu()), tag
            assert torch.equal(_bits(eng.resid), _bits(twin.resid)), tag
            assert torch.equal(_bits(eng.mom), _bits(twin.mom)), tag
        eng.close()
        twin.close()


@pytest.mark.parametrize("config", ["shard", "noshard"])
@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("mode", ["bloom_leftmost", "topk", "randomk", "rle"])
def test_clip_multirank_vs_oracle(monkeypatch, mode, W, config):
    monkeypatch.setenv("DR_DETERMINISTIC", "1")
    plan, owner, _ = _setup(mode, torch.float32, split=True)
    shard = config == "shard"
    arenas = [torch.zeros(plan.arena_words(W, shard), dtype=torch.int32, device="cuda:0") for _ in range(W)]
    engs = [_RankEngine(plan, arenas, r, momentum=M, clip_norm=C, owner=owner, average=False, spin_limit=4_000_000,
                        peer_timeout_ms=5000, shard=shard) for r in range(W)]
    assert engs[0].clip_thr == C / math.sqrt(W)
    gen = torch.Generator().manual_seed(4)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    mom = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in range(1, 4):
        grads = [_fill(plan, gen) * (0.5 + 0.5 * r) for r in range(W)]
        for r in range(W):
            engs[r].grad.copy_(grads[r].cuda())
        _run_step(engs, config, epoch)
        out, res, slots, mom = engine_oracle(plan, grads, res, epoch=epoch, average=False, momentum=M, moms=mom,
                                             clip_norm=C, owner=owner)
        for r in range(W):
            tag = f"{mode} W={W} {config} epoch {epoch} rank {r}"
            assert not _compare_slot(plan, engs[r].slot(), slots[r], tag), tag
            assert torch.equal(_bits(engs[r].resid), _bits(res[r])), tag
            assert torch.equal(_bits(engs[r].mom), _bits(mom[r])), tag
            assert torch.equal(_bits(engs[r].grad), _bits(out)), tag
    for e in engs:
        e.close()


def _cl_grads(model, gen):
    """Seeded gradients in each parameter's layout (channels_last for the conv weights): conv2.weight (norm ~0.19) is
    clipped at c = 0.05, conv1.weight (~0.04), fc and the biases are not."""
    return {n: (torch.randn(p.shape, generator=gen) * 1e-3).contiguous(
                memory_format=torch.channels_last if p.dim() == 4 else torch.contiguous_format)
            for n, p in model.named_parameters()}


def test_ddp_fused_channels_last_matches_grace_route():
    """DeepReduceDDP on CUDA (fused) with 'clip_norm' on a channels_last conv net: every p.grad equals, bit for bit,
    what the per-tensor GRACE route computes from the same gradients, which it sums in their storage order.  Plain
    top-k pairs: the selection is a set, so the routes' different index orders (storage, logical) do not matter; the
    seed has no 22-bit tie at K (where the fused select would ship more than K)."""
    from deepreduce_b200.parallel import DeepReduceDDP
    from deepreduce_b200.parallel.ddp import fused_path
    cfg = {'compressor': 'topk', 'memory': 'dgc', 'momentum': M, 'clip_norm': 0.05, 'communicator': 'allgather',
           'compress_ratio': 0.01, 'calibrate_partition': False, 'min_numel': 100}
    assert fused_path(cfg)
    torch.manual_seed(0)
    model = _ConvNet().cuda().to(memory_format=torch.channels_last)
    assert not model.conv2.weight.is_contiguous()
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    assert ddp.fused and len(ddp.engines) == 1
    grc = dr.deepreduce_from_params(cfg)
    gen = torch.Generator().manual_seed(1)
    clipped = 0
    for step in range(3):
        grads = _cl_grads(model, gen)
        with torch.no_grad():
            for n, p in model.named_parameters():
                p.grad.copy_(grads[n])                                 # p.grad is the parameter's view of the bucket
        ddp.finish()
        for n, p in model.named_parameters():
            g = grads[n]
            acc = copy.deepcopy(grc.memory).compensate(g.clone(), n)
            assert not _prefix_tie(acc.as_strided((acc.numel(),), (1,)).contiguous(),
                                   min(spec.topk_k(g.numel(), 0.01), g.numel())), (step, n)
            clipped += int(not torch.equal(grc.memory._clip(g), g))
            want = grc.step(g.clone(), n).view_as(p)
            assert torch.equal(p.grad.cpu(), want), (step, n, int((p.grad.cpu() != want).sum()))
    assert clipped == 3
    ddp.close()


def test_ddp_hook_clip_channels_last(nccl_world1):
    """torch DDP + the DeepReduce hook with 'clip_norm' on a channels_last conv net: every bucket layout's result equals
    ``engine_oracle`` fed the gradients in bucket (storage) order, across DDP's bucket rebuild."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    torch.manual_seed(0)
    cfg = {'compressor': 'topk', 'memory': 'dgc', 'momentum': M, 'clip_norm': 0.05, 'communicator': 'allgather',
           'compress_ratio': 0.01, 'calibrate_partition': False, 'min_numel': 100}
    model = _ConvNet().cuda().to(memory_format=torch.channels_last)
    ddp = DDP(model, device_ids=[0], bucket_cap_mb=0.05)
    st = DeepReduceHookState(cfg, model)
    named = dict(model.named_parameters())
    by_id = {id(p): n for n, p in named.items()}
    local = {}

    def spy_hook(state, bucket):
        buf = bucket.buffer()
        for p, (d, k) in zip(bucket.parameters(), bucket_segments(bucket)):
            local[by_id[id(p)]] = buf[d:d + k].detach().float().cpu().clone()
        return deepreduce_hook(state, bucket)
    ddp.register_comm_hook(st, spy_hook)
    u = {n: torch.zeros(p.numel()) for n, p in named.items()}
    r = {n: torch.zeros(p.numel()) for n, p in named.items()}
    gen = torch.Generator(device="cuda").manual_seed(5)
    clipped = 0
    try:
        for step in range(3):
            for p in model.parameters():
                p.grad = None
            x = torch.randn(4, 3, 8, 8, device="cuda", generator=gen).contiguous(memory_format=torch.channels_last)
            ddp(x).float().pow(2).mean().backward()
            torch.cuda.synchronize()
            st.check()
            for lay in set(st._by_index.values()):
                plan = lay.plan
                assert lay.engine.clip_thr == 0.05
                fg, fr, fu = (torch.zeros(plan.total_elems) for _ in range(3))
                rows = [(by_id[id(p)], p, lay.eng_off[i], k) for i, (p, (_, k)) in enumerate(zip(lay.params, lay.segments))]
                for n, p, off, k in rows:
                    fg[off:off + k], fr[off:off + k], fu[off:off + k] = local[n], r[n], u[n]
                clipped += int(not torch.equal(clip_oracle(plan, fg, 0.05, lay.engine.owner), fg))
                out, res, _, mom = engine_oracle(plan, [fg], [fr], epoch=lay.engine.epoch, momentum=M, moms=[fu],
                                                 clip_norm=0.05, owner=lay.engine.owner)
                for n, p, off, k in rows:
                    tag = f"step {step} {n}"
                    assert torch.equal(_bits(_storage(p.grad)), _bits(out[off:off + k])), tag
                    assert torch.equal(_bits(lay.resid_of(p)), _bits(res[0][off:off + k])), tag
                    assert torch.equal(_bits(lay.mom_of(p)), _bits(mom[0][off:off + k])), tag
                    r[n], u[n] = res[0][off:off + k].clone(), mom[0][off:off + k].clone()
            with torch.no_grad():
                for p in model.parameters():
                    p -= 0.05 * p.grad
        assert clipped > 0
    finally:
        st.close()
