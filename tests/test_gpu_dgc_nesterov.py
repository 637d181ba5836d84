"""The fused engine's 'dgc' memory with Nesterov momentum and per-parameter weight decay (a factor of 0 for the
parameters 'weight_decay_exclude' names) on the GPU.

Phase 0 reads each plan tensor's decay factor once per tensor run and adds v = fl(d + fl(m * u)) to the residual
instead of u.  The exact modes are checked bit for bit against ``engine_oracle(nesterov=True, weight_decays=...)``, the
others against a momentum-0 'dgc' twin fed v; then the default against an engine built without the new arguments,
NaN parameters on excluded tensors, W = 2 and 4 ranks in one process, DeepReduceDDP against the per-tensor memory on
channels_last ResNet-20, the DDP hook across its bucket rebuild, and a sparsity warm-up stage switch."""
import os
import tempfile

import pytest
import torch

from deepreduce_b200.grace import DgcMemory
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import decay_oracle, tensor_decays
from deepreduce_b200.parallel.plan import split_large
from test_engine_multirank import _RankEngine, _run_step
from test_gpu_engine import SIZES, _compare_slot, _fill

pytestmark = pytest.mark.gpu
M, WD, C = 0.9, 0.05, 60.0
# parameters 1, 5 and 8 (589824 elements: split into chunks) are excluded from the decay
EXCLUDED = (1, 5, 8)

MODES = {
    "plain": dict(index=None),
    "threshold": dict(index=None, sparsifier="threshold", threshold=1.5),
    "bloom_leftmost": dict(index="bloom"),
    "bloom_random": dict(index="bloom", policy="random", fpr=0.02),
    "bloom_p0": dict(index="bloom", policy="p0"),
    "rle": dict(index="rle"),
    "elias_fano": dict(index="elias_fano"),
    "bloom_bf16": dict(index="bloom", value="bf16"),
    "rle_sign": dict(index="rle", value="sign"),
    "ef_fp8": dict(index="elias_fano", value="fp8"),
    "randomk": dict(index=None, sparsifier="randomk"),
    "randomk_fp8": dict(index=None, sparsifier="randomk", value="fp8"),
    # value codecs whose oracle is not bit-exact against the device: checked against the twin
    "bloom_qsgd": dict(index="bloom", value="qsgd"),
    "rle_qsgd": dict(index="rle", value="qsgd"),
    "bloom_polyfit": dict(index="bloom", value="polyfit", poly_min_k=300),
    "bloom_dexp": dict(index="bloom", value="dexp"),
    "randomk_qsgd": dict(index=None, sparsifier="randomk", value="qsgd"),
}
INEXACT = ("bloom_qsgd", "rle_qsgd", "bloom_polyfit", "bloom_dexp", "randomk_qsgd")
EXACT = [m for m in MODES if m not in INEXACT]
LAUNCH = [dict(use_tma=True, blocks_per_sm=2), dict(use_tma=False, blocks_per_sm=1)]


def _bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


def _placed(w, i):
    """w itself for even i; for odd i a copy that starts one element past an aligned address."""
    if i % 2 == 0:
        return w
    buf = torch.empty(w.numel() + 1, dtype=w.dtype, device=w.device)
    buf[1:].copy_(w)
    return buf[1:]


def _setup(mode, dtype, sizes=SIZES, nan_excluded=False, seed=0):
    """Plan (parameters past two tiles as 8192-element chunks), owner, parameters and per-parameter decays."""
    numels, names, shapes, owner = split_large(sizes, [f"t{i}" for i in range(len(sizes))], [(n,) for n in sizes], 8192)
    plan = BucketPlan(numels, names, shapes, compress_ratio=0.01, **MODES[mode])
    gen = torch.Generator().manual_seed(seed)
    params = []
    for i, n in enumerate(sizes):
        w = torch.randn(n, generator=gen)
        if nan_excluded and i in EXCLUDED:
            w.fill_(float('nan'))
        params.append(_placed(w.to(dtype).cuda(), i))
    decays = [0.0 if i in EXCLUDED else WD for i in range(len(sizes))]
    return plan, owner, params, decays


def _weights(plan, owner, params):
    """The parameters flat in plan layout, widened to fp32, zeros in the padding."""
    w = torch.zeros(plan.total_elems)
    done = [0] * len(params)
    for j, t in enumerate(plan.tensors):
        i = owner[j]
        w[t.elem_off:t.elem_off + t.numel] = params[i].detach().float().cpu()[done[i]:done[i] + t.numel]
        done[i] += t.numel
    return w


def _nudge(params, step):
    for p in params:                      # the parameters move between steps, in place: every step reads new values
        p.mul_(1.0 - 0.01 * (step + 1))


def _grad(plan, gen, dtype, step):
    return (_fill(plan, gen) * (0.5 + step)).to(dtype).float()      # the widened gradient the engine receives


def _check(eng, out, res, mom, tag):
    if eng.grad_dtype == torch.float32:
        assert torch.equal(_bits(eng.grad), _bits(out)), tag
    else:                                 # the fp32 aggregate, rounded once
        assert torch.equal(eng.grad.cpu(), out.to(torch.bfloat16)), tag
    assert torch.equal(_bits(eng.resid), _bits(res)), tag
    if mom is not None:
        assert torch.equal(_bits(eng.mom), _bits(mom)), tag


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", EXACT)
def test_engine_vs_oracle(mode, dtype):
    """Three steps against the oracle; the launch (TMA ring or cp.async) and clipping alternate over the cases."""
    k = EXACT.index(mode) + (dtype == torch.bfloat16)
    launch, clip = LAUNCH[k % 2], (C if (k // 2) % 2 == 0 else None)
    plan, owner, params, decays = _setup(mode, dtype)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, nesterov=True, weight_decays=decays,
                       owner=owner, clip_norm=clip, grad_dtype=dtype, spin_limit=2_000_000, **launch)
    assert eng.decays == tensor_decays(plan, 0.0, decays, owner)
    eng.bind_parameters(params, owner)
    gen = torch.Generator().manual_seed(2)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(3):
        g = _grad(plan, gen, dtype, step)
        w = _weights(plan, owner, params)
        eng.grad.copy_(g.to(dtype).cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom, weights=[w],
                                             weight_decays=decays, owner=owner, nesterov=True, clip_norm=clip)
        tag = f"{mode} {dtype} {launch} clip={clip} step {step}"
        assert not _compare_slot(plan, eng.slot(), slots[0], tag), tag
        _check(eng, out, res[0], mom[0], tag)
        _nudge(params, step)
    eng.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", list(MODES))
def test_engine_vs_momentum_free_twin(mode, dtype):
    """Every mode, the coded values included: the Nesterov engine against a momentum-0 'dgc' engine fed v, which it
    adds to the residual unchanged (v = fl(fl(0 * u) + v)); u is tracked from the engine's own momentum buffer, and is
    cleared exactly where the twin's own decoded contribution is not zero."""
    launch = LAUNCH[(list(MODES).index(mode) + (dtype == torch.bfloat16)) % 2]
    plan, owner, params, decays = _setup(mode, dtype)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, nesterov=True, weight_decays=decays,
                       owner=owner, grad_dtype=dtype, spin_limit=2_000_000, **launch)
    eng.bind_parameters(params, owner)
    twin = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=0.0, spin_limit=2_000_000, **launch)
    tdec = tensor_decays(plan, 0.0, decays, owner)
    gen = torch.Generator().manual_seed(3)
    for step in range(3):
        g = _grad(plan, gen, dtype, step)
        d = decay_oracle(plan, g, _weights(plan, owner, params), tdec)
        u = (M * eng.mom.cpu()) + d
        v = d + (M * u)
        eng.grad.copy_(g.to(dtype).cuda())
        twin.grad.copy_(v.cuda())
        eng.step()
        twin.step()
        torch.cuda.synchronize()
        eng.check_status()
        twin.check_status()
        tag = f"{mode} {dtype} {launch} step {step}"
        assert torch.equal(eng.slot().cpu(), twin.slot().cpu()), tag
        own = twin.grad.cpu()
        if dtype == torch.float32:
            assert torch.equal(_bits(eng.grad), _bits(own)), tag
        else:
            assert torch.equal(eng.grad.cpu(), own.to(torch.bfloat16)), tag
        assert torch.equal(_bits(eng.resid), _bits(twin.resid)), tag
        assert torch.equal(_bits(eng.mom), _bits(torch.where(own != 0, torch.zeros_like(u), u))), tag
        _nudge(params, step)
    eng.close()
    twin.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", ["plain", "bloom_leftmost", "rle_qsgd", "bloom_polyfit", "randomk", "ef_fp8"])
def test_default_is_todays_engine(mode, dtype):
    """nesterov=False with one decay factor for every parameter computes bit for bit what an engine built without the
    new arguments computes, -0.0 gradients included."""
    plan, owner, params, _ = _setup(mode, dtype)
    new = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, nesterov=False,
                       weight_decays=[WD] * len(params), owner=owner, grad_dtype=dtype)
    ref = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, weight_decay=WD, grad_dtype=dtype)
    for e in (new, ref):
        e.bind_parameters(params, owner)
    gen = torch.Generator().manual_seed(4)
    ibits = torch.int16 if dtype == torch.bfloat16 else torch.int32
    for step in range(3):
        g = _fill(plan, gen).to(dtype)
        g[::5] = -0.0
        for e in (new, ref):
            e.grad.copy_(g.cuda())
            e.step()
        torch.cuda.synchronize()
        tag = f"{mode} {dtype} step {step}"
        assert torch.equal(new.slot().cpu(), ref.slot().cpu()), tag
        assert torch.equal(new.grad.cpu().view(ibits), ref.grad.cpu().view(ibits)), tag
        assert torch.equal(_bits(new.resid), _bits(ref.resid)), tag
        assert torch.equal(_bits(new.mom), _bits(ref.mom)), tag
        _nudge(params, step)
    new.close()
    ref.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", ["plain", "bloom_leftmost", "rle_sign", "bloom_qsgd"])
def test_excluded_parameters_are_never_read(mode, dtype):
    """NaN parameters bound to the excluded tensors give the bits of a twin whose excluded parameters are finite, and on
    the excluded tensors the bits of a twin without any weight decay (each tensor selects and codes on its own at
    W = 1), -0.0 gradients included."""
    plan, owner, params, decays = _setup(mode, dtype, nan_excluded=True)
    _, _, finite, _ = _setup(mode, dtype)
    engs = []
    for ps in (params, finite):
        e = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, nesterov=True, weight_decays=decays,
                         owner=owner, grad_dtype=dtype)
        e.bind_parameters(ps, owner)
        engs.append(e)
    engs.append(BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, nesterov=True, grad_dtype=dtype))
    gen = torch.Generator().manual_seed(5)
    excluded = torch.zeros(plan.total_elems, dtype=torch.bool)
    for t, o in zip(plan.tensors, owner):
        excluded[t.elem_off:t.elem_off + t.numel] = o in EXCLUDED
    for step in range(3):
        g = _fill(plan, gen).to(dtype)
        g[::7] = -0.0
        for e in engs:
            e.grad.copy_(g.cuda())
            e.step()
        torch.cuda.synchronize()
        a, b, free = engs
        tag = f"{mode} {dtype} step {step}"
        assert torch.equal(a.slot().cpu(), b.slot().cpu()), tag
        assert torch.isfinite(a.grad.cpu().float()).all() and torch.isfinite(a.mom.cpu()).all(), tag
        assert torch.equal(_bits(a.resid), _bits(b.resid)) and torch.equal(_bits(a.mom), _bits(b.mom)), tag
        assert torch.equal(_bits(a.grad), _bits(b.grad)), tag
        for x, y in ((a.resid, free.resid), (a.mom, free.mom), (a.grad, free.grad)):
            assert torch.equal(_bits(x)[excluded], _bits(y)[excluded]), tag
    for e in engs:
        e.close()


@pytest.mark.parametrize("config", ["shard", "noshard"])
@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("mode", ["bloom_leftmost", "plain", "randomk", "elias_fano"])
def test_multirank_vs_oracle(monkeypatch, mode, W, config):
    # rank-ordered sums without averaging: the aggregate is the oracle's bit for bit
    monkeypatch.setenv("DR_DETERMINISTIC", "1")
    plan, owner, params0, decays = _setup(mode, torch.float32)
    shard = config == "shard"
    arenas = [torch.zeros(plan.arena_words(W, shard), dtype=torch.int32, device="cuda:0") for _ in range(W)]
    engs = [_RankEngine(plan, arenas, r, momentum=M, nesterov=True, weight_decays=decays, owner=owner, average=False,
                        spin_limit=4_000_000, peer_timeout_ms=5000, shard=shard) for r in range(W)]
    params = [[_placed(p * (1.0 + 0.1 * r), i) for i, p in enumerate(params0)] for r in range(W)]
    for e, ps in zip(engs, params):
        e.bind_parameters(ps, owner)
    gen = torch.Generator().manual_seed(6)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    mom = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in range(1, 4):
        grads = [_fill(plan, gen) for _ in range(W)]
        ws = [_weights(plan, owner, ps) for ps in params]
        for r in range(W):
            engs[r].grad.copy_(grads[r].cuda())
        _run_step(engs, config, epoch)
        out, res, slots, mom = engine_oracle(plan, grads, res, epoch=epoch, average=False, momentum=M, moms=mom,
                                             weights=ws, weight_decays=decays, owner=owner, nesterov=True)
        for r in range(W):
            tag = f"{mode} W={W} {config} epoch {epoch} rank {r}"
            assert not _compare_slot(plan, engs[r].slot(), slots[r], tag), tag
            assert torch.equal(_bits(engs[r].resid), _bits(res[r])), tag
            assert torch.equal(_bits(engs[r].mom), _bits(mom[r])), tag
            assert torch.equal(_bits(engs[r].grad), _bits(out)), tag
        for ps in params:
            _nudge(ps, epoch)
    for e in engs:
        e.close()


class _Own:
    """A compressor whose 'compressed' form is the decoded contribution itself."""

    def decompress(self, c, ctx):
        return c


CFG = {'compressor': 'topk', 'memory': 'dgc', 'momentum': M, 'nesterov': True, 'weight_decay': WD,
       'weight_decay_exclude': ['*.bias', '*bn*'], 'communicator': 'allgather', 'compress_ratio': 0.01,
       'calibrate_partition': False, 'min_numel': 100}


def _excluded(n):
    return n.endswith(".bias") or "bn" in n


def test_ddp_fused_channels_last_resnet20_matches_per_tensor_memory():
    """DeepReduceDDP on CUDA (fused, plain top-k pairs, clipping on) on channels_last ResNet-20 against the per-tensor
    DgcMemory of the GRACE route with the same keys, bit for bit: the memory is fed each parameter's gradient in its
    layout and, as its own contribution, what the engine shipped (at W = 1 the aggregate), and must end with the
    engine's residual and momentum; every shipped value is the memory's compensated value."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel import DeepReduceDDP
    from deepreduce_b200.parallel.ddp import fused_path
    cfg = dict(CFG, clip_norm=0.05)
    assert fused_path(cfg)
    torch.manual_seed(0)
    model = resnet20().cuda().to(memory_format=torch.channels_last)
    named = list(model.named_parameters())
    assert any(not p.is_contiguous() for _, p in named)
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    (eng,) = ddp.engines
    (items,) = ddp.buckets
    assert eng.nesterov and len(items) == len(eng.plan.tensors)
    assert eng.decays == [0.0 if _excluded(n) else WD for n, _ in items]
    mem = DgcMemory(M, WD, 0.05, 1, nesterov=True, weight_decay_exclude=cfg['weight_decay_exclude'])
    mem.bind_parameters(named)
    gen = torch.Generator().manual_seed(1)
    for step in range(3):
        grads = {n: (torch.randn(p.shape, generator=gen) * 1e-3).cuda().contiguous(
                     memory_format=torch.channels_last if p.dim() == 4 else torch.contiguous_format)
                 for n, p in named}
        with torch.no_grad():
            for n, p in named:
                p.grad.copy_(grads[n])                                 # p.grad is the parameter's view of the bucket
        ddp.finish()
        torch.cuda.synchronize()
        for (n, p), t in zip(items, eng.plan.tensors):
            v = mem.compensate(grads[n].clone(), n)
            own = p.grad.detach().clone()
            mem.update(v, n, _Own(), own, None)
            tag = (step, n)
            shipped = own != 0
            assert int(shipped.sum()) > 0 and torch.equal(_bits(own[shipped]), _bits(v[shipped])), tag
            for buf, want in ((eng.resid, mem.residuals[n]), (eng.mom, mem.momenta[n])):
                got = buf[t.elem_off:t.elem_off + t.numel].as_strided(p.size(), p.stride())
                assert torch.equal(_bits(got), _bits(want)), tag
        with torch.no_grad():
            for _, p in named:
                p -= 0.05 * p.grad
    ddp.close()


@pytest.fixture
def nccl_world1():
    import torch.distributed as dist
    f = tempfile.NamedTemporaryFile(delete=False)
    f.close()
    os.unlink(f.name)
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method=f"file://{f.name}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


class _ConvNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = torch.nn.Conv2d(3, 64, 3, padding=1)
        self.bn1 = torch.nn.BatchNorm2d(64)
        self.conv2 = torch.nn.Conv2d(64, 64, 3, padding=1)
        self.fc = torch.nn.Linear(64, 10)

    def forward(self, x):
        x = torch.relu(self.conv2(torch.relu(self.bn1(self.conv1(x)))))
        return self.fc(x.mean(dim=(2, 3)))


def _storage(t):
    """The elements of a dense tensor in storage order."""
    return t.detach().as_strided((t.numel(),), (1,)).float().cpu()


def test_ddp_hook_across_bucket_rebuild(nccl_world1):
    """torch DDP + the DeepReduce hook with both keys on a channels_last conv net: every bucket layout's result equals
    ``engine_oracle`` fed the gradients and parameters in bucket (storage) order, across DDP's bucket rebuild."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    torch.manual_seed(0)
    model = _ConvNet().cuda().to(memory_format=torch.channels_last)
    ddp = DDP(model, device_ids=[0], bucket_cap_mb=0.05)
    st = DeepReduceHookState(CFG, model)
    named = dict(model.named_parameters())
    by_id = {id(p): n for n, p in named.items()}
    local, wseen = {}, {}

    def spy_hook(state, bucket):
        buf = bucket.buffer()
        for p, (d, k) in zip(bucket.parameters(), bucket_segments(bucket)):
            n = by_id[id(p)]
            local[n] = buf[d:d + k].detach().float().cpu().clone()
            wseen[n] = _storage(p)
        return deepreduce_hook(state, bucket)
    ddp.register_comm_hook(st, spy_hook)
    n_layouts = []
    new_layout = st._new_layout

    def spy_layout(*a, **k):
        n_layouts.append(1)
        return new_layout(*a, **k)
    st._new_layout = spy_layout
    u = {n: torch.zeros(p.numel()) for n, p in named.items()}
    r = {n: torch.zeros(p.numel()) for n, p in named.items()}
    gen = torch.Generator(device="cuda").manual_seed(5)
    try:
        for step in range(4):
            for p in model.parameters():
                p.grad = None
            x = torch.randn(4, 3, 8, 8, device="cuda", generator=gen).contiguous(memory_format=torch.channels_last)
            ddp(x).float().pow(2).mean().backward()
            torch.cuda.synchronize()
            st.check()
            for lay in set(st._by_index.values()):
                plan, eng = lay.plan, lay.engine
                decays = [0.0 if _excluded(n) else WD for n in lay.names]
                assert eng.nesterov and eng.decays == tensor_decays(plan, 0.0, decays, eng.owner)
                fg, fr, fu, fw = (torch.zeros(plan.total_elems) for _ in range(4))
                rows = [(by_id[id(p)], p, lay.eng_off[i], k) for i, (p, (_, k)) in enumerate(zip(lay.params, lay.segments))]
                for n, p, off, k in rows:
                    fg[off:off + k], fr[off:off + k], fu[off:off + k], fw[off:off + k] = local[n], r[n], u[n], wseen[n]
                out, res, _, mom = engine_oracle(plan, [fg], [fr], epoch=eng.epoch, momentum=M, moms=[fu],
                                                 weights=[fw], weight_decays=decays, owner=eng.owner, nesterov=True)
                for n, p, off, k in rows:
                    tag = f"step {step} {n}"
                    assert torch.equal(_bits(_storage(p.grad)), _bits(out[off:off + k])), tag
                    assert torch.equal(_bits(lay.resid_of(p)), _bits(res[0][off:off + k])), tag
                    assert torch.equal(_bits(lay.mom_of(p)), _bits(mom[0][off:off + k])), tag
                    r[n], u[n] = res[0][off:off + k].clone(), mom[0][off:off + k].clone()
            with torch.no_grad():
                for p in model.parameters():
                    p -= 0.05 * p.grad
        assert len(n_layouts) >= 2, "DDP's bucket rebuild was not met"
    finally:
        st.close()


def test_warmup_stage_switch_keeps_both_keys(monkeypatch):
    """A sparsity warm-up stage switch builds new engines: they keep Nesterov and the per-parameter decays, and every
    exchange before and after the switch equals the oracle."""
    from deepreduce_b200.parallel import DeepReduceDDP
    seen = []
    orig = BucketEngine.step

    def spy(self, epoch=None):
        seen.append((self, self.grad.detach().cpu().clone(), self.resid.cpu().clone(), self.mom.cpu().clone(),
                     self.parameter_buffer().cpu()))
        orig(self, epoch)
    monkeypatch.setattr(BucketEngine, "step", spy)
    cfg = dict(CFG, warmup_ratios=[0.1, 0.05], warmup_steps=1)
    torch.manual_seed(0)
    model = _ConvNet().cuda()
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    named = list(model.named_parameters())
    gen = torch.Generator(device="cuda").manual_seed(7)
    engines = []
    for step in range(4):
        with torch.no_grad():
            for _, p in named:
                p.grad.copy_(torch.randn(p.shape, device="cuda", generator=gen))
        seen.clear()
        ddp.finish()
        torch.cuda.synchronize()
        assert len(seen) == len(ddp.buckets) == 1
        eng, g, r, u, w = seen[0]
        engines.append(eng)
        assert eng.nesterov and eng.decays == [0.0 if _excluded(n) else WD for n, _ in ddp.buckets[0]]
        out, res, _, mom = engine_oracle(eng.plan, [g], [r], epoch=eng.epoch, momentum=M, moms=[u], weights=[w],
                                         weight_decays=eng.decays, nesterov=True)
        tag = f"step {step} ratio {eng.plan.tensors[0].k}"
        _check(eng, out, res[0], mom[0], tag)
    assert len({id(e) for e in engines}) == 3, "the warm-up did not switch stages"
    for e in ddp.engines:
        assert e.nesterov and any(e.decays) and not all(e.decays)
    ddp.close()


def test_engine_refuses_mixed_decay_factors():
    """The engine takes one decay factor for every parameter, or 0 to exclude one; other per-parameter values raise."""
    plan, owner, params, decays = _setup("plain", torch.float32)
    with pytest.raises(ValueError, match="one factor"):
        BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, owner=owner,
                     weight_decays=[WD * (1 + (i % 2)) for i in range(len(params))])
    with pytest.raises(ValueError):
        BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, owner=owner, weight_decay=WD,
                     weight_decays=decays)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, owner=owner,
                       weight_decays=[0.0] * len(params))                 # everything excluded: nothing is read
    eng.step()
    torch.cuda.synchronize()
    eng.check_status()
    eng.close()
