"""The fused engine's 'dgc' memory with weight decay on the GPU: phase 0 reads the parameters and adds
fl(wd * w) to the gradient ahead of the momentum.

In every fused mode a weight-decay engine is checked bit for bit against a 'dgc' engine without weight decay fed
d = fl(g + fl(wd * w)) computed in torch, and where ``engine_oracle``'s values are exact (fp32 and bf16 values) against
``engine_oracle(weight_decay=..., weights=...)`` directly.  The parameters have tensors whose numel is not a multiple
of 4, chunks of split parameters, and storage that is not 16-byte aligned."""
import pytest
import torch

from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.plan import split_large
from test_engine_multirank import _RankEngine, _run_step
from test_gpu_engine import SIZES, _compare_slot, _fill

pytestmark = pytest.mark.gpu
M, WD = 0.9, 0.05

MODES = {
    "topk": dict(index=None),
    "threshold": dict(index=None, sparsifier="threshold", threshold=1.5),
    "randomk": dict(index=None, sparsifier="randomk"),
    "bloom_leftmost": dict(index="bloom"),
    "bloom_random": dict(index="bloom", policy="random", fpr=0.02),
    "bloom_p0": dict(index="bloom", policy="p0"),
    "bloom_p2": dict(index="bloom", policy="conflict_sets"),
    "rle": dict(index="rle"),
    "rle_qsgd": dict(index="rle", value="qsgd"),
    "bloom_polyfit": dict(index="bloom", value="polyfit", poly_min_k=300),
    "bloom_dexp": dict(index="bloom", value="dexp"),
    "value_dexp": dict(index=None, value="dexp"),
    "bloom_bf16": dict(index="bloom", value="bf16"),
    "randomk_bf16": dict(index=None, sparsifier="randomk", value="bf16"),
}
EXACT = ("topk", "threshold", "randomk", "bloom_leftmost", "bloom_random", "bloom_p0", "rle", "bloom_bf16",
         "randomk_bf16")


def _bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


def _setup(mode, dtype, split=False, sizes=SIZES, seed=0):
    """Plan, owner and parameters of the bucket: every other parameter starts one element past an aligned address
    (4 bytes for fp32, 2 for bf16), so its vector loads fall back to element loads; ``split`` cuts the parameters
    larger than two tiles into 8192-element chunks."""
    numels, names, shapes, owner = split_large(sizes, [f"t{i}" for i in range(len(sizes))], [(n,) for n in sizes],
                                               8192 if split else None)
    plan = BucketPlan(numels, names, shapes, compress_ratio=0.01, **MODES[mode])
    gen = torch.Generator().manual_seed(seed)
    return plan, owner, [_placed(torch.randn(n, generator=gen).to(dtype).cuda(), i) for i, n in enumerate(sizes)]


def _placed(w, i):
    """w itself for even i; for odd i a copy that starts one element past an aligned address."""
    if i % 2 == 0:
        return w
    buf = torch.empty(w.numel() + 1, dtype=w.dtype, device=w.device)
    buf[1:].copy_(w)
    return buf[1:]


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


@pytest.mark.parametrize("split", [False, True], ids=["whole", "split"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", list(MODES))
def test_weight_decay_engine_vs_decay_free_twin(mode, dtype, split):
    plan, owner, params = _setup(mode, dtype, split)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, weight_decay=WD, grad_dtype=dtype,
                       spin_limit=2_000_000)
    eng.bind_parameters(params, owner)
    twin = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, spin_limit=2_000_000)
    gen = torch.Generator().manual_seed(1)
    for step in range(3):
        g = _fill(plan, gen).to(dtype).float()
        w = _weights(plan, owner, params)
        assert torch.equal(_bits(eng.parameter_buffer()), _bits(w))
        eng.grad.copy_(g.to(dtype).cuda())
        twin.grad.copy_((g + (WD * w)).cuda())            # d = fl(g + fl(wd * w)), fp32
        eng.step()
        twin.step()
        torch.cuda.synchronize()
        eng.check_status()
        twin.check_status()
        tag = f"{mode} {dtype} split={split} step {step}"
        assert torch.equal(eng.slot().cpu(), twin.slot().cpu()), tag
        assert torch.equal(_bits(eng.resid), _bits(twin.resid)), tag
        assert torch.equal(_bits(eng.mom), _bits(twin.mom)), tag
        if dtype == torch.float32:
            assert torch.equal(_bits(eng.grad), _bits(twin.grad)), tag
        else:                           # the fp32 aggregate, rounded once
            assert torch.equal(eng.grad.cpu(), twin.grad.cpu().to(torch.bfloat16)), tag
        _nudge(params, step)
    eng.close()
    twin.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", EXACT)
def test_weight_decay_engine_vs_oracle(mode, dtype):
    split = True                          # the parameters past two tiles as 8192-element chunks, the others whole
    plan, owner, params = _setup(mode, dtype, split)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, weight_decay=WD, grad_dtype=dtype,
                       spin_limit=2_000_000)
    eng.bind_parameters(params, owner)
    gen = torch.Generator().manual_seed(2)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(3):
        g = _fill(plan, gen).to(dtype).float()
        w = _weights(plan, owner, params)
        eng.grad.copy_(g.to(dtype).cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom, weight_decay=WD,
                                             weights=[w])
        tag = f"{mode} {dtype} split={split} step {step}"
        assert not _compare_slot(plan, eng.slot(), slots[0], tag), tag
        if dtype == torch.float32:
            assert torch.equal(_bits(eng.grad), _bits(out)), tag
        else:
            assert torch.equal(eng.grad.cpu(), out.to(torch.bfloat16)), tag
        assert torch.equal(_bits(eng.resid), _bits(res[0])), tag
        assert torch.equal(_bits(eng.mom), _bits(mom[0])), tag
        _nudge(params, step)
    eng.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", ["topk", "bloom_leftmost", "bloom_p2", "rle_qsgd", "bloom_polyfit", "randomk",
                                  "bloom_bf16"])
def test_zero_weight_decay_is_todays_engine(mode, dtype):
    plan, owner, params = _setup(mode, dtype)
    zero = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, weight_decay=0.0, grad_dtype=dtype)
    zero.bind_parameters(params, owner)
    ref = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, grad_dtype=dtype)
    gen = torch.Generator().manual_seed(3)
    ibits = torch.int16 if dtype == torch.bfloat16 else torch.int32
    for step in range(3):
        g = _fill(plan, gen).to(dtype)
        g[::5] = -0.0                                    # -0.0 stays -0.0: nothing is added at wd = 0
        for e in (zero, ref):
            e.grad.copy_(g.cuda())
            e.step()
        torch.cuda.synchronize()
        tag = f"{mode} {dtype} step {step}"
        assert torch.equal(zero.slot().cpu(), ref.slot().cpu()), tag
        assert torch.equal(zero.grad.cpu().view(ibits), ref.grad.cpu().view(ibits)), tag
        assert torch.equal(_bits(zero.resid), _bits(ref.resid)), tag
        assert torch.equal(_bits(zero.mom), _bits(ref.mom)), tag
    zero.close()
    ref.close()


def test_engine_refuses_unbound_and_foreign_parameters():
    plan, owner, params = _setup("topk", torch.float32, True)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, weight_decay=WD)
    with pytest.raises(RuntimeError, match="bind_parameters"):
        eng.step()
    with pytest.raises(ValueError):
        eng.bind_parameters([p.bfloat16() for p in params], owner)          # not the bucket's dtype
    with pytest.raises(ValueError):
        eng.bind_parameters([p.cpu() for p in params], owner)               # not on the engine's device
    with pytest.raises(ValueError):
        eng.bind_parameters(params[:-1], owner[:-1])                        # does not cover the plan
    flat = [torch.randn(n, device="cuda") for n in (64, 72)]
    eng2 = BucketEngine(BucketPlan([64, 72], index=None), device="cuda:0", world=1, rank=0, momentum=M,
                        weight_decay=WD)
    with pytest.raises(ValueError, match="dense"):
        eng2.bind_parameters([flat[0], torch.randn(144, device="cuda")[::2]])         # every other element
    eng2.bind_parameters(flat)
    with pytest.raises(ValueError):
        BucketEngine(plan, device="cuda:0", world=1, rank=0, weight_decay=WD)          # needs the 'dgc' momentum
    # a parameter that moves to another layout after it was bound (e.g. model.to(memory_format=...) after the buckets
    # were built): the bucket keeps its gradient in the old storage order, so the next step refuses to read it
    conv = torch.randn(8, 4, 3, 3, device="cuda").contiguous(memory_format=torch.channels_last)
    eng3 = BucketEngine(BucketPlan([conv.numel()], index=None), device="cuda:0", world=1, rank=0, momentum=M,
                        weight_decay=WD)
    eng3.bind_parameters([conv])
    conv.data = conv.data.clone()                        # moved, same layout: rebound silently
    eng3.step()
    conv.data = conv.data.contiguous()                   # moved to another layout
    with pytest.raises(ValueError, match="layout"):
        eng3.step()
    torch.cuda.synchronize()
    for e in (eng, eng2, eng3):
        e.close()


@pytest.mark.parametrize("config", ["shard", "noshard"])
@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("mode", ["bloom_leftmost", "topk", "randomk", "rle"])
def test_weight_decay_multirank_vs_oracle(monkeypatch, mode, W, config):
    # rank-ordered sums without averaging: the aggregate is the oracle's bit for bit (test_gpu_bf16_values.py)
    monkeypatch.setenv("DR_DETERMINISTIC", "1")
    plan, owner, params0 = _setup(mode, torch.float32, True)
    shard = config == "shard"
    arenas = [torch.zeros(plan.arena_words(W, shard), dtype=torch.int32, device="cuda:0") for _ in range(W)]
    engs = [_RankEngine(plan, arenas, r, momentum=M, weight_decay=WD, average=False, spin_limit=4_000_000,
                        peer_timeout_ms=5000, shard=shard) for r in range(W)]
    # every rank holds its own copy of the parameters (replicas in training; here they differ, which checks that each
    # rank reads its own)
    params = [[_placed(p * (1.0 + 0.1 * r), i) for i, p in enumerate(params0)] for r in range(W)]
    for e, ps in zip(engs, params):
        e.bind_parameters(ps, owner)
    gen = torch.Generator().manual_seed(4)
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    mom = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in range(1, 4):
        grads = [_fill(plan, gen) for _ in range(W)]
        ws = [_weights(plan, owner, ps) for ps in params]
        for r in range(W):
            engs[r].grad.copy_(grads[r].cuda())
        _run_step(engs, config, epoch)
        out, res, slots, mom = engine_oracle(plan, grads, res, epoch=epoch, average=False, momentum=M, moms=mom,
                                             weight_decay=WD, weights=ws)
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


def test_trainer_resnet20_weight_decay_fused_vs_oracle():
    """ResNet-20 through ``Trainer`` with 'dgc' + 'weight_decay' on the fused path: SGD without momentum and without
    weight decay, and every step's aggregate, residual and momentum equal to ``engine_oracle`` fed the gradients the
    engine received and the parameters as they were at the exchange."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel.ddp import fused_path
    from deepreduce_b200.trainer import Trainer
    torch.manual_seed(0)
    cfg = {'compressor': 'topk', 'communicator': 'allgather', 'deepreduce': 'index', 'index': 'bloom',
           'memory': 'dgc', 'momentum': M, 'weight_decay': WD, 'compress_ratio': 0.01, 'calibrate_partition': False}
    assert fused_path(cfg)
    tr = Trainer(resnet20().cuda(), cfg, lr=0.05, amp_dtype=None, overlap=False, weight_decay=1e-4)
    assert tr.opt.param_groups[0]["momentum"] == 0.0 and tr.opt.param_groups[0]["weight_decay"] == 0.0
    (eng,) = tr.ddp.engines
    assert eng.weight_decay == WD
    (items,) = tr.ddp.buckets
    assert len(items) == len(eng.plan.tensors)                       # nothing split: one plan tensor per parameter
    res, mom = [torch.zeros(eng.plan.total_elems)], [torch.zeros(eng.plan.total_elems)]
    orig = eng.step
    seen = []

    def spy(epoch=None):
        w = torch.zeros(eng.plan.total_elems)
        for (_, p), t in zip(items, eng.plan.tensors):
            w[t.elem_off:t.elem_off + t.numel] = p.detach().cpu().reshape(-1)
        seen.append((eng.grad.detach().cpu().clone(), w))
        orig(epoch)
    eng.step = spy
    gen = torch.Generator(device="cuda").manual_seed(1)
    for step in range(3):
        x = torch.randn(8, 3, 32, 32, device="cuda", generator=gen)
        y = torch.randint(0, 10, (8,), device="cuda", generator=gen)
        tr.step(x, target=y)
        torch.cuda.synchronize()
        g, w = seen[-1]
        out, res, _, mom = engine_oracle(eng.plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom, weight_decay=WD,
                                         weights=[w])
        assert torch.equal(_bits(eng.grad), _bits(out)), step
        assert torch.equal(_bits(eng.resid), _bits(res[0])), step
        assert torch.equal(_bits(eng.mom), _bits(mom[0])), step
    tr.close()


@pytest.fixture
def nccl_world1():
    import os
    import tempfile
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
        self.conv2 = torch.nn.Conv2d(64, 64, 3, padding=1)
        self.fc = torch.nn.Linear(64, 10)

    def forward(self, x):
        x = torch.relu(self.conv2(torch.relu(self.conv1(x))))
        return self.fc(x.mean(dim=(2, 3)))


def _storage(t):
    """The elements of a dense tensor in storage order."""
    return t.detach().as_strided((t.numel(),), (1,)).float().cpu()


def test_ddp_hook_weight_decay_channels_last_and_moved_storage(nccl_world1):
    """torch DDP + the DeepReduce hook with 'dgc' + 'weight_decay' on a channels_last conv net, against
    ``engine_oracle`` per bucket layout, across DDP's bucket rebuild; between two steps every parameter's storage is
    replaced (``p.data = ...``) and the next step must read the new values."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    torch.manual_seed(0)
    cfg = {'compressor': 'topk', 'memory': 'dgc', 'momentum': M, 'weight_decay': WD, 'communicator': 'allgather',
           'compress_ratio': 0.01, 'calibrate_partition': False, 'min_numel': 100}
    model = _ConvNet().cuda().to(memory_format=torch.channels_last)
    assert not model.conv2.weight.is_contiguous()
    ddp = DDP(model, device_ids=[0], bucket_cap_mb=0.05)
    st = DeepReduceHookState(cfg, model)
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
    old = []
    gen = torch.Generator(device="cuda").manual_seed(5)
    try:
        for step in range(4):
            if step == 2:
                for p in model.parameters():
                    old.append(p.data)                   # keep the old storage alive: a stale read would see it
                    p.data = p.data.clone() * 0.5
            for p in model.parameters():
                p.grad = None
            x = torch.randn(4, 3, 8, 8, device="cuda", generator=gen).contiguous(memory_format=torch.channels_last)
            ddp(x).float().pow(2).mean().backward()
            torch.cuda.synchronize()
            st.check()
            for lay in set(st._by_index.values()):
                plan = lay.plan
                fg, fr, fu, fw = (torch.zeros(plan.total_elems) for _ in range(4))
                rows = [(by_id[id(p)], p, lay.eng_off[i], k) for i, (p, (_, k)) in enumerate(zip(lay.params, lay.segments))]
                for n, p, off, k in rows:
                    fg[off:off + k], fr[off:off + k], fu[off:off + k], fw[off:off + k] = local[n], r[n], u[n], wseen[n]
                out, res, _, mom = engine_oracle(plan, [fg], [fr], epoch=lay.engine.epoch, momentum=M, moms=[fu],
                                                 weight_decay=WD, weights=[fw])
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
