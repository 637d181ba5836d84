"""The fused engine's 'dgc' memory (momentum correction + momentum factor masking) on the GPU.

Each step of a 'dgc' engine is checked bit for bit against two references: a residual-memory engine of the same plan
(whose kernels the other GPU tests check against ``engine_oracle``) fed the compensated momentum
u' = fl(fl(m * u) + g), which must produce the same slot, aggregate and residual; and the momentum u' cleared wherever
the rank's own slot decodes (``decode_slot_oracle``) to a non-zero value.  Modes with fp32 values are also checked
against ``engine_oracle(momentum=...)`` directly."""
import pytest
import torch

from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import decode_slot_oracle
from test_engine_multirank import _RankEngine, _run_step
from test_gpu_engine import SIZES, _compare_slot, _fill

pytestmark = pytest.mark.gpu
M = 0.9

MODES = {
    "topk": dict(index=None),
    "threshold": dict(index=None, sparsifier="threshold", threshold=1.5),
    "randomk": dict(index=None, sparsifier="randomk"),
    "randomk_qsgd": dict(index=None, sparsifier="randomk", value="qsgd"),
    "bloom_leftmost": dict(index="bloom"),
    "bloom_random": dict(index="bloom", policy="random", fpr=0.02),
    "bloom_p0": dict(index="bloom", policy="p0"),
    "bloom_p2": dict(index="bloom", policy="conflict_sets"),
    "rle": dict(index="rle"),
    "bloom_polyfit": dict(index="bloom", value="polyfit", poly_min_k=300),
    "bloom_qsgd": dict(index="bloom", value="qsgd"),
    "bloom_dexp": dict(index="bloom", value="dexp"),
    "rle_polyfit": dict(index="rle", value="polyfit", poly_min_k=300),
    "rle_qsgd": dict(index="rle", value="qsgd"),
    "rle_dexp": dict(index="rle", value="dexp"),
    "value_qsgd": dict(index=None, value="qsgd"),
    "value_polyfit": dict(index=None, value="polyfit", poly_min_k=300),
    "value_dexp": dict(index=None, value="dexp"),
}
FP32_VALUES = ("topk", "threshold", "randomk", "bloom_leftmost", "bloom_random", "bloom_p0", "rle")


def _plan(mode, sizes=SIZES):
    return BucketPlan(sizes, compress_ratio=0.01, **MODES[mode])


def _bits(t):
    return t.detach().float().cpu().view(torch.int32)


def _masked(plan, u, slot):
    own = decode_slot_oracle(plan, slot)
    return torch.where(own != 0, torch.zeros_like(u), u)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", list(MODES))
def test_dgc_engine_vs_residual_twin_and_mask(mode, dtype):
    plan = _plan(mode)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, grad_dtype=dtype, spin_limit=2_000_000)
    twin = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000)
    gen = torch.Generator().manual_seed(1)
    u = torch.zeros(plan.total_elems)
    for step in range(4):
        g = (_fill(plan, gen) * (0.3 if step == 2 else 1.0)).to(dtype).float()    # bf16: the widened gradient
        u_new = M * u + g
        eng.grad.copy_(g.to(dtype).cuda())
        twin.grad.copy_(u_new.cuda())
        eng.step()
        twin.step()
        torch.cuda.synchronize()
        eng.check_status()
        twin.check_status()
        tag = f"{mode} {dtype} step {step}"
        assert torch.equal(eng.slot().cpu(), twin.slot().cpu()), tag
        assert torch.equal(_bits(eng.resid), _bits(twin.resid)), tag
        if dtype == torch.float32:
            assert torch.equal(_bits(eng.grad), _bits(twin.grad)), tag
        else:                           # the fp32 aggregate, rounded once
            assert torch.equal(eng.grad.cpu(), twin.grad.cpu().to(torch.bfloat16)), tag
        u = _masked(plan, u_new, eng.slot().cpu())
        assert torch.equal(_bits(eng.mom), _bits(u)), tag
        assert int((u == 0).sum()) > int((u_new == 0).sum()), tag         # something was masked
    eng.close()
    twin.close()


@pytest.mark.parametrize("mode", FP32_VALUES)
def test_dgc_engine_vs_oracle(mode):
    plan = _plan(mode, SIZES + [2359296])
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, spin_limit=2_000_000)
    gen = torch.Generator().manual_seed(2)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(4):
        g = _fill(plan, gen)
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom)
        tag = f"{mode} step {step}"
        assert not _compare_slot(plan, eng.slot(), slots[0], tag), tag
        assert torch.equal(_bits(eng.grad), _bits(out)), tag
        assert torch.equal(_bits(eng.resid), _bits(res[0])), tag
        assert torch.equal(_bits(eng.mom), _bits(mom[0])), tag
    eng.close()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", ["topk", "bloom_leftmost", "bloom_p2", "rle_qsgd", "bloom_polyfit", "randomk"])
def test_zero_momentum_is_residual_engine(mode, dtype):
    plan = _plan(mode)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=0.0, grad_dtype=dtype)
    ref = BucketEngine(plan, device="cuda:0", world=1, rank=0, grad_dtype=dtype)
    gen = torch.Generator().manual_seed(3)
    for step in range(3):
        g = _fill(plan, gen).to(dtype)
        eng.grad.copy_(g.cuda())
        ref.grad.copy_(g.cuda())
        eng.step()
        ref.step()
        torch.cuda.synchronize()
        tag = f"{mode} {dtype} step {step}"
        assert torch.equal(eng.slot().cpu(), ref.slot().cpu()), tag
        assert torch.equal(eng.grad.cpu().view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                           ref.grad.cpu().view(torch.int16 if dtype == torch.bfloat16 else torch.int32)), tag
        assert torch.equal(_bits(eng.resid), _bits(ref.resid)), tag
        u = eng.mom.cpu()
        off = u != 0
        assert torch.equal(u[off], g.float()[off]), tag                    # u = g off the masked set
    eng.close()
    ref.close()


@pytest.mark.parametrize("config", ["shard", "noshard"])
@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("mode", ["bloom_leftmost", "rle_qsgd", "randomk", "topk"])
def test_dgc_multirank_vs_residual_twins(monkeypatch, mode, W, config):
    # rank-ordered decode sums: the default bloom apply adds the senders with RED.ADD in launch-dependent order at
    # W > 2, so two engine groups would differ in the last bits of the aggregate; ordered, with W a power of two, the
    # sum is determined bit for bit (test_engine_multirank.py::_exact_tensor)
    monkeypatch.setenv("DR_DETERMINISTIC", "1")
    plan = _plan(mode, SIZES)
    kw = dict(spin_limit=4_000_000, peer_timeout_ms=5000, shard=config == "shard")
    arenas = [torch.zeros(plan.arena_words(W, kw["shard"]), dtype=torch.int32, device="cuda:0") for _ in range(W)]
    tarenas = [torch.zeros(plan.arena_words(W, kw["shard"]), dtype=torch.int32, device="cuda:0") for _ in range(W)]
    engs = [_RankEngine(plan, arenas, r, momentum=M, **kw) for r in range(W)]
    twins = [_RankEngine(plan, tarenas, r, **kw) for r in range(W)]
    gen = torch.Generator().manual_seed(4)
    us = [torch.zeros(plan.total_elems) for _ in range(W)]
    for epoch in range(1, 5):
        u_new = []
        for r in range(W):
            g = _fill(plan, gen)
            u_new.append(M * us[r] + g)
            engs[r].grad.copy_(g.cuda())
            twins[r].grad.copy_(u_new[r].cuda())
        _run_step(engs, config, epoch)
        _run_step(twins, config, epoch)
        for r in range(W):
            tag = f"{mode} W={W} {config} epoch {epoch} rank {r}"
            assert torch.equal(engs[r].slot().cpu(), twins[r].slot().cpu()), tag
            assert torch.equal(_bits(engs[r].grad), _bits(twins[r].grad)), tag
            assert torch.equal(_bits(engs[r].resid), _bits(twins[r].resid)), tag
            assert torch.equal(_bits(engs[r].grad), _bits(engs[0].grad)), tag            # the ranks agree
            us[r] = _masked(plan, u_new[r], engs[r].slot().cpu())
            assert torch.equal(_bits(engs[r].mom), _bits(us[r])), tag


def test_dgc_engine_state_resume_and_calibration():
    plan = _plan("bloom_leftmost")
    gen = torch.Generator().manual_seed(5)
    gs = [_fill(plan, gen) for _ in range(4)]
    a = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M)
    for g in gs[:2]:
        a.grad.copy_(g.cuda())
        a.step()
    st = a.state_dict()
    assert "mom" in st and bool((st["mom"] != 0).any())
    b = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M)
    b.load_state_dict(st)
    for g in gs[2:]:
        for e in (a, b):
            e.grad.copy_(g.cuda())
            e.step()
        torch.cuda.synchronize()
        for x, y in ((a.grad, b.grad), (a.resid, b.resid), (a.mom, b.mom)):
            assert torch.equal(_bits(x), _bits(y))
        assert torch.equal(a.slot().cpu(), b.slot().cpu())
    # memory kinds do not mix
    plain = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    with pytest.raises(ValueError):
        plain.load_state_dict(st)
    with pytest.raises(ValueError):
        b.load_state_dict(plain.state_dict())
    # the partition calibration runs synthetic steps and leaves u at zero, as it leaves the residual
    b.calibrate_partition(steps=1, rounds=1)
    assert not bool(b.mom.any()) and not bool(b.resid.any())
    for e in (a, b, plain):
        e.close()


@pytest.mark.parametrize("cfg", [
    {'compressor': 'topk', 'communicator': 'allgather', 'deepreduce': 'index', 'index': 'bloom'},
    {'compressor': 'randomk', 'communicator': 'allreduce'},
], ids=["bloom", "randomk_allreduce"])
def test_trainer_resnet20_dgc_fused_vs_oracle(cfg):
    """ResNet-20 through ``Trainer`` with 'dgc' on the fused path: SGD without momentum, and every step's aggregate,
    residual and momentum equal to ``engine_oracle`` fed the gradients the engine received."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel.ddp import fused_path
    from deepreduce_b200.trainer import Trainer
    torch.manual_seed(0)
    cfg = {**cfg, 'memory': 'dgc', 'momentum': M, 'compress_ratio': 0.01, 'calibrate_partition': False}
    assert fused_path(cfg)
    tr = Trainer(resnet20().cuda(), cfg, lr=0.05, amp_dtype=None, overlap=False)
    assert tr.opt.param_groups[0]["momentum"] == 0.0
    (eng,) = tr.ddp.engines
    assert eng.mom is not None
    res, mom = [torch.zeros(eng.plan.total_elems)], [torch.zeros(eng.plan.total_elems)]
    orig = eng.step
    seen = []

    def spy(epoch=None):
        seen.append(eng.grad.detach().cpu().clone())
        orig(epoch)
    eng.step = spy
    gen = torch.Generator(device="cuda").manual_seed(1)
    for step in range(3):
        x = torch.randn(8, 3, 32, 32, device="cuda", generator=gen)
        y = torch.randint(0, 10, (8,), device="cuda", generator=gen)
        tr.step(x, target=y)
        torch.cuda.synchronize()
        out, res, _, mom = engine_oracle(eng.plan, [seen[-1]], res, epoch=eng.epoch, momentum=M, moms=mom)
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


def test_ddp_hook_dgc_across_bucket_rebuild(nccl_world1):
    """torch DDP + the DeepReduce hook with 'dgc', against ``engine_oracle`` per bucket layout: every step's gradients,
    residuals and momenta bit for bit, across DDP's bucket rebuild (the momentum is carried with the residual), and
    the hook's checkpoint holds both by parameter name."""
    from test_gpu_comm_hook import MLP, _inputs
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    torch.manual_seed(0)
    cfg = {'compressor': 'topk', 'memory': 'dgc', 'momentum': M, 'communicator': 'allgather', 'compress_ratio': 0.01,
           'calibrate_partition': False}
    model = MLP().cuda()
    ddp = DDP(model, device_ids=[0], bucket_cap_mb=0.5)
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
    n_layouts = []
    new_layout = st._new_layout

    def spy_layout(*a, **k):
        n_layouts.append(1)
        return new_layout(*a, **k)
    st._new_layout = spy_layout
    u = {n: torch.zeros(p.numel()) for n, p in named.items()}
    r = {n: torch.zeros(p.numel()) for n, p in named.items()}
    try:
        for step in range(4):
            for p in model.parameters():
                p.grad = None
            ddp(_inputs("mlp", step, 0, torch.float32)).float().pow(2).mean().backward()
            torch.cuda.synchronize()
            st.check()
            for lay in set(st._by_index.values()):
                plan = lay.plan
                fg, fr, fu = (torch.zeros(plan.total_elems) for _ in range(3))
                rows = [(by_id[id(p)], p, lay.eng_off[i], k) for i, (p, (_, k)) in enumerate(zip(lay.params, lay.segments))]
                for n, p, off, k in rows:
                    fg[off:off + k], fr[off:off + k], fu[off:off + k] = local[n], r[n], u[n]
                out, res, _, mom = engine_oracle(plan, [fg], [fr], epoch=lay.engine.epoch, momentum=M, moms=[fu])
                for n, p, off, k in rows:
                    tag = f"step {step} {n}"
                    assert torch.equal(_bits(p.grad.flatten()), _bits(out[off:off + k])), tag
                    assert torch.equal(_bits(lay.resid_of(p)), _bits(res[0][off:off + k])), tag
                    assert torch.equal(_bits(lay.mom_of(p)), _bits(mom[0][off:off + k])), tag
                    r[n], u[n] = res[0][off:off + k].clone(), mom[0][off:off + k].clone()
        assert len(n_layouts) >= 2, "DDP's bucket rebuild was not met"
        sd = st.state_dict()
        assert set(sd["momentum"]) == set(sd["residuals"]) == set(named)
        for n in named:
            assert torch.equal(sd["momentum"][n], u[n]) and torch.equal(sd["residuals"][n], r[n])
    finally:
        st.close()
