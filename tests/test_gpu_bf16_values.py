"""bf16 values on the wire ('value': 'bf16', vmode 4) in the fused engine, on the GPU.

Every slot word is checked against ``engine_oracle`` (the encode oracle) bit for bit, and at W = 1 so are the output,
the residual and the 'dgc' momentum: emit rounds each value as it gathers it, so nothing here is approximate.  W = 2-4
run in one process through the multi-rank harness of ``test_engine_multirank.py``."""
import numpy as np
import pytest
import torch

from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import decode_slot_oracle
from test_engine_multirank import _engines, _run_step
from test_gpu_engine import SIZES, _compare_slot, _fill

pytestmark = pytest.mark.gpu
M = 0.9

INDEX = {"plain": dict(index=None), "bloom": dict(index="bloom"),
         "bloom_random": dict(index="bloom", policy="random", fpr=0.02), "bloom_p0": dict(index="bloom", policy="p0"),
         "bloom_p2": dict(index="bloom", policy="conflict_sets"), "rle": dict(index="rle")}
SPARSIFIER = {"topk": dict(), "threshold": dict(sparsifier="threshold", threshold=1.0, capacity_ratio=0.2)}
CASES = [(i, s) for i in INDEX for s in SPARSIFIER if not (i == "bloom_p2" and s == "threshold")] + [("randomk", None)]


def _plan(index, sparsifier, sizes=SIZES):
    if index == "randomk":
        return BucketPlan(sizes, compress_ratio=0.01, index=None, sparsifier="randomk", value="bf16")
    return BucketPlan(sizes, compress_ratio=0.01, value="bf16", **INDEX[index], **SPARSIFIER[sparsifier])


def _bits(t):
    return t.detach().float().cpu().view(torch.int32)


def _same_payload(plan, slot_gpu, slot_ref, tag):
    a = slot_gpu.cpu().numpy().view(np.uint32)[:plan.payload_words]
    if not np.array_equal(a, slot_ref[:plan.payload_words]):
        bad = _compare_slot(plan, slot_gpu, slot_ref, tag)
        where = np.nonzero(a != slot_ref[:plan.payload_words])[0]
        raise AssertionError(f"{tag}: {where.size} slot words differ, first at {where[:8].tolist()}; {bad[:4]}")


@pytest.mark.parametrize("memory", ["residual", "dgc"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("index,sparsifier", CASES)
def test_engine_vs_oracle_w1(index, sparsifier, dtype, memory):
    plan = _plan(index, sparsifier)
    assert sum(t.vmode == 4 for t in plan.tensors) >= 4
    dgc = memory == "dgc"
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, grad_dtype=dtype, spin_limit=2_000_000,
                       momentum=M if dgc else None)
    gen = torch.Generator().manual_seed(11)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(3):
        g = (_fill(plan, gen) * (1e-3 if step == 1 else 1.0)).to(dtype).float()
        eng.grad.copy_(g.to(dtype).cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        if dgc:
            out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom)
        else:
            out, res, slots = engine_oracle(plan, [g], res, epoch=eng.epoch)
        tag = f"{index} {sparsifier} {dtype} {memory} step {step}"
        _same_payload(plan, eng.slot(), slots[0], tag)
        if dtype == torch.float32:
            assert torch.equal(_bits(eng.grad), _bits(out)), tag
        else:
            assert torch.equal(eng.grad.cpu(), out.to(torch.bfloat16)), tag
        assert torch.equal(_bits(eng.resid), _bits(res[0])), tag
        if dgc:
            assert torch.equal(_bits(eng.mom), _bits(mom[0])), tag
        assert bool((res[0] != 0).any())
    eng.close()


@pytest.mark.parametrize("index", ["plain", "bloom", "rle"])
def test_engine_edge_values_w1(index):
    """Planted values at the rounding rule's branch points: ties, subnormals that round to 0 and to the smallest bf16
    subnormal, just below and above the overflow point, and +-inf, with the 'dgc' memory."""
    plan = BucketPlan([8192, 5000], ks=[64, 50], value="bf16", **INDEX[index])
    edge = np.array([0x00004000, 0x80007FFF, 0x00008001, 0x3F808000, 0x3F818000, 0x7F7F7FFF, 0x7F7F8000, 0xFF7F8000,
                     0x7F800000, 0xFF800000, 0x7F7FFFFF], dtype=np.uint32)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, spin_limit=2_000_000)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    gen = torch.Generator().manual_seed(12)
    t1 = plan.tensors[1]
    for step in range(2):
        # fewer non-zeros than K: every planted value is shipped (the select never ships an exact zero)
        g = torch.zeros(plan.total_elems)
        pos = torch.randperm(8192, generator=gen)[:edge.size + 40]
        g[pos[:edge.size]] = torch.from_numpy(edge.view(np.float32).copy())
        g[pos[edge.size:]] = torch.randn(40, generator=gen)
        g[t1.elem_off:t1.elem_off + t1.numel] = torch.randn(t1.numel, generator=gen)
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom)
        tag = f"{index} step {step}"
        _same_payload(plan, eng.slot(), slots[0], tag)
        assert torch.equal(_bits(eng.grad), _bits(out)), tag
        assert torch.equal(_bits(eng.resid), _bits(res[0])), tag
        assert torch.equal(_bits(eng.mom), _bits(mom[0])), tag
    eng.close()


@pytest.mark.parametrize("index,W,config", [
    ("plain", 2, "shard"), ("plain", 3, "noshard"), ("bloom", 2, "noshard"), ("bloom", 3, "shard"),
    ("bloom", 4, "shard"), ("bloom_p0", 4, "noshard"), ("rle", 3, "shard"), ("rle", 4, "noshard"),
    ("randomk", 2, "shard"), ("randomk", 4, "noshard")])
def test_multirank(monkeypatch, index, W, config):
    """Rank-ordered sums (DR_DETERMINISTIC=1) without averaging are the oracle's aggregate bit for bit; the default
    RED.ADD apply is within a few roundings of it and identical on every rank."""
    plan = _plan(index, "topk")
    gen = torch.Generator().manual_seed(13 + W)
    for det in (True, False):
        monkeypatch.setenv("DR_DETERMINISTIC", "1" if det else "0")
        engs = _engines(plan, W, config, average=not det)
        res = [torch.zeros(plan.total_elems) for _ in range(W)]
        for epoch in range(1, 4):
            grads = [_fill(plan, gen) for _ in range(W)]
            for r in range(W):
                engs[r].grad.copy_(grads[r].cuda())
            _run_step(engs, config, epoch)
            out, res, slots = engine_oracle(plan, grads, res, epoch=epoch, average=not det)
            for r in range(W):
                tag = f"{index} W={W} {config} det={det} epoch {epoch} rank {r}"
                _same_payload(plan, engs[r].slot(), slots[r], tag)
                assert torch.equal(_bits(engs[r].resid), _bits(res[r])), tag
                assert torch.equal(_bits(engs[r].grad), _bits(engs[0].grad)), tag        # the ranks agree
            if det:
                assert torch.equal(_bits(engs[0].grad), _bits(out)), tag
            else:
                mag = sum(decode_slot_oracle(plan, s).abs() for s in slots) / W
                err = (engs[0].grad.cpu() - out).abs()
                assert bool((err <= 4 * W * 2.0 ** -24 * mag + 1e-30).all()), (tag, float(err.max()))
        for e in engs:
            e.close()


def test_trainer_step_vs_oracle():
    """ResNet-20 through ``Trainer`` with rle + bf16 values on the fused path: every step's aggregate and residual
    equal to ``engine_oracle`` fed the gradients the engine received."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel.ddp import fused_path
    from deepreduce_b200.trainer import Trainer
    torch.manual_seed(0)
    cfg = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
           'deepreduce': 'both', 'index': 'rle', 'value': 'bf16', 'calibrate_partition': False}
    assert fused_path(cfg)
    tr = Trainer(resnet20().cuda(), cfg, lr=0.05, amp_dtype=None, overlap=False)
    (eng,) = tr.ddp.engines
    assert any(t.vmode == 4 for t in eng.plan.tensors)
    res = [torch.zeros(eng.plan.total_elems)]
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
        out, res, _ = engine_oracle(eng.plan, [seen[-1]], res, epoch=eng.epoch)
        assert torch.equal(_bits(eng.grad), _bits(out)), step
        assert torch.equal(_bits(eng.resid), _bits(res[0])), step
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


def test_ddp_hook_across_bucket_rebuild(nccl_world1):
    """torch DDP + the DeepReduce hook with bloom + bf16 values, against ``engine_oracle`` per bucket layout: every
    step's gradients and residuals bit for bit, across DDP's bucket rebuild."""
    from test_gpu_comm_hook import MLP, _inputs
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    torch.manual_seed(0)
    cfg = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
           'deepreduce': 'both', 'index': 'bloom', 'value': 'bf16', 'calibrate_partition': False}
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
                assert any(t.vmode == 4 for t in plan.tensors)
                fg, fr = torch.zeros(plan.total_elems), torch.zeros(plan.total_elems)
                rows = [(by_id[id(p)], p, lay.eng_off[i], k) for i, (p, (_, k)) in enumerate(zip(lay.params, lay.segments))]
                for n, p, off, k in rows:
                    fg[off:off + k], fr[off:off + k] = local[n], r[n]
                out, res, _ = engine_oracle(plan, [fg], [fr], epoch=lay.engine.epoch)
                for n, p, off, k in rows:
                    tag = f"step {step} {n}"
                    assert torch.equal(_bits(p.grad.flatten()), _bits(out[off:off + k])), tag
                    assert torch.equal(_bits(lay.resid_of(p)), _bits(res[0][off:off + k])), tag
                    r[n] = res[0][off:off + k].clone()
        assert len(n_layouts) >= 2, "DDP's bucket rebuild was not met"
    finally:
        st.close()
