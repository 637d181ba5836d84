"""The conflict-sets (P2) bloom policy in the fused engine, on the GPU: the sender stage (p2_pick_kernel), the header
words after emit and the receiver's thinning of the probed masks (p2_thin_kernel), against the CPU oracle."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import test_engine_multirank as multirank
from deepreduce_b200 import spec
from deepreduce_b200.codecs.bloom import bloom_query_oracle
from deepreduce_b200.parallel import BucketEngine, BucketPlan, DeepReduceDDP, engine_oracle
from deepreduce_b200.parallel.engine import decode_slot_oracle
from deepreduce_b200.parallel.plan import MODE_BLOOM, auto_split_numel, split_large
from test_gpu_engine import _compare_slot, _fill
from test_train_step_reference import ref_flat, unflatten

pytestmark = pytest.mark.gpu

# ResNet-50-like shapes: a 1x1 conv, a 3x3 conv, a bias below the 1000-element bypass, the fc layer, and layer4's
# 3x3 conv cut by auto_split_numel (for a 16 KB filter stage) into chunks (each chunk its own P2 tensor)
RN50 = [16384, 36864, 147456, 512, 2048000, 2359296]


def _plan(ratio=0.01, split=True, sizes=RN50, **kw):
    if split:
        sizes = split_large(RN50, [f"t{i}" for i in range(len(RN50))], [(n,) for n in RN50],
                            auto_split_numel(ratio, kw.get("fpr"), filter_smem_bytes=16 * 1024))[0]
    return BucketPlan(sizes, compress_ratio=ratio, policy="conflict_sets", **kw)


def _check_p2_words(plan, a, b, tag):
    for t in plan.tensors:
        if t.pos_cap:
            for off, n in ((t.off_pos_prefix, t.n_tiles), (t.off_pick, (t.pos_cap + 31) // 32)):
                assert np.array_equal(a[off:off + n], b[off:off + n]), (tag, t.name, off)


W1_CASES = [(True, 2, torch.float32, None), (False, 2, torch.float32, None), (True, 1, torch.float32, None),
            (False, 1, torch.bfloat16, None), (True, 2, torch.bfloat16, None), (True, 2, torch.float32, "qsgd"),
            (False, 1, torch.float32, "polyfit")]


@pytest.mark.parametrize("tma,bps,dtype,value", W1_CASES)
def test_engine_vs_oracle_w1(tma, bps, dtype, value):
    plan = _plan(value=value, poly_min_k=64)
    assert len(plan.tensors) > len(RN50)                      # the auto split cut at least one tensor
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, use_tma=tma, blocks_per_sm=bps, grad_dtype=dtype)
    resid = torch.zeros(plan.total_elems)
    for step in range(5):
        g = _fill(plan, torch.Generator().manual_seed(step)).to(dtype)
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        tag = f"tma={tma} bps={bps} {dtype} {value} step {step}"
        out, new_res, slots = engine_oracle(plan, [g.float()], [resid], average=True, epoch=eng.epoch)
        resid = new_res[0]
        a = eng.slot().cpu().numpy().view(np.uint32)
        bad = _compare_slot(plan, eng.slot(), slots[0], tag)
        assert not bad, bad
        _check_p2_words(plan, a, slots[0], tag)
        got = eng.grad.cpu()
        if dtype == torch.bfloat16:
            assert torch.equal(got, out.to(torch.bfloat16)), tag
        elif value is None:
            assert torch.equal(got, out), tag
        else:
            assert torch.allclose(got, out, rtol=1e-5, atol=1e-6), tag
        # value codecs: the residual keeps value - decoded value, whose fp32 rounding may differ from the oracle's by ulps
        tol = 1e-6 if value is None else 1e-5 * float(resid.abs().max())
        assert torch.allclose(eng.resid.cpu(), resid, rtol=1e-5, atol=tol), tag
    eng.close()


def test_device_pick_equals_host_conflict_sets():
    """The device draw alone: the pick the engine shipped equals ops.cpu.conflict_sets on the same positives."""
    from deepreduce_b200 import ops
    plan = _plan(hint=False)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    for step in range(3):
        g = _fill(plan, torch.Generator().manual_seed(50 + step))
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        a = eng.slot().cpu().numpy().view(np.uint32)
        for ti, t in enumerate(plan.tensors):
            if t.mode != MODE_BLOOM:
                continue
            words = torch.from_numpy(a[t.off_filter:t.off_filter + t.n_filter_words].view(np.int32).copy())
            pos = bloom_query_oracle(words, t.numel, t.n_hash, t.m_bits)[:t.pos_cap]
            want = ops.cpu.conflict_sets(pos, t.k, t.n_hash, t.m_bits, spec.DEFAULT_SEED,
                                         spec.policy_seed(eng.epoch, t.salt))
            q = np.arange(pos.numel())
            pick = a[t.off_pick:t.off_pick + (t.pos_cap + 31) // 32].astype(np.int64)
            got = pos[torch.from_numpy(((pick[q >> 5] >> (q & 31)) & 1).astype(bool))]
            assert torch.equal(got, want), (step, t.name)
    eng.close()


def test_high_fpr_and_beyond_cap():
    """Most positives false (fpr 0.3, one hash), and a tensor whose positives run past pos_cap."""
    plan = _plan(fpr=0.3, max_hash=1, hint=False, split=False, sizes=RN50[:4] + [589824])
    big = max(range(len(plan.tensors)), key=lambda i: plan.tensors[i].numel)
    plan.tensors[big].pos_cap = plan.tensors[big].k + 100
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    resid = torch.zeros(plan.total_elems)
    for step in range(3):
        g = _fill(plan, torch.Generator().manual_seed(70 + step))
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, new_res, slots = engine_oracle(plan, [g], [resid], average=True, epoch=eng.epoch)
        resid = new_res[0]
        assert not _compare_slot(plan, eng.slot(), slots[0], step)
        _check_p2_words(plan, eng.slot().cpu().numpy().view(np.uint32), slots[0], step)
        assert torch.equal(eng.grad.cpu(), out), step
        st = eng.stats()
        assert st["tensors"][big]["beyond_cap"] > 0
        assert st["total"]["n_pos"] > 3 * st["total"]["n_sel"]
    eng.close()


MR = pytest.param
MR_CASES = [
    MR("shard", 2, None, False, torch.float32, id="shard-W2"),
    MR("shard", 3, None, True, torch.float32, id="shard-W3-det"),
    MR("shard", 4, "qsgd", False, torch.float32, id="shard-W4-qsgd"),
    MR("shard", 8, None, False, torch.bfloat16, id="shard-W8-bf16"),
    MR("noshard", 3, None, False, torch.float32, id="noshard-W3"),
    MR("noshard", 2, "polyfit", True, torch.bfloat16, id="noshard-W2-polyfit-det-bf16"),
    MR("nccl", 4, None, False, torch.float32, id="nccl-W4"),
    MR("nccl", 3, "qsgd", True, torch.bfloat16, id="nccl-W3-qsgd-det-bf16"),
]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,W,value,deterministic,dtype", MR_CASES)
def test_multirank_vs_oracle(monkeypatch, config, W, value, deterministic, dtype):
    monkeypatch.setenv("DR_DETERMINISTIC", "1" if deterministic else "0")
    plan = _plan(value=value, poly_min_k=64)
    kw = dict(average=True, spin_limit=4_000_000, peer_timeout_ms=5000, grad_dtype=dtype)
    if config == "nccl":
        engs = [BucketEngine(plan, device="cuda:0", world=W, rank=r, transport="nccl", **kw) for r in range(W)]
    else:
        arenas = [torch.zeros(plan.arena_words(W, config == "shard"), dtype=torch.int32, device="cuda:0") for _ in range(W)]
        engs = [multirank._RankEngine(plan, arenas, r, shard=config == "shard", **kw) for r in range(W)]
    resid = [torch.zeros(plan.total_elems) for _ in range(W)]
    for step in range(3):
        epoch = step + 1
        grads = [_fill(plan, torch.Generator().manual_seed(100 * step + r)).to(dtype).float() for r in range(W)]
        for e, g in zip(engs, grads):
            e.grad.copy_(g.to(dtype).cuda())
        multirank._run_step(engs, config, epoch)
        tag = f"{config} W{W} {value} det={deterministic} {dtype} step {step}"
        out, resid, slots = engine_oracle(plan, grads, resid, average=True, epoch=epoch)
        for r, e in enumerate(engs):
            assert not _compare_slot(plan, e.slot(r), slots[r], (tag, r))
            _check_p2_words(plan, e.slot(r).cpu().numpy().view(np.uint32), slots[r], (tag, r))
            for s in range(W):                                     # every arena holds every sender's slot
                assert torch.equal(e.slot(s).cpu(), engs[s].slot(s).cpu()), (tag, r, s)
        # the aggregate against the decode of the slots actually shipped (sum order: rank-major)
        dec = torch.zeros(plan.total_elems)
        for s in range(W):
            dec += decode_slot_oracle(plan, engs[0].slot(s)) * (1.0 / W)
        outs = [e.grad.cpu() for e in engs]
        for r in range(1, W):
            assert torch.equal(outs[r].view(torch.int16) if dtype == torch.bfloat16 else outs[r].view(torch.int32),
                               outs[0].view(torch.int16) if dtype == torch.bfloat16 else outs[0].view(torch.int32)), (tag, r)
        tol = 1e-6 * float(dec.abs().max())
        if dtype == torch.bfloat16:
            assert torch.allclose(outs[0].float(), dec, rtol=2.0 ** -7, atol=tol), tag
        else:
            assert torch.allclose(outs[0], dec, rtol=1e-6, atol=tol), tag
            if value is None:
                assert torch.allclose(outs[0], out, rtol=1e-6, atol=tol), tag
    for e in engs:
        e.close()


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(64, 512)
        self.b = nn.Linear(512, 512)
        self.c = nn.Linear(512, 10)

    def forward(self, x):
        return self.c(torch.relu(self.b(torch.relu(self.a(x)))))


@pytest.mark.parametrize("dr", ["index", "both"])
def test_ddp_two_buckets_scheduler(dr):
    """DeepReduceDDP with the key: fused, several buckets through the background Scheduler, against plain torch + the oracle;
    without the key the same params take the per-tensor path."""
    cfg = {'compressor': 'topk', 'compress_ratio': 0.01, 'memory': 'residual', 'communicator': 'allgather',
           'deepreduce': dr, 'index': 'bloom', 'value': 'qsgd', 'policy': 'conflict_sets', 'calibrate_partition': False}
    torch.manual_seed(0)
    model, ref = _Net().cuda(), _Net().cuda()
    ref.load_state_dict(model.state_dict())
    assert not DeepReduceDDP(_Net().cuda(), dict(cfg), overlap=False).fused
    ddp = DeepReduceDDP(model, dict(cfg, p2_pick_mask=True), bucket_cap_mb=0.5, overlap=True)
    assert ddp.fused and len(ddp.engines) >= 2
    opt, ref_opt = torch.optim.SGD(model.parameters(), lr=0.1), torch.optim.SGD(ref.parameters(), lr=0.1)
    resid = [torch.zeros(e.plan.total_elems) for e in ddp.engines]
    gen = torch.Generator(device="cuda").manual_seed(1)
    for step in range(3):
        x = torch.randn(32, 64, device="cuda", generator=gen)
        y = torch.randint(0, 10, (32,), device="cuda", generator=gen)
        ddp.zero_grad()
        nn.functional.cross_entropy(model(x), y).backward()
        ddp.finish()
        ref_opt.zero_grad()
        nn.functional.cross_entropy(ref(x), y).backward()
        grads = {}
        for b, (eng, items) in enumerate(zip(ddp.engines, ddp.buckets)):
            names = dict(ref.named_parameters())
            params = {n: names[n] for n, _ in items}
            flat = ref_flat(eng.plan, params, {n: q.grad for n, q in params.items()})
            out, new_res, _ = engine_oracle(eng.plan, [flat], [resid[b]], average=True, epoch=eng.epoch)
            resid[b] = new_res[0]
            assert torch.allclose(eng.grad.cpu(), out, rtol=1e-6, atol=1e-7), (step, b)
            grads.update(unflatten(eng.plan, params, eng.grad.cpu()))
        for n, q in ref.named_parameters():
            q.grad = grads[n].cuda()
        opt.step()
        ref_opt.step()
        for p, q in zip(model.parameters(), ref.parameters()):
            assert torch.equal(p, q), step
    ddp.close()
