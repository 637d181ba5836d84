"""QSGD and polyfit values over the fused run-length index ('fused_rle_values') on the GPU, against the oracle.

W = 1 through ``test_gpu_engine._run_vs_oracle`` (fp32) and a bf16-bucket loop; W = 2 ... 16 through the one-GPU W-rank
harness of ``test_engine_multirank`` (sharded, unsharded, the NCCL transport, rank-ordered and RED.ADD sums); and the
public entry points: the benchmark's ResNet-50 and NCF training steps, the DDP communication hook across DDP's bucket
rebuild, and a checkpoint round trip."""
import os
import tempfile

import pytest
import torch
import torch.distributed as dist

import bench
import test_engine_multirank as multirank
import test_gpu_comm_hook as hook
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.plan import DYN_WORDS, MODE_RLE, SLOT_HEADER_WORDS
from test_gpu_engine import SIZES, _compare_slot, _fill, _run_vs_oracle
from test_train_step_reference import run_case

pytestmark = pytest.mark.gpu

BIG = SIZES + [2359296]
CODECS = {"qsgd8": dict(value="qsgd"), "qsgd16": dict(value="qsgd", quantum_num=1000), "polyfit": dict(value="polyfit")}


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("tma,bps", [(True, 2), (False, 2), (True, 1)])
def test_single_rank_vs_oracle(codec, tma, bps):
    """W = 1 (emit scatters nothing that is value-coded, so the run-length apply runs on the own slot), three epochs,
    the second through the unfused phase chain: slots against the oracle, output and residual within the value
    codecs' tolerances."""
    kw = dict(CODECS[codec])
    value = kw.pop("value")
    for kind in ("randn", "sparse"):
        _run_vs_oracle(kind, "rle", "leftmost", True, tma, value, bps=bps, **kw)


@pytest.mark.parametrize("codec,threshold", [("qsgd8", 0.0), ("qsgd16", 0.0), ("polyfit", 1.0)])
def test_single_rank_threshold_full_capacity(codec, threshold):
    """The threshold sparsifier with the slot provisioned for every element: at threshold 0 every non-zero of a tile is
    shipped (4096 run-length entries in one tile).  The slot is checked against the oracle; the output against the
    decode of the engine's own slot, and the residual against accumulated - output, because with every element shipped
    the few QSGD levels that a different norm summation order flips are each one whole quantum of the output."""
    from deepreduce_b200.parallel.engine import decode_slot_oracle
    plan = BucketPlan(BIG, index="rle", poly_min_k=300, sparsifier="threshold", threshold=threshold, capacity_ratio=1.0,
                      **CODECS[codec])
    assert max(t.val_cap for t in plan.tensors) == 2359296
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000)
    gen = torch.Generator().manual_seed(6)
    resid = torch.zeros(plan.total_elems)
    for step in range(3):
        g = _fill(plan, gen) * (0.2 if step == 2 else 1.0)
        acc = resid + g
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        _, _, slots = engine_oracle(plan, [g], [resid], epoch=eng.epoch)
        bad = _compare_slot(plan, eng.slot(), slots[0], f"rle_threshold_{codec}_s{step}")
        assert not bad, bad[:4]
        out, resid = eng.grad.cpu(), eng.resid.cpu().clone()
        sc = float(acc.abs().max())
        assert torch.allclose(out, decode_slot_oracle(plan, eng.slot()), rtol=0, atol=1e-6 * sc), step
        assert torch.allclose(resid + out, acc, rtol=0, atol=1e-6 * sc), step
        if threshold == 0.0:                     # every non-zero of the largest tensor is shipped
            t = plan.tensors[-1]
            n_sel = int(slots[0][SLOT_HEADER_WORDS + DYN_WORDS * (len(plan.tensors) - 1)])
            assert n_sel == int((acc[t.elem_off:t.elem_off + t.numel] != 0).sum()), step
    eng.close()


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("bps", [2, 1])
def test_single_rank_bf16_bucket(codec, bps):
    """bf16 gradient buckets: the engine computes what an fp32 engine fed the widened gradient computes, and rounds the
    aggregate once."""
    plan = BucketPlan(BIG, compress_ratio=0.01, index="rle", poly_min_k=300, **CODECS[codec])
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000, blocks_per_sm=bps,
                       grad_dtype=torch.bfloat16)
    gen = torch.Generator().manual_seed(4)
    resid_ref = torch.zeros(plan.total_elems)
    for step in range(3):
        g = (_fill(plan, gen) * (0.2 if step == 2 else 1.0)).bfloat16()
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out_ref, new_res, slots = engine_oracle(plan, [g.float()], [resid_ref], epoch=eng.epoch)
        bad = _compare_slot(plan, eng.slot(), slots[0], f"rle_bf16_{codec}_{bps}_s{step}")
        assert not bad, bad[:4]
        sc = float(out_ref.abs().max())
        assert torch.allclose(eng.grad.float().cpu(), out_ref, atol=2e-3 * sc, rtol=1e-2), step
        assert torch.allclose(eng.resid.cpu(), new_res[0], atol=2e-3 * sc, rtol=1e-2), step
        resid_ref = eng.resid.cpu().clone()
    eng.close()


C = pytest.param
# (configuration, W, sizes, codec, DR_DETERMINISTIC, average, rank with an all-zero gradient, claims)
MR_CASES = [
    C("shard", 2, BIG, "qsgd8", False, True, 1, {"rle", "qsgd8"}, id="shard-qsgd8-W2-fast"),
    C("shard", 2, SIZES, "polyfit", True, True, None, {"rle", "polyfit"}, id="shard-polyfit-W2-det"),
    C("shard", 3, SIZES, "polyfit", False, True, 0, {"rle", "polyfit", "split"}, id="shard-polyfit-W3-fast"),
    C("shard", 3, SIZES, "qsgd16", True, True, None, {"rle", "qsgd16", "split"}, id="shard-qsgd16-W3-det"),
    C("shard", 4, SIZES, "qsgd8", True, False, 2, {"rle", "qsgd8"}, id="shard-qsgd8-W4-det-sum"),
    C("shard", 4, SIZES, "qsgd16", False, True, None, {"rle", "qsgd16"}, id="shard-qsgd16-W4-fast"),
    C("shard", 8, multirank.SMALL, "qsgd8", False, True, 3, {"rle", "qsgd8", "empty"}, id="shard-small-qsgd8-W8-fast"),
    C("shard", 8, multirank.SMALL, "qsgd16", True, True, None, {"rle", "qsgd16", "empty"}, id="shard-small-qsgd16-W8-det"),
    C("shard", 16, multirank.SMALL, "qsgd8", True, True, None, {"rle", "qsgd8", "empty"}, id="shard-small-qsgd8-W16-det"),
    C("shard", 16, multirank.SMALL, "qsgd16", False, True, 5, {"rle", "qsgd16", "empty"},
      id="shard-small-qsgd16-W16-fast"),
    C("noshard", 3, SIZES, "polyfit", False, True, None, {"rle", "polyfit"}, id="noshard-polyfit-W3-fast"),
    C("noshard", 2, SIZES, "qsgd8", True, False, 0, {"rle", "qsgd8"}, id="noshard-qsgd8-W2-det-sum"),
    C("noshard", 4, SIZES, "qsgd16", False, True, 1, {"rle", "qsgd16"}, id="noshard-qsgd16-W4-fast"),
    C("nccl", 3, SIZES, "qsgd8", True, True, 2, {"rle", "qsgd8"}, id="nccl-qsgd8-W3-det"),
    C("nccl", 2, SIZES, "polyfit", False, True, None, {"rle", "polyfit"}, id="nccl-polyfit-W2-fast"),
    C("nccl", 4, SIZES, "qsgd16", False, False, None, {"rle", "qsgd16"}, id="nccl-qsgd16-W4-fast-sum"),
]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,W,sizes,codec,deterministic,average,zero_rank,claims", MR_CASES)
def test_multirank_vs_oracle(monkeypatch, config, W, sizes, codec, deterministic, average, zero_rank, claims):
    """W ranks on one GPU: slots and residuals against ``engine_oracle``, delivery of every slot, the aggregate against
    the decode of the shipped slots, identical bits on every rank and (sharded) the stage-2 lists.  A rank with an
    all-zero gradient ships no value at all (n_sel = 0 in every header) next to senders at capacity."""
    kw = dict(index="rle", poly_min_k=300, **CODECS[codec])
    multirank.test_engine_multirank_vs_oracle(monkeypatch, config, W, sizes, kw, deterministic, average, zero_rank,
                                              claims)


RLE_QSGD = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
            'deepreduce': 'both', 'index': 'rle', 'value': 'qsgd', 'fused_rle_values': True}


def _rle_coded(tr):
    assert tr.ddp.fused and tr.ddp.grc is None
    ts = [t for e in tr.ddp.engines for t in e.plan.tensors]
    assert any(t.mode == MODE_RLE and t.vmode for t in ts)


@pytest.mark.timeout(900)
def test_resnet50_train_step(monkeypatch):
    """ResNet-50, batch 16, the benchmark's ``Trainer`` with rle + QSGD against plain torch + ``engine_oracle``."""
    monkeypatch.setitem(bench.CONFIGS, "rle_qsgd", dict(RLE_QSGD))
    run_case(monkeypatch, "image", "rle_qsgd", 16, check=_rle_coded)


@pytest.mark.timeout(600)
def test_ncf_train_step(monkeypatch):
    """NCF, top-k 0.1 % + run-length index + polyfit values (the benchmark's NCF config with a value codec)."""
    monkeypatch.setitem(bench.CONFIGS, "rle_polyfit", {**bench.CONFIGS["rle"], 'deepreduce': 'both', 'value': 'polyfit',
                                                       'fused_rle_values': True})
    run_case(monkeypatch, "ncf", "rle_polyfit", 4096, check=_rle_coded)


@pytest.fixture
def nccl_world1():
    f = tempfile.NamedTemporaryFile(delete=False)
    f.close()
    os.unlink(f.name)
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method=f"file://{f.name}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("value", ["qsgd", "polyfit"])
def test_ddp_hook_resnet20(monkeypatch, nccl_world1, value):
    """torch DDP + the communication hook on ResNet-20, four steps across DDP's bucket rebuild, against the oracle."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel.ddp import plan_kwargs_from_params
    name = f"rle_{value}"
    # 5 %: ResNet-20's largest convs ship more than poly_min_k values, so polyfit is on the wire too
    cfg = {**hook.CONFIGS["rle"], 'compress_ratio': 0.05, 'deepreduce': 'both', 'value': value, 'fused_rle_values': True}
    plan = BucketPlan([p.numel() for p in resnet20().parameters()], **plan_kwargs_from_params(cfg))
    assert any(t.mode == MODE_RLE and t.vmode for t in plan.tensors)
    monkeypatch.setitem(hook.CONFIGS, name, cfg)
    st = hook.run_ddp_case(name, "resnet20")
    assert st.fused_params


def test_checkpoint_round_trip():
    """A DeepReduceDDP checkpoint of the fused route holds the engines' state; a fresh wrapper that loads it continues
    bit for bit."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel import DeepReduceDDP

    def make():
        torch.manual_seed(0)
        m = resnet20().cuda()
        return m, DeepReduceDDP(m, dict(RLE_QSGD), bucket_cap_mb=0.5, overlap=False)

    def step(m, ddp, i):
        x = torch.randn(8, 3, 32, 32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(i))
        m.zero_grad()
        m(x).float().pow(2).mean().backward()
        ddp.finish()
        torch.cuda.synchronize()
        ddp.check()
        return [p.grad.clone() for p in m.parameters()]

    ma, a = make()
    assert a.fused and len(a.engines) > 1
    for i in range(2):
        step(ma, a, i)
    ckpt = a.state_dict()
    assert "engines" in ckpt
    mb, b = make()
    b.load_state_dict(ckpt)
    for i in (2, 3):
        ga, gb = step(ma, a, i), step(mb, b, i)
        assert all(torch.equal(x, y) for x, y in zip(ga, gb)), i
    for e, f in zip(a.engines, b.engines):
        assert torch.equal(e.resid, f.resid) and e.epoch == f.epoch
    a.close(); b.close()
