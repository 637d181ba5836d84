"""The DDP communication hook (``parallel/comm_hook.py``) without a GPU: routing, the segment tables of real DDP
buckets before and after DDP's bucket rebuild, the torch reference of the repack, the GRACE per-tensor path at W = 2
against ``DeepReduceDDP``'s, and checkpoints that move between bucket sizes."""
import os
import socket
import tempfile
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
from torch.nn.parallel import DistributedDataParallel as DDP

from deepreduce_b200.parallel import BucketPlan, DeepReduceHookState, register_deepreduce_hook
from deepreduce_b200.parallel.comm_hook import (bucket_segments, pack_reference, segment_table, unpack_reference)
from deepreduce_b200.parallel.ddp import fused_path
from deepreduce_b200.parallel.plan import split_large

BLOOM = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.05,
         'deepreduce': 'index', 'index': 'bloom'}


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _mlp():
    torch.manual_seed(0)
    return nn.Sequential(nn.Linear(33, 70), nn.ReLU(), nn.Linear(70, 50), nn.ReLU(), nn.Linear(50, 5), nn.Linear(5, 3))


@pytest.fixture
def gloo_world1():
    f = tempfile.NamedTemporaryFile(delete=False)
    f.close()
    os.unlink(f.name)
    dist.init_process_group("gloo", init_method=f"file://{f.name}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


# ---------------------------------------------------------------------------
# routing
# ---------------------------------------------------------------------------
class _FakeBucket:
    def __init__(self, buf):
        self.buf = buf

    def buffer(self):
        return self.buf

    def index(self):
        return 0

    def is_last(self):
        return True


ROUTES = [
    (BLOOM, "fused", "grace"),
    ({'compressor': 'topk', 'memory': 'residual', 'compress_ratio': 0.01}, "fused", "grace"),
    ({'compressor': 'randomk', 'memory': 'residual', 'compress_ratio': 0.01}, "fused", "grace"),
    ({'compressor': 'threshold', 'threshold': 0.01, 'memory': 'residual'}, "fused", "grace"),
    ({'compressor': 'topk', 'deepreduce': 'index', 'index': 'huffman'}, "grace", "grace"),
    ({'compressor': 'topk', 'deepreduce': 'both', 'index': 'rle'}, "grace", "grace"),
    ({'compressor': 'topk', 'communicator': 'allreduce'}, "grace", "grace"),
    ({'compressor': 'none', 'memory': 'none', 'communicator': 'allreduce'}, "dense", "dense"),
]


@pytest.mark.parametrize("params,on_cuda,on_cpu", ROUTES)
def test_routing(params, on_cuda, on_cpu):
    st = DeepReduceHookState(params, _mlp())
    assert st.path(SimpleNamespace(is_cuda=True)) == on_cuda
    assert st.path(torch.zeros(4)) == on_cpu
    assert (on_cuda == "fused") == (params['compressor'] != 'none' and fused_path(params))


def test_fused_bucket_dtype_raises():
    st = DeepReduceHookState(BLOOM, _mlp())
    with pytest.raises(ValueError, match="fp32 or bf16"):
        st._run(_FakeBucket(SimpleNamespace(is_cuda=True, dtype=torch.float16)))


def test_parameter_outside_module_raises():
    st = DeepReduceHookState(BLOOM, _mlp())
    with pytest.raises(ValueError, match="not one of the module's"):
        st._name(nn.Parameter(torch.zeros(3)))


# ---------------------------------------------------------------------------
# segment tables of real DDP buckets
# ---------------------------------------------------------------------------
def test_segment_tables_across_rebuild(gloo_world1):
    model = _mlp()
    ddp = DDP(model, bucket_cap_mb=0.01)
    seen = []

    def hook(state, bucket):
        buf = bucket.buffer()
        segs = bucket_segments(bucket)
        for (d, n), g in zip(segs, bucket.gradients()):
            assert g.numel() == n and buf[d:].data_ptr() == g.data_ptr()
        # DDP packs the bucket without gaps
        assert sorted(segs)[0][0] == 0 and sum(n for _, n in segs) == buf.numel()
        names = [state[id(p)] for p in bucket.parameters()]
        numels, nm, shapes, owner = split_large([n for _, n in segs], names, [tuple(p.shape) for p in bucket.parameters()],
                                                4096)
        plan = BucketPlan(numels, nm, shapes, index=None)
        table = segment_table(segs, plan, owner)
        assert table.shape == (len(segs), 3)
        for (d, e, n), (d0, n0) in zip(table.tolist(), segs):
            assert (d, n) == (d0, n0) and e % 32 == 0 and e + n <= plan.total_elems
        seen.append((bucket.index(), [id(p) for p in bucket.parameters()], segs))
        fut = torch.futures.Future()
        fut.set_result(buf)
        return fut

    ddp.register_comm_hook({id(p): n for n, p in model.named_parameters()}, hook)
    n_buckets = []
    for it in range(3):
        before = len(seen)
        ddp(torch.randn(4, 33)).sum().backward()
        n_buckets.append(len(seen) - before)
    it0, it1, it2 = (seen[sum(n_buckets[:i]):sum(n_buckets[:i + 1])] for i in range(3))
    assert it0 != it1, "DDP did not rebuild its buckets after the first iteration"
    assert it1 == it2, "the rebuilt layout must stay fixed"
    assert [b[0] for b in it1] == list(range(len(it1)))           # hooks run in bucket-index order


# ---------------------------------------------------------------------------
# the torch reference of the repack
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_reference_repack_round_trip(dtype):
    gen = torch.Generator().manual_seed(3)
    numels = [1, 3, 4097, 1, 70, 2310, 5, 33]
    segs, off = [], 0
    for n in numels:
        segs.append((off, n))
        off += n
    plan = BucketPlan(numels, index=None)
    table = segment_table(segs, plan, list(range(len(numels))))
    ddp = torch.randn(off, generator=gen).to(dtype)
    eng = torch.full((plan.total_elems,), float("nan"), dtype=dtype)
    pack_reference(ddp, eng, table)
    covered = torch.zeros(plan.total_elems, dtype=torch.bool)
    for d, e, n in table.tolist():
        covered[e:e + n] = True
    assert torch.isnan(eng[~covered]).all(), "padding was written"
    back = torch.zeros_like(ddp)
    unpack_reference(eng, back, table)
    assert torch.equal(back, ddp)


# ---------------------------------------------------------------------------
# W = 2 gloo: DDP + hook on the GRACE path == DeepReduceDDP's GRACE path
# ---------------------------------------------------------------------------
def _grace_worker(rank, world, port, cfg, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from deepreduce_b200.parallel import DeepReduceDDP
    a, b = _mlp(), _mlp()
    ddp = DDP(a, bucket_cap_mb=0.01)
    st = register_deepreduce_hook(ddp, cfg)
    ref = DeepReduceDDP(b, cfg)
    oa, ob = torch.optim.SGD(a.parameters(), lr=0.1), torch.optim.SGD(b.parameters(), lr=0.1)
    ok, layouts = True, set()
    for step in range(3):
        x = torch.randn(8, 33, generator=torch.Generator().manual_seed(10 * step + rank))
        ddp(x).pow(2).sum().backward()
        b(x).pow(2).sum().backward()
        ref.finish()
        for (n, p), q in zip(a.named_parameters(), b.parameters()):
            ok = ok and torch.equal(p.grad, q.grad)
        layouts.add(tuple(sorted(st.grc.memory.residuals)))
        oa.step(); ob.step(); oa.zero_grad(); ob.zero_grad()
    flat = torch.cat([p.detach().flatten() for p in a.parameters()])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    if rank == 0:
        ret["ok"] = bool(ok)
        ret["same"] = all(torch.equal(gathered[0], g) for g in gathered)
        ret["path"] = st.path(flat)
        ret["steps"] = st.step_count
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_grace_path_matches_deepreduce_ddp_world2():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_grace_worker, args=(2, _free_port(), BLOOM, ret), nprocs=2, join=True)
    assert ret["path"] == "grace"
    assert ret["ok"], "DDP + hook and DeepReduceDDP disagree on the gradient bits"
    assert ret["same"], "ranks diverged"
    assert ret["steps"] == 3


# ---------------------------------------------------------------------------
# checkpoints keyed by parameter name
# ---------------------------------------------------------------------------
def _step(ddp, step):
    x = torch.randn(8, 33, generator=torch.Generator().manual_seed(step))
    for p in ddp.module.parameters():
        p.grad = None
    ddp(x).pow(2).sum().backward()
    return [p.grad.clone() for p in ddp.module.parameters()]


def test_state_dict_into_other_bucket_cap(gloo_world1):
    a = DDP(_mlp(), bucket_cap_mb=0.01)
    st_a = register_deepreduce_hook(a, BLOOM)
    for s in range(2):
        _step(a, s)
    ckpt = st_a.state_dict()
    assert ckpt["step"] == 2 and set(ckpt["memory"]["residuals"]) == {n for n, _ in a.module.named_parameters()}
    b = DDP(_mlp(), bucket_cap_mb=25)
    st_b = register_deepreduce_hook(b, BLOOM)
    st_b.load_state_dict(ckpt)
    ga, gb = _step(a, 2), _step(b, 2)
    assert all(torch.equal(x, y) for x, y in zip(ga, gb))
    assert st_b.step_count == 3
