"""'dgc' memory with weight decay inside the momentum ('weight_decay'): config, the per-tensor DgcMemory against the
formula, wd = 0 against today's memory, the fused engine's oracle, two gloo ranks through ``Trainer``, and the
regularisation against dense momentum SGD.  CPU only."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from deepreduce_b200 import deepreduce_from_params
from deepreduce_b200.config import KNOWN_KEYS, ConfigError, DeepReduceConfig
from deepreduce_b200.grace import DgcMemory
from deepreduce_b200.grace.sparsifiers import TopKCompressor
from deepreduce_b200.parallel import BucketPlan, engine_oracle

BASE = {'compressor': 'topk', 'memory': 'dgc', 'communicator': 'allgather', 'compress_ratio': 0.05}


def _bits(t):
    return t.detach().float().contiguous().view(torch.int32)


def test_config_accepts_and_rejects():
    assert "weight_decay" in KNOWN_KEYS
    for ok in (dict(BASE, weight_decay=1e-4), dict(BASE, weight_decay=0), dict(BASE, weight_decay=0.0),
               dict(BASE, weight_decay=5, momentum=0.5), dict(BASE, compressor='randomk', communicator='allreduce',
                                                             weight_decay=1e-4)):
        assert DeepReduceConfig.from_params(ok, strict=True).memory == 'dgc'
    for bad in (dict(BASE, memory='residual', weight_decay=1e-4), dict(BASE, memory='none', weight_decay=1e-4),
                {k: v for k, v in dict(BASE, weight_decay=1e-4).items() if k != 'memory'},
                dict(BASE, weight_decay=-1e-4), dict(BASE, weight_decay=float('nan')),
                dict(BASE, weight_decay=float('inf')), dict(BASE, weight_decay=True), dict(BASE, weight_decay=False),
                dict(BASE, weight_decay='1e-4'), dict(BASE, weight_decay=None)):
        with pytest.raises(ConfigError):
            DeepReduceConfig.from_params(bad)
    mem = deepreduce_from_params(dict(BASE, weight_decay=0.25)).memory
    assert isinstance(mem, DgcMemory) and mem.weight_decay == 0.25
    assert deepreduce_from_params(BASE).memory.weight_decay == 0.0


def _step(grc, g, name):
    return grc.step(g.clone(), name)


def test_dgc_memory_three_step_formula():
    torch.manual_seed(0)
    m, wd, n = 0.9, 0.05, 1000
    grc = deepreduce_from_params(dict(BASE, momentum=m, weight_decay=wd))
    w = torch.randn(n)
    grc.memory.bind_parameters([("w", w)])
    comp = TopKCompressor(0.05)
    u = v = None
    for s in range(3):
        g = torch.randn(n)
        _step(grc, g, "w")
        # the formula, written out: d = g + (wd * w), u = m*u + d, v = v + u, own = decode(encode(v)), v -= own,
        # u[own != 0] = 0; the first step starts from u = v = d
        d = g + (wd * w)
        if s == 0:
            u, v = d.clone(), d.clone()
        else:
            u = (m * u) + d
            v = v + u
        own = comp.decompress(*comp.compress(v, "w"))
        v = v - own
        u = torch.where(own != 0, torch.zeros_like(u), u)
        assert torch.equal(_bits(grc.memory.momenta["w"]), _bits(u)), s
        assert torch.equal(_bits(grc.memory.residuals["w"]), _bits(v)), s
        w = w - 0.01 * own                               # the memory reads the parameter's value at every step
        grc.memory.parameters["w"].copy_(w)


def test_unbound_name_raises():
    grc = deepreduce_from_params(dict(BASE, weight_decay=1e-4))
    grc.memory.bind_parameters([("a", torch.zeros(10))])
    with pytest.raises(KeyError, match="'b'"):
        grc.step(torch.randn(10), "b")
    # without weight decay nothing is read, so nothing has to be bound
    assert _step(deepreduce_from_params(BASE), torch.randn(10), "b").shape == (10,)


def test_zero_weight_decay_is_todays_memory_bitwise():
    torch.manual_seed(1)
    today = deepreduce_from_params(dict(BASE, momentum=0.9))
    zero = deepreduce_from_params(dict(BASE, momentum=0.9, weight_decay=0.0))
    zero.memory.bind_parameters([("t", torch.randn(2000))])
    for s in range(3):
        g = torch.randn(2000)
        g[::7] = -0.0                                     # -0.0 must survive: wd * w is not added at all
        a, b = _step(today, g, "t"), _step(zero, g, "t")
        assert torch.equal(_bits(a), _bits(b)), s
        assert torch.equal(_bits(today.memory.momenta["t"]), _bits(zero.memory.momenta["t"])), s
        assert torch.equal(_bits(today.memory.residuals["t"]), _bits(zero.memory.residuals["t"])), s
        if s == 0:
            assert bool((_bits(zero.memory.momenta["t"])[::7] == _bits(torch.tensor(-0.0))).all())


PLANS = [dict(index="bloom"), dict(index="rle"), dict(index=None), dict(index="bloom", value="qsgd"),
         dict(index=None, sparsifier="randomk")]


@pytest.mark.parametrize("mode", PLANS)
def test_oracle_weight_decay_formula_and_zero(mode):
    torch.manual_seed(2)
    m, wd, W = 0.9, 0.03, 2
    plan = BucketPlan([20000, 5000, 301], compress_ratio=0.02, min_numel=100, **mode)
    pad = torch.ones(plan.total_elems, dtype=torch.bool)
    for t in plan.tensors:
        pad[t.elem_off:t.elem_off + t.numel] = False
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    mom = [torch.zeros(plan.total_elems) for _ in range(W)]
    res0, mom0 = [r.clone() for r in res], [u.clone() for u in mom]
    for e in range(1, 4):
        grads = [torch.randn(plan.total_elems).masked_fill(pad, 0.0) for _ in range(W)]
        grads[0][::11] = -0.0
        weights = [torch.randn(plan.total_elems).masked_fill(pad, 0.0) for _ in range(W)]
        us = [m * mom[r] + (grads[r] + (wd * weights[r])) for r in range(W)]
        accs = [res[r] + us[r] for r in range(W)]
        out, res, slots, mom = engine_oracle(plan, grads, res, epoch=e, momentum=m, moms=mom, weight_decay=wd,
                                             weights=weights)
        # the compensated accumulator equals what the residual memory ships when fed it directly
        ref_out, ref_res, ref_slots = engine_oracle(plan, accs, [torch.zeros(plan.total_elems)] * W, epoch=e)
        assert torch.equal(_bits(out), _bits(ref_out))
        for r in range(W):
            assert torch.equal(_bits(res[r]), _bits(ref_res[r]))
            assert (slots[r] == ref_slots[r]).all()
            off = mom[r] != 0
            assert torch.equal(_bits(mom[r][off]), _bits(us[r][off]))
        # wd = 0 returns exactly what the oracle without the argument returns, weights or not
        a = engine_oracle(plan, grads, res0, epoch=e, momentum=m, moms=mom0)
        b = engine_oracle(plan, grads, res0, epoch=e, momentum=m, moms=mom0, weight_decay=0.0, weights=weights)
        assert torch.equal(_bits(a[0]), _bits(b[0]))
        for r in range(W):
            assert torch.equal(_bits(a[1][r]), _bits(b[1][r])) and torch.equal(_bits(a[3][r]), _bits(b[3][r]))
            assert (a[2][r] == b[2][r]).all()
        res0, mom0 = a[1], a[3]
    with pytest.raises(ValueError):
        engine_oracle(plan, grads, res, weight_decay=wd, weights=weights)            # needs the 'dgc' momentum
    with pytest.raises(ValueError):
        engine_oracle(plan, grads, res, momentum=m, moms=mom, weight_decay=wd)       # needs the parameters


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, cfg, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(0)
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.trainer import Trainer
    model = resnet20()
    tr = Trainer(model, cfg, lr=0.05, amp_dtype=None, weight_decay=1e-4)
    torch.manual_seed(100 + rank)
    x = torch.randn(8, 3, 32, 32)
    y = torch.randint(0, 10, (8,))
    losses = [float(tr.step(x, target=y)) for _ in range(3)]
    flat = torch.cat([p.detach().flatten() for p in model.parameters()])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    if rank == 0:
        ret["losses"] = losses
        ret["same"] = all(torch.equal(gathered[0], g) for g in gathered)
        ret["opt_wd"] = tr.opt.param_groups[0]["weight_decay"]
        ret["opt_momentum"] = tr.opt.param_groups[0]["momentum"]
        ret["mem_wd"] = tr.ddp.grc.memory.weight_decay
        ret["bound"] = len(tr.ddp.grc.memory.parameters)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_resnet20_world2_gloo_weight_decay():
    mgr = mp.Manager()
    ret = mgr.dict()
    cfg = dict(BASE, compress_ratio=0.01, deepreduce='index', index='bloom', momentum=0.9, weight_decay=5e-4)
    mp.spawn(_worker, args=(2, _free_port(), cfg, ret), nprocs=2, join=True)
    assert ret["same"], "ranks diverged"
    assert all(l == l and l < 20 for l in ret["losses"])
    assert ret["opt_wd"] == 0.0 and ret["opt_momentum"] == 0.0
    assert ret["mem_wd"] == 5e-4 and ret["bound"] > 0


def _mlp():
    return nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 64), nn.ReLU(), nn.Linear(64, 8))


def _data(n=512, d=64, classes=8, seed=0):
    gen = torch.Generator().manual_seed(seed)
    centers = torch.randn(classes, d, generator=gen) * 2.0
    y = torch.randint(0, classes, (n,), generator=gen)
    x = centers[y] + torch.randn(n, d, generator=gen)
    return x, y


def test_trainer_optimizer_weight_decay():
    from deepreduce_b200.trainer import Trainer
    for cfg, wd in ((dict(BASE, weight_decay=0.01), 0.0), (BASE, 1e-3),
                    ({'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather'}, 1e-3)):
        tr = Trainer(_mlp(), cfg, lr=0.05, weight_decay=1e-3, amp_dtype=None)
        assert tr.opt.param_groups[0]["weight_decay"] == wd, cfg
        tr.close()


@pytest.mark.timeout(300)
def test_weight_decay_in_memory_tracks_dense_momentum_sgd():
    """The motivation: with the decay in the memory the parameters shrink as under dense momentum SGD with the same
    decay; with the decay in the optimizer (no momentum there) it is about 1 / (1 - m) = 10 times weaker."""
    from deepreduce_b200.trainer import Trainer
    wd, m, lr = 0.02, 0.9, 0.05
    x, y = _data()

    def train(cfg, opt_wd, momentum, steps=150):
        torch.manual_seed(0)
        tr = Trainer(_mlp(), cfg, lr=lr, momentum=momentum, weight_decay=opt_wd, amp_dtype=None)
        for s in range(steps):
            i = (s * 64) % 512
            tr.step(x[i:i + 64], target=y[i:i + 64])
        norm = float(torch.cat([p.detach().flatten() for p in tr.model.parameters()]).norm())
        tr.close()
        return norm

    dense = train({'compressor': 'none', 'memory': 'none', 'communicator': 'allreduce'}, wd, m)
    cfg = dict(BASE, min_numel=100, momentum=m)
    in_memory = train(dict(cfg, weight_decay=wd), wd, m)        # the dict's value wins: the optimizer gets 0
    in_optimizer = train(cfg, wd, m)                              # the optimizer's decay, without its momentum
    assert abs(in_memory - dense) < abs(in_optimizer - dense), (dense, in_memory, in_optimizer)
    assert in_memory < in_optimizer


def test_ddp_hook_per_tensor_route_reads_parameters_in_bucket_order():
    """The DDP hook's per-tensor route hands the memory DDP's gradients as plain reshapes of the flat bucket, which
    holds a channels_last conv weight's gradient in the weight's storage order: the memory must read w in that order
    too.  Checked against the formula on the first step's momentum u = d = g + (wd * w) (u is cleared where it
    was shipped), for a channels_last conv and a contiguous linear layer; then a layout change is refused."""
    import tempfile
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.parallel import DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    f = tempfile.NamedTemporaryFile(delete=False)
    f.close()
    os.unlink(f.name)
    dist.init_process_group("gloo", init_method=f"file://{f.name}", rank=0, world_size=1)
    try:
        torch.manual_seed(0)
        wd = 0.5
        model = nn.Sequential(nn.Conv2d(4, 16, 3), nn.Flatten(), nn.Linear(16 * 4 * 4, 5))
        model = model.to(memory_format=torch.channels_last)
        conv = model[0].weight
        assert not conv.is_contiguous() and conv.is_contiguous(memory_format=torch.channels_last)
        ddp = DDP(model)
        st = DeepReduceHookState(dict(BASE, momentum=0.9, weight_decay=wd, min_numel=10), model)
        named = dict(model.named_parameters())
        by_id = {id(p): n for n, p in named.items()}
        seen = {}

        def spy_hook(state, bucket):
            buf = bucket.buffer()
            for p, (d, k) in zip(bucket.parameters(), bucket_segments(bucket)):
                seen[by_id[id(p)]] = buf[d:d + k].detach().clone()         # the gradient in bucket order
            return deepreduce_hook(state, bucket)
        ddp.register_comm_hook(st, spy_hook)
        x = torch.randn(2, 4, 6, 6).contiguous(memory_format=torch.channels_last)
        ddp(x).pow(2).mean().backward()
        assert st.path(torch.zeros(1)) == "grace"
        for n, p in named.items():
            w = p.detach().as_strided((p.numel(),), (1,))                   # storage order
            d = seen[n] + (wd * w)
            u = st.grc.memory.momenta[n].reshape(-1)
            kept = u != 0
            assert int(kept.sum()) > p.numel() // 2, n
            assert torch.equal(_bits(u[kept]), _bits(d[kept])), n
        # the conv weight moves to another layout after DDP built its buckets: reading it would permute w
        conv.data = conv.data.contiguous()
        with pytest.raises(ValueError, match="layout"):
            st.grc.memory.compensate(torch.zeros(conv.shape), "0.weight")
    finally:
        dist.destroy_process_group()
