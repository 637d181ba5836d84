"""'dgc' memory with DGC's local gradient clipping ('clip_norm'): config, the per-tensor DgcMemory against a
hand-written fp64 formula (clipped, untouched, exactly at the threshold, NaN and +-inf, W = 2 and 4), the pairwise
order of the norm, the fused engine's oracle against the per-tensor route, two gloo ranks and checkpoints.  CPU only."""
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from deepreduce_b200 import deepreduce_from_params
from deepreduce_b200.config import KNOWN_KEYS, ConfigError, DeepReduceConfig
from deepreduce_b200.grace import DgcMemory
from deepreduce_b200.grace.memory import pairwise_sumsq
from deepreduce_b200.parallel import BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import clip_oracle, owner_spans
from deepreduce_b200.parallel.plan import split_large

BASE = {'compressor': 'topk', 'memory': 'dgc', 'communicator': 'allgather', 'compress_ratio': 0.05}


def _bits(t):
    return t.detach().float().contiguous().view(torch.int32)


def _formula(g, c, W):
    """The specification in numpy: fp64 squares, zero-padded to 4096 * 2^ceil(log2 ceil(n / 4096)), summed by
    adjacent pairs; thr = c / sqrt(W); where sqrt(sum) is finite and > thr, g * fl32(thr / nrm) in fp32."""
    x = g.detach().numpy().astype(np.float32).reshape(-1).astype(np.float64)
    n = x.size
    tiles = max(1, -(-n // 4096))
    pad = 4096
    while pad < 4096 * tiles:
        pad *= 2
    s = np.zeros(pad)
    s[:n] = x * x
    while s.size > 1:
        s = s[0::2] + s[1::2]
    thr = c / math.sqrt(W)
    nrm = math.sqrt(float(s[0]))
    if math.isfinite(nrm) and nrm > thr:
        f = np.float32(thr / nrm)
        return torch.from_numpy((g.detach().numpy().astype(np.float32) * f).astype(np.float32))
    return g.clone()


def test_config_accepts_and_rejects():
    assert "clip_norm" in KNOWN_KEYS
    for ok in (dict(BASE, clip_norm=1.0), dict(BASE, clip_norm=5), dict(BASE, clip_norm=1e-30),
               dict(BASE, clip_norm=2.0, weight_decay=1e-4, momentum=0.5),
               dict(BASE, compressor='randomk', communicator='allreduce', clip_norm=0.5)):
        assert DeepReduceConfig.from_params(ok, strict=True).memory == 'dgc'
    for bad in (dict(BASE, memory='residual', clip_norm=1.0), dict(BASE, memory='none', clip_norm=1.0),
                {k: v for k, v in dict(BASE, clip_norm=1.0).items() if k != 'memory'},
                dict(BASE, clip_norm=0.0), dict(BASE, clip_norm=0), dict(BASE, clip_norm=-1.0),
                dict(BASE, clip_norm=float('nan')), dict(BASE, clip_norm=float('inf')), dict(BASE, clip_norm=True),
                dict(BASE, clip_norm=False), dict(BASE, clip_norm='1.0'), dict(BASE, clip_norm=None)):
        with pytest.raises(ConfigError):
            DeepReduceConfig.from_params(bad)
    # GRACE's element-wise clamp stays refused, and the refusal names the key that clips
    with pytest.raises(ConfigError, match="clip_norm"):
        DeepReduceConfig.from_params(dict(BASE, gradient_clipping=True))
    mem = deepreduce_from_params(dict(BASE, clip_norm=2.5)).memory
    assert isinstance(mem, DgcMemory) and mem.clip_norm == 2.5 and mem.world_size == 1 and mem.clip_thr == 2.5
    assert deepreduce_from_params(BASE).memory.clip_thr is None


def _cases():
    gen = torch.Generator().manual_seed(0)
    big = torch.randn(10000, generator=gen) * 3.0                        # norm ~300: clipped at every c below
    small = torch.randn(50, generator=gen) * 1e-3                        # norm ~7e-3: untouched
    at_thr = torch.tensor([3.0, 4.0, 0.0, 0.0])                          # norm exactly 5
    nan = big.clone(); nan[17] = float('nan')
    pinf = big.clone(); pinf[3] = float('inf')
    ninf = big.clone(); ninf[9999] = float('-inf')
    return {"big": big, "small": small, "at_thr": at_thr, "nan": nan, "pinf": pinf, "ninf": ninf,
            "matrix": (torch.randn(70, 130, generator=gen) * 0.2), "tiles3": torch.randn(3 * 4096 + 5, generator=gen)}


@pytest.mark.parametrize("W", [1, 2, 4])
def test_dgc_memory_against_formula(W):
    c = 5.0 * math.sqrt(W)                        # thr = 5 at every W: the 3-4-5 tensor sits exactly at it
    for name, g in _cases().items():
        mem = DgcMemory(momentum=0.9, clip_norm=c, world_size=W)
        assert mem.clip_thr == 5.0
        out = mem.compensate(g.clone(), name)     # first step: u = v = the clipped gradient
        ref = _formula(g, c, W)
        assert torch.equal(_bits(out), _bits(ref)), name
        if name in ("small", "at_thr", "nan", "pinf", "ninf"):
            assert torch.equal(_bits(out), _bits(g)), name           # untouched, NaN and inf bits included
        else:
            assert not torch.equal(out, g), name
            assert abs(float(out.double().norm()) - 5.0) < 1e-5, name
    # thr = c / sqrt(W): the same tensor is clipped harder on more ranks
    g = _cases()["big"]
    outs = [DgcMemory(clip_norm=10.0, world_size=w).compensate(g.clone(), "x") for w in (1, 2, 4)]
    assert [round(float(o.double().norm()), 4) for o in outs] == [10.0, round(10.0 / math.sqrt(2), 4), 5.0]


def test_clip_then_weight_decay_then_momentum_three_steps():
    """Per step: g = clip(g), d = g + wd * w, u = m * u + d, v = v + u (the fused engine's order)."""
    from deepreduce_b200.grace.sparsifiers import TopKCompressor
    gen = torch.Generator().manual_seed(1)
    m, wd, c, n = 0.9, 0.01, 2.0, 3000
    w = torch.randn(n, generator=gen)
    grc = deepreduce_from_params(dict(BASE, momentum=m, weight_decay=wd, clip_norm=c))
    grc.memory.bind_parameters([("p", w)])
    comp = TopKCompressor(0.05)
    u = v = None
    for s in range(3):
        g = torch.randn(n, generator=gen) * (0.5 + s)
        grc.step(g.clone(), "p")
        d = _formula(g, c, 1) + wd * w
        if s == 0:
            u = v = d
        else:
            u = m * u + d
            v = v + u
        own = comp.decompress(*comp.compress(v, "p"))
        v = v - own
        u = torch.where(own != 0, torch.zeros_like(u), u)
        assert torch.equal(_bits(grc.memory.residuals["p"]), _bits(v)), s
        assert torch.equal(_bits(grc.memory.momenta["p"]), _bits(u)), s


def test_pairwise_order_decides_the_factor():
    """A tensor whose sequential fp64 sum of squares differs from the pairwise one (one 2^27 and 4095 ones: each 1
    vanishes next to 2^54, but the ones summed among themselves do not), and a c between the two norms' fp32 factors:
    the pairwise order gives the other factor, and the memory follows the pairwise order."""
    x = torch.ones(4096)
    x[0] = 2.0 ** 27
    seq = 0.0
    for v in x.double().tolist():
        seq += v * v
    pair = pairwise_sumsq(x)
    assert seq == 2.0 ** 54 and pair > seq
    # midpoint of two fp32 neighbours, so thr / nrm_seq and thr / nrm_pair round to different fp32 factors
    f_mid = (0.5 + 2.0 ** -25)
    c = f_mid * math.sqrt(0.5 * (seq + pair))
    f_seq, f_pair = np.float32(c / math.sqrt(seq)), np.float32(c / math.sqrt(pair))
    assert f_seq != f_pair
    out = DgcMemory(clip_norm=c).compensate(x.clone(), "x")
    assert torch.equal(_bits(out), _bits(x * torch.tensor(float(f_pair))))
    assert not torch.equal(_bits(out), _bits(x * torch.tensor(float(f_seq))))


def test_channels_last_norm_in_storage_order():
    """A dense non-contiguous gradient (channels_last) is summed in its storage order, the order it has in a flat
    gradient bucket; the clipped values keep its layout."""
    gen = torch.Generator().manual_seed(2)
    g = (torch.randn(16, 8, 5, 5, generator=gen) * 4).contiguous(memory_format=torch.channels_last)
    out = DgcMemory(clip_norm=1.0).compensate(g, "conv")
    flat = g.as_strided((g.numel(),), (1,))
    ref = _formula(flat.clone(), 1.0, 1)
    assert torch.equal(_bits(out.as_strided((g.numel(),), (1,))), _bits(ref))
    assert out.stride() == g.stride()


def test_oracle_clip_spans_split_parameters():
    numels, names, shapes, owner = split_large([20000, 300, 3 * 4096], ["a", "b", "c"], [(20000,), (300,), (12288,)],
                                               8192)
    plan = BucketPlan(numels, names, shapes, index=None)
    spans = owner_spans(plan, owner)
    assert spans[0] == spans[1] == spans[2] == (0, 5) and spans[3] == (5, 1) and spans[4] == spans[5] == (6, 3)
    with pytest.raises(ValueError):
        owner_spans(plan, [0, 1, 0, 2, 3, 3])                            # chunks of one parameter apart
    gen = torch.Generator().manual_seed(3)
    g = torch.zeros(plan.total_elems)
    for v in plan.views(g):
        v.copy_(torch.randn(v.shape, generator=gen))
    out = clip_oracle(plan, g, 3.0, owner)
    vs, os_ = plan.views(g), plan.views(out)
    whole_a = torch.cat([vs[0], vs[1], vs[2]])
    assert torch.equal(_bits(torch.cat([os_[0], os_[1], os_[2]])), _bits(_formula(whole_a, 3.0, 1)))
    assert torch.equal(_bits(os_[3]), _bits(_formula(vs[3], 3.0, 1)))
    # per chunk instead of per parameter would differ
    assert not torch.equal(_bits(os_[0]), _bits(_formula(vs[0], 3.0, 1)))


@pytest.mark.parametrize("m", [0.9, 0.0])
def test_oracle_equals_per_tensor_route(m):
    """engine_oracle with 'clip_norm', weight decay and a split parameter equals the per-tensor GRACE route bit for
    bit over three steps (the threshold sparsifier selects per element, so chunking does not change the selection)."""
    wd, c, thr = 0.01, 4.0, 1.5
    sizes = [20000, 300, 5000]
    numels, names, shapes, owner = split_large(sizes, ["a", "b", "c"], [(n,) for n in sizes], 8192)
    plan = BucketPlan(numels, names, shapes, index=None, sparsifier="threshold", threshold=thr, capacity_ratio=1.0)
    cfg = dict(BASE, compressor='threshold', threshold=thr, momentum=m, weight_decay=wd, clip_norm=c)
    grc = deepreduce_from_params(cfg)
    gen = torch.Generator().manual_seed(4)
    params = [torch.randn(n, generator=gen) for n in sizes]
    grc.memory.bind_parameters(zip(["a", "b", "c"], params))
    w = torch.zeros(plan.total_elems)
    done = [0, 0, 0]
    for t, i in zip(plan.tensors, owner):
        w[t.elem_off:t.elem_off + t.numel] = params[i][done[i]:done[i] + t.numel]
        done[i] += t.numel
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(3):
        grads = [torch.randn(n, generator=gen) * (0.3 + step) for n in sizes]
        g = torch.zeros(plan.total_elems)
        done = [0, 0, 0]
        for t, i in zip(plan.tensors, owner):
            g[t.elem_off:t.elem_off + t.numel] = grads[i][done[i]:done[i] + t.numel]
            done[i] += t.numel
        out, res, _, mom = engine_oracle(plan, [g], res, epoch=step + 1, momentum=m, moms=mom, weight_decay=wd,
                                         weights=[w], clip_norm=c, owner=owner)
        for i, name in enumerate(["a", "b", "c"]):
            ref = grc.step(grads[i].clone(), name)
            js = [j for j, o in enumerate(owner) if o == i]
            got = torch.cat([out[plan.tensors[j].elem_off:plan.tensors[j].elem_off + plan.tensors[j].numel] for j in js])
            r = torch.cat([res[0][plan.tensors[j].elem_off:plan.tensors[j].elem_off + plan.tensors[j].numel]
                           for j in js])
            u = torch.cat([mom[0][plan.tensors[j].elem_off:plan.tensors[j].elem_off + plan.tensors[j].numel]
                           for j in js])
            assert torch.equal(_bits(got), _bits(ref)), (step, name)
            assert torch.equal(_bits(r), _bits(grc.memory.residuals[name])), (step, name)
            assert torch.equal(_bits(u), _bits(grc.memory.momenta[name])), (step, name)
    with pytest.raises(ValueError):
        engine_oracle(plan, [g], res, clip_norm=c)                       # needs the 'dgc' momentum


def test_oracle_thr_scales_with_world():
    plan = BucketPlan([5000, 700], index=None)
    gen = torch.Generator().manual_seed(5)
    W, c = 4, 3.0
    grads = []
    for _ in range(W):
        g = torch.zeros(plan.total_elems)
        for v in plan.views(g):
            v.copy_(torch.randn(v.shape, generator=gen))
        grads.append(g)
    zeros = [torch.zeros(plan.total_elems) for _ in range(W)]
    _, res, _, _ = engine_oracle(plan, grads, zeros, momentum=0.9, moms=zeros, clip_norm=c, average=False)
    _, res_c, _, _ = engine_oracle(plan, [clip_oracle(plan, g, c / 2.0) for g in grads], zeros, momentum=0.9,
                                   moms=zeros, average=False)
    for a, b in zip(res, res_c):
        assert torch.equal(_bits(a), _bits(b))


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
    tr = Trainer(model, cfg, lr=0.05, amp_dtype=None)
    torch.manual_seed(100 + rank)
    x = torch.randn(8, 3, 32, 32)
    y = torch.randint(0, 10, (8,))
    losses = [float(tr.step(x, target=y)) for _ in range(3)]
    flat = torch.cat([p.detach().flatten() for p in model.parameters()])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    # every residual + momentum norm is bounded by what three clipped steps can put there
    u_max = max(float(u.double().norm()) for u in tr.ddp.grc.memory.momenta.values())
    if rank == 0:
        ret["losses"] = losses
        ret["same"] = all(torch.equal(gathered[0], g) for g in gathered)
        ret["thr"] = tr.ddp.grc.memory.clip_thr
        ret["u_max"] = u_max
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_resnet20_world2_gloo_clip():
    mgr = mp.Manager()
    ret = mgr.dict()
    c = 0.05
    cfg = dict(BASE, compress_ratio=0.01, deepreduce='index', index='bloom', momentum=0.9, clip_norm=c)
    mp.spawn(_worker, args=(2, _free_port(), cfg, ret), nprocs=2, join=True)
    assert ret["same"], "ranks diverged"
    assert all(l == l and l < 20 for l in ret["losses"])
    assert ret["thr"] == c / math.sqrt(2)
    assert ret["u_max"] <= (1 + 0.9 + 0.81) * ret["thr"] * (1 + 1e-5)


def _mlp():
    return nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 64), nn.ReLU(), nn.Linear(64, 8))


def test_checkpoint_round_trip_with_and_without_key():
    """'clip_norm' adds no state: a checkpoint of a clipping memory has the keys of one without, and loads into
    memories with and without the key; the clipping memory then continues bit for bit."""
    from deepreduce_b200.parallel import DeepReduceDDP
    cfg = dict(BASE, momentum=0.9, min_numel=100, clip_norm=0.5)
    torch.manual_seed(5)
    model = _mlp()
    ddp = DeepReduceDDP(model, cfg)
    for _ in range(2):
        for p in model.parameters():
            p.grad = torch.randn_like(p)
        ddp.finish()
    st = ddp.state_dict()
    plain = DeepReduceDDP(_mlp(), {k: v for k, v in cfg.items() if k != 'clip_norm'})
    for p in plain.module.parameters():
        p.grad = torch.randn_like(p)
    plain.finish()
    assert set(st["memory"]) == set(plain.state_dict()["memory"])
    plain.load_state_dict(st)
    model2 = _mlp()
    ddp2 = DeepReduceDDP(model2, cfg)
    ddp2.load_state_dict(st)
    ddp.load_state_dict(plain.state_dict())          # a checkpoint taken without the key loads too
    g = {n: torch.randn_like(p) * 3 for n, p in model.named_parameters()}
    for mdl, d in ((model, ddp), (model2, ddp2)):
        for n, p in mdl.named_parameters():
            p.grad = g[n].clone()
        d.finish()
    for (n, p), (_, q) in zip(model.named_parameters(), model2.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
        assert torch.equal(ddp.grc.memory.momenta[n], ddp2.grc.memory.momenta[n])
        assert torch.equal(ddp.grc.memory.residuals[n], ddp2.grc.memory.residuals[n])
