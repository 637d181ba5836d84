"""'dgc' memory (momentum correction + momentum factor masking, Deep Gradient Compression): config, the per-tensor
DgcMemory against the formula, m = 0 against the residual memory, the fused engine's oracle, checkpoints, two gloo
ranks, and convergence against dense momentum SGD.  CPU only."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from deepreduce_b200 import deepreduce_from_params, spec
from deepreduce_b200.config import ConfigError, DeepReduceConfig
from deepreduce_b200.grace import DgcMemory, ResidualMemory
from deepreduce_b200.grace.sparsifiers import TopKCompressor
from deepreduce_b200.parallel import BucketPlan, engine_oracle

BASE = {'compressor': 'topk', 'memory': 'dgc', 'communicator': 'allgather', 'compress_ratio': 0.05}


def test_config_accepts_and_rejects():
    for ok in (BASE, dict(BASE, momentum=0.0), dict(BASE, momentum=0.99), dict(BASE, momentum=0),
               dict(BASE, compressor='randomk', communicator='allreduce'), dict(BASE, gradient_clipping=False),
               dict(BASE, deepreduce='index', index='bloom')):
        assert DeepReduceConfig.from_params(ok, strict=True).memory == 'dgc'
    for bad in (dict(BASE, memory='residual', momentum=0.9), dict(BASE, memory='none', momentum=0.9),
                dict(BASE, compressor='none', communicator='allreduce'), dict(BASE, beta=0.5), dict(BASE, gamma=2.0),
                dict(BASE, gradient_clipping=True), dict(BASE, momentum=1.0), dict(BASE, momentum=-0.1),
                dict(BASE, momentum='0.9'), dict(BASE, momentum=True), {**BASE, 'memory': 'momentum'}):
        with pytest.raises(ConfigError):
            DeepReduceConfig.from_params(bad)
    assert isinstance(deepreduce_from_params(dict(BASE, momentum=0.5)).memory, DgcMemory)
    assert deepreduce_from_params(dict(BASE, momentum=0.5)).memory.momentum == 0.5
    assert deepreduce_from_params(BASE).memory.momentum == 0.9


def _step(grc, g, name):
    return grc.step(g.clone(), name)


def test_dgc_memory_three_step_formula():
    torch.manual_seed(0)
    m, n = 0.9, 1000
    grc = deepreduce_from_params(dict(BASE, momentum=m))
    comp = TopKCompressor(0.05)
    u = v = None
    for s in range(3):
        g = torch.randn(n)
        _step(grc, g, "w")
        # the formula, written out: u = m*u + g, v = v + u, own = decode(encode(v)), v -= own, u[own != 0] = 0
        if s == 0:
            u, v = g.clone(), g.clone()
        else:
            u = (m * u) + g
            v = v + u
        own = comp.decompress(*comp.compress(v, "w"))
        v = v - own
        u = torch.where(own != 0, torch.zeros_like(u), u)
        assert torch.equal(grc.memory.momenta["w"], u) and torch.equal(grc.memory.residuals["w"], v)
        assert int((u == 0).sum()) >= spec.topk_k(n, 0.05)      # the shipped coordinates lost their momentum


def test_dgc_masking_skips_zero_decoded_values():
    # QSGD: a level of 0 decodes to 0.0, so the coordinate keeps its momentum although its index was shipped
    torch.manual_seed(1)
    m = 0.5
    grc = deepreduce_from_params(dict(BASE, momentum=m, deepreduce='value', value='qsgd', quantum_num=2,
                                      min_numel=100))
    g1, g2 = torch.randn(4096), torch.randn(4096)
    _step(grc, g1, "q")
    u1 = grc.memory.momenta["q"].clone()
    _step(grc, g2, "q")
    u2 = m * u1 + g2
    kept = grc.memory.momenta["q"] != 0
    assert torch.equal(grc.memory.momenta["q"][kept], u2[kept])
    # some selected coordinates decoded to 0 (level 0): u keeps its value there, so more than numel - K survive
    assert int(kept.sum()) > 4096 - spec.topk_k(4096, 0.05), "no shipped coordinate decoded to 0"

    # top-k padding: fewer non-zeros than K, the padding (index 0, value 0.0) must not clear u[0]
    grc = deepreduce_from_params(dict(BASE, compress_ratio=0.25, momentum=0.5))
    _step(grc, torch.tensor([0.5, 4.0, 3.0, 0, 0, 0, 0, 0]), "p")     # ships 1 and 2: u = r = [0.5, 0, ...]
    assert grc.memory.momenta["p"].tolist() == [0.5, 0, 0, 0, 0, 0, 0, 0]
    _step(grc, torch.tensor([-0.75, 0, 0, 2.0, 0, 0, 0, 0]), "p")     # u = [-0.5, 0, 0, 2], v = [0, 0, 0, 2]
    assert grc.memory.momenta["p"].tolist() == [-0.5, 0, 0, 0, 0, 0, 0, 0]
    assert grc.memory.residuals["p"].tolist() == [0.0] * 8
    out = _step(grc, torch.tensor([0, 1.0, 0, 0, 0, 0, 0, 0]), "p")   # u = [-0.25, 1], v = u: both shipped
    assert out.tolist() == [-0.25, 1.0, 0, 0, 0, 0, 0, 0]
    assert grc.memory.momenta["p"].tolist() == [0.0] * 8


@pytest.mark.parametrize("extra", [
    {}, dict(compressor='threshold', threshold=0.5), dict(compressor='randomk'),
    dict(deepreduce='index', index='bloom'), dict(deepreduce='index', index='rle'),
    dict(deepreduce='both', index='bloom', value='polyfit'), dict(deepreduce='value', value='qsgd'),
])
def test_zero_momentum_is_residual_bitwise(extra):
    torch.manual_seed(2)
    res = deepreduce_from_params(dict(BASE, memory='residual', min_numel=100, **extra))
    dgc = deepreduce_from_params(dict(BASE, momentum=0.0, min_numel=100, **extra))
    assert isinstance(res.memory, ResidualMemory)
    for s in range(3):
        for name, n in (("a", 3000), ("b", 700)):
            g = torch.randn(n)
            assert torch.equal(_step(res, g, name), _step(dgc, g, name)), (extra, s, name)
            assert torch.equal(res.memory.residuals[name], dgc.memory.residuals[name])
            u = dgc.memory.momenta[name]
            assert torch.equal(u[u != 0], g[u != 0])                 # u = g off the masked set


PLANS = [dict(index="bloom"), dict(index="bloom", policy="p0"), dict(index="bloom", policy="random"),
         dict(index="rle"), dict(index=None), dict(index="bloom", value="polyfit", poly_min_k=64),
         dict(index="bloom", value="qsgd"), dict(index=None, sparsifier="randomk")]


@pytest.mark.parametrize("mode", PLANS)
def test_oracle_zero_momentum_is_residual_oracle(mode):
    torch.manual_seed(3)
    plan = BucketPlan([30000, 5000, 300], compress_ratio=0.02, min_numel=100, **mode)
    W = 2
    res_r = [torch.zeros(plan.total_elems) for _ in range(W)]
    res_d = [torch.zeros(plan.total_elems) for _ in range(W)]
    mom = [torch.zeros(plan.total_elems) for _ in range(W)]
    for e in range(1, 4):
        grads = [torch.randn(plan.total_elems) for _ in range(W)]
        out_r, res_r, slots_r = engine_oracle(plan, grads, res_r, epoch=e)
        out_d, res_d, slots_d, mom = engine_oracle(plan, grads, res_d, epoch=e, momentum=0.0, moms=mom)
        assert torch.equal(out_r, out_d)
        for r in range(W):
            assert torch.equal(res_r[r], res_d[r])
            assert (slots_r[r] == slots_d[r]).all()
            off = mom[r] != 0
            assert torch.equal(mom[r][off], grads[r][off])


def test_oracle_momentum_formula():
    torch.manual_seed(4)
    m = 0.9
    plan = BucketPlan([20000, 400], compress_ratio=0.01, min_numel=100, index="bloom")
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for e in range(1, 4):
        g = torch.randn(plan.total_elems)
        u = m * mom[0] + g
        acc = res[0] + u
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=e, momentum=m, moms=mom)
        own = out                                            # W = 1, averaged over one rank: the own decode
        assert torch.equal(res[0] + own, acc)
        assert torch.equal(mom[0], torch.where(own != 0, torch.zeros_like(u), u))


def _mlp():
    return nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 64), nn.ReLU(), nn.Linear(64, 8))


def test_ddp_checkpoint_round_trip():
    from deepreduce_b200.parallel import DeepReduceDDP
    cfg = dict(BASE, momentum=0.9, min_numel=100)
    torch.manual_seed(5)
    model = _mlp()
    ddp = DeepReduceDDP(model, cfg)
    for _ in range(2):
        for p in model.parameters():
            p.grad = torch.randn_like(p)
        ddp.finish()
    st = ddp.state_dict()
    assert set(st["memory"]["momenta"]) == set(st["memory"]["residuals"]) == {n for n, _ in model.named_parameters()}
    model2 = _mlp()
    ddp2 = DeepReduceDDP(model2, cfg)
    ddp2.load_state_dict(st)
    g = {n: torch.randn_like(p) for n, p in model.named_parameters()}
    for mdl, d in ((model, ddp), (model2, ddp2)):
        for n, p in mdl.named_parameters():
            p.grad = g[n].clone()
        d.finish()
    for (n, p), (_, q) in zip(model.named_parameters(), model2.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
        assert torch.equal(ddp.grc.memory.momenta[n], ddp2.grc.memory.momenta[n])
        assert torch.equal(ddp.grc.memory.residuals[n], ddp2.grc.memory.residuals[n])
    # a residual memory's state does not load into a dgc memory
    with pytest.raises(ValueError):
        DgcMemory().load_state_dict(ResidualMemory().state_dict())


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
    if rank == 0:
        ret["losses"] = losses
        ret["same"] = all(torch.equal(gathered[0], g) for g in gathered)
        ret["opt_momentum"] = tr.opt.param_groups[0]["momentum"]
        ret["moms"] = len(tr.ddp.grc.memory.momenta)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_resnet20_world2_gloo_dgc():
    mgr = mp.Manager()
    ret = mgr.dict()
    cfg = dict(BASE, compress_ratio=0.01, deepreduce='index', index='bloom', momentum=0.9)
    mp.spawn(_worker, args=(2, _free_port(), cfg, ret), nprocs=2, join=True)
    assert ret["same"], "ranks diverged"
    assert all(l == l and l < 20 for l in ret["losses"])
    assert ret["opt_momentum"] == 0.0 and ret["moms"] > 0


def _data(n=512, d=64, classes=8, seed=0):
    gen = torch.Generator().manual_seed(seed)
    centers = torch.randn(classes, d, generator=gen) * 2.0
    y = torch.randint(0, classes, (n,), generator=gen)
    x = centers[y] + torch.randn(n, d, generator=gen)
    return x, y


@pytest.mark.timeout(300)
def test_dgc_tracks_dense_momentum_sgd_per_tensor():
    from deepreduce_b200.trainer import Trainer

    def train(cfg, momentum, steps=150):
        torch.manual_seed(0)
        tr = Trainer(_mlp(), cfg, lr=0.05, momentum=momentum, weight_decay=0.0, amp_dtype=None)
        x, y = _data()
        losses = [float(tr.step(x[(s * 64) % 512:(s * 64) % 512 + 64], target=y[(s * 64) % 512:(s * 64) % 512 + 64]))
                  for s in range(steps)]
        assert tr.opt.param_groups[0]["momentum"] == (0.0 if cfg.get('memory') == 'dgc' else momentum)
        tr.close()
        return losses

    dense = train({'compressor': 'none', 'memory': 'none', 'communicator': 'allreduce'}, 0.9)
    d_end = sum(dense[-10:]) / 10
    assert d_end < 0.25 * dense[0]
    for extra in ({}, dict(deepreduce='index', index='bloom'), dict(deepreduce='both', index='bloom', value='qsgd')):
        comp = train(dict(BASE, min_numel=100, momentum=0.9, **extra), 0.9)
        c_end = sum(comp[-10:]) / 10
        assert c_end < 0.35 * comp[0] and c_end < 2.0 * d_end + 0.15, (extra, d_end, c_end)


@pytest.mark.timeout(600)
def test_dgc_tracks_dense_momentum_sgd_fused_oracle_two_ranks():
    x, y = _data(n=1024, seed=1)
    lr, m = 0.05, 0.9

    def run(mode, steps=120):
        torch.manual_seed(0)
        model = _mlp()
        ps = list(model.parameters())
        plan = None
        if mode is not None:
            plan = BucketPlan([p.numel() for p in ps], compress_ratio=0.05, min_numel=100, **mode)
            resid = [torch.zeros(plan.total_elems) for _ in range(2)]
            mom = [torch.zeros(plan.total_elems) for _ in range(2)]
        buf = [torch.zeros_like(p) for p in ps]              # dense run: SGD momentum buffers
        losses = []
        for s in range(steps):
            grads, ls = [], 0.0
            for r in range(2):
                i = ((2 * s + r) * 64) % 1024
                model.zero_grad()
                loss = nn.functional.cross_entropy(model(x[i:i + 64]), y[i:i + 64])
                loss.backward()
                ls += float(loss.detach()) / 2
                if plan is None:
                    grads.append([p.grad.clone() for p in ps])
                else:
                    flat = torch.zeros(plan.total_elems)
                    for v, p in zip(plan.views(flat), ps):
                        v.copy_(p.grad.reshape(v.shape))
                    grads.append(flat)
            with torch.no_grad():
                if plan is None:
                    for p, b, a, c in zip(ps, buf, *grads):
                        b.mul_(m).add_((a + c) / 2)
                        p -= lr * b
                else:
                    out, resid, _, mom = engine_oracle(plan, grads, resid, epoch=s + 1, momentum=m, moms=mom)
                    for v, p in zip(plan.views(out), ps):
                        p -= lr * v.reshape(p.shape)              # SGD without momentum: it lives in the memory
            losses.append(ls)
        return losses

    dense = run(None)
    d_end = sum(dense[-10:]) / 10
    assert d_end < 0.25 * dense[0]
    for mode in (dict(index="bloom"), dict(index=None), dict(index="bloom", value="qsgd")):
        comp = run(mode)
        c_end = sum(comp[-10:]) / 10
        assert c_end < 0.3 * comp[0] and c_end < 2.0 * d_end + 0.15, (mode, d_end, c_end)
