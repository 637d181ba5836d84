"""'dgc' memory with Nesterov momentum ('nesterov') and weight-decay exclusions by parameter name
('weight_decay_exclude'): config, the per-tensor DgcMemory against the formula, the momentum buffer against torch's
SGD, the fused engine's oracle against the per-tensor memory in every fused mode, convergence against dense
SGD(nesterov=True) with a no-decay param group, two gloo ranks, and the pattern checks of DeepReduceDDP and the DDP
hook.  CPU only."""
import os
import socket
import tempfile

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
from deepreduce_b200.parallel.engine import decode_slot_oracle, tensor_decays
from deepreduce_b200.parallel.plan import split_large

BASE = {'compressor': 'topk', 'memory': 'dgc', 'communicator': 'allgather', 'compress_ratio': 0.05}
EXCL = ['*.bias', '*bn*']


def _bits(t):
    return t.detach().float().contiguous().view(torch.int32)


def test_config_accepts_and_rejects():
    assert {"nesterov", "weight_decay_exclude"} <= KNOWN_KEYS
    for ok in (dict(BASE, nesterov=True), dict(BASE, nesterov=False), dict(BASE, nesterov=False, momentum=0.0),
               dict(BASE, nesterov=True, momentum=0.5), dict(BASE, weight_decay=1e-4, weight_decay_exclude=EXCL),
               dict(BASE, weight_decay=1e-4, weight_decay_exclude=[]),
               dict(BASE, weight_decay=1e-4, weight_decay_exclude=('*.bias',)),
               dict(BASE, compressor='randomk', communicator='allreduce', nesterov=True, weight_decay=1e-4,
                    weight_decay_exclude=EXCL)):
        with __import__("warnings").catch_warnings():
            __import__("warnings").simplefilter("error")          # no unknown-key warning for either key
            assert DeepReduceConfig.from_params(ok, strict=True).memory == 'dgc'
    for bad in (dict(BASE, nesterov=1), dict(BASE, nesterov='True'), dict(BASE, nesterov=None),
                dict(BASE, nesterov=0.0),
                dict(BASE, memory='residual', nesterov=True), dict(BASE, memory='none', nesterov=False),
                {k: v for k, v in dict(BASE, nesterov=True).items() if k != 'memory'},
                dict(BASE, nesterov=True, momentum=0), dict(BASE, nesterov=True, momentum=0.0),
                dict(BASE, memory='residual', weight_decay_exclude=EXCL),
                dict(BASE, weight_decay_exclude=EXCL), dict(BASE, weight_decay=0.0, weight_decay_exclude=EXCL),
                dict(BASE, weight_decay=1e-4, weight_decay_exclude='*.bias'),
                dict(BASE, weight_decay=1e-4, weight_decay_exclude=['*.bias', 3]),
                dict(BASE, weight_decay=1e-4, weight_decay_exclude=None),
                dict(BASE, weight_decay=1e-4, weight_decay_exclude={'*.bias': True})):
        with pytest.raises(ConfigError):
            DeepReduceConfig.from_params(bad)
    mem = deepreduce_from_params(dict(BASE, nesterov=True, weight_decay=0.1, weight_decay_exclude=EXCL)).memory
    assert isinstance(mem, DgcMemory) and mem.nesterov and mem.weight_decay_exclude == tuple(EXCL)
    mem = deepreduce_from_params(BASE).memory
    assert not mem.nesterov and mem.weight_decay_exclude == ()
    with pytest.raises(ValueError):
        DgcMemory(momentum=0.0, nesterov=True)


def test_dgc_memory_nesterov_three_step_formula():
    torch.manual_seed(0)
    m, wd, n = 0.9, 0.05, 1000
    grc = deepreduce_from_params(dict(BASE, momentum=m, weight_decay=wd, nesterov=True))
    w = torch.randn(n)
    grc.memory.bind_parameters([("w", w)])
    comp = TopKCompressor(0.05)
    u = r = None
    for s in range(3):
        g = torch.randn(n)
        out = grc.step(g.clone(), "w")
        # the formula, written out: d = g + (wd * w), u = m*u + d, v = d + (m * u), r = r + v, own = decode(encode(r)),
        # r -= own, u[own != 0] = 0; the first step starts from u = d, so r = d + (m * d)
        d = g + (wd * w)
        if s == 0:
            u = d.clone()
            r = d + (m * u)
        else:
            u = (m * u) + d
            r = r + (d + (m * u))
        own = comp.decompress(*comp.compress(r, "w"))
        r = r - own
        u = torch.where(own != 0, torch.zeros_like(u), u)
        assert torch.equal(_bits(grc.memory.momenta["w"]), _bits(u)), s
        assert torch.equal(_bits(grc.memory.residuals["w"]), _bits(r)), s
        assert torch.equal(_bits(out), _bits(own)), s
        w = w - 0.01 * own
        grc.memory.parameters["w"].copy_(w)


def test_excluded_name_is_the_decay_free_memory():
    """An excluded name computes bit for bit what a weight_decay = 0 memory computes (-0.0 in g stays -0.0: nothing is
    added), and its parameter is never read: a NaN parameter bound to it leaves everything finite, and an unbound
    excluded name is fine."""
    torch.manual_seed(1)
    for nesterov in (False, True):
        cfg = dict(BASE, momentum=0.9, nesterov=nesterov)
        excl = deepreduce_from_params(dict(cfg, weight_decay=0.5, weight_decay_exclude=['bn*', '*.bias']))
        free = deepreduce_from_params(cfg)
        excl.memory.bind_parameters([("bn1.weight", torch.full((2000,), float('nan'))), ("fc.weight", torch.randn(10))])
        for s in range(3):
            for name in ("bn1.weight", "fc.bias"):                     # bound to NaN / not bound at all
                g = torch.randn(2000)
                g[::7] = -0.0
                a, b = excl.step(g.clone(), name), free.step(g.clone(), name)
                assert torch.equal(_bits(a), _bits(b)), (nesterov, s, name)
                assert torch.isfinite(a).all()
                for k in ("momenta", "residuals"):
                    x, y = getattr(excl.memory, k)[name], getattr(free.memory, k)[name]
                    assert torch.equal(_bits(x), _bits(y)) and torch.isfinite(x).all(), (nesterov, s, name, k)
                if s == 0:
                    assert bool((_bits(excl.memory.momenta[name])[::7] == _bits(torch.tensor(-0.0))).all())
        # a name that is not excluded still reads its parameter
        with pytest.raises(KeyError):
            excl.step(torch.randn(10), "fc2.weight")


@pytest.mark.parametrize("foreach", [False, True])
def test_momentum_buffer_is_torchs_nesterov_sgd(foreach):
    """u is torch's momentum_buffer bit for bit, on the coordinates that are never shipped (masking clears the
    others); torch's buffer starts from the first gradient, as DgcMemory's u does."""
    torch.manual_seed(2)
    m, n = 0.9, 4000
    p = nn.Parameter(torch.randn(n))
    opt = torch.optim.SGD([p], lr=0.0, momentum=m, nesterov=True, foreach=foreach)
    mem = DgcMemory(momentum=m, nesterov=True)
    comp = TopKCompressor(0.01)
    shipped = torch.zeros(n, dtype=torch.bool)
    for s in range(4):
        g = torch.randn(n)
        p.grad = g.clone()
        opt.step()                                           # lr = 0: p stays, the buffer moves
        v = mem.compensate(g.clone(), "p")
        c, ctx = comp.compress(v, "p")
        mem.update(v, "p", comp, c, ctx)
        shipped |= comp.decompress(c, ctx) != 0
        keep = ~shipped
        assert int(keep.sum()) > n // 2
        buf = opt.state[p]["momentum_buffer"]
        assert torch.equal(_bits(mem.momenta["p"][keep]), _bits(buf[keep])), s


class _Stub:
    """A compressor whose 'compressed' form is the decoded contribution itself: it lets the per-tensor DgcMemory run on
    exactly what a fused engine slot ships."""

    def decompress(self, c, ctx):
        return c


MODES = {
    "plain": dict(index=None),
    "bloom_leftmost": dict(index="bloom"),
    "bloom_random": dict(index="bloom", policy="random", fpr=0.02),
    "bloom_p0": dict(index="bloom", policy="p0"),
    "rle": dict(index="rle"),
    "elias_fano": dict(index="elias_fano"),
    "qsgd": dict(index="bloom", value="qsgd"),
    "polyfit": dict(index="bloom", value="polyfit"),
    "dexp": dict(index="bloom", value="dexp"),
    "bf16": dict(index="bloom", value="bf16"),
    "sign": dict(index="rle", value="sign"),
    "fp8": dict(index="elias_fano", value="fp8"),
    "randomk": dict(index=None, sparsifier="randomk"),
    "randomk_qsgd": dict(index=None, sparsifier="randomk", value="qsgd"),
}


def _to_plan(plan, owner, per_param):
    out = torch.zeros(plan.total_elems)
    done = [0] * len(per_param)
    for t, i in zip(plan.tensors, owner):
        out[t.elem_off:t.elem_off + t.numel] = per_param[i][done[i]:done[i] + t.numel]
        done[i] += t.numel
    return out


def _of_param(plan, owner, flat, i):
    return torch.cat([flat[t.elem_off:t.elem_off + t.numel] for t, o in zip(plan.tensors, owner) if o == i])


@pytest.mark.parametrize("clip", [None, 30.0], ids=["noclip", "clip"])
@pytest.mark.parametrize("mode", list(MODES))
def test_oracle_equals_per_tensor_memory(mode, clip):
    """engine_oracle(nesterov=True, weight_decays=...) against the per-tensor DgcMemory with the same keys, over three
    steps, bit for bit: the memory is fed, per parameter, what the oracle's slot ships for it (decode_slot_oracle).
    Parameter 'bn.weight' is split into chunks and excluded; its bound values are NaN, which must never be read."""
    m, wd = 0.9, 0.03
    sizes = [20000, 300, 5000, 9000]
    pnames = ["fc.weight", "fc.bias", "conv.weight", "bn.weight"]
    numels, names, shapes, owner = split_large(sizes, pnames, [(n,) for n in sizes], 8192)
    assert owner.count(3) == 2 and owner.count(0) == 3
    plan = BucketPlan(numels, names, shapes, compress_ratio=0.02, min_numel=100, **MODES[mode])
    gen = torch.Generator().manual_seed(3)
    params = [torch.randn(n, generator=gen) for n in sizes]
    params[3] = torch.full((sizes[3],), float('nan'))
    mem = DgcMemory(momentum=m, weight_decay=wd, clip_norm=clip, nesterov=True, weight_decay_exclude=EXCL)
    mem.bind_parameters(zip(pnames, params))
    decays = [0.0 if n.endswith(".bias") or "bn" in n else wd for n in pnames]
    assert tensor_decays(plan, 0.0, decays, owner) == [decays[o] for o in owner]
    w = _to_plan(plan, owner, params)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(3):
        grads = [torch.randn(n, generator=gen) * (0.5 + step) for n in sizes]
        g = _to_plan(plan, owner, grads)
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=step + 1, momentum=m, moms=mom, weights=[w],
                                             weight_decays=decays, owner=owner, nesterov=True, clip_norm=clip)
        own = decode_slot_oracle(plan, torch.from_numpy(slots[0].view("int32")))
        assert torch.equal(_bits(own), _bits(out)), (mode, step)         # W = 1: the aggregate is the own decode
        for i, name in enumerate(pnames):
            v = mem.compensate(grads[i].clone(), name)
            mem.update(v, name, _Stub(), _of_param(plan, owner, own, i), None)
            tag = (mode, step, name)
            assert torch.equal(_bits(mem.residuals[name]), _bits(_of_param(plan, owner, res[0], i))), tag
            assert torch.equal(_bits(mem.momenta[name]), _bits(_of_param(plan, owner, mom[0], i))), tag
            assert torch.isfinite(mem.momenta[name]).all(), tag


def test_oracle_default_is_unchanged_and_refusals():
    """nesterov=False and all-equal weight_decays compute what the oracle computed without the arguments."""
    plan = BucketPlan([20000, 5000, 301], compress_ratio=0.02, min_numel=100, index="bloom")
    gen = torch.Generator().manual_seed(4)
    g = [torch.randn(plan.total_elems, generator=gen)]
    w = [torch.randn(plan.total_elems, generator=gen)]
    z = [torch.zeros(plan.total_elems)]
    a = engine_oracle(plan, g, z, momentum=0.9, moms=z, weight_decay=0.1, weights=w)
    b = engine_oracle(plan, g, z, momentum=0.9, moms=z, weights=w, weight_decays=[0.1] * 3, nesterov=False)
    assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(_bits(a[1][0]), _bits(b[1][0]))
    assert torch.equal(_bits(a[3][0]), _bits(b[3][0])) and (a[2][0] == b[2][0]).all()
    with pytest.raises(ValueError):
        engine_oracle(plan, g, z, momentum=0.0, moms=z, nesterov=True)            # torch refuses it too
    with pytest.raises(ValueError):
        engine_oracle(plan, g, z, nesterov=True)                                   # needs the 'dgc' momentum
    with pytest.raises(ValueError):
        engine_oracle(plan, g, z, momentum=0.9, moms=z, weights=w, weight_decays=[0.1] * 2)   # not one per parameter
    with pytest.raises(ValueError):
        engine_oracle(plan, g, z, momentum=0.9, moms=z, weights=w, weight_decay=0.1, weight_decays=[0.1] * 3)
    with pytest.raises(ValueError):
        engine_oracle(plan, g, z, momentum=0.9, moms=z, weights=w, weight_decays=[0.1, -1.0, 0.0])


def test_threshold_route_equals_oracle_with_split_excluded_owner():
    """The real per-tensor route (grc.step, threshold sparsifier: the selection is per element, so chunks select what
    the whole tensor selects) against the oracle, with a split parameter whose owner is excluded, and clipping."""
    m, wd, c, thr = 0.9, 0.01, 4.0, 1.5
    sizes = [20000, 300, 9000]
    pnames = ["a.weight", "a.bias", "bn.weight"]
    numels, names, shapes, owner = split_large(sizes, pnames, [(n,) for n in sizes], 8192)
    plan = BucketPlan(numels, names, shapes, index=None, sparsifier="threshold", threshold=thr, capacity_ratio=1.0)
    grc = deepreduce_from_params(dict(BASE, compressor='threshold', threshold=thr, momentum=m, weight_decay=wd,
                                      clip_norm=c, nesterov=True, weight_decay_exclude=EXCL))
    gen = torch.Generator().manual_seed(5)
    params = [torch.randn(n, generator=gen) for n in sizes]
    grc.memory.bind_parameters([("a.weight", params[0])])                 # the excluded ones need no binding
    w = _to_plan(plan, owner, [params[0], torch.zeros(300), torch.zeros(9000)])
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(3):
        grads = [torch.randn(n, generator=gen) * (0.3 + step) for n in sizes]
        out, res, _, mom = engine_oracle(plan, [_to_plan(plan, owner, grads)], res, epoch=step + 1, momentum=m,
                                         moms=mom, weights=[w], weight_decays=[wd, 0.0, 0.0], clip_norm=c,
                                         owner=owner, nesterov=True)
        for i, name in enumerate(pnames):
            ref = grc.step(grads[i].clone(), name)
            assert torch.equal(_bits(_of_param(plan, owner, out, i)), _bits(ref)), (step, name)
            assert torch.equal(_bits(_of_param(plan, owner, res[0], i)), _bits(grc.memory.residuals[name]))
            assert torch.equal(_bits(_of_param(plan, owner, mom[0], i)), _bits(grc.memory.momenta[name]))


class _BnMlp(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc1, self.bn1 = nn.Linear(64, 128), nn.BatchNorm1d(128)
        self.fc2, self.bn2 = nn.Linear(128, 64), nn.BatchNorm1d(64)
        self.fc3 = nn.Linear(64, 8)

    def forward(self, x):
        x = torch.relu(self.bn1(self.fc1(x)))
        x = torch.relu(self.bn2(self.fc2(x)))
        return self.fc3(x)


def _data(n=512, d=64, classes=8, seed=0):
    gen = torch.Generator().manual_seed(seed)
    centers = torch.randn(classes, d, generator=gen) * 2.0
    y = torch.randint(0, classes, (n,), generator=gen)
    x = centers[y] + torch.randn(n, d, generator=gen)
    return x, y


def _groups(model, wd):
    decay = [p for n, p in model.named_parameters() if not (n.endswith(".bias") or "bn" in n)]
    free = [p for n, p in model.named_parameters() if n.endswith(".bias") or "bn" in n]
    assert decay and free
    return [{"params": decay, "weight_decay": wd}, {"params": free, "weight_decay": 0.0}]


@pytest.mark.timeout(300)
def test_nesterov_tracks_dense_nesterov_sgd_trainer():
    from deepreduce_b200.trainer import Trainer
    lr, m, wd = 0.05, 0.9, 0.01
    x, y = _data()

    def batches(steps):
        return [(x[(s * 64) % 512:(s * 64) % 512 + 64], y[(s * 64) % 512:(s * 64) % 512 + 64]) for s in range(steps)]

    torch.manual_seed(0)
    model = _BnMlp()
    opt = torch.optim.SGD(_groups(model, wd), lr=lr, momentum=m, nesterov=True)
    dense = []
    for xb, yb in batches(150):
        opt.zero_grad()
        loss = nn.functional.cross_entropy(model(xb), yb)
        loss.backward()
        opt.step()
        dense.append(float(loss.detach()))
    d_end = sum(dense[-10:]) / 10
    assert d_end < 0.25 * dense[0]
    torch.manual_seed(0)
    cfg = dict(BASE, min_numel=100, momentum=m, nesterov=True, weight_decay=wd, weight_decay_exclude=EXCL)
    tr = Trainer(_BnMlp(), cfg, lr=lr, momentum=m, weight_decay=wd, amp_dtype=None)
    assert tr.opt.param_groups[0]["momentum"] == 0.0 and tr.opt.param_groups[0]["weight_decay"] == 0.0
    comp = [float(tr.step(xb, target=yb)) for xb, yb in batches(150)]
    tr.close()
    c_end = sum(comp[-10:]) / 10
    assert c_end < 0.35 * comp[0] and c_end < 2.0 * d_end + 0.15, (d_end, c_end)


@pytest.mark.timeout(600)
def test_nesterov_tracks_dense_nesterov_sgd_fused_oracle_two_ranks():
    x, y = _data(n=1024, seed=1)
    lr, m, wd = 0.05, 0.9, 0.01

    def run(mode, steps=120):
        torch.manual_seed(0)
        model = _BnMlp()
        named = list(model.named_parameters())
        ps = [p for _, p in named]
        decays = [0.0 if n.endswith(".bias") or "bn" in n else wd for n, _ in named]
        if mode is None:
            opt = torch.optim.SGD(_groups(model, wd), lr=lr, momentum=m, nesterov=True)
        else:
            plan = BucketPlan([p.numel() for p in ps], compress_ratio=0.05, min_numel=100, **mode)
            resid = [torch.zeros(plan.total_elems) for _ in range(2)]
            mom = [torch.zeros(plan.total_elems) for _ in range(2)]
        losses = []
        for s in range(steps):
            grads, ls = [], 0.0
            for r in range(2):
                i = ((2 * s + r) * 64) % 1024
                model.zero_grad()
                loss = nn.functional.cross_entropy(model(x[i:i + 64]), y[i:i + 64])
                loss.backward()
                ls += float(loss.detach()) / 2
                grads.append([p.grad.clone() for p in ps])
            if mode is None:
                for p, a, b in zip(ps, *grads):
                    p.grad = (a + b) / 2
                opt.step()
            else:
                flat = [_to_plan(plan, list(range(len(ps))), [t.reshape(-1) for t in gr]) for gr in grads]
                w = _to_plan(plan, list(range(len(ps))), [p.detach().reshape(-1) for p in ps])
                out, resid, _, mom = engine_oracle(plan, flat, resid, epoch=s + 1, momentum=m, moms=mom,
                                                   weights=[w, w], weight_decays=decays, nesterov=True)
                with torch.no_grad():
                    for v, p in zip(plan.views(out), ps):
                        p -= lr * v.reshape(p.shape)          # SGD without momentum and decay: both live in the memory
            losses.append(ls)
        return losses

    dense = run(None)
    d_end = sum(dense[-10:]) / 10
    assert d_end < 0.25 * dense[0]
    for mode in (dict(index="bloom"), dict(index=None), dict(index="bloom", value="qsgd")):
        comp = run(mode)
        c_end = sum(comp[-10:]) / 10
        assert c_end < 0.3 * comp[0] and c_end < 2.0 * d_end + 0.15, (mode, d_end, c_end)


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
        mem = tr.ddp.grc.memory
        ret["losses"] = losses
        ret["same"] = all(torch.equal(gathered[0], g) for g in gathered)
        ret["opt"] = (tr.opt.param_groups[0]["weight_decay"], tr.opt.param_groups[0]["momentum"])
        ret["mem"] = (mem.nesterov, mem.weight_decay_exclude)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_resnet20_world2_gloo_nesterov_exclude():
    mgr = mp.Manager()
    ret = mgr.dict()
    cfg = dict(BASE, compress_ratio=0.01, deepreduce='index', index='bloom', momentum=0.9, nesterov=True,
               weight_decay=5e-4, weight_decay_exclude=EXCL)
    mp.spawn(_worker, args=(2, _free_port(), cfg, ret), nprocs=2, join=True)
    assert ret["same"], "ranks diverged"
    assert all(l == l and l < 20 for l in ret["losses"])
    assert ret["opt"] == (0.0, 0.0)
    assert ret["mem"] == (True, tuple(EXCL))


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


def test_patterns_select_the_same_parameters_in_ddp_and_hook(gloo_world1):
    """The same patterns select the same parameters in DeepReduceDDP (named_parameters names) and in the DDP hook (the
    names its state_dict keys): one step from the same gradients leaves the same momenta, and an excluded parameter's
    first momentum is its gradient (nothing added).  A pattern that matches nothing raises in both."""
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.parallel import DeepReduceDDP, DeepReduceHookState
    from deepreduce_b200.parallel.comm_hook import deepreduce_hook
    cfg = dict(BASE, momentum=0.9, nesterov=True, weight_decay=0.5, weight_decay_exclude=EXCL, min_numel=10)
    torch.manual_seed(6)
    model = _BnMlp()
    twin = _BnMlp()
    twin.load_state_dict(model.state_dict())
    x = torch.randn(16, 64)
    ddp = DeepReduceDDP(model, cfg)
    model(x).pow(2).mean().backward()
    grads = {n: p.grad.clone() for n, p in model.named_parameters()}
    ddp.finish()
    hook_model = DDP(twin)
    st = DeepReduceHookState(cfg, twin)
    hook_model.register_comm_hook(st, deepreduce_hook)
    hook_model(x).pow(2).mean().backward()
    excluded = set()
    for n, p in model.named_parameters():
        a, b = ddp.grc.memory.momenta[n], st.grc.memory.momenta[n]
        assert torch.equal(_bits(a), _bits(b.reshape(a.shape))), n
        kept = a.reshape(-1) != 0
        if torch.equal(_bits(a.reshape(-1)[kept]), _bits(grads[n].reshape(-1)[kept])):
            excluded.add(n)
    assert excluded == {n for n, _ in model.named_parameters() if n.endswith(".bias") or "bn" in n}
    ddp.close()
    st.close()
    for bad in (['*.bias', 'batchnorm*'], ['nothing']):
        cfg_bad = dict(cfg, weight_decay_exclude=bad)
        with pytest.raises(ValueError, match="match none"):
            DeepReduceDDP(_BnMlp(), cfg_bad)
        with pytest.raises(ValueError, match="match none"):
            DeepReduceHookState(cfg_bad, _BnMlp())


def test_patterns_over_frozen_parameters_raise_in_ddp_and_hook(gloo_world1):
    """Both routes match the patterns against the parameters they exchange, those that require a gradient: a pattern
    that matches only a frozen parameter matches nothing they exchange, and both refuse it."""
    from deepreduce_b200.parallel import DeepReduceDDP, DeepReduceHookState
    cfg = dict(BASE, momentum=0.9, weight_decay=0.5, min_numel=10)
    for frozen_only in (['fc1.weight'], ['*.bias', 'fc1.*']):
        model = _BnMlp()
        for p in model.fc1.parameters():
            p.requires_grad_(False)
        bad = dict(cfg, weight_decay_exclude=frozen_only)
        with pytest.raises(ValueError, match="match none"):
            DeepReduceDDP(model, bad)
        with pytest.raises(ValueError, match="match none"):
            DeepReduceHookState(bad, model)
    model = _BnMlp()
    model.fc1.weight.requires_grad_(False)
    ok = dict(cfg, weight_decay_exclude=['fc1.*', '*bn*'])          # fc1.bias still requires a gradient
    DeepReduceDDP(model, ok).close()
    DeepReduceHookState(ok, model).close()
