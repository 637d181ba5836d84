"""The Elias-Fano index ('index': 'elias_fano') in the fused engine on the GPU.

W = 1 through ``test_gpu_engine._run_vs_oracle`` in every value mode, both copy paths and both launch variants; bf16
buckets, the 'dgc' memory with weight decay and clipping, and the threshold sparsifier at full capacity (L = 0, 4096
entries in one tile) against the oracle and against a run-length engine fed the same gradients; W = 2 ... 16 through
the one-GPU W-rank harness of ``test_engine_multirank`` (sharded, unsharded, the NCCL transport, rank-ordered and
RED.ADD sums), again against the oracle and against run-length engines; the per-tensor codec on CUDA; and the public
entry points: the benchmark's ResNet-50 step, the DDP hook across DDP's bucket rebuild, a checkpoint round trip and a
sparsity warm-up through its stage switches."""
import copy
import dataclasses

import numpy as np
import pytest
import torch

import bench
import test_engine_multirank as multirank
import test_gpu_comm_hook as hook
import test_gpu_engine
from deepreduce_b200 import spec
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import decode_slot_oracle
from deepreduce_b200.parallel.plan import DYN_WORDS, MODE_EF, MODE_RAW, MODE_RLE, SLOT_HEADER_WORDS, split_large
from test_gpu_dgc_weight_decay import _placed, nccl_world1  # noqa: F401
from test_gpu_engine import SIZES, _fill, _run_vs_oracle
from test_train_step_reference import run_case

pytestmark = pytest.mark.gpu

BIG = SIZES + [2359296]
VALUES = {"fp32": dict(), "bf16": dict(value="bf16"), "qsgd8": dict(value="qsgd"),
          "qsgd16": dict(value="qsgd", quantum_num=1000), "polyfit": dict(value="polyfit"), "dexp": dict(value="dexp")}
_compare_shared = test_gpu_engine._compare_slot


def compare_slot(plan, slot_gpu, slot_ref, tag):
    """``test_gpu_engine._compare_slot`` with the Elias-Fano index: each such tensor's counts and its two streams word
    for word; its header and values through the shared comparison, which sees it as plain pairs whose index lies in
    a zero pad appended to both slots."""
    a = slot_gpu.cpu().numpy().view(np.uint32)[:len(slot_ref)]
    b = np.asarray(slot_ref, dtype=np.uint32)
    bad, shown = [], copy.copy(plan)
    tensors = []
    for t in plan.tensors:
        if t.mode == MODE_EF:
            _, lo, hi = spec.ef_layout(t.val_cap, t.n_tiles)
            for what, off, n in (("counts", t.off_prefix, (t.n_tiles + 1) // 2), ("streams", t.off_idx, lo + hi)):
                if not np.array_equal(a[off:off + n], b[off:off + n]):
                    bad.append(f"{t.name} ef {what} differ in {int((a[off:off + n] != b[off:off + n]).sum())}/{n} words")
            t = dataclasses.replace(t, mode=MODE_RAW, off_idx=len(b))
        tensors.append(t)
    shown.tensors = tensors
    pad = np.zeros(max(t.val_cap for t in plan.tensors), dtype=np.uint32)
    bad += _compare_shared(shown, torch.from_numpy(np.concatenate([a, pad]).view(np.int32)), np.concatenate([b, pad]),
                           tag)
    return bad


@pytest.fixture
def ef_harness(monkeypatch):
    """The shared harnesses with the Elias-Fano slot comparison, and its decode sums (SMEM ``acc += v * scale`` in rank
    order) classed as the run-length index's."""
    monkeypatch.setattr(test_gpu_engine, "_compare_slot", compare_slot)
    monkeypatch.setattr(multirank, "_compare_slot", compare_slot)
    exact = multirank._exact_tensor
    monkeypatch.setattr(multirank, "_exact_tensor",
                        lambda t, *a: exact(dataclasses.replace(t, mode=MODE_RLE) if t.mode == MODE_EF else t, *a))


def _bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


@pytest.mark.parametrize("value", list(VALUES))
@pytest.mark.parametrize("tma,bps", [(True, 2), (False, 2), (True, 1), (False, 1)])
def test_single_rank_vs_oracle(ef_harness, value, tma, bps):
    """W = 1, three epochs (the second through the unfused phase chain): slots against the oracle; fp32 values give
    the output and residual bit for bit, the value codecs within their tolerances."""
    for kind in ("randn", "sparse"):
        _run_vs_oracle(kind, "elias_fano", "leftmost", True, tma, VALUES[value].get("value"),
                       bps=bps, **{k: v for k, v in VALUES[value].items() if k != "value"})


def _twins(plan_kw, sizes=BIG, steps=3, grad_dtype=torch.float32, **eng_kw):
    """An Elias-Fano engine and a run-length engine fed the same gradients: the Elias-Fano slot against the oracle
    each step; returns the per-step (ef, rle) engine states."""
    ef = BucketPlan(sizes, index="elias_fano", **plan_kw)
    rle = BucketPlan(sizes, index="rle", **plan_kw)
    assert any(t.mode == MODE_EF for t in ef.tensors)
    kw = dict(device="cuda:0", world=1, rank=0, spin_limit=2_000_000, grad_dtype=grad_dtype, **eng_kw)
    engs = [BucketEngine(ef, **kw), BucketEngine(rle, **kw)]
    gen = torch.Generator().manual_seed(5)
    resid = torch.zeros(ef.total_elems)
    states = []
    for step in range(steps):
        g = (_fill(ef, gen) * (0.2 if step == 2 else 1.0)).to(grad_dtype)
        for e in engs:
            e.grad.copy_(g.cuda())
            e.step()
        torch.cuda.synchronize()
        for e in engs:
            e.check_status()
        if "momentum" not in eng_kw:
            _, _, slots = engine_oracle(ef, [g.float()], [resid], epoch=engs[0].epoch)
            bad = compare_slot(ef, engs[0].slot(), slots[0], f"ef_twin_s{step}")
            assert not bad, bad[:4]
            resid = engs[0].resid.cpu().clone()
        states.append([(e.grad.cpu().clone(), e.resid.cpu().clone(),
                        e.mom.cpu().clone() if e.mom is not None else None, e.slot().cpu()) for e in engs])
    for e in engs:
        e.close()
    return ef, states


@pytest.mark.parametrize("value", ["fp32", "bf16", "qsgd8", "polyfit"])
@pytest.mark.parametrize("bps", [2, 1])
def test_bf16_bucket_equals_rle(value, bps):
    """bf16 gradient buckets: output and residual equal a run-length engine's bit for bit (coded values: within the
    codec's tolerance, the fit's fp32 sums are the same code on both), and the slot is the oracle's."""
    _, states = _twins(dict(compress_ratio=0.01, poly_min_k=300, **VALUES[value]), grad_dtype=torch.bfloat16,
                       blocks_per_sm=bps)
    for step, ((ga, ra, _, _), (gb, rb, _, _)) in enumerate(states):
        if value in ("fp32", "bf16"):
            assert torch.equal(ga, gb) and torch.equal(_bits(ra), _bits(rb)), step
        else:
            sc = float(gb.float().abs().max())
            assert torch.allclose(ga.float(), gb.float(), atol=2e-3 * sc, rtol=1e-2), step


@pytest.mark.parametrize("value", ["fp32", "bf16"])
@pytest.mark.parametrize("threshold,cr", [(0.0, None), (1.0, 0.3)])
def test_threshold_full_and_partial_capacity(threshold, cr, value):
    """The threshold sparsifier with the slot provisioned for every element (L = 0: at threshold 0 every non-zero of a
    tile is shipped, 4096 entries) and with 'capacity_ratio': slots against the oracle, output and residual equal the
    run-length engine's bit for bit and the decode of the engine's own slot (bf16 values: the W = 1 output is that
    decode, fp32 values are scattered by emit)."""
    ef, states = _twins(dict(sparsifier="threshold", threshold=threshold, capacity_ratio=cr, **VALUES[value]))
    t = ef.tensors[-1]
    assert (t.ef_low_bits == 0) == (cr is None)
    for step, ((ga, ra, _, sa), (gb, rb, _, _)) in enumerate(states):
        assert torch.equal(_bits(ga), _bits(gb)) and torch.equal(_bits(ra), _bits(rb)), step
        assert torch.equal(_bits(ga), _bits(decode_slot_oracle(ef, sa))), step
        if cr is None:
            n_sel = int(sa[SLOT_HEADER_WORDS + DYN_WORDS * (len(ef.tensors) - 1)])
            assert n_sel > 4096 * (t.n_tiles - 1), step


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_dgc_weight_decay_and_clip_equal_rle(dtype):
    """The 'dgc' memory with weight decay and clipping: output, residual and momentum equal a run-length engine's bit
    for bit, and the Elias-Fano slot is the oracle's (``engine_oracle`` with the same memory)."""
    from test_gpu_dgc_weight_decay import _weights
    sizes = BIG
    numels, names, shapes, owner = split_large(sizes, [f"t{i}" for i in range(len(sizes))], [(n,) for n in sizes], 8192)
    gen = torch.Generator().manual_seed(0)
    params = [_placed(torch.randn(n, generator=gen).to(dtype).cuda(), i) for i, n in enumerate(sizes)]
    engs, plans = [], []
    for index in ("elias_fano", "rle"):
        plan = BucketPlan(numels, names, shapes, compress_ratio=0.01, index=index)
        e = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=0.9, weight_decay=0.05, clip_norm=60.0,
                         owner=owner, grad_dtype=dtype, spin_limit=2_000_000)
        e.bind_parameters(params, owner)
        engs.append(e)
        plans.append(plan)
    w = _weights(plans[0], owner, params)
    res, mom = [torch.zeros(plans[0].total_elems)], [torch.zeros(plans[0].total_elems)]
    for step in range(3):
        g = (_fill(plans[0], gen) * (0.5 + step)).to(dtype)
        for e in engs:
            e.grad.copy_(g.cuda())
            e.step()
        torch.cuda.synchronize()
        for e in engs:
            e.check_status()
        out, res, slots, mom = engine_oracle(plans[0], [g.float()], res, epoch=engs[0].epoch, momentum=0.9, moms=mom,
                                             weight_decay=0.05, weights=[w], clip_norm=60.0, owner=owner)
        bad = compare_slot(plans[0], engs[0].slot(), slots[0], f"ef_dgc_s{step}")
        assert not bad, bad[:4]
        a, b = engs
        assert torch.equal(_bits(a.grad), _bits(b.grad)), step
        assert torch.equal(_bits(a.resid), _bits(b.resid)) and torch.equal(_bits(a.mom), _bits(b.mom)), step
        res, mom = [a.resid.cpu().clone()], [a.mom.cpu().clone()]
    for e in engs:
        e.close()


C = pytest.param
# (configuration, W, sizes, plan keyword arguments, DR_DETERMINISTIC, average, rank with an all-zero gradient, claims)
MR_CASES = [
    C("shard", 2, BIG, {}, False, True, None, set(), id="shard-fp32-W2-fast"),
    C("shard", 3, SIZES, {}, True, True, None, {"split"}, id="shard-fp32-W3-det"),
    C("shard", 4, BIG, dict(value="qsgd"), False, True, 1, {"qsgd8"}, id="shard-qsgd8-W4-fast"),
    C("shard", 3, SIZES, dict(value="polyfit", poly_min_k=300), True, False, None, {"polyfit", "split"},
      id="shard-polyfit-W3-det-sum"),
    C("shard", 2, SIZES, dict(value="bf16"), True, True, 0, set(), id="shard-bf16-W2-det"),
    C("shard", 3, SIZES, dict(sparsifier="threshold", threshold=1.0, capacity_ratio=0.2), False, True, 2, set(),
      id="shard-threshold-W3-fast"),
    C("shard", 8, multirank.SMALL, {}, False, True, 3, {"empty"}, id="shard-small-W8-fast"),
    C("shard", 16, multirank.SMALL, dict(value="qsgd", quantum_num=1000), True, True, None, {"empty", "qsgd16"},
      id="shard-small-qsgd16-W16-det"),
    C("noshard", 3, SIZES, {}, False, True, None, set(), id="noshard-fp32-W3-fast"),
    C("noshard", 2, SIZES, dict(value="qsgd"), True, False, 0, {"qsgd8"}, id="noshard-qsgd8-W2-det-sum"),
    C("nccl", 3, SIZES, {}, True, True, 2, set(), id="nccl-fp32-W3-det"),
    C("nccl", 4, SIZES, dict(value="polyfit", poly_min_k=300), False, True, None, {"polyfit"}, id="nccl-polyfit-W4-fast"),
]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,W,sizes,kw,deterministic,average,zero_rank,claims", MR_CASES)
def test_multirank_vs_oracle(ef_harness, monkeypatch, config, W, sizes, kw, deterministic, average, zero_rank, claims):
    """W ranks on one GPU through the shared harness: slots and residuals against ``engine_oracle``, delivery of every
    slot, the aggregate against the decode of the shipped slots, identical bits on every rank, the stage-2 lists."""
    multirank.test_engine_multirank_vs_oracle(monkeypatch, config, W, sizes, dict(index="elias_fano", **kw),
                                              deterministic, average, zero_rank, claims)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,W,deterministic", [("shard", 2, False), ("shard", 3, True), ("shard", 16, False),
                                                    ("noshard", 4, False), ("nccl", 3, False), ("nccl", 4, True)])
@pytest.mark.parametrize("value", ["fp32", "bf16"])
def test_multirank_equals_rle(monkeypatch, config, W, deterministic, value):
    """W Elias-Fano ranks and W run-length ranks fed the same gradients: every rank's output and residual are the
    run-length group's bit for bit, three steps."""
    monkeypatch.setenv("DR_DETERMINISTIC", "1" if deterministic else "0")
    sizes = SIZES if W <= 5 else multirank.SMALL
    groups = []
    for index in ("elias_fano", "rle"):
        plan = BucketPlan(sizes, compress_ratio=0.01, index=index, **VALUES[value])
        groups.append(multirank._engines(plan, W, config, True))
    for step in range(3):
        for engs in groups:
            for r, e in enumerate(engs):
                g = _fill(e.plan, torch.Generator().manual_seed(1000 * step + r)) * (0.2 if step == 2 else 1.0)
                e.grad.copy_(g.cuda())
            multirank._run_step(engs, config, step + 1)
        for a, b in zip(*groups):
            assert torch.equal(_bits(a.grad), _bits(b.grad)), (step, a.rank)
            assert torch.equal(_bits(a.resid), _bits(b.resid)), (step, a.rank)
    for engs in groups:
        for e in engs:
            e.close()


def test_codec_cuda_words_equal_cpu():
    from deepreduce_b200.codecs.elias_fano import EliasFano
    gen = torch.Generator().manual_seed(2)
    for numel, n in ((1001, 1), (4097, 4097), (5 * 4096 + 3, 700), (2359296, 23592), (40000, 39000)):
        idx = torch.randperm(numel, generator=gen)[:n]
        vals = torch.randn(n, generator=gen)
        vc, ec, sc = EliasFano.compress((vals, idx, torch.Size([numel])), {})
        vg, eg, sg = EliasFano.compress((vals.cuda(), idx.cuda(), torch.Size([numel])), {})
        assert eg.is_cuda and torch.equal(eg.cpu(), ec) and torch.equal(vg.cpu(), vc), (numel, n)
        _, ig, _ = EliasFano.decompress((vg, eg, sg), {})
        assert torch.equal(ig.cpu(), idx.sort().values), (numel, n)


# ---- public entry points ------------------------------------------------------------------------------------------
EF_CFG = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
          'deepreduce': 'index', 'index': 'elias_fano'}


def _ef_fused(tr):
    assert tr.ddp.fused and tr.ddp.grc is None
    assert any(t.mode == MODE_EF for e in tr.ddp.engines for t in e.plan.tensors)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("extra", [{}, {'deepreduce': 'both', 'value': 'qsgd'}], ids=["fp32", "qsgd"])
def test_resnet50_train_step(monkeypatch, extra):
    """ResNet-50, batch 16, the benchmark's ``Trainer`` with the Elias-Fano index against plain torch +
    ``engine_oracle``."""
    monkeypatch.setitem(bench.CONFIGS, "ef", {**EF_CFG, **extra})
    run_case(monkeypatch, "image", "ef", 16, check=_ef_fused)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("extra", [{}, {'deepreduce': 'both', 'value': 'qsgd', 'compress_ratio': 0.05}],
                         ids=["fp32", "qsgd"])
def test_ddp_hook_resnet20(monkeypatch, nccl_world1, extra):  # noqa: F811
    """torch DDP + the communication hook on ResNet-20, four steps across DDP's bucket rebuild, against the oracle."""
    monkeypatch.setitem(hook.CONFIGS, "ef", {**hook.CONFIGS["rle"], 'index': 'elias_fano', **extra})
    st = hook.run_ddp_case("ef", "resnet20")
    assert st.fused_params


def test_checkpoint_round_trip():
    """A DeepReduceDDP checkpoint of the fused route holds the engines' state; a fresh wrapper that loads it continues
    bit for bit."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel import DeepReduceDDP

    def make():
        torch.manual_seed(0)
        m = resnet20().cuda()
        return m, DeepReduceDDP(m, {**EF_CFG, 'deepreduce': 'both', 'value': 'bf16'}, bucket_cap_mb=0.5, overlap=False)

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
    assert any(t.mode == MODE_EF for e in a.engines for t in e.plan.tensors)
    for i in range(2):
        step(ma, a, i)
    ckpt = a.state_dict()
    mb, b = make()
    b.load_state_dict(ckpt)
    for i in (2, 3):
        ga, gb = step(ma, a, i), step(mb, b, i)
        assert all(torch.equal(x, y) for x, y in zip(ga, gb)), i
    for e, f in zip(a.engines, b.engines):
        assert torch.equal(e.resid, f.resid) and e.epoch == f.epoch
    a.close(); b.close()


def test_warmup_schedule_switches_plans():
    """A sparsity warm-up through two stage switches: each stage's engine has its own plan and its own L, and every
    exchange's aggregate equals ``engine_oracle`` on that stage's plan bit for bit."""
    from deepreduce_b200.config import warmup_from_params
    from deepreduce_b200.parallel import DeepReduceDDP
    from test_gpu_dgc_weight_decay import _ConvNet
    cfg = {**EF_CFG, 'calibrate_partition': False, 'min_numel': 100, 'warmup_ratios': [0.25, 0.0625],
           'warmup_steps': 2}
    wu = warmup_from_params(cfg)
    torch.manual_seed(0)
    model = _ConvNet().cuda()
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    assert ddp.fused and len(ddp.engines) == 1
    res = [torch.zeros(ddp.engines[0].plan.total_elems)]
    gen = torch.Generator().manual_seed(1)
    Ls = []
    for e in range(6):
        eng = ddp.engines[0]
        assert eng.plan.compress_ratio == wu.ratio_at(e)
        Ls.append(tuple(t.ef_low_bits for t in eng.plan.tensors if t.mode == MODE_EF))
        with torch.no_grad():
            for p in model.parameters():
                p.grad.copy_(torch.randn(p.shape, generator=gen) * 1e-3)
        g = eng.grad.float().cpu()
        ddp.finish()
        torch.cuda.synchronize()
        ddp.check()
        out, res, _ = engine_oracle(eng.plan, [g], res, epoch=eng.epoch)
        assert torch.equal(_bits(ddp.flat[0]), _bits(out)), e
        assert torch.equal(_bits(ddp.engines[0].resid), _bits(res[0])), e
    assert Ls[0] != Ls[2] != Ls[4]
    ddp.close()
