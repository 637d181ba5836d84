"""Sparsity warm-up ('warmup_ratios', 'warmup_steps'): config, the schedule at its stage boundaries, the per-tensor
sparsifiers against a run that swaps 'compress_ratio' by hand, checkpoints mid-stage and at a boundary, the plans of the
stages, Trainer's exchange counting and two gloo ranks.  CPU only."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from deepreduce_b200 import deepreduce_from_params
from deepreduce_b200.config import KNOWN_KEYS, ConfigError, DeepReduceConfig, warmup_from_params
from deepreduce_b200.grace.helper import sparsifier_of
from deepreduce_b200.parallel.ddp import engine_split_numel, plan_kwargs_from_params, stage_plans
from deepreduce_b200.parallel.plan import BucketPlan, split_large

DGC = [0.25, 0.0625, 0.015625, 0.004]
TOPK = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.001}
WU = dict(TOPK, warmup_ratios=DGC, warmup_steps=3)


def _bits(t):
    return t.detach().float().contiguous().view(torch.int32)


# ---- config ---------------------------------------------------------------------------------------------------------
def test_config_accepts():
    assert {"warmup_ratios", "warmup_steps"} <= KNOWN_KEYS
    cfg = DeepReduceConfig.from_params(WU, strict=True)
    assert cfg.warmup_ratios == tuple(DGC) and cfg.warmup_steps == 3
    for ok in (dict(WU, compressor='randomk', communicator='allreduce'), dict(WU, memory='dgc', momentum=0.9),
               dict(WU, memory='none'), dict(WU, warmup_ratios=[1, 0.5], warmup_steps=1),
               dict(WU, warmup_ratios=(0.5,)), dict(WU, deepreduce='index', index='bloom')):
        DeepReduceConfig.from_params(ok, strict=True)


@pytest.mark.parametrize("bad", [
    dict(TOPK, warmup_ratios=DGC), dict(TOPK, warmup_steps=2),                        # one key without the other
    dict(WU, compressor='none', communicator='allreduce'), dict(WU, compressor='threshold'),
    {k: v for k, v in WU.items() if k != 'compressor'},
    dict(WU, warmup_ratios=[]), dict(WU, warmup_ratios=0.25), dict(WU, warmup_ratios="0.25"),
    dict(WU, warmup_ratios=[0.25, 0.0]), dict(WU, warmup_ratios=[1.5]), dict(WU, warmup_ratios=[-0.1]),
    dict(WU, warmup_ratios=[True]), dict(WU, warmup_ratios=["0.1"]), dict(WU, warmup_ratios=[None]),
    dict(WU, warmup_steps=0), dict(WU, warmup_steps=-1), dict(WU, warmup_steps=1.0), dict(WU, warmup_steps=True),
    dict(WU, warmup_steps="2"),
])
def test_config_rejects(bad):
    with pytest.raises(ConfigError):
        DeepReduceConfig.from_params(bad)
    with pytest.raises(ConfigError):
        deepreduce_from_params(bad)


def test_no_keys_unchanged():
    """Without the keys the parsed config, its params and the sparsifier are what they were."""
    cfg = DeepReduceConfig.from_params(TOPK, strict=True)
    assert cfg.warmup_ratios is None and cfg.warmup_steps is None
    p = cfg.to_params()
    assert "warmup_ratios" not in p and "warmup_steps" not in p
    assert set(p) == set(DeepReduceConfig.from_params(dict(TOPK)).to_params())
    assert warmup_from_params(TOPK) is None
    assert all(cfg.ratio_at(e) == 0.001 for e in (0, 1, 10 ** 6))
    sp = sparsifier_of(deepreduce_from_params(TOPK))
    assert sp.warmup is None
    sp.compress(torch.randn(5000), "w")
    assert sp.exchanges == {}


# ---- schedule ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e,ratio", [(0, 0.25), (2, 0.25), (3, 0.0625), (5, 0.0625), (6, 0.015625), (8, 0.015625),
                                     (9, 0.004), (11, 0.004), (12, 0.001), (13, 0.001), (10 ** 9, 0.001)])
def test_schedule_table(e, ratio):
    cfg = DeepReduceConfig.from_params(WU)
    wu = warmup_from_params(WU)
    assert cfg.ratio_at(e) == ratio == wu.ratio_at(e)
    assert wu.stage(e) == min(e // 3, 4) and wu.n_stages == 5


def test_schedule_one_step_stages():
    wu = warmup_from_params(dict(TOPK, warmup_ratios=[0.5, 0.1], warmup_steps=1))
    assert [wu.ratio_at(e) for e in range(4)] == [0.5, 0.1, 0.001, 0.001]


# ---- per-tensor route ------------------------------------------------------------------------------------------------
SHAPES = {"a": (64, 80), "b": (3000,), "c": (17, 19, 3)}


def _grads(steps, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [{n: torch.randn(s, generator=g) for n, s in SHAPES.items()} for _ in range(steps)]


def _by_hand(params, grads):
    """The specification: a run without the keys whose 'compress_ratio' is set to the stage's ratio before every
    exchange."""
    wu = warmup_from_params(params)
    grc = deepreduce_from_params({k: v for k, v in params.items() if k not in ("warmup_ratios", "warmup_steps")})
    out = []
    for e, step in enumerate(grads):
        sparsifier_of(grc).compress_ratio = wu.ratio_at(e)
        out.append({n: grc.step(t.clone(), n) for n, t in step.items()})
    return out


MEMORIES = [dict(memory='residual'), dict(memory='dgc', momentum=0.9), dict(memory='none'),
            dict(memory='dgc', momentum=0.5, clip_norm=2.0)]


@pytest.mark.parametrize("comp", ["topk", "randomk"])
@pytest.mark.parametrize("mem", MEMORIES, ids=lambda m: "-".join(f"{k}={v}" for k, v in m.items()))
def test_per_tensor_equals_hand_swapped(comp, mem):
    params = dict(WU, compressor=comp, **mem, warmup_steps=2)
    if comp == 'randomk':
        params['communicator'] = 'allreduce'
    grads = _grads(11)
    want = _by_hand(params, grads)
    grc = deepreduce_from_params(params)
    for e, step in enumerate(grads):
        for n, t in step.items():
            got = grc.step(t.clone(), n)
            assert torch.equal(_bits(got), _bits(want[e][n])), (e, n)
    assert sparsifier_of(grc).exchanges == {n: 11 for n in SHAPES}


def test_per_tensor_k_follows_stage():
    grc = deepreduce_from_params(dict(WU, warmup_steps=1))
    x = torch.randn(10000)
    ks = [sparsifier_of(grc).compress(x, "w")[0][0].numel() for _ in range(6)]
    assert ks == [2500, 625, 156, 40, 10, 10]


def test_counts_per_name_and_wrapped_sparsifier():
    """Counts are kept per tensor name; under a DeepReduce codec wrapper the inner sparsifier keeps them."""
    params = dict(WU, deepreduce='index', index='bloom', min_numel=100)
    grc = deepreduce_from_params(params)
    sp = sparsifier_of(grc)
    assert sp is not grc.compressor and sp.warmup is not None
    for _ in range(4):
        grc.step(torch.randn(5000), "x")
    grc.step(torch.randn(5000), "y")
    assert sp.state_dict() == {"exchanges": {"x": 4, "y": 1}}


def test_randomk_seed_counter_untouched():
    params = dict(WU, compressor='randomk', communicator='allreduce')
    a = sparsifier_of(deepreduce_from_params(params))
    b = sparsifier_of(deepreduce_from_params({k: v for k, v in params.items() if not k.startswith("warmup")}))
    for s in (a, b):
        for n in ("p", "q", "p"):
            s.compress(torch.randn(3000), n)
    assert a.global_step == b.global_step == 3


# ---- checkpoints -------------------------------------------------------------------------------------------------------
def _mlp():
    torch.manual_seed(7)
    return nn.Sequential(nn.Linear(64, 96), nn.ReLU(), nn.Linear(96, 48), nn.ReLU(), nn.Linear(48, 8))


def _run(ddp, grads):
    out = []
    for g in grads:
        for (n, p), t in zip(ddp.module.named_parameters(), g):
            p.grad = t.clone()
        ddp.finish()
        out.append([p.grad.clone() for p in ddp.module.parameters()])
    return out


def _mlp_grads(steps):
    gen = torch.Generator().manual_seed(3)
    return [[torch.randn(p.shape, generator=gen) for p in _mlp().parameters()] for _ in range(steps)]


@pytest.mark.parametrize("mem", [dict(memory='residual'), dict(memory='dgc', momentum=0.9, weight_decay=1e-3)],
                         ids=["residual", "dgc"])
@pytest.mark.parametrize("cut", [2, 3, 4])          # at a boundary (2, 4) and mid-stage (3); stages of 2 exchanges
def test_checkpoint_resume_equals_uninterrupted(mem, cut):
    from deepreduce_b200.parallel import DeepReduceDDP
    params = dict(WU, **mem, warmup_steps=2, min_numel=100)
    grads = _mlp_grads(8)
    ref = _run(DeepReduceDDP(_mlp(), params), grads)
    first = DeepReduceDDP(_mlp(), params)
    _run(first, grads[:cut])
    st = first.state_dict()
    assert st["step"] == cut and st["sparsifier"]["exchanges"]["0.weight"] == cut
    resumed = DeepReduceDDP(_mlp(), params)
    resumed.load_state_dict(st)
    got = _run(resumed, grads[cut:])
    for e, (a, b) in enumerate(zip(ref[cut:], got)):
        for x, y in zip(a, b):
            assert torch.equal(_bits(x), _bits(y)), (cut, e)


def test_checkpoint_without_key_loads_at_count_zero():
    from deepreduce_b200.parallel import DeepReduceDDP
    params = dict(WU, min_numel=100)
    old = DeepReduceDDP(_mlp(), {k: v for k, v in params.items() if not k.startswith("warmup")})
    _run(old, _mlp_grads(2))
    st = old.state_dict()
    assert "sparsifier" not in st
    ddp = DeepReduceDDP(_mlp(), params)
    _run(ddp, _mlp_grads(1))
    ddp.load_state_dict(st)
    assert sparsifier_of(ddp.grc).exchanges == {}
    assert ddp.step_count == 2
    # and without the keys the checkpoint keeps its keys
    assert set(st) == {"step", "memory"}


def test_hook_state_records_exchanges():
    """The DDP hook's checkpoint carries the exchange count ('step') and, on the per-tensor route, the counts."""
    from deepreduce_b200.parallel.comm_hook import DeepReduceHookState
    st = DeepReduceHookState(dict(WU, min_numel=100), _mlp())
    st._make_grc()
    for _ in range(3):
        sparsifier_of(st.grc).compress(torch.randn(6144), "0.weight")
    st.step_count = 3
    sd = st.state_dict()
    assert sd["step"] == 3 and sd["sparsifier"] == {"exchanges": {"0.weight": 3}}
    st2 = DeepReduceHookState(dict(WU, min_numel=100), _mlp())
    st2.load_state_dict(sd)
    assert st2.step_count == 3 and sparsifier_of(st2.grc).exchanges == {"0.weight": 3}
    sd.pop("sparsifier")
    st2.load_state_dict(sd)
    assert sparsifier_of(st2.grc).exchanges == {}


# ---- stage plans ---------------------------------------------------------------------------------------------------
RESNETISH = [64 * 3 * 7 * 7, 64, 256 * 64, 256 * 64 * 9, 512 * 256 * 9, 2048 * 512, 1000 * 2048, 1000, 2048 * 1024]


@pytest.mark.parametrize("extra", [dict(deepreduce='index', index='bloom'), dict(deepreduce='index', index='rle'),
                                   dict(), dict(deepreduce='both', index='bloom', value='qsgd'),
                                   dict(compressor='randomk', communicator='allreduce'),
                                   dict(deepreduce='index', index='bloom', policy='conflict_sets', p2_pick_mask=True)],
                         ids=["bloom", "rle", "plain", "bloom-qsgd", "randomk", "p2"])
def test_stage_plans_share_layout(extra):
    params = dict(WU, **extra)
    wu = warmup_from_params(params)
    sn = engine_split_numel(params, 2)
    numels, names, shapes, _ = split_large(RESNETISH, [f"t{i}" for i in range(len(RESNETISH))],
                                           [(n,) for n in RESNETISH], sn)
    plans = stage_plans(numels, names, shapes, params, wu)
    final = BucketPlan(numels, names, shapes, **plan_kwargs_from_params(params))
    assert len(plans) == 5
    for s, pl in enumerate(plans):
        assert pl.compress_ratio == wu.ratio(s)
        assert [t.numel for t in pl.tensors] == [t.numel for t in final.tensors]
        assert [t.elem_off for t in pl.tensors] == [t.elem_off for t in final.tensors]
        assert [t.tile_begin for t in pl.tensors] == [t.tile_begin for t in final.tensors]
        assert pl.total_elems == final.total_elems and pl.n_tiles == final.n_tiles
    assert plans[-1].wire_bytes() == final.wire_bytes()
    assert plans[0].wire_bytes() > plans[1].wire_bytes() > plans[-1].wire_bytes()
    assert [t.k for t in plans[0].tensors] == [max(1, min(t.numel, int(t.numel * 0.25))) for t in final.tensors]


def test_no_warmup_one_plan():
    numels = [5000, 70000]
    plans = stage_plans(numels, ["a", "b"], [(5000,), (70000,)], dict(TOPK, deepreduce='index', index='bloom'), None)
    ref = BucketPlan(numels, ["a", "b"], [(5000,), (70000,)], **plan_kwargs_from_params(dict(TOPK, deepreduce='index',
                                                                                             index='bloom')))
    assert len(plans) == 1 and plans[0].tensor_table().equal(ref.tensor_table())
    assert plans[0].wire_bytes() == ref.wire_bytes()


def test_stage_a_plan_refuses_raises_up_front():
    """P2 draws over at most 2^20 positives per tensor: fine at 0.1 %, refused at 25 %, and refused when the stage
    plans are built, before any exchange."""
    params = dict(WU, deepreduce='index', index='bloom', policy='conflict_sets', p2_pick_mask=True,
                  split_numel=0)
    numels = [8 * 1024 * 1024]
    BucketPlan(numels, ["w"], [(numels[0],)], **plan_kwargs_from_params(params))           # the final ratio is fine
    with pytest.raises(ValueError, match="positives"):
        stage_plans(numels, ["w"], [(numels[0],)], params, warmup_from_params(params))


# ---- Trainer counts exchanges ------------------------------------------------------------------------------------------
def test_trainer_accumulation_counts_exchanges():
    from deepreduce_b200.trainer import Trainer
    model = _mlp()
    tr = Trainer(model, dict(WU, min_numel=100, warmup_steps=2), lr=0.01, amp_dtype=None, accum_steps=2)
    x, y = torch.randn(4, 64), torch.randint(0, 8, (4,))
    for _ in range(6):
        tr.step(x, target=y)
    assert tr.ddp.step_count == 3
    assert set(sparsifier_of(tr.ddp.grc).exchanges.values()) == {3}


# ---- two gloo ranks -------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, params, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from deepreduce_b200.parallel import DeepReduceDDP
    wu = warmup_from_params(params)
    ddp = DeepReduceDDP(_mlp(), params)
    hand = DeepReduceDDP(_mlp(), {k: v for k, v in params.items() if not k.startswith("warmup")})
    gen = torch.Generator().manual_seed(50 + rank)
    same, shipped = True, []
    for e in range(7):
        g = [torch.randn(p.shape, generator=gen) for p in ddp.module.parameters()]
        sparsifier_of(hand.grc).compress_ratio = wu.ratio_at(e)
        sent = ddp.grc.bytes_sent
        a, b = _run(ddp, [g])[0], _run(hand, [g])[0]
        shipped.append(ddp.grc.bytes_sent - sent)
        same = same and all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))
    flat = torch.cat([p.grad.flatten() for p in ddp.module.parameters()])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    ret[rank] = (same, shipped, all(torch.equal(gathered[0], x) for x in gathered))
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("mem", [dict(memory='residual'), dict(memory='dgc', momentum=0.9, clip_norm=1.0)],
                         ids=["residual", "dgc"])
def test_gloo_world2_across_two_boundaries(mem):
    params = dict(TOPK, **mem, compress_ratio=0.01, warmup_ratios=[0.25, 0.0625], warmup_steps=2, min_numel=100)
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), params, ret), nprocs=2, join=True)
    for r in range(2):
        same, shipped, agree = ret[r]
        assert same and agree, r
        # two exchanges per stage, then the final ratio: what a rank ships shrinks at each boundary
        assert shipped[0] == shipped[1] > shipped[2] == shipped[3] > shipped[4] == shipped[5] == shipped[6]
