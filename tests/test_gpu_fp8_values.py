"""FP8 values ('value': 'fp8', VMODE_FP8) in the fused engine and the per-tensor kernels, on the GPU.

The block rule is integer arithmetic, one exact multiply by a power of two and one round-to-nearest-even conversion, so
nothing here is approximate: every shipped slot word, and at W = 1 the output, the residual and the 'dgc' momentum, are
``engine_oracle``'s bit for bit (NaN compared as NaN).  W = 2-16 run in one process through the harness of
``test_engine_multirank.py``.  The conversion instruction itself is checked against torch's CUDA ``float8_e4m3fn``
cast for every fp32 pattern of magnitude at most 448."""
import numpy as np
import pytest
import torch

import bench
import test_engine_multirank as multirank
import test_gpu_comm_hook as hook
from deepreduce_b200.codecs.fp8 import FP8, fp8_decode_oracle, fp8_encode_oracle
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import decode_slot_oracle
from deepreduce_b200.parallel.plan import VMODE_FP8, split_large
from test_gpu_dgc_weight_decay import _placed, _weights, nccl_world1  # noqa: F401
from test_gpu_engine import SIZES, _compare_slot, _fill
from test_train_step_reference import run_case

pytestmark = pytest.mark.gpu
M, WD, C = 0.9, 0.05, 60.0

INDEX = {"plain": dict(index=None), "bloom": dict(index="bloom"),
         "bloom_random": dict(index="bloom", policy="random", fpr=0.02), "bloom_p0": dict(index="bloom", policy="p0"),
         "bloom_p2": dict(index="bloom", policy="conflict_sets"), "rle": dict(index="rle"),
         "elias_fano": dict(index="elias_fano"), "randomk": dict(index=None, sparsifier="randomk")}
SPARSIFIER = {"topk": dict(), "thr_full": dict(sparsifier="threshold", threshold=1.0),
              "thr_partial": dict(sparsifier="threshold", threshold=1.0, capacity_ratio=0.2)}
# index x sparsifier, each with a bucket dtype, a memory and a launch variant so that every pair of the last three
# axes (and each of them with every index) occurs
LAUNCH = [dict(use_tma=True, blocks_per_sm=2), dict(use_tma=False, blocks_per_sm=1),
          dict(use_tma=True, blocks_per_sm=1), dict(use_tma=False, blocks_per_sm=2)]
_AXES = [(d, m, l) for d in (torch.float32, torch.bfloat16) for m in ("residual", "dgc") for l in range(2)]
CASES = []
for _i, _ix in enumerate(INDEX):
    for _j, _sp in enumerate(SPARSIFIER):
        if (_ix in ("bloom_p2", "randomk")) and _sp != "topk":
            continue
        _d, _m, _l = _AXES[(_i + 3 * _j) % len(_AXES)]
        CASES.append(pytest.param(_ix, _sp, _d, _m, LAUNCH[(_l + _i) % 4], id=f"{_ix}-{_sp}-{_d}-{_m}-{(_l + _i) % 4}"))


def _bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


def _same(a, b):
    """Bit-equal fp32 tensors, where a NaN matches any NaN (the device's arithmetic NaN is 0x7FFFFFFF, torch's CPU one
    0x7FC00000)."""
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(_bits(a)[~na], _bits(b)[~nb])


def _same_payload(plan, slot_gpu, slot_ref, tag):
    a = slot_gpu.cpu().numpy().view(np.uint32)[:plan.payload_words]
    if not np.array_equal(a, slot_ref[:plan.payload_words]):
        bad = _compare_slot(plan, slot_gpu, slot_ref, tag)
        where = np.nonzero(a != slot_ref[:plan.payload_words])[0]
        raise AssertionError(f"{tag}: {where.size} slot words differ, first at {where[:8].tolist()}; {bad[:4]}")


def _setup(plan_kw, dtype, sizes=SIZES):
    numels, names, shapes, owner = split_large(sizes, [f"t{i}" for i in range(len(sizes))], [(n,) for n in sizes], 8192)
    plan = BucketPlan(numels, names, shapes, compress_ratio=0.01, value="fp8", **plan_kw)
    gen = torch.Generator().manual_seed(3)
    return plan, owner, [_placed(torch.randn(n, generator=gen).to(dtype).cuda(), i) for i, n in enumerate(sizes)]


@pytest.mark.parametrize("index,sparsifier,dtype,memory,launch", CASES)
def test_engine_vs_oracle_w1(index, sparsifier, dtype, memory, launch):
    plan, owner, params = _setup({**INDEX[index], **SPARSIFIER[sparsifier]}, dtype)
    assert sum(t.vmode == VMODE_FP8 for t in plan.tensors) >= 4
    dgc = memory == "dgc"
    kw = dict(momentum=M, weight_decay=WD, clip_norm=C, owner=owner) if dgc else {}
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, grad_dtype=dtype, spin_limit=2_000_000, **launch, **kw)
    if dgc:
        eng.bind_parameters(params, owner)
    w = _weights(plan, owner, params)
    gen = torch.Generator().manual_seed(11)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    for step in range(3):
        g = (_fill(plan, gen) * (1e-3 if step == 1 else 1.0 + step)).to(dtype).float()
        eng.grad.copy_(g.to(dtype).cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        if dgc:
            out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom,
                                                 weight_decay=WD, weights=[w], clip_norm=C, owner=owner)
        else:
            out, res, slots = engine_oracle(plan, [g], res, epoch=eng.epoch)
        tag = f"{index} {sparsifier} {dtype} {memory} {launch} step {step}"
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


def _f(bits):
    return torch.from_numpy(np.asarray(bits, dtype=np.uint32).view(np.float32).copy())


@pytest.mark.parametrize("index", ["plain", "bloom", "rle", "elias_fano"])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 511, 512, 513, 1025])
def test_engine_edge_values_w1(index, n):
    """n shipped values (every non-zero of a tensor of K = n) holding fp32 subnormals, values near FLT_MAX, values that
    round to 0 beside a large one, and from n > 40 a NaN in block 1 and an inf in the last block, with the 'dgc'
    memory: the blocks' edges and the non-finite rule."""
    plan = BucketPlan([8192, 5000], ks=[n, 50], value="fp8", min_numel=0, **INDEX[index])
    edge = _f([0x00000200, 0x80000201, 0x007FFFFF, 0x807FFFFF, 0x7F7FFFFF, 0xFF77FFFE, 0x00800000,
               0x447A0000, 0x38D1B717, 0xB8D1B717])       # keys >= 2^9; 1000.0 beside +-1e-4, which round to 0
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, momentum=M, spin_limit=2_000_000)
    res, mom = [torch.zeros(plan.total_elems)], [torch.zeros(plan.total_elems)]
    gen = torch.Generator().manual_seed(12 + n)
    t1 = plan.tensors[1]
    for step in range(2):
        g = torch.zeros(plan.total_elems)
        pos = torch.randperm(8192, generator=gen)[:n].sort().values
        v = torch.randn(n, generator=gen)
        m = min(n, edge.numel())
        v[:m] = edge[:m]                                  # block 0 holds the edge values, in this order
        if n > 40:
            v[40] = float("nan") if step == 0 else -float("inf")
            v[-1] = float("inf") if step == 0 else -float("nan")
        g[pos] = v
        g[t1.elem_off:t1.elem_off + t1.numel] = torch.randn(t1.numel, generator=gen)
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, res, slots, mom = engine_oracle(plan, [g], res, epoch=eng.epoch, momentum=M, moms=mom)
        tag = f"{index} n={n} step {step}"
        _same_payload(plan, eng.slot(), slots[0], tag)
        # a NaN that is not shipped stays in the residual and the momentum, where its bits follow the arithmetic
        assert _same(eng.grad, out) and _same(eng.resid, res[0]) and _same(eng.mom, mom[0]), tag
        if n > 40 and step == 0 and index != "bloom":     # bloom also ships false positives: slots != pos
            assert bool(torch.isnan(out[pos[32:64]]).all()) and bool(torch.isfinite(out[pos[64:(n - 1) // 32 * 32]]).all())
    eng.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("index,W,config", [
    ("plain", 2, "shard"), ("bloom", 3, "noshard"), ("bloom_p0", 4, "shard"), ("rle", 3, "nccl"),
    ("elias_fano", 4, "noshard"), ("elias_fano", 16, "shard"), ("randomk", 2, "nccl"), ("bloom", 8, "shard")])
def test_multirank(monkeypatch, index, W, config):
    """Rank-ordered sums (DR_DETERMINISTIC=1) without averaging are the oracle's aggregate bit for bit; the default
    RED.ADD apply is within a few roundings of it and identical on every rank."""
    sizes = SIZES if W <= 5 else multirank.SMALL
    plan = BucketPlan(sizes, compress_ratio=0.01, value="fp8", **INDEX[index])
    gen = torch.Generator().manual_seed(13 + W)
    for det in (True, False):
        monkeypatch.setenv("DR_DETERMINISTIC", "1" if det else "0")
        engs = multirank._engines(plan, W, config, average=not det)
        res = [torch.zeros(plan.total_elems) for _ in range(W)]
        for epoch in range(1, 4):
            grads = [_fill(plan, gen) for _ in range(W)]
            for r in range(W):
                engs[r].grad.copy_(grads[r].cuda())
            multirank._run_step(engs, config, epoch)
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


@pytest.mark.parametrize("K", [1, 31, 33, 127, 128, 129, 511, 512, 513, 1025, 70000, 1_300_001])
def test_per_tensor_kernels_equal_the_cpu_codec(K):
    from deepreduce_b200 import ops
    gen = torch.Generator().manual_seed(K)
    v = torch.randn(K, generator=gen) * torch.exp(torch.randn(K, generator=gen) * 4)
    v[torch.rand(K, generator=gen) < 0.01] = 0.0
    if K > 2000:
        v[1500] = -0.0
        sub = (np.arange(32, dtype=np.uint32) * 261631) | ((np.arange(32, dtype=np.uint32) % 2) << 31)
        v[1600:1632] = _f(sub)                            # block 50: fp32 subnormals and +-0 only
        v[1700] = float("nan")                            # block 53: NaN, the other blocks unaffected
        v[1800] = -float("inf")
        v[1900] = 3.3e38                                  # block 59: its maximum decodes to inf
    sc, ec = fp8_encode_oracle(v)
    sg, eg = ops.fp8_encode(v.cuda())
    assert torch.equal(sg.cpu(), sc) and torch.equal(eg.cpu(), ec), K
    dec = ops.fp8_decode(sg, eg, K)
    assert _same(dec, fp8_decode_oracle(sc, ec, K)), K
    idx = torch.randperm(4 * K, generator=gen)[:K]
    wc, ic, _ = FP8.compress((v, idx, torch.Size([4 * K])), {})
    wg, ig, shape = FP8.compress((v.cuda(), idx.cuda(), torch.Size([4 * K])), {})
    assert torch.equal(wg.cpu(), wc) and torch.equal(ig.cpu(), ic), K
    back, _, _ = FP8.decompress((wg, None, shape), {})
    assert _same(back, FP8.decompress((wc, None, shape), {})[0]), K


@pytest.mark.timeout(600)
def test_conversion_equals_torch_cast_for_every_fp32_pattern():
    """Every fp32 bit pattern of magnitude at most 448 (both signs, +-0, subnormals and 448 itself) goes through the
    encode kernel in blocks whose maximum is 448, so e = 0 and the element byte is the conversion of the value itself;
    it must equal torch's CUDA float8_e4m3fn cast."""
    from deepreduce_b200 import ops
    top = 0x43E00000                                      # 448.0
    rows = 1 << 22                                        # 31 patterns per block, 2^22 blocks per chunk
    per = 31 * rows
    checked = 0
    for neg in (False, True):
        for start in range(0, top + 1, per):
            p = torch.arange(start, min(start + per, top + 1), dtype=torch.int64, device="cuda")
            n = p.numel()
            bits = torch.zeros(per, dtype=torch.int64, device="cuda")
            bits[:n] = p - (1 << 31) if neg else p         # the sign bit set, as an int32 pattern
            x = bits.to(torch.int32).view(torch.float32).view(rows, 31)
            blk = torch.cat([torch.full((rows, 1), 448.0, device="cuda"), x], dim=1).contiguous()
            scales, elems = ops.fp8_encode(blk.view(-1))
            assert bool((scales == 0x7F7F7F7F).all())     # scale byte 127 (e = 0) everywhere
            got = elems.view(torch.uint8).view(rows, 32)[:, 1:]
            want = x.to(torch.float8_e4m3fn).view(torch.uint8)
            bad = torch.nonzero(got.reshape(-1)[:n] != want.reshape(-1)[:n])
            assert bad.numel() == 0, (neg, start, bad[:4].flatten().tolist())
            checked += n
    assert checked == 2 * (top + 1)


# ---- public entry points ------------------------------------------------------------------------------------------
FP8_CFG = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
           'deepreduce': 'both', 'index': 'elias_fano', 'value': 'fp8'}


def _fp8_fused(tr):
    assert tr.ddp.fused and tr.ddp.grc is None
    assert any(t.vmode == VMODE_FP8 for e in tr.ddp.engines for t in e.plan.tensors)


@pytest.mark.timeout(900)
def test_resnet50_train_step(monkeypatch):
    """ResNet-50, batch 16, the benchmark's ``Trainer`` with Elias-Fano + fp8 values against plain torch +
    ``engine_oracle``."""
    monkeypatch.setitem(bench.CONFIGS, "fp8", FP8_CFG)
    run_case(monkeypatch, "image", "fp8", 16, check=_fp8_fused)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("extra", [{'index': 'rle'}, {'index': 'bloom'}], ids=["rle", "bloom"])
def test_ddp_hook_resnet20(monkeypatch, nccl_world1, extra):  # noqa: F811
    """torch DDP + the communication hook on ResNet-20, four steps across DDP's bucket rebuild, against the oracle."""
    monkeypatch.setitem(hook.CONFIGS, "fp8", {**hook.CONFIGS["rle"], 'deepreduce': 'both', 'value': 'fp8', **extra})
    st = hook.run_ddp_case("fp8", "resnet20")
    assert st.fused_params


def test_checkpoint_round_trip():
    """A DeepReduceDDP checkpoint of the fused route with fp8 values; a fresh wrapper that loads it continues bit for
    bit."""
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.parallel import DeepReduceDDP

    def make():
        torch.manual_seed(0)
        m = resnet20().cuda()
        return m, DeepReduceDDP(m, FP8_CFG, bucket_cap_mb=0.5, overlap=False)

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
    assert any(t.vmode == VMODE_FP8 for e in a.engines for t in e.plan.tensors)
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
    """A sparsity warm-up through two stage switches with fp8 values: every exchange's aggregate equals
    ``engine_oracle`` on that stage's plan bit for bit."""
    from deepreduce_b200.config import warmup_from_params
    from deepreduce_b200.parallel import DeepReduceDDP
    from test_gpu_dgc_weight_decay import _ConvNet
    cfg = {**FP8_CFG, 'calibrate_partition': False, 'min_numel': 100, 'warmup_ratios': [0.25, 0.0625],
           'warmup_steps': 2}
    wu = warmup_from_params(cfg)
    torch.manual_seed(0)
    model = _ConvNet().cuda()
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    assert ddp.fused and len(ddp.engines) == 1
    res = [torch.zeros(ddp.engines[0].plan.total_elems)]
    gen = torch.Generator().manual_seed(1)
    caps = []
    for e in range(6):
        eng = ddp.engines[0]
        assert eng.plan.compress_ratio == wu.ratio_at(e)
        assert any(t.vmode == VMODE_FP8 for t in eng.plan.tensors)
        caps.append(tuple(t.val_cap for t in eng.plan.tensors))
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
    assert caps[0] != caps[2] != caps[4]
    ddp.close()
