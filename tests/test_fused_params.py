"""The fused engine away from its default memory settings, K and filter sizes.

* ``beta`` / ``gamma`` of the residual memory: the engine's phase 0 must round ``beta * r + gamma * g`` as torch does
  (three roundings: ``ResidualMemory``, ``engine_oracle``), never as one contracted FMA, and ``'memory': 'none'`` must
  not scale the gradient by ``gamma`` (GRACE's ``NoneMemory`` ignores it).
* K = 1, K = d - 1, K = d and one tile's worth of K, on tensors of 1 to ~10^6 elements, with the selection checked
  against an fp64 sort as well as against the oracle.
* Bloom filters larger than the kernel's SMEM staging buffer, which the query and decode phases probe from L2, and
  the false-positive rate extremes (one hash function; the ``max_hash`` cap).

CPU tests pin the reference side (oracle == per-tensor route, the rounding the kernel must make); the GPU tests
compare the kernel with the oracle word for word over three steps with the residual carried."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import deepreduce_b200 as dr
from deepreduce_b200 import spec
from deepreduce_b200.codecs.bloom import bloom_query_oracle
from deepreduce_b200.parallel import BucketPlan, engine_oracle
from deepreduce_b200.parallel.ddp import engine_kwargs
from deepreduce_b200.parallel.engine import shipped_index_oracle
from deepreduce_b200.parallel.plan import DYN_WORDS, MODE_BLOOM, SLOT_HEADER_WORDS

PAIRS = [(0.9, 1.0), (0.99, 0.5), (0.5, 0.3), (0.9, 0.7)]          # (beta, gamma)
GRACE = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}


def _keys(x):
    """|x| bit patterns (the engine's select keys), int64."""
    return x.contiguous().view(torch.int32).to(torch.int64) & 0x7FFFFFFF


def _prefix_tie(acc, k):
    """True if the K-th and the (K+1)-th largest |acc| share their 22-bit key prefix.  The fused select then ships
    both (DESIGN.md, 'insert'), while the per-tensor top-k ships exactly K: the two routes agree only without a tie."""
    if k >= acc.numel():
        return False
    top = torch.topk(_keys(acc), k + 1, sorted=True).values
    return int(top[k - 1]) >> 9 == int(top[k]) >> 9


# ---------------------------------------------------------------------------
# CPU: the reference side
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("index", ["bloom", None], ids=["bloom", "plain"])
@pytest.mark.parametrize("beta,gamma", PAIRS)
def test_oracle_matches_grace_path_beta_gamma(index, beta, gamma):
    """engine_oracle at beta, gamma != 1 equals the per-tensor GRACE route (ResidualMemory) bit for bit, output and
    residual, over three steps with the residual carried."""
    plan = BucketPlan([36864, 500, 9408], compress_ratio=0.01, hint=False, index=index)
    cfg = dict(GRACE, beta=beta, gamma=gamma)
    if index:
        cfg.update(deepreduce='index', index=index)
    grc = dr.deepreduce_from_params(cfg)
    gen = torch.Generator().manual_seed(4)             # a seed whose steps have no 22-bit tie at K
    res = torch.zeros(plan.total_elems)
    for step in range(3):
        g = torch.zeros(plan.total_elems)
        for v in plan.views(g):
            v.copy_(torch.randn(v.shape, generator=gen))
        acc = beta * res + gamma * g
        for t in plan.tensors:
            assert not _prefix_tie(acc[t.elem_off:t.elem_off + t.numel], t.k), (step, t.name)
        out, resids, _ = engine_oracle(plan, [g], [res], beta=beta, gamma=gamma, epoch=step + 1)
        for t, v, o, r in zip(plan.tensors, plan.views(g), plan.views(out), plan.views(resids[0])):
            ref = grc.step(v.clone().flatten(), t.name)
            assert torch.equal(o.flatten(), ref), (step, t.name)
            assert torch.equal(r.flatten(), grc.memory.residuals[t.name]), (step, t.name)
        res = resids[0]


def test_engine_kwargs_follow_grace_memory():
    """gamma scales the gradient only under 'residual' memory, as GRACE's memories do; beta is 0 without a residual."""
    base = dict(GRACE, deepreduce='index', index='bloom')
    kw = engine_kwargs(dict(base, memory='none', beta=0.9, gamma=0.5))
    assert (kw['beta'], kw['gamma'], kw['momentum']) == (0.0, 1.0, None)
    kw = engine_kwargs(dict(base, memory='residual', beta=0.9, gamma=0.5))
    assert (kw['beta'], kw['gamma'], kw['momentum']) == (0.9, 0.5, None)
    kw = engine_kwargs(dict(base, memory='dgc', momentum=0.8))
    assert (kw['beta'], kw['gamma'], kw['momentum']) == (1.0, 1.0, 0.8)
    assert engine_kwargs(dict(base, average=False))['average'] is False


def test_memory_none_gamma_matches_grace_path():
    """{'memory': 'none', 'gamma': 0.5}: the oracle run with the engine arguments make_engine builds equals the
    per-tensor NoneMemory route, which ignores gamma; the oracle at gamma = 0.5 does not."""
    cfg = dict(GRACE, memory='none', gamma=0.5, deepreduce='index', index='bloom', hint=False)
    kw = engine_kwargs(cfg)
    plan = BucketPlan([36864, 500, 9408], compress_ratio=0.01, hint=False)
    grc = dr.deepreduce_from_params(cfg)
    gen = torch.Generator().manual_seed(3)
    for step in range(2):
        g = torch.zeros(plan.total_elems)
        for v in plan.views(g):
            v.copy_(torch.randn(v.shape, generator=gen))
        zero = torch.zeros_like(g)
        out, _, _ = engine_oracle(plan, [g], [zero], beta=kw['beta'], gamma=kw['gamma'], epoch=step + 1)
        halved, _, _ = engine_oracle(plan, [g], [zero], beta=0.0, gamma=0.5, epoch=step + 1)
        for t, v, o in zip(plan.tensors, plan.views(g), plan.views(out)):
            assert torch.equal(o.flatten(), grc.step(v.clone().flatten(), t.name)), (step, t.name)
        assert not torch.equal(out, halved)


@pytest.mark.parametrize("beta,gamma", [(0.9, 1.0), (0.99, 0.5), (0.5, 0.3), (0.9, 0.7), (1.0, 1.0), (0.5, 0.5)])
def test_phase0_needs_separately_rounded_products(beta, gamma):
    """Why phase 0 spells out __fmul_rn / __fadd_rn.  Left to itself nvcc contracts ``beta * r + gamma * g`` into one
    FMUL and one FFMA: fl(x * c + fl(y * b)), one product rounded and the other fused into the sum (sm_90a, -O3: the
    product with gamma is the fused one).  Emulated in fp64 (the product of two fp32 values is exact there; the sum is
    rounded once more only when it lands on an fp32 rounding boundary), each contraction differs from the oracle's
    fl(fl(beta * r) + fl(gamma * g)) in a large share of the elements when its fused factor is not 0 or a power of
    two, and nowhere when it is.  The three-rounding form computed in fp32 matches the oracle's torch expression."""
    rng = np.random.default_rng(0)
    n = 1_000_000
    r = rng.standard_normal(n).astype(np.float32)
    g = rng.standard_normal(n).astype(np.float32)
    b, c = np.float32(beta), np.float32(gamma)
    oracle = (beta * torch.from_numpy(r) + gamma * torch.from_numpy(g)).numpy().view(np.uint32)
    assert np.array_equal(((b * r) + (c * g)).view(np.uint32), oracle)        # numpy fp32: every operation rounded
    for fused, x, y, other in ((b, r, g, c), (c, g, r, b)):
        fma = (fused.astype(np.float64) * x.astype(np.float64) + (other * y).astype(np.float64)).astype(np.float32)
        n_diff = int((fma.view(np.uint32) != oracle).sum())
        exact = float(fused) == 0.0 or np.frexp(float(fused))[0] == 0.5           # 0 or a power of two
        if exact:
            assert n_diff == 0, (float(fused), n_diff)
        else:
            assert n_diff > n // 10, (float(fused), n_diff)


def _selection_reference(acc, k):
    """Independent of the oracle: the exact top-K of a stable fp64 sort of |acc| (exact zeros and keys with a 22-bit
    prefix of 0, |x| < 2^-140, left out: the select never takes them) and the set the 22-bit rule takes (everything
    whose key prefix is at least the K-th's).  Returns (top-K set, candidate set, K-th prefix)."""
    a = acc.double()
    keys = _keys(acc)
    eligible = torch.nonzero((keys >> 9) > 0).flatten()
    order = eligible[torch.sort(a[eligible].abs(), descending=True, stable=True).indices]
    top = order[:k]
    if top.numel() == 0:
        return set(), set(), None
    kth = int(keys[top[-1]]) >> 9
    cand = torch.nonzero((keys >> 9) >= kth).flatten()
    return set(top.tolist()), set(cand.tolist()), kth


def _check_selection(plan, slot, acc, tag):
    """The shipped index set of every tensor against ``_selection_reference``: every shipped index is a candidate, or
    (bloom) a filter positive; every candidate left of the last shipped index is shipped; when the slot is not full, the
    whole candidate set (so the exact top-K) is shipped."""
    a = slot.cpu().numpy().view(np.uint32)
    for ti, t in enumerate(plan.tensors):
        seg = acc[t.elem_off:t.elem_off + t.numel]
        top, cand, _ = _selection_reference(seg, t.k)
        assert top <= cand, (tag, t.name)
        shipped = shipped_index_oracle(plan, a, ti)
        s = set(shipped.tolist())
        n_sel = int(a[SLOT_HEADER_WORDS + DYN_WORDS * ti])
        assert len(s) == n_sel == shipped.numel(), (tag, t.name)
        if t.mode == MODE_BLOOM:
            words = torch.from_numpy(a[t.off_filter:t.off_filter + t.n_filter_words].view(np.int32).copy())
            pos = set(bloom_query_oracle(words, t.numel, t.n_hash, t.m_bits).tolist())
            assert cand <= pos, (tag, t.name, len(cand - pos))           # every candidate was inserted
            assert s <= pos, (tag, t.name)
        else:
            assert s <= cand, (tag, t.name, sorted(s - cand)[:4])
        last = max(s) if s else -1
        left = {i for i in cand if i <= last}
        if t.mode != MODE_BLOOM or plan.policy in ("leftmost", "p0"):
            assert left <= s, (tag, t.name, sorted(left - s)[:4])
        if n_sel < t.val_cap and (t.mode != MODE_BLOOM or plan.policy in ("leftmost", "p0")):
            assert top <= s and cand <= s, (tag, t.name)


def test_selection_reference_on_the_oracle():
    """The independent selection check agrees with the oracle's slots (K = 1, d - 1, d; ties; tiny non-zeros)."""
    sizes = [1, 31, 4096, 4097, 20000]
    for kw in (dict(index=None), dict(index="bloom"), dict(index="bloom", policy="p0"), dict(index="rle")):
        for ks in ([1] * 5, [max(1, d - 1) for d in sizes], list(sizes)):
            plan = BucketPlan(sizes, ks=ks, min_numel=0, **kw)
            for kind in ("randn", "ties", "tiny"):
                g = _fill_kind(plan, torch.Generator().manual_seed(5), kind)
                _, _, slots = engine_oracle(plan, [g], [torch.zeros_like(g)])
                _check_selection(plan, torch.from_numpy(slots[0].view(np.int32)), g, f"{kw}-{kind}")


def _fill_kind(plan, gen, kind):
    """_fill's kinds plus 'tiny': randn with a tenth of the elements replaced by +-2^-145, non-zeros with a 22-bit key
    prefix of 0 (they stay below 2^-140 after beta, gamma <= 1)."""
    from test_gpu_engine import _fill
    if kind != "tiny":
        return _fill(plan, gen, kind)
    g = _fill(plan, gen, "randn")
    for v in plan.views(g):
        tiny = torch.rand(v.shape, generator=gen) < 0.1
        v[tiny] = torch.where(v[tiny] < 0, -1.0, 1.0) * 2.0 ** -145
    return g


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
def _new_engine(plan, **kw):
    from deepreduce_b200.parallel import BucketEngine
    return BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000, **kw)


def _run_w1(plan, kinds=("randn", "ties", "randn"), *, beta=1.0, gamma=1.0, tma=True, bps=2, seed=0, check_sel=False,
            l2=None):
    """One step per entry of ``kinds`` (the fill of that step) against engine_oracle(beta, gamma), the residual
    carried and the third step shrunk (history fallback).  Exact modes: slot word for word, residual and output bit for
    bit.  Value codecs: the slot within _compare_slot's tolerances and the output near the oracle's; the residual equal to
    the accumulator minus the output, to the bit (polyfit, dexp), or near the oracle's (QSGD).  Returns the last slot and
    accumulator."""
    from test_gpu_engine import _compare_slot
    eng = _new_engine(plan, beta=beta, gamma=gamma, use_tma=tma, blocks_per_sm=bps)
    if l2 is not None:                      # the branch this run must take: a filter in L2 (True) or all in SMEM (False)
        words = (160 if bps < 2 else 80) * 1024 // 4                   # BucketEngine's default filter_smem_bytes / 4
        assert any(t.mode == MODE_BLOOM and t.n_filter_words > words for t in plan.tensors) == l2
    coded = any(t.vmode in (1, 2, 3) for t in plan.tensors)
    fitted = any(t.vmode in (1, 3) for t in plan.tensors)
    gen = torch.Generator().manual_seed(seed)
    resid_ref = torch.zeros(plan.total_elems)
    slot = None
    for step, kind in enumerate(kinds):
        g = _fill_kind(plan, gen, kind) * (0.2 if step == 2 else 1.0)
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        acc = beta * resid_ref + gamma * g if beta != 0.0 else gamma * g
        out_ref, new_res, slots = engine_oracle(plan, [g], [resid_ref], beta=beta, gamma=gamma, epoch=eng.epoch)
        tag = f"w1_{kind}_b{beta}_g{gamma}_tma{int(tma)}_bps{bps}_s{step}"
        slot = eng.slot()
        bad = _compare_slot(plan, slot, slots[0], tag)
        assert not bad, (tag, bad[:4])
        out, res = eng.grad.cpu(), eng.resid.cpu()
        if check_sel:
            _check_selection(plan, slot, acc, tag)
        if not coded:
            assert torch.equal(res, new_res[0]), (tag, int((res != new_res[0]).sum()))
            assert torch.equal(out, out_ref), (tag, int((out != out_ref).sum()))
            resid_ref = new_res[0]
        else:
            sc = float(out_ref.abs().max())
            assert torch.allclose(out, out_ref, atol=2e-3 * sc, rtol=1e-2), tag
            if fitted:
                assert torch.equal(res, acc - out), (tag, int((res != acc - out).sum()))
            else:                                                      # QSGD: _run_vs_oracle's tolerance
                assert torch.allclose(res, new_res[0], atol=2e-3 * sc, rtol=1e-2), tag
            resid_ref = res.clone()
    eng.close()
    return slot, acc


def _sweep_plan(kw):
    from test_gpu_engine import SIZES
    return BucketPlan(SIZES, compress_ratio=0.01, **kw)


S = pytest.param
# (plan keyword arguments, TMA, blocks per SM, bucket dtype)
SWEEP = [
    S(dict(index="bloom"), True, 2, torch.float32, id="bloom-hint-tma-bps2"),
    S(dict(index="bloom", hint=False), False, 1, torch.float32, id="bloom-nohint-cpasync-bps1"),
    S(dict(index="bloom", policy="p0"), True, 1, torch.float32, id="p0-tma-bps1"),
    S(dict(index="bloom", policy="random", fpr=0.02), False, 2, torch.float32, id="random-cpasync-bps2"),
    S(dict(index=None), True, 2, torch.float32, id="plain-tma"),
    S(dict(index="rle"), False, 2, torch.float32, id="rle-cpasync"),
    S(dict(index="bloom", value="qsgd"), True, 2, torch.float32, id="bloom-qsgd"),
    S(dict(index=None, value="bf16"), False, 1, torch.float32, id="plain-bf16values-cpasync-bps1"),
    S(dict(index="bloom", value="polyfit", poly_min_k=300), True, 2, torch.float32, id="bloom-polyfit"),
    S(dict(index="rle", value="dexp", dexp_min_numel=1000), True, 1, torch.float32, id="rle-dexp-bps1"),
    S(dict(index="bloom"), False, 2, torch.bfloat16, id="bf16bucket-bloom-cpasync"),
    S(dict(index="rle"), True, 1, torch.bfloat16, id="bf16bucket-rle-bps1"),
    S(dict(index=None, value="qsgd"), True, 2, torch.bfloat16, id="bf16bucket-plain-qsgd"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("beta,gamma", PAIRS)
@pytest.mark.parametrize("kw,tma,bps,dtype", SWEEP)
def test_beta_gamma_vs_oracle_w1(kw, tma, bps, dtype, beta, gamma):
    """Phase 0 at beta, gamma != 1 (the residual update's three roundings) through every index mode, value codec and
    kernel variant.  bf16 buckets: the engine on g equals the fp32 engine on g.float(), which equals the oracle."""
    plan = _sweep_plan(kw)
    if dtype == torch.float32:
        _run_w1(plan, beta=beta, gamma=gamma, tma=tma, bps=bps)
        return
    from test_gpu_bf16 import _check_pair, _pair
    from test_gpu_engine import _compare_slot, _fill
    e16, e32 = _pair(plan, use_tma=tma, blocks_per_sm=bps, beta=beta, gamma=gamma)
    gen = torch.Generator().manual_seed(7)
    resid_ref = torch.zeros(plan.total_elems)
    coded = plan.tensors and any(t.vmode in (1, 2, 3) for t in plan.tensors)
    for step in range(3):
        g = (_fill(plan, gen) * (0.2 if step == 2 else 1.0)).to(torch.bfloat16)
        e16.grad.copy_(g.cuda())
        e32.grad.copy_(g.float().cuda())
        e16.step()
        e32.step()
        torch.cuda.synchronize()
        tag = f"bf16 {kw} b{beta} g{gamma} s{step}"
        _check_pair(e16, e32, tag)
        out_ref, new_res, slots = engine_oracle(plan, [g.float()], [resid_ref], beta=beta, gamma=gamma, epoch=e32.epoch)
        assert not _compare_slot(plan, e32.slot(), slots[0], tag.replace(" ", "_"))
        if coded:                                                      # QSGD here: _run_vs_oracle's tolerance
            sc = float(out_ref.abs().max())
            assert torch.allclose(e32.resid.cpu(), new_res[0], atol=2e-3 * sc, rtol=1e-2), tag
            resid_ref = e32.resid.cpu().clone()
        else:
            assert torch.equal(e32.resid.cpu(), new_res[0]) and torch.equal(e32.grad.cpu(), out_ref), tag
            resid_ref = new_res[0]
    e16.close()
    e32.close()


EDGE_SIZES = [1, 31, 4096, 4097, 1000000]
EDGE_MODES = [S(dict(index=None), id="plain"), S(dict(index="bloom"), id="bloom"),
              S(dict(index="bloom", policy="p0"), id="p0"), S(dict(index="bloom", policy="random"), id="random"),
              S(dict(index="rle"), id="rle")]
EDGE_KS = {"k1": [1] * 5, "kd-1": [max(1, d - 1) for d in EDGE_SIZES], "kd": None, "ktile": [min(d, spec.TILE) for d in EDGE_SIZES]}


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("k_case", list(EDGE_KS))
@pytest.mark.parametrize("kw", EDGE_MODES)
def test_k_extremes_vs_oracle_and_fp64_sort(kw, k_case):
    """K = 1, d - 1, d (compress_ratio 1.0) and one tile's worth, on one-tile and multi-tile tensors, with exact
    ties (K = d then ships fewer than K: exact zeros are never selected), sparse input and non-zeros below 2^-140.
    Against the oracle and against the fp64-sort reference of the selection."""
    ks = EDGE_KS[k_case]
    plan = (BucketPlan(EDGE_SIZES, compress_ratio=1.0, min_numel=0, **kw) if ks is None
            else BucketPlan(EDGE_SIZES, ks=ks, min_numel=0, **kw))
    if ks is None:
        assert [t.k for t in plan.tensors] == EDGE_SIZES
    slot, acc = _run_w1(plan, ["randn", "ties", "sparse", "tiny"], beta=0.9, gamma=0.5, check_sel=True, seed=1)
    if k_case == "kd":                   # the 'tiny' step: K = d non-zeros, those below 2^-140 never selected
        a = slot.cpu().numpy().view(np.uint32)
        t = plan.tensors[-1]
        seg = acc[t.elem_off:t.elem_off + t.numel]
        n_big = int((seg.abs() >= 2.0 ** -140).sum())
        assert int((seg != 0).sum()) == t.k and n_big < t.k
        if t.mode != MODE_BLOOM:
            assert int(a[SLOT_HEADER_WORDS + DYN_WORDS * (len(EDGE_SIZES) - 1)]) == n_big


BIG_FILTER = 1310720                     # at ratio 0.1: 39 261 filter words, between the 2- and 1-CTA/SM SMEM limits


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kw", [S(dict(index="bloom"), id="leftmost"), S(dict(index="bloom", hint=False), id="nohint"),
                                S(dict(index="bloom", policy="p0"), id="p0"),
                                S(dict(index="bloom", policy="random"), id="random"),
                                S(dict(index="bloom", value="qsgd"), id="qsgd")])
def test_filter_beyond_smem_w1(kw):
    """Filters that do not fit the SMEM staging buffer: the same plan at 2 CTAs/SM (filter probed from L2) and at
    1 CTA/SM (from SMEM) must both equal the oracle; K = d on 10^6 elements fits neither."""
    plan = BucketPlan([BIG_FILTER, 4097], compress_ratio=0.1, **kw)
    assert plan.tensors[0].n_filter_words == 39261
    for bps, l2 in ((2, True), (1, False)):
        _run_w1(plan, beta=0.9, gamma=0.5, bps=bps, l2=l2)
    if kw.get("value"):
        # QSGD at K = d: _compare_slot admits n_sel / 2000 level flips (fp32 vs fp64 norms), each of which moves one
        # output by a whole level, more than the output tolerance; the 39 261-word plan above covers the codec
        return
    plan = BucketPlan([1000000], compress_ratio=1.0, **kw)
    assert plan.tensors[0].n_filter_words > 40960
    for bps in (2, 1):
        _run_w1(plan, ["randn", "sparse", "randn"], bps=bps, l2=True)


M = pytest.param
MR_FILTER = [
    M("shard", 2, dict(index="bloom"), False, id="shard-W2-fast"),
    M("shard", 3, dict(index="bloom"), True, id="shard-W3-det"),
    M("shard", 4, dict(index="bloom", policy="p0"), False, id="shard-p0-W4-fast"),
    M("shard", 4, dict(index="bloom", hint=False), True, id="shard-nohint-W4-det"),
    M("noshard", 3, dict(index="bloom"), False, id="noshard-W3"),
    M("nccl", 2, dict(index="bloom", policy="random"), False, id="nccl-random-W2"),
    M("nccl", 4, dict(index="bloom"), True, id="nccl-W4-det"),
]


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("config,W,kw,deterministic", MR_FILTER)
def test_filter_beyond_smem_multirank(monkeypatch, config, W, kw, deterministic):
    """The decode side of the L2 branch (W > 1): test_engine_multirank's harness and checks (every slot, delivery,
    the aggregate against the decode of the shipped slots, identical bits on every rank, the stage-2 lists) on a plan
    with a 39 261-word filter and a K = d filter of 149 767 words, both above the 2-CTA/SM limit of 20 480."""
    from test_engine_multirank import test_engine_multirank_vs_oracle
    sizes = [64, 4097, 36864, BIG_FILTER, 1000000]
    ks = [spec.topk_k(d, 0.01) for d in sizes[:3]] + [spec.topk_k(BIG_FILTER, 0.1), 1000000]
    plan = BucketPlan(sizes, ks=ks, **kw)
    assert sum(t.n_filter_words > 80 * 1024 // 4 for t in plan.tensors if t.mode == MODE_BLOOM) == 2
    test_engine_multirank_vs_oracle(monkeypatch, config, W, sizes, dict(kw, ks=ks), deterministic, True, None, set())


FPR_CASES = [S(dict(policy="leftmost"), id="leftmost"), S(dict(policy="leftmost", hint=False), id="leftmost-nohint"),
             S(dict(policy="p0"), id="p0"), S(dict(policy="random"), id="random")]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("fpr", [0.5, 1e-6])
@pytest.mark.parametrize("kw", FPR_CASES)
def test_fpr_extremes(monkeypatch, kw, fpr):
    """fpr = 0.5 (one hash function, false positives far beyond K: the leftmost cutoff, the p0 capacity, the random
    acceptance threshold, the hint) and fpr = 1e-6 (n_hash capped at max_hash = 16), at W = 1 and W = 2."""
    from test_engine_multirank import test_engine_multirank_vs_oracle
    from test_gpu_engine import SIZES
    plan = _sweep_plan(dict(kw, index="bloom", fpr=fpr))
    hashes = {t.n_hash for t in plan.tensors if t.mode == MODE_BLOOM}
    assert hashes == ({1} if fpr == 0.5 else {16}), hashes
    _run_w1(plan, ["randn", "sparse", "randn"], beta=0.9, gamma=0.5, check_sel=True)
    test_engine_multirank_vs_oracle(monkeypatch, "shard", 2, SIZES, dict(kw, index="bloom", fpr=fpr), False, True,
                                    None, set())


class _MLP(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(32, 64)                  # weights of 2 048 and 3 072 elements take the bloom index, the
        self.b = nn.Linear(64, 48)                  # rest plain pairs; small enough that a 22-bit tie at K is rare
        self.c = nn.Linear(48, 10)

    def forward(self, x):
        return self.c(torch.relu(self.b(torch.relu(self.a(x)))))


@pytest.mark.gpu
@pytest.mark.parametrize("memory", ["residual", "none"])
def test_ddp_fused_matches_grace_route(memory):
    """DeepReduceDDP on CUDA (the fused route) with beta = 0.9, gamma = 0.5: every p.grad equals, bit for bit, what the
    per-tensor GRACE route computes from the same gradients with the same dict, over three steps."""
    from deepreduce_b200.parallel import DeepReduceDDP
    from deepreduce_b200.parallel.ddp import fused_path
    cfg = dict(GRACE, memory=memory, beta=0.9, gamma=0.5, deepreduce='index', index='bloom', hint=False,
               calibrate_partition=False)
    assert fused_path(cfg)
    torch.manual_seed(0)
    model = _MLP().cuda()
    ref = _MLP().cuda()
    ref.load_state_dict(model.state_dict())
    ddp = DeepReduceDDP(model, cfg, overlap=False)
    assert ddp.fused and len(ddp.engines) == 1
    grc = dr.deepreduce_from_params(cfg)
    gen = torch.Generator(device="cuda").manual_seed(1)
    for step in range(3):
        x = torch.randn(64, 32, device="cuda", generator=gen)
        y = torch.randint(0, 10, (64,), device="cuda", generator=gen)
        ddp.zero_grad()
        nn.functional.cross_entropy(model(x), y).backward()
        ref.zero_grad()
        nn.functional.cross_entropy(ref(x), y).backward()
        for (n, p), q in zip(model.named_parameters(), ref.parameters()):
            assert torch.equal(p.grad, q.grad), (step, n)              # the same local gradients go in
        ddp.finish()
        for (n, p), q in zip(model.named_parameters(), ref.parameters()):
            g = q.grad.detach().cpu().flatten()
            if memory == 'residual' and n in grc.memory.residuals:    # the route agrees only without a 22-bit tie
                acc = 0.9 * grc.memory.residuals[n] + 0.5 * g
            else:
                acc = 0.5 * g if memory == 'residual' else g
            k = spec.topk_k(g.numel(), 0.01)
            assert not _prefix_tie(acc, min(k, g.numel())), (step, n)
            want = grc.step(g.clone(), n).view_as(p)
            assert torch.equal(p.grad.cpu(), want), (step, n, int((p.grad.cpu() != want).sum()))
    ddp.close()
