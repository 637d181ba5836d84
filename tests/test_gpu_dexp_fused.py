"""Double-exponential values in the fused engine ('fused_dexp') on the GPU, against the oracle.

Every shipped word of the kernel's slot equals the oracle's (headers, rank map, {num_pos, n}, indices, fp32 values of
the uncoded tensors) except the eight coefficient words of each 'dexp' tensor: the kernel's fp64 sums run in another
order than torch's, so each run's curve is compared within the tolerance of test_dexp_fit_vs_fp64_oracle.  At W = 1
the residual is v - fitted to the bit, where fitted is the output, i.e. the decode of the engine's own slot.  Also:
``ops.dexp_fit`` against the bits the per-tensor kernel gave before the regression moved into dexp_fit.cuh."""
import os

import numpy as np
import pytest
import torch

import test_engine_multirank as multirank
import test_gpu_comm_hook as hook
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import decode_slot_oracle, shipped_index_oracle
from deepreduce_b200.parallel.plan import DEXP_COEF_WORDS, MODE_BLOOM, MODE_RAW, MODE_RLE
from test_gpu_codec_kernels import _gen
from test_gpu_engine import SIZES, _fill
from test_gpu_fused_values import _acc, _grad, _rank_map, _rng, _step_both

pytestmark = pytest.mark.gpu
F = np.float32
BIG = SIZES + [2359296]
INDEX = {None: MODE_RAW, "bloom": MODE_BLOOM, "rle": MODE_RLE}


# ---------------------------------------------------------------------------
# the per-tensor kernel keeps its bits
# ---------------------------------------------------------------------------
def test_dexp_fit_kernel_bits_unchanged():
    """ops.dexp_fit on the seeded inputs of test_gpu_codec_kernels (random |randn| and an exact double exponential
    at K = 2 ... 10^6, then K = 1, a constant and zeros) returns the bits recorded from the kernel as it was before
    its body became the shared block function (tests/golden/dexp_fit_parent.npy).  One row moves on purpose: random
    data at K = 2, where p == q.  The old kernel solved the singular 2x2 system for a, b through the rounding residue
    of a contracted determinant (a == b, a curve through neither point); it now takes the one-exponential fallback
    a = sum(e^{px} y) / sum(e^{2px}), b = 0, as the oracle does.  p and q keep their bits."""
    from deepreduce_b200 import ops
    ops.require()
    want = np.load(os.path.join(os.path.dirname(__file__), "golden", "dexp_fit_parent.npy"))
    ys = []
    for K in [2, 1023, 1024, 1025, 2049, 1_000_000]:
        ys.append(torch.sort(torch.randn(K, generator=_gen("dexp", K)).abs()).values)
        x = np.arange(1, K + 1, dtype=np.float64) / K
        ys.append(torch.from_numpy(2.0 * np.exp(3.0 * x) - 0.5 * np.exp(-1.0 * x)).float())
    ys += [torch.tensor([0.37]), torch.full((3000,), 0.37), torch.zeros(3000)]
    got = np.stack([ops.dexp_fit(y.cuda()).cpu().numpy() for y in ys])
    assert np.array_equal(got[1:].view(np.uint64), want[1:].view(np.uint64)), np.flatnonzero(got[1:] != want[1:])
    a, b, p, q = got[0]
    assert want[0][2] == want[0][3] and np.array_equal(got[0][2:].view(np.uint64), want[0][2:].view(np.uint64))
    e = np.exp(p * np.array([0.5, 1.0]))
    assert b == 0.0 and abs(a - (e * ys[0].double().numpy()).sum() / (e * e).sum()) <= 1e-14 * abs(a), got[0]


# ---------------------------------------------------------------------------
# slot against the oracle
# ---------------------------------------------------------------------------
def _curve(c, n):
    a, b, p, q = (float(t) for t in c)
    x = np.arange(1, n + 1, dtype=np.float64) / n
    return a * np.exp(p * x) + b * np.exp(q * x)


def compare_dexp_slot(plan, slot_gpu, slot_ref, tag=""):
    """[] if the kernel's slot matches the oracle's: every shipped word exact except the 'dexp' coefficients, whose
    curves (fp64, from the shipped fp32 words) agree to 1e-3 relative and 1e-4 of the run's largest magnitude.  Runs
    shorter than 3 are underdetermined (test_dexp_fit_vs_fp64_oracle): only finiteness is required there."""
    a = (slot_gpu.cpu().numpy() if torch.is_tensor(slot_gpu) else np.asarray(slot_gpu)).view(np.uint32)
    b = np.asarray(slot_ref, dtype=np.uint32)
    P = plan.payload_words
    mask = np.ones(P, bool)
    bad = []
    for t in plan.tensors:
        if t.vmode != 3:
            continue
        mask[t.off_coef:t.off_coef + DEXP_COEF_WORDS] = False
        ca = a[t.off_coef:t.off_coef + DEXP_COEF_WORDS].view(np.float32)
        cb = b[t.off_coef:t.off_coef + DEXP_COEF_WORDS].view(np.float32)
        num_pos, n = int(b[t.off_coef + DEXP_COEF_WORDS]), int(b[t.off_coef + DEXP_COEF_WORDS + 1])
        if not np.isfinite(ca).all():
            bad.append(f"{t.name} non-finite coefficients {ca}")
            continue
        for r, ln in ((0, num_pos), (1, n - num_pos)):
            if ln < 3:
                continue
            fa, fb = _curve(ca[4 * r:4 * r + 4], ln), _curve(cb[4 * r:4 * r + 4], ln)
            scale = float(np.abs(fb).max())
            if not np.allclose(fa, fb, rtol=1e-3, atol=1e-4 * scale):
                bad.append(f"{t.name} run {r} (len {ln}) curve max diff {float(np.abs(fa - fb).max())} scale {scale}: "
                           f"gpu {ca[4 * r:4 * r + 4]} ref {cb[4 * r:4 * r + 4]}")
    diff = np.flatnonzero((a[:P] != b[:P]) & mask)
    if diff.size:
        bad.append(f"{diff.size} shipped words differ, first at {diff[:8].tolist()}")
    return bad


def _check_w1(plan, eng, acc, tag):
    """W = 1: output and residual of the engine's own slot.  The output is the decode of that slot (the receiver's
    evaluation); the residual on the shipped set is v - output to the bit, elsewhere acc itself."""
    slot = eng.slot().cpu()
    out = eng.grad.float().cpu()
    res = eng.resid.cpu()
    ref = decode_slot_oracle(plan, slot)
    sc = float(ref.abs().max())
    bf16 = eng.grad.dtype == torch.bfloat16
    assert torch.allclose(out, ref, rtol=2.0 ** -8 if bf16 else 1e-6, atol=1e-6 * sc), tag
    shipped = torch.zeros(plan.total_elems, dtype=torch.bool)
    for ti, t in enumerate(plan.tensors):
        shipped[t.elem_off + shipped_index_oracle(plan, slot, ti)] = True
    assert torch.equal(res[~shipped], acc[~shipped]), tag
    coded = torch.zeros(plan.total_elems, dtype=torch.bool)
    for t in plan.tensors:
        if t.vmode == 3:
            coded[t.elem_off:t.elem_off + t.numel] = True
    m = shipped & coded
    if not bf16:
        assert bool((res[m] == acc[m] - out[m]).all()), (tag, int((res[m] != acc[m] - out[m]).sum()))
    else:   # the bf16 output is rounded once from the fitted value; the residual keeps v - fitted in fp32
        assert torch.allclose(acc[m] - res[m], ref[m], rtol=1e-6, atol=1e-6 * sc), tag
    assert bool(torch.isfinite(res).all()) and bool(torch.isfinite(out).all()), tag


def _run_single(plan, tag, steps=3, bf16=False, **kw):
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000,
                       grad_dtype=torch.bfloat16 if bf16 else torch.float32, **kw)
    gen = torch.Generator().manual_seed(0)
    resid = torch.zeros(plan.total_elems)
    try:
        for step in range(steps):
            g = _fill(plan, gen) * (0.2 if step == 2 else 1.0)
            if bf16:
                g = g.bfloat16().float()
            acc = resid + g
            eng.grad.copy_(g.to(eng.grad.dtype).cuda())
            (eng.run_unfused if step == 1 else eng.step)()
            torch.cuda.synchronize()
            eng.check_status()
            _, _, slots = engine_oracle(plan, [g], [resid], epoch=eng.epoch)
            bad = compare_dexp_slot(plan, eng.slot(), slots[0], f"{tag}_s{step}")
            assert not bad, bad[:4]
            _check_w1(plan, eng, acc, f"{tag}_s{step}")
            resid = eng.resid.cpu().clone()          # follow the GPU trajectory
    finally:
        eng.close()


P = pytest.param
SINGLE = [
    P("topk", "rle", "leftmost", {}, id="topk-rle"),
    P("topk", "bloom", "leftmost", {}, id="topk-bloom-leftmost"),
    P("topk", "bloom", "random", dict(fpr=0.02), id="topk-bloom-random"),
    P("topk", "bloom", "p0", {}, id="topk-bloom-p0"),
    P("topk", "bloom", "conflict_sets", {}, id="topk-bloom-p2mask"),
    P("topk", None, "leftmost", {}, id="topk-value"),
    P("threshold", "rle", "leftmost", dict(threshold=1.5, capacity_ratio=0.05), id="threshold-rle"),
    P("threshold", "bloom", "leftmost", dict(threshold=1.5, capacity_ratio=0.05), id="threshold-bloom"),
    P("threshold", None, "leftmost", dict(threshold=2.0, capacity_ratio=0.05), id="threshold-value"),
]


@pytest.mark.parametrize("sparsifier,index,policy,kw", SINGLE)
def test_single_rank_vs_oracle(sparsifier, index, policy, kw):
    """W = 1, three steps (the second through the unfused phase chain), fp32 buckets."""
    plan = BucketPlan(BIG, compress_ratio=0.01, index=index, policy=policy, value="dexp", sparsifier=sparsifier, **kw)
    assert sum(t.vmode == 3 for t in plan.tensors) >= 3 and any(t.mode == INDEX[index] and t.vmode for t in plan.tensors)
    _run_single(plan, f"dexp_{sparsifier}_{index}_{policy}")


@pytest.mark.parametrize("index,bps", [("rle", 2), ("bloom", 1), (None, 2)])
def test_single_rank_bf16_bucket(index, bps):
    plan = BucketPlan(BIG, compress_ratio=0.01, index=index, value="dexp")
    _run_single(plan, f"dexp_bf16_{index}", bf16=True, blocks_per_sm=bps)


# ---------------------------------------------------------------------------
# degenerate runs, and a non-finite tensor
# ---------------------------------------------------------------------------
# (id, K, num_pos, values, index, signed zeros with beta = 0)
DEGENERATE = [
    P(600, 0, "randn", "rle", False, id="no-positives"),
    P(600, 600, "randn", None, False, id="no-rest"),
    P(600, 1, "randn", "rle", False, id="pos-len1"),
    P(600, 2, "randn", None, False, id="pos-len2"),
    P(600, 599, "randn", "rle", False, id="rest-len1"),
    P(600, 598, "randn", None, False, id="rest-len2"),
    P(4097, 2000, "equal", "rle", False, id="all-equal"),
    P(3000, 3000, "randn", "bloom", True, id="rest-all-signed-zeros"),
    P(3000, 1500, "randn", "bloom", True, id="signed-zeros-among-negatives"),
]


@pytest.mark.parametrize("K,num_pos,kind,index,signed_zeros", DEGENERATE)
def test_degenerate_runs(K, num_pos, kind, index, signed_zeros):
    """Runs of length 0, 1 and 2, all equal values, and runs of exact zeros of both signs (bloom false positives
    with beta = 0): finite coefficients, finite output, the rank map the stable descending sort, the residual
    v - output to the bit."""
    d = 200_000
    plan = BucketPlan([d], ks=[K], index=index, value="dexp", fpr=0.05 if index == "bloom" else None)
    t = plan.tensors[0]
    assert t.vmode == 3 and t.mode == INDEX[index]
    g = _grad(plan, d, K, num_pos, kind, ("dexp", K, num_pos, kind, index), signed_zeros=signed_zeros)
    beta = 0.0 if signed_zeros else 1.0
    a, out, res = _step_both(plan, g, beta=beta)
    acc = _acc(g, beta)
    idx = shipped_index_oracle(plan, a, 0).numpy()
    v = acc[idx]
    n = idx.size
    coef = a[t.off_coef:t.off_coef + DEXP_COEF_WORDS].view(np.float32)
    assert np.isfinite(coef).all(), coef
    assert [int(a[t.off_coef + 8]), int(a[t.off_coef + 9])] == [int((v > 0).sum()), n]
    order = torch.sort(torch.from_numpy(v.astype(np.float64)), descending=True, stable=True).indices.numpy()
    assert np.array_equal(_rank_map(a, t, n)[order], np.arange(n))
    assert np.isfinite(out).all() and np.isfinite(res).all()
    assert np.all(res[idx] == v - out[idx])
    if signed_zeros:
        z = v == 0
        assert z.sum() >= 10 and (z & np.signbit(v)).sum() >= 1, int(z.sum())
        if num_pos == K:                   # the non-positive run is all zeros: so is its curve
            assert not coef[4:].any() and not out[idx][z].any()
    if kind == "equal":
        for r, ln in ((0, num_pos), (1, n - num_pos)):
            assert np.abs(_curve(coef[4 * r:4 * r + 4], ln) - 0.37).max() <= 1e-6


def test_nonfinite_tensor_is_isolated():
    """NaN, +-inf and -0.0 among tensor 0's values: the step finishes with a clean status, tensors 1 and 2 get the
    bits they get next to a finite tensor 0, and tensor 0's rank map is still a permutation."""
    sizes, ks = [20_000, 30_000, 40_000], [600, 700, 800]
    plan = BucketPlan(sizes, ks=ks, index="bloom", value="dexp")
    assert all(t.vmode == 3 for t in plan.tensors)
    rnd = torch.from_numpy(_rng("iso", "dexp").standard_normal(plan.total_elems).astype(F))
    g = torch.zeros(plan.total_elems)
    for t in plan.tensors:
        g[t.elem_off:t.elem_off + t.numel] = rnd[t.elem_off:t.elem_off + t.numel]
    bad = g.clone()
    t0 = plan.tensors[0]
    bad[t0.elem_off + torch.tensor([5, 77, 900, 4000, 4001])] = torch.tensor([float("nan"), float("inf"), -float("inf"),
                                                                               float("nan"), -0.0])
    _, out_ok, res_ok = _step_both(plan, g, check_unfused=False, beta=0.0)
    a, out_bad, res_bad = _step_both(plan, bad, check_unfused=False, beta=0.0)
    for t in plan.tensors[1:]:
        seg = slice(t.elem_off, t.elem_off + t.numel)
        assert np.array_equal(out_ok[seg].view(np.uint32), out_bad[seg].view(np.uint32)), t.name
        assert np.array_equal(res_ok[seg].view(np.uint32), res_bad[seg].view(np.uint32)), t.name
    idx = shipped_index_oracle(plan, a, 0).numpy()
    assert {5, 77, 900, 4000} <= set(idx.tolist())
    assert np.array_equal(np.sort(_rank_map(a, t0, idx.size)), np.arange(idx.size))


# ---------------------------------------------------------------------------
# W = 2, 3, 4 ranks in one process
# ---------------------------------------------------------------------------
C = pytest.param
MR_CASES = [
    C("shard", 2, BIG, dict(index="rle"), False, True, 1, {"rle"}, id="shard-rle-W2-fast"),
    C("shard", 3, SIZES, dict(index="bloom"), True, True, None, {"split"}, id="shard-bloom-W3-det"),
    C("shard", 4, SIZES, dict(index=None), False, False, None, set(), id="shard-value-W4-fast-sum"),
    C("noshard", 3, SIZES, dict(index="rle"), False, True, 0, {"rle"}, id="noshard-rle-W3-fast"),
    C("nccl", 2, SIZES, dict(index="bloom", policy="p0"), True, True, None, set(), id="nccl-p0-W2-det"),
]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config,W,sizes,kw,deterministic,average,zero_rank,claims", MR_CASES)
def test_multirank_vs_oracle(monkeypatch, config, W, sizes, kw, deterministic, average, zero_rank, claims):
    """W ranks on one GPU (test_engine_multirank's harness): slots against engine_oracle as above, delivery of every
    slot, the aggregate against decode_slot_oracle of the shipped slots, identical bits on every rank and (sharded)
    the stage-2 lists."""
    plan_kw = dict(kw, value="dexp")
    assert any(t.vmode == 3 for t in BucketPlan(sizes, compress_ratio=0.01, **plan_kw).tensors)
    monkeypatch.setattr(multirank, "_compare_slot", compare_dexp_slot)
    multirank.test_engine_multirank_vs_oracle(monkeypatch, config, W, sizes, plan_kw, deterministic, average,
                                              zero_rank, claims)


# ---------------------------------------------------------------------------
# the DDP communication hook, and its checkpoint
# ---------------------------------------------------------------------------
RLE_DEXP = {**hook.CONFIGS["rle"], 'deepreduce': 'both', 'value': 'dexp', 'fused_dexp': True}


@pytest.mark.timeout(600)
def test_ddp_hook_vs_oracle(monkeypatch, nccl_world1):
    """torch DDP + the hook on the MLP (two 'dexp' tensors), four steps across DDP's bucket rebuild."""
    monkeypatch.setitem(hook.CONFIGS, "rle_dexp", dict(RLE_DEXP))
    from deepreduce_b200.parallel.ddp import plan_kwargs_from_params
    plan = BucketPlan([p.numel() for p in hook.MLP().parameters()], **plan_kwargs_from_params(RLE_DEXP))
    assert sum(t.vmode == 3 for t in plan.tensors) == 2
    st = hook.run_ddp_case("rle_dexp", "mlp")
    assert st.fused_params


@pytest.mark.timeout(600)
def test_ddp_hook_state_dict_round_trip(nccl_world1):
    """Two steps, a checkpoint, a fresh hook at another bucket size that loads it: the third step's gradients and
    residuals equal those of the run that kept going."""
    from torch.nn.parallel import DistributedDataParallel as DDP

    from deepreduce_b200.parallel import register_deepreduce_hook

    def make(cap):
        m = hook._model("mlp", torch.float32, False)
        d = DDP(m, device_ids=[0], bucket_cap_mb=cap)
        return m, d, register_deepreduce_hook(d, dict(RLE_DEXP))

    def step(m, d, s):
        for p in m.parameters():
            p.grad = None
        d(hook._inputs("mlp", s, 0, torch.float32)).pow(2).mean().backward()
        torch.cuda.synchronize()
        return {n: p.grad.clone() for n, p in m.named_parameters()}

    ma, da, sa = make(0.01)
    mb, db, sb = make(25.0)
    try:
        for s in range(2):
            step(ma, da, s)
        assert any(t.vmode == 3 for e in sa.engines for t in e.plan.tensors)
        ckpt = sa.state_dict()
        sb.load_state_dict(ckpt)
        ga, gb = step(ma, da, 2), step(mb, db, 2)
        for n in ga:
            assert torch.equal(ga[n], gb[n]), n
        ra, rb = sa.state_dict()["residuals"], sb.state_dict()["residuals"]
        for n in ra:
            assert torch.equal(ra[n], rb[n]), n
    finally:
        sa.close()
        sb.close()


nccl_world1 = hook.nccl_world1
