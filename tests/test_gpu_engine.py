"""sm_90a kernels vs the plain-torch oracle (GPU).  SURVEY §4 "Golden parity":
set equality for S~ / bit-exact slots, allclose for values."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from deepreduce_b200 import spec

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_OUT = []


def _out_dir():
    """Diagnostics and timings of this test run: a fresh private directory outside the tree, made on first use."""
    if not _OUT:
        _OUT.append(tempfile.mkdtemp(prefix="deepreduce_b200_tests_"))
        print(f"[tests] diagnostics in {_OUT[0]}")
    return _OUT[0]


def _diag(name, text):
    with open(os.path.join(_out_dir(), f"diag_{name}.txt"), "a") as f:
        f.write(text + "\n")


def _fill(plan, gen, kind="randn"):
    g = torch.zeros(plan.total_elems)
    for v in plan.views(g):
        if kind == "randn":
            v.copy_(torch.randn(v.shape, generator=gen))
        elif kind == "sparse":          # mostly zeros -> threshold 0, massive ties
            x = torch.randn(v.shape, generator=gen)
            x[torch.rand(v.shape, generator=gen) < 0.997] = 0
            v.copy_(x)
        elif kind == "ties":            # few distinct magnitudes
            v.copy_(torch.randint(-3, 4, v.shape, generator=gen).float())
    return g


def _compare_slot(plan, slot_gpu, slot_ref, tag):
    bad = []
    a = slot_gpu.cpu().numpy().view(np.uint32)
    b = slot_ref
    from deepreduce_b200.parallel.plan import SLOT_HEADER_WORDS, DYN_WORDS, MODE_BLOOM, MODE_RLE, rle_stream_words
    if not np.array_equal(a[:5], b[:5]):
        bad.append(f"header {a[:5]} vs {b[:5]}")
    for ti, t in enumerate(plan.tensors):
        d0 = SLOT_HEADER_WORDS + DYN_WORDS * ti
        if not np.array_equal(a[d0:d0 + 4], b[d0:d0 + 4]):
            bad.append(f"{t.name} dyn gpu={a[d0:d0+4].tolist()} ref={b[d0:d0+4].tolist()} (d={t.numel},k={t.k},mode={t.mode})")
        n_sel = int(b[d0])
        if t.mode == MODE_BLOOM:
            fa, fb = a[t.off_filter:t.off_filter + t.n_filter_words], b[t.off_filter:t.off_filter + t.n_filter_words]
            if not np.array_equal(fa, fb):
                bad.append(f"{t.name} filter differs in {int((fa != fb).sum())}/{t.n_filter_words} words; popcount gpu={int(np.unpackbits(fa.view(np.uint8)).sum())} ref={int(np.unpackbits(fb.view(np.uint8)).sum())}")
            pa, pb = a[t.off_prefix:t.off_prefix + t.n_tiles], b[t.off_prefix:t.off_prefix + t.n_tiles]
            if not np.array_equal(pa, pb):
                bad.append(f"{t.name} prefix gpu={pa[:8].tolist()} ref={pb[:8].tolist()}")
            if t.off_hint:
                ha, hb = a[t.off_hint:t.off_hint + 4 * t.n_tiles], b[t.off_hint:t.off_hint + 4 * t.n_tiles]
                if not np.array_equal(ha, hb):
                    bad.append(f"{t.name} hint differs in {int((ha != hb).sum())}/{4 * t.n_tiles} words")
        elif t.mode == MODE_RLE:
            nc = (t.n_tiles + 1) // 2
            if not np.array_equal(a[t.off_prefix:t.off_prefix + nc], b[t.off_prefix:t.off_prefix + nc]):
                bad.append(f"{t.name} rle tile counts differ gpu={a[t.off_prefix:t.off_prefix+4].tolist()} ref={b[t.off_prefix:t.off_prefix+4].tolist()}")
            nw = rle_stream_words(t.val_cap)
            sa, sb = a[t.off_idx:t.off_idx + nw], b[t.off_idx:t.off_idx + nw]
            if not np.array_equal(sa, sb):
                bad.append(f"{t.name} rle stream differs in {int((sa != sb).sum())}/{nw} words")
        else:
            ia, ib = a[t.off_idx:t.off_idx + n_sel], b[t.off_idx:t.off_idx + n_sel]
            if not np.array_equal(ia, ib):
                bad.append(f"{t.name} raw idx gpu={ia[:8].tolist()} ref={ib[:8].tolist()}")
        if t.vmode == 2:
            nb = (n_sel + 511) // 512
            na, nbb = a[t.off_coef:t.off_coef + nb].view(np.float32), b[t.off_coef:t.off_coef + nb].view(np.float32)
            if not np.allclose(na, nbb, rtol=1e-5):
                bad.append(f"{t.name} qsgd norms differ {float(np.abs(na - nbb).max())}")
            la = a[t.off_rankmap:t.off_rankmap + (n_sel + 3) // 4].view(np.int8)[:n_sel]
            lb = b[t.off_rankmap:t.off_rankmap + (n_sel + 3) // 4].view(np.int8)[:n_sel]
            if int((la != lb).sum()) > max(2, n_sel // 2000):       # rounding-boundary flips from reduction order only
                bad.append(f"{t.name} qsgd levels differ in {int((la != lb).sum())}/{n_sel}")
            continue
        if t.vmode == 1:
            nc = 22 * (t.poly_degree + 1)
            ca, cb = a[t.off_coef:t.off_coef + nc].view(np.float32), b[t.off_coef:t.off_coef + nc].view(np.float32)
            if not np.allclose(ca, cb, rtol=2e-3, atol=2e-4 * float(np.abs(cb).max() + 1e-30)):
                bad.append(f"{t.name} coef max abs diff {float(np.abs(ca - cb).max())} (scale {float(np.abs(cb).max())})")
            if not np.array_equal(a[t.off_coef + nc:t.off_coef + nc + 2], b[t.off_coef + nc:t.off_coef + nc + 2]):
                bad.append(f"{t.name} coef tail gpu={a[t.off_coef+nc:t.off_coef+nc+2].tolist()} ref={b[t.off_coef+nc:t.off_coef+nc+2].tolist()}")
            nw = n_sel if t.rank_u32 else n_sel // 2          # compare whole words only
            ra, rb = a[t.off_rankmap:t.off_rankmap + nw], b[t.off_rankmap:t.off_rankmap + nw]
            if not np.array_equal(ra, rb):
                bad.append(f"{t.name} rank map differs in {int((ra != rb).sum())}/{nw} words")
            continue
        va, vb = a[t.off_vals:t.off_vals + n_sel], b[t.off_vals:t.off_vals + n_sel]
        if not np.array_equal(va, vb):
            bad.append(f"{t.name} vals differ in {int((va != vb).sum())}/{n_sel}")
    if bad:
        _diag(tag, "\n".join(bad))
    return bad


SIZES = [64, 1000, 1001, 4096, 4097, 36864, 147456, 10, 589824]


@pytest.mark.parametrize("kind", ["randn", "sparse", "ties"])
@pytest.mark.parametrize("index,policy,hint,tma,value", [
    ("bloom", "leftmost", True, True, None), ("bloom", "leftmost", False, False, None), ("bloom", "p0", True, True, None),
    (None, "leftmost", True, True, None), ("rle", "leftmost", True, True, None),
    ("bloom", "leftmost", True, True, "polyfit"),
    ("bloom", "leftmost", True, True, "qsgd")])
def test_engine_vs_oracle_single_rank(kind, index, policy, hint, tma, value):
    _run_vs_oracle(kind, index, policy, hint, tma, value)


@pytest.mark.parametrize("hist_shift,bps", [(23, 2), (22, 1), (20, 2)])
@pytest.mark.parametrize("index,policy,value", [("bloom", "leftmost", None), ("bloom", "p0", None), (None, "leftmost", None),
                                                ("rle", "leftmost", None), ("bloom", "leftmost", "polyfit")])
def test_engine_option_flags_vs_oracle(hist_shift, bps, index, policy, value):
    """The history bound (how many elements become candidates; 20 = tight -> frequent fallbacks) and the register /
    occupancy variant of the kernel must not change a single bit of the slot / output / residual."""
    for kind in ("randn", "ties"):
        _run_vs_oracle(kind, index, policy, True, True, value, hist_shift=hist_shift, bps=bps)


def _run_vs_oracle(kind, index, policy, hint, tma, value, hist_shift=22, bps=2, **plan_kw):
    from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
    plan = BucketPlan(SIZES + [2359296], compress_ratio=0.01, index=index, policy=policy, hint=hint, value=value,
                      poly_min_k=300, **plan_kw)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000, use_tma=tma, hist_shift=hist_shift,
                       blocks_per_sm=bps)
    gen = torch.Generator().manual_seed(0)
    resid_ref = torch.zeros(plan.total_elems)
    for step in range(3):                       # step 0: no history; steps 1,2: history lower bound (+fallback)
        g = _fill(plan, gen, kind) * (0.2 if step == 2 else 1.0)    # step 2 shrinks -> exercises the fallback
        eng.grad.copy_(g.cuda())
        if step == 1:
            eng.run_unfused()                   # the debug chain must agree with the fused launch
        else:
            eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out_ref, new_res, slots = engine_oracle(plan, [g], [resid_ref], epoch=eng.epoch)
        tag = f"single_{kind}_{index}_{policy}_{hint}_{value}_s{step}"
        bad = _compare_slot(plan, eng.slot(), slots[0], tag)
        assert not bad, bad[:4]
        if value is None:
            assert torch.equal(eng.resid.cpu(), new_res[0]), tag
            assert torch.allclose(eng.grad.cpu(), out_ref, atol=0, rtol=0), tag
            resid_ref = new_res[0]
        else:       # fp32 Gram sums on the GPU vs fp64 in the oracle
            scale = float(out_ref.abs().max())
            assert torch.allclose(eng.grad.cpu(), out_ref, atol=2e-3 * scale, rtol=1e-2), tag
            assert torch.allclose(eng.resid.cpu(), new_res[0], atol=2e-3 * scale, rtol=1e-2), tag
            resid_ref = eng.resid.cpu().clone()      # follow the GPU trajectory so later steps compare like with like
    eng.close()


@pytest.mark.parametrize("index,policy,value,kw", [
    (None, "leftmost", "polyfit", {}),                                         # value-only mode: coded values + plain indices
    (None, "leftmost", "qsgd", {}),
    ("bloom", "leftmost", "qsgd", dict(quantum_num=1000)),                     # int16 QSGD levels
    ("bloom", "leftmost", None, dict(sparsifier="threshold", threshold=0.0, capacity_ratio=0.5)),
    (None, "leftmost", None, dict(sparsifier="threshold", threshold=1.5)),
    ("bloom", "p0", None, dict(sparsifier="threshold", threshold=0.0, fpr=0.01, capacity_ratio=0.3)),
    ("rle", "leftmost", None, dict(sparsifier="threshold", threshold=2.0, capacity_ratio=0.1)),
    ("bloom", "leftmost", "qsgd", dict(sparsifier="threshold", threshold=1.0, capacity_ratio=0.5)),
    ("bloom", "random", None, dict(fpr=0.02)),                                 # P1: seeded draw among the positives
    ("bloom", "random", None, dict(fpr=0.05, hint=False)),
    ("bloom", "random", "qsgd", dict(sparsifier="threshold", threshold=1.0, capacity_ratio=0.5, fpr=0.01)),   # run_deepreduce.sh:73
    ("bloom", "random", "polyfit", dict(fpr=0.02)),
])
def test_engine_fused_recipe_modes(index, policy, value, kw):
    """The reference's launch recipes beyond top-k + bloom (run_deepreduce.sh:66-74): threshold sparsifier (variable K),
    value-only mode, QSGD with >= 128 levels, policy 'random' (P1, :73-74) — all inside the fused kernel, bit-exact against the oracle."""
    kw = dict(kw)
    hint = kw.pop("hint", True)
    for kind in ("randn", "sparse"):
        _run_vs_oracle(kind, index, policy, hint, True, value, **kw)


def test_topk_select_exact_with_ties_and_sparse():
    """ops.topk_select is exact: ties at the threshold go to the smaller index, fewer than k non-zeros pad with zeros."""
    from deepreduce_b200 import ops
    x = torch.tensor([1.0] * 1000 + [100.0])
    v, i = ops.topk_select(x.cuda(), 2)                 # massive ties: falls back to torch.topk
    assert sorted(i.cpu().tolist())[-1] == 1000 and float(v.abs().max()) == 100.0
    g = torch.Generator().manual_seed(5)
    y = torch.randint(-50, 51, (300000,), generator=g).float()      # many equal magnitudes around the threshold
    v, i = ops.topk_select(y.cuda(), 3000)
    ref = torch.sort(y.abs(), descending=True, stable=True).indices[:3000].sort().values
    assert torch.equal(i.cpu(), ref) and torch.equal(v.cpu(), y[ref])
    z = torch.zeros(200000); z[[5, 77, 1999]] = torch.tensor([1.0, -2.0, 3.0])
    v, i = ops.topk_select(z.cuda(), 100)
    assert v.numel() == 100 and set(i.cpu().tolist()) == {0, 5, 77, 1999} and float(v.abs().sum()) == 6.0
    from deepreduce_b200.grace.sparsifiers import _desparsify
    assert torch.equal(_desparsify((v, i), torch.Size([200000])).cpu(), z)


def test_calibrated_partition_is_bit_exact():
    """Per-phase tile partitions re-cut from measured per-CTA speeds (BucketEngine.calibrate_partition) change which CTA
    handles which tile in every phase, never a bit of the slot, the output or the residual; and the state is fresh
    afterwards.  Also with deliberately skewed speeds (some CTAs get almost nothing)."""
    from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
    plan = BucketPlan(SIZES + [2359296, 1048576], compress_ratio=0.01, index="bloom")
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    assert eng.cuts is not None
    log = eng.calibrate_partition(steps=2, rounds=1)
    assert len(log) == 2 and float(eng.resid.abs().max()) == 0.0 and int(eng.sel.abs().max()) == 0
    gen = torch.Generator().manual_seed(3)
    resid_ref = torch.zeros(plan.total_elems)
    for step in range(3):
        if step == 2:                                    # skewed cut: a few CTAs own most of the tiles
            sp = np.ones((4, eng.grid())); sp[:, ::3] = 0.05; sp[:, 7] = 30.0
            eng.cta_speeds = sp; eng._set_cuts()
        g = _fill(plan, gen, "randn")
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out_ref, new_res, slots = engine_oracle(plan, [g], [resid_ref], epoch=eng.epoch)
        assert not _compare_slot(plan, eng.slot(), slots[0], f"calib_s{step}")
        assert torch.equal(eng.grad.cpu(), out_ref) and torch.equal(eng.resid.cpu(), new_res[0])
        resid_ref = new_res[0]
    eng.close()


@pytest.mark.timeout(300)
def test_both_adversarial_ties_is_bounded():
    """Worst case of the exact in-bin rank of the 'both' mode (ops/csrc/engine.cu::phase_rank_exact is all-pairs
    inside a counting-sort bin): every shipped value has the same magnitude, so the K = 131072 values (the largest K
    that takes the polynomial fit, plan.MAX_POLY_K) fall into two bins.  The step must finish without tripping a
    watchdog, agree with the oracle, and its time is written to adversarial_ties.json in _out_dir()."""
    import json
    import time
    from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
    d = 1310720
    plan = BucketPlan([d], compress_ratio=0.1, index="bloom", value="polyfit")
    assert plan.tensors[0].vmode == 1 and plan.tensors[0].k == 131072
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    gen = torch.Generator().manual_seed(0)
    g = torch.where(torch.rand(plan.total_elems, generator=gen) < 0.5, -1.0, 1.0)
    g[d:] = 0
    times = []
    for step in range(3):
        eng.resid.zero_()
        eng.grad.copy_(g.cuda())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        eng.check_status()
    out_ref, new_res, slots = engine_oracle(plan, [g], [torch.zeros_like(g)], epoch=eng.epoch)
    assert not _compare_slot(plan, eng.slot(), slots[0], "ties131072")
    assert torch.allclose(eng.grad.cpu(), out_ref, atol=2e-3, rtol=1e-2)
    with open(os.path.join(_out_dir(), "adversarial_ties.json"), "w") as f:
        json.dump({"K": 131072, "d": d, "values": "all +-1 (two rank bins of ~65536)", "step_ms": times}, f)
    assert min(times) < 2000.0, times
    eng.close()


def test_engine_resnet50_shapes_and_volume():
    from deepreduce_b200.models import resnet50
    from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
    m = resnet50()
    named = list(reversed([(n, p) for n, p in m.named_parameters()]))
    plan = BucketPlan([p.numel() for _, p in named], [n for n, _ in named], compress_ratio=0.01)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    gen = torch.Generator().manual_seed(1)
    g = _fill(plan, gen)
    eng.grad.copy_(g.cuda())
    eng.step()
    torch.cuda.synchronize()
    eng.check_status()
    out_ref, new_res, slots = engine_oracle(plan, [g], [torch.zeros_like(g)], epoch=1)
    assert not _compare_slot(plan, eng.slot(), slots[0], "resnet50")
    assert torch.equal(eng.grad.cpu(), out_ref)
    assert plan.wire_bytes() < 0.02 * plan.dense_bytes()
    eng.close()


def test_per_tensor_ops_vs_oracle():
    from deepreduce_b200 import ops
    from deepreduce_b200.codecs import bloom as B, bitpack, polyfit, qsgd
    torch.manual_seed(0)
    d, K = 300000, 3000
    idx = torch.randperm(d)[:K].sort().values
    k, m_bits, _ = spec.bloom_layout(K, d)
    w_ref = B.bloom_insert_oracle(idx, k, m_bits)
    w = ops.bloom_insert(idx.cuda(), k, m_bits)
    assert torch.equal(w.cpu(), w_ref)
    pos_ref = B.bloom_query_oracle(w_ref, d, k, m_bits)
    assert torch.equal(ops.bloom_select(w, d, K, k, m_bits, "p0").cpu(), pos_ref)
    assert torch.equal(ops.bloom_select(w, d, K, k, m_bits, "leftmost").cpu(), pos_ref[:K])
    assert torch.equal(ops.bloom_select(w, d, K, k, m_bits, "random", 9).cpu(),
                       B.apply_policy_oracle(pos_ref, K, "random", 9))
    # top-k
    x = torch.randn(1_000_003)
    v, i = ops.topk_select(x.cuda(), 5000)
    ref_i = torch.topk(x.abs(), 5000).indices.sort().values
    assert torch.equal(i.cpu(), ref_i) and torch.equal(v.cpu(), x[ref_i])
    # bit packing
    vals = torch.randint(0, 2 ** 13, (10001,))
    p = ops.pack_bits(vals.cuda(), 13)
    assert torch.equal(p.cpu(), bitpack.pack_bits_oracle(vals, 13))
    assert torch.equal(ops.unpack_bits(p, 10001, 13).cpu(), vals)
    # qsgd
    y = torch.randn(5000)
    lvl, nrm = ops.qsgd_encode(y.cuda(), 127, 512, 77)
    lvl_ref, nrm_ref = qsgd.qsgd_encode_oracle(y, 127, 512, 77)
    assert torch.allclose(nrm.cpu(), nrm_ref, rtol=1e-5)
    assert (lvl.cpu().float() != lvl_ref).sum() <= 5          # rounding-boundary flips from reduction order only
    assert torch.allclose(ops.qsgd_decode(lvl, nrm, 127, 512).cpu(), qsgd.qsgd_decode_oracle(lvl.cpu(), nrm.cpu(), 127, 512))
    # polyfit
    ys = torch.sort(torch.randn(23592), descending=True).values
    seg = polyfit.get_segments(23592, int((ys > 0).sum()))
    c = ops.polyfit_fit(ys.cuda(), seg, 5)
    c_ref = polyfit.polyfit_fit_oracle(ys, seg, 5)
    fit = ops.polyfit_eval(c, seg, 5, 23592).cpu()
    fit_ref = polyfit.polyfit_eval_oracle(c_ref, seg, 5)
    assert torch.allclose(fit, fit_ref, atol=2e-3), float((fit - fit_ref).abs().max())
    # delta + bp128
    enc = ops.delta_bp128_encode(idx.cuda())
    assert torch.equal(ops.delta_bp128_decode(enc, K).cpu(), idx)
    from deepreduce_b200.codecs.integer import int_encode
    ref = int_encode(np.diff(idx.numpy().astype(np.uint32), prepend=np.uint32(0)).astype(np.uint32), "bp128")
    assert np.array_equal(enc.cpu().numpy().view(np.uint32), ref)
    # run-length kernels
    from deepreduce_b200.codecs import rle as R
    blocks = torch.cat([torch.arange(100, 160), torch.arange(5000, 5003), idx[idx > 6000]]).unique()
    for ix, dd in ((idx, d), (blocks, d), (torch.arange(0, 50), 50), (torch.tensor([d - 1]), d)):
        runs = ops.rle_runs(ix.cuda(), dd)
        assert torch.equal(runs.cpu(), R.runs_from_sorted_oracle(ix, dd)), (ix[:5], dd)
        assert torch.equal(ops.rle_indices(runs, ix.numel()).cpu(), ix)
    # input normalisation kernel
    img = torch.randint(0, 256, (4, 32, 32, 3), dtype=torch.uint8)
    o = ops.u8_to_nhwc_norm(img.cuda()).float().cpu()
    m = torch.tensor([0.485, 0.456, 0.406]); s = torch.tensor([0.229, 0.224, 0.225])
    assert torch.allclose(o, (img.float() / 255 - m) / s, atol=2e-2)
    assert ops.launch_count() > 0


@pytest.mark.parametrize("cfg", [
    dict(deepreduce='index', index='bloom'), dict(deepreduce='index', index='bloom', policy='p0'),
    dict(deepreduce='both'), dict(deepreduce='both', min_numel=100), dict(deepreduce='value', value='polyfit'), dict(deepreduce='value', value='qsgd'),
    dict(deepreduce='index', index='rle'), dict(deepreduce='index', index='integer'), dict()])
def test_grace_path_cuda_matches_cpu(cfg):
    import deepreduce_b200 as dr
    base = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
    torch.manual_seed(0)
    g = torch.randn(147456)
    out_cpu = dr.deepreduce_from_params(dict(base, **cfg)).step(g.clone(), 'w')
    out_gpu = dr.deepreduce_from_params(dict(base, **cfg)).step(g.cuda(), 'w').cpu()
    # the CUDA top-k resolves its threshold to 22 bits (>= K selected, left-most K kept), so the support
    # may differ from torch.topk in a handful of coordinates whose |value| sits at the threshold
    sc, sg = set(out_cpu.nonzero().flatten().tolist()), set(out_gpu.nonzero().flatten().tolist())
    assert len(sc ^ sg) <= 12, len(sc ^ sg)
    both = torch.tensor(sorted(sc & sg))
    if cfg.get('index') != 'bloom' and cfg.get('deepreduce') != 'both' and cfg.get('value') != 'qsgd':   # qsgd buckets follow value order
        assert torch.allclose(out_cpu[both], out_gpu[both], atol=5e-3, rtol=1e-3)
    assert torch.nn.functional.cosine_similarity(out_cpu, out_gpu, dim=0) > 0.98


def test_trainer_cuda_resnet20_overlap():
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.trainer import Trainer
    torch.manual_seed(0)
    cfg = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
           'deepreduce': 'index', 'index': 'bloom'}
    tr = Trainer(resnet20().cuda(), cfg, lr=0.05, bucket_cap_mb=0.25, channels_last=True)   # several buckets + thread
    assert len(tr.ddp.engines) > 1
    x = torch.randn(32, 3, 32, 32, device="cuda"); y = torch.randint(0, 10, (32,), device="cuda")
    losses = [float(tr.step(x, target=y)) for _ in range(8)]
    tr.ddp.check()
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
    xh = torch.randn(32, 3, 32, 32).pin_memory(); yh = torch.randint(0, 10, (32,)).pin_memory()
    l = tr.step_host((xh,), yh)
    assert np.isfinite(l) and tr.h2d_bytes == xh.numel() * 4 + yh.numel() * 8
    tr.close()


@pytest.mark.timeout(600)
def test_multi_gpu_engine():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    W = min(n, 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={W}",
           "--master-addr", "127.0.0.1", "--master-port", "29533", os.path.join(ROOT, "tests", "run_multigpu.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=550)
    _diag("multigpu", r.stdout[-4000:] + r.stderr[-4000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "MULTIGPU_OK" in r.stdout


def test_engine_state_roundtrip_and_accumulation():
    from deepreduce_b200.parallel import BucketEngine, BucketPlan
    plan = BucketPlan([50000, 700, 9000], compress_ratio=0.02)
    gen = torch.Generator().manual_seed(3)
    a = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    for _ in range(2):
        a.grad.copy_(_fill(plan, gen).cuda()); a.step()
    st = a.state_dict()
    b = BucketEngine(plan, device="cuda:0", world=1, rank=0)
    b.load_state_dict(st)
    g = _fill(plan, gen).cuda()
    a.grad.copy_(g); b.grad.copy_(g)
    a.step(); b.step()
    torch.cuda.synchronize()
    assert torch.equal(a.grad, b.grad) and torch.equal(a.resid, b.resid) and a.epoch == b.epoch
    a.close(); b.close()
    # gradient accumulation on the fused path: exchange only on the last micro-step
    from deepreduce_b200.models import resnet20
    from deepreduce_b200.trainer import Trainer
    cfg = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
           'deepreduce': 'index', 'index': 'bloom'}
    tr = Trainer(resnet20().cuda(), cfg, lr=0.05, accum_steps=2)
    x = torch.randn(16, 3, 32, 32, device="cuda"); y = torch.randint(0, 10, (16,), device="cuda")
    w0 = [p.detach().clone() for p in tr.model.parameters()]
    tr.step(x, target=y)
    assert all(torch.equal(p, q) for p, q in zip(w0, tr.model.parameters()))
    tr.step(x, target=y)
    tr.ddp.check()
    assert tr.ddp.step_count == 1 and any(not torch.equal(p, q) for p, q in zip(w0, tr.model.parameters()))
    tr.close()


def test_tf_compat_on_device_and_dexp_kernel():
    """The TF-side compressors keep CUDA gradients on the device (Fit-DExp / PolySeg are GPU ops upstream,
    tensorflow/deepreduce.py:376-557) and the double-exponential fit runs in the hand-written one-CTA kernel."""
    from deepreduce_b200 import ops, tf_compat as T
    from deepreduce_b200.codecs import dexp
    g = torch.Generator().manual_seed(0)
    y = torch.sort(torch.randn(50000, generator=g).abs()).values
    ref = torch.stack(dexp.double_exponential_fit_oracle(y))
    got = ops.dexp_fit(y.cuda()).cpu()
    curve_ref = dexp.double_exponential_eval(ref.float(), y.numel())
    curve_got = dexp.double_exponential_eval(got.float(), y.numel())
    assert torch.allclose(curve_got, curve_ref, rtol=1e-3, atol=1e-4 * float(y.max())), (got, ref)
    assert ops.launch_count() > 0
    x = torch.randn(20000, generator=g)
    for cls, params in ((T.DoubleExpCompressor, {"compress_ratio": 0.05}),
                        (T.PolySegCompressor, {"compress_ratio": 0.05, "polynomial_degree": 5}),
                        (T.BloomFilterCompressor, {"compress_ratio": 0.01, "bloom_fpr": 0.01, "bloom_policy": "leftmostK"})):
        pc, pg = dict(params), dict(params)
        comp_c, ctx_c = cls.compress(x.clone(), pc)
        comp_g, ctx_g = cls.compress(x.cuda(), pg)
        out_c = cls.decompress(comp_c, ctx_c, pc)
        out_g = cls.decompress(comp_g, ctx_g, pg)
        assert out_g.is_cuda, cls.__name__
        assert torch.allclose(out_g.cpu(), out_c, rtol=2e-3, atol=2e-3), cls.__name__


def test_conflict_sets_p2_on_device_matches_host():
    """P2 (conflict sets) runs on the GPU — set construction by sort, the sequential draw in a one-warp kernel — and
    returns exactly what the host C++ routine (the reference's policies.hpp semantics) returns."""
    from deepreduce_b200 import ops
    from deepreduce_b200.codecs import bloom as B
    torch.manual_seed(0)
    for d, K in ((36864, 368), (589824, 5898), (20000, 2000)):
        idx = torch.randperm(d)[:K].sort().values
        k, m_bits, _ = spec.bloom_layout(K, d)
        words = B.bloom_insert_oracle(idx, k, m_bits)
        pos = B.bloom_query_oracle(words, d, k, m_bits)
        for pseed in (7, 12345):
            ref = ops.cpu.conflict_sets(pos, K, k, m_bits, spec.DEFAULT_SEED, pseed)
            got = B.conflict_sets_cuda(pos.cuda(), K, k, m_bits, spec.DEFAULT_SEED, pseed)
            assert got is not None and torch.equal(got.cpu(), ref), (d, K, pseed)
            sel = B.bloom_select(words.cuda(), d, K, k, m_bits, "conflict_sets", pseed)
            assert torch.equal(sel.cpu(), ref)
