"""Bucket plan + engine oracle (CPU): the specification the fused kernel is tested against."""
import pytest
import numpy as np
import torch

from deepreduce_b200 import spec
from deepreduce_b200.parallel import BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import select_topk_oracle
from deepreduce_b200.parallel.plan import MODE_BLOOM, MODE_RAW, SLOT_HEADER_WORDS, DYN_WORDS
import deepreduce_b200 as dr

SIZES = [64, 1000, 1001, 4096, 4097, 36864, 147456, 10]


def test_plan_layout():
    plan = BucketPlan(SIZES, compress_ratio=0.01)
    assert [t.mode for t in plan.tensors] == [MODE_RAW, MODE_RAW, MODE_BLOOM, MODE_BLOOM, MODE_BLOOM, MODE_BLOOM, MODE_BLOOM, MODE_RAW]
    assert plan.n_tiles == sum((d + spec.TILE - 1) // spec.TILE for d in SIZES)
    tt = plan.tile_table()
    assert tuple(tt.shape) == (plan.n_tiles, 4)
    for i, t in enumerate(plan.tensors):
        assert t.elem_off % 32 == 0 and t.k == max(1, int(t.numel * 0.01))
        rows = tt[t.tile_begin:t.tile_begin + t.n_tiles]
        assert rows[:, 0].tolist() == [i] * t.n_tiles
        assert rows[0, 1] == t.elem_off and int((rows[:, 2] & 0xFFFF).sum()) == t.numel and rows[-1, 3] == (t.n_tiles - 1) * spec.TILE
        assert bool(rows[0, 2] < 0) == (t.n_tiles == 1)                 # bit 31 flags one-tile tensors
    # regions do not overlap and fit in the payload
    regions = []
    for t in plan.tensors:
        regions.append((t.off_vals, t.val_cap))
        if t.mode == MODE_BLOOM:
            regions += [(t.off_filter, t.n_filter_words), (t.off_prefix, t.n_tiles), (t.off_hint, 4 * t.n_tiles)]
        else:
            regions.append((t.off_idx, t.k))
    regions.sort()
    assert regions[0][0] >= SLOT_HEADER_WORDS + DYN_WORDS * len(SIZES)
    for (a, n), (b, _) in zip(regions[:-1], regions[1:]):
        assert a + n <= b
    assert regions[-1][0] + regions[-1][1] <= plan.payload_words <= plan.slot_words
    assert plan.tensor_table().numel() == 32 * len(SIZES)
    # bloom wire is smaller than plain (fp32,int64) pairs: the paper's headline for index compression
    assert plan.wire_bytes() < plan.topk_pair_bytes()


def test_select_rule_22bit_threshold():
    # rule: (key >> 9) >= max(T22, 1) with T22 = 22-bit prefix of the K-th largest |x|
    x = torch.tensor([0.0, 1.0, -1.0, 1.0, 0.5, -1.0, 2.0])
    idx, thr = select_topk_oracle(x, 3)
    assert idx.tolist() == [1, 2, 3, 5, 6]           # everything sharing the threshold's prefix comes along
    assert thr == (torch.tensor(1.0).view(torch.int32).item() >> 9) << 9
    x = torch.zeros(100); x[7] = 3.0
    idx, thr = select_topk_oracle(x, 5)
    assert idx.tolist() == [7]                       # exact zeros are never shipped
    torch.manual_seed(0)
    x = torch.randn(100000)
    idx, _ = select_topk_oracle(x, 1000)
    ref = set(torch.topk(x.abs(), 1000).indices.tolist())
    assert ref <= set(idx.tolist()) and idx.numel() <= 1010      # >= K, plus at most a handful at the threshold


def test_oracle_matches_grace_path_single_rank():
    torch.manual_seed(0)
    plan = BucketPlan([36864, 500, 9408], compress_ratio=0.01, hint=False)      # pure bloom == the per-tensor API
    g = torch.zeros(plan.total_elems)
    for v in plan.views(g):
        v.copy_(torch.randn_like(v))
    out, resids, slots = engine_oracle(plan, [g], [torch.zeros_like(g)])
    grc = dr.deepreduce_from_params({'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather',
                                     'compress_ratio': 0.01, 'deepreduce': 'index', 'index': 'bloom'})
    for t, v, o, r in zip(plan.tensors, plan.views(g), plan.views(out), plan.views(resids[0])):
        ref = grc.step(v.clone().flatten(), t.name)
        assert torch.equal(o.flatten(), ref), t.name              # same S~, same values as the per-tensor API
        assert torch.equal(r.flatten(), grc.memory.residuals[t.name])
    assert slots[0][0] == 0xD33B2000 and slots[0].dtype == np.uint32


def test_oracle_multi_rank_average_and_residual():
    torch.manual_seed(1)
    plan = BucketPlan([20000, 300], compress_ratio=0.02)
    W = 3
    grads = [torch.randn(plan.total_elems) for _ in range(W)]
    for g in grads:                                     # padding must stay zero
        mask = torch.zeros(plan.total_elems, dtype=torch.bool)
        for t in plan.tensors:
            mask[t.elem_off:t.elem_off + t.numel] = True
        g[~mask] = 0
    res = [torch.zeros(plan.total_elems) for _ in range(W)]
    out, new_res, slots = engine_oracle(plan, grads, res)
    total = sum(g - r for g, r in zip(grads, new_res)) / W
    assert torch.allclose(out, total, atol=1e-6)        # what was shipped == grad - residual, averaged
    out2, _, _ = engine_oracle(plan, grads, new_res)
    assert not torch.equal(out, out2)                   # residual feeds the next step


def test_p0_capacity_and_header():
    torch.manual_seed(2)
    plan = BucketPlan([50000], compress_ratio=0.01, policy="p0")
    t = plan.tensors[0]
    assert t.val_cap > t.k
    g = torch.randn(plan.total_elems)
    out, res, slots = engine_oracle(plan, [g], [torch.zeros_like(g)])
    dyn = SLOT_HEADER_WORDS
    n_sel, cutoff, thr, n_pos = slots[0][dyn:dyn + 4].tolist()
    assert n_sel == n_pos and n_sel >= t.k and cutoff == 0xFFFFFFFF
    true = set(torch.topk(g[:50000].abs(), t.k).indices.tolist())
    assert true <= set(out[:50000].nonzero().flatten().tolist())        # P0 is lossless w.r.t. top-k


def test_occupancy_hint_removes_false_positives():
    torch.manual_seed(5)
    g = torch.randn(200000)
    outs = {}
    for hint in (False, True):
        plan = BucketPlan([200000], compress_ratio=0.01, hint=hint)
        gg = torch.zeros(plan.total_elems); gg[:200000] = g
        out, res, slots = engine_oracle(plan, [gg], [torch.zeros_like(gg)])
        outs[hint] = out[:200000]
        if hint:
            assert plan.tensors[0].off_hint > 0 and plan.wire_bytes() < 1.09 * plan_nohint_bytes
        else:
            plan_nohint_bytes = plan.wire_bytes()
    true = set(torch.topk(g.abs(), 2000).indices.tolist())
    kept = {h: len(true & set(outs[h].nonzero().flatten().tolist())) for h in outs}
    assert kept[True] > kept[False]                 # fewer false positives displace true top-k entries
    assert kept[True] >= 1940


def test_oracle_both_polyfit():
    torch.manual_seed(7)
    plan = BucketPlan([300000, 5000], compress_ratio=0.01, value="polyfit")
    t0, t1 = plan.tensors
    assert t0.vmode == 1 and t0.rank_u32 == 0 and t1.vmode == 0          # K=50 stays fp32 (fit header would be larger)
    plain = BucketPlan([300000, 5000], compress_ratio=0.01)
    assert plan.wire_bytes() < 0.75 * plain.wire_bytes()                 # values: 4 B -> 2 B (+ coefficients)
    g = torch.zeros(plan.total_elems)
    for v in plan.views(g):
        v.copy_(torch.randn_like(v))
    out, res, slots = engine_oracle(plan, [g], [torch.zeros_like(g)])
    out_p, res_p, _ = engine_oracle(plain, [g], [torch.zeros_like(g)])
    seg = slice(0, 300000)
    assert torch.equal(out[seg] != 0, out_p[seg] != 0)                   # same support, fitted values
    rel = (out[seg] - out_p[seg]).norm() / out_p[seg].norm()
    assert rel < 0.08
    assert torch.allclose(out[seg] + res[0][seg], g[seg], atol=1e-6)     # residual keeps the fit error


def test_oracle_both_qsgd():
    torch.manual_seed(8)
    plan = BucketPlan([300000], compress_ratio=0.01, value="qsgd")
    plain = BucketPlan([300000], compress_ratio=0.01)
    assert plan.tensors[0].vmode == 2 and plan.poly_tables()[3] == (3000 + 511) // 512
    assert plan.wire_bytes() < 0.6 * plain.wire_bytes()                  # values: 4 B -> 1 B (+ a norm per 512)
    g = torch.zeros(plan.total_elems); g[:300000] = torch.randn(300000)
    out, res, _ = engine_oracle(plan, [g], [torch.zeros_like(g)])
    out_p, _, _ = engine_oracle(plain, [g], [torch.zeros_like(g)])
    assert torch.equal(out != 0, out_p != 0) or (out != 0).sum() >= 0.98 * (out_p != 0).sum()   # level 0 can zero a value
    assert (out - out_p).norm() / out_p.norm() < 0.12
    assert torch.allclose(out + res[0], g, atol=1e-6)


def test_oracle_rle_index_is_lossless_and_smaller_than_pairs():
    """Fused 'rle' index mode (kModeRle): same selection / output / residual as plain top-k pairs, smaller wire,
    and the bit stream decodes back to the selected indices (tile count + 12-bit in-tile offsets)."""
    from deepreduce_b200.parallel import BucketPlan, engine_oracle
    from deepreduce_b200.parallel.engine import rle_unpack12
    from deepreduce_b200.parallel.plan import DYN_WORDS, MODE_RLE, SLOT_HEADER_WORDS
    sizes = [64, 5000, 20000, 100000]
    rle = BucketPlan(sizes, compress_ratio=0.01, index="rle")
    raw = BucketPlan(sizes, compress_ratio=0.01, index=None)
    assert rle.tensors[0].mode != MODE_RLE and all(t.mode == MODE_RLE for t in rle.tensors[1:])
    assert rle.wire_bytes() < 0.75 * raw.wire_bytes()
    gen = torch.Generator().manual_seed(5)
    g = [torch.randn(rle.total_elems, generator=gen) for _ in range(3)]
    r = [torch.zeros(rle.total_elems) for _ in range(3)]
    o1, r1, s1 = engine_oracle(rle, g, r)
    o2, r2, s2 = engine_oracle(raw, g, r)
    assert torch.equal(o1, o2) and all(torch.equal(a, b) for a, b in zip(r1, r2))
    for ti, (ta, tb) in enumerate(zip(rle.tensors, raw.tensors)):
        if ta.mode != MODE_RLE:
            continue
        n = int(s1[0][SLOT_HEADER_WORDS + DYN_WORDS * ti])
        cnt = s1[0][ta.off_prefix:ta.off_prefix + (ta.n_tiles + 1) // 2].view(np.uint16)[:ta.n_tiles].astype(np.int64)
        assert cnt.sum() == n
        tile_of = np.repeat(np.arange(ta.n_tiles), cnt)
        idx = tile_of * 4096 + rle_unpack12(s1[0][ta.off_idx:], n)
        assert np.array_equal(idx, s2[0][tb.off_idx:tb.off_idx + n].astype(np.int64))


def test_stats_from_slot_counts_and_bytes():
    """Counters read back from the slot's dynamic headers (SURVEY §5: per-step device counters)."""
    from deepreduce_b200.parallel import stats_from_slot
    sizes = [64, 5000, 20000, 100000]
    for index in ("bloom", "rle", None):
        plan = BucketPlan(sizes, compress_ratio=0.01, index=index)
        gen = torch.Generator().manual_seed(9)
        g = [torch.randn(plan.total_elems, generator=gen)]
        _, _, slots = engine_oracle(plan, g, [torch.zeros(plan.total_elems)])
        st = stats_from_slot(plan, slots[0])
        tot = st["total"]
        assert tot["k"] == sum(t.k for t in plan.tensors)
        assert tot["n_sel"] == sum(r["n_sel"] for r in st["tensors"]) and tot["n_sel"] >= 0.9 * tot["k"]
        assert tot["value_bytes"] + tot["index_bytes"] + tot["header_bytes"] <= tot["wire_bytes"] + 64 * len(sizes)
        assert 0 < tot["relative_volume"] < 0.05
        big = st["tensors"][-1]
        assert big["threshold"] > 1.5          # top 1 % of |N(0,1)| starts near 2.57 (22-bit threshold rounds down)
        if index == "bloom":
            assert big["n_pos"] >= big["n_sel"] and big["false_pos"] >= 0
        else:
            assert big["false_pos"] == 0


def test_stage2_layout_never_overflows_by_construction(monkeypatch):
    """Sharded decode: the stage-2 slot holds the worst case (all W senders' selections inside one slice)."""
    sizes = [64, 5000, 20000, 100000, 2359296]
    plan = BucketPlan(sizes, compress_ratio=0.01)
    k_total = sum(t.val_cap for t in plan.tensors)
    for W in (2, 4, 8):
        cap, words = plan.stage2_layout(W)
        slice_elems = (plan.n_tiles + W - 1) // W * 4096
        assert cap % 4 == 0 and words % 64 == 0 and words >= 4 + 2 * cap
        assert cap >= min(W * k_total, slice_elems)
        assert plan.arena_words(W, True) == plan.arena_words(W, False) + 2 * W * words
        assert plan.arena_words(W, True) < 2 ** 32            # word offsets are uint32-safe
    assert plan.arena_words(1, True) == plan.arena_words(1, False)
    monkeypatch.setenv("DR_S2_SLACK", "2")
    assert plan.stage2_layout(8)[0] == ((2 * k_total + 8192 + 3) // 4) * 4


@pytest.mark.parametrize("seed", [0, 1])
def test_wire_format_is_self_sufficient(seed):
    """Sender spec (`engine_oracle`) vs an independent receiver (`decode_slot_oracle`, slot words + plan only):
    every mode, hint on/off, P0, sizes around tile boundaries, ties / sparse gradients, 1-3 ranks, two steps."""
    import random

    from deepreduce_b200.parallel import decode_slot_oracle
    rnd = random.Random(seed)
    for it in range(25):
        sizes = [rnd.choice([1, 2, 10, 64, 999, 1000, 1001, 4095, 4096, 4097, 8193, 20000, 50000])
                 for _ in range(rnd.randint(1, 5))]
        mode = rnd.choice([dict(index='bloom'), dict(index='bloom', policy='p0'), dict(index='bloom', hint=False),
                           dict(index='rle'), dict(index=None), dict(index='bloom', value='polyfit', poly_min_k=32),
                           dict(index='bloom', value='qsgd'), dict(index='bloom', policy='random', fpr=0.05),
                           dict(index='bloom', policy='random', value='qsgd', sparsifier='threshold', threshold=1.0,
                                capacity_ratio=0.5, fpr=0.01)])
        W = rnd.choice([1, 2, 3])
        plan = BucketPlan(sizes, compress_ratio=rnd.choice([0.001, 0.01, 0.1, 0.5]), min_numel=rnd.choice([0, 1000]), **mode)
        kind = rnd.choice(['randn', 'ties', 'sparse'])
        gen = torch.Generator().manual_seed(100 * seed + it)

        def mk():
            g = torch.randn(plan.total_elems, generator=gen)
            if kind == 'ties':
                g = torch.randint(-2, 3, (plan.total_elems,), generator=gen).float()
            if kind == 'sparse':
                g[torch.rand(plan.total_elems, generator=gen) < 0.99] = 0
            return g
        grads = [mk() for _ in range(W)]
        res = [torch.zeros(plan.total_elems) for _ in range(W)]
        for step in range(2):
            out, res, slots = engine_oracle(plan, grads, res, epoch=step + 1)
            rec = sum(decode_slot_oracle(plan, s) for s in slots) / W
            tol = (1e-4 if 'value' in mode else 1e-6) * float(out.abs().max() + 1e-30)
            assert torch.allclose(rec, out, atol=tol, rtol=1e-5), (sizes, mode, W, kind, step)


def test_split_large_chunks_are_contiguous_tile_multiples():
    from deepreduce_b200.parallel.plan import split_large
    numels, names, shapes = [64, 31254528, 4096 * 3 + 5, 1000], ["b", "emb", "w", "s"], [(64,), (30522, 1024), (12293,), (1000,)]
    n2, nm2, sh2, owner = split_large(numels, names, shapes, 4_000_000)
    step = (4_000_000 // 4096) * 4096
    assert sum(n2) == sum(numels) and owner == [0] + [1] * 8 + [2, 3]
    assert n2[1:8] == [step] * 7 and n2[8] == 31254528 - 7 * step and nm2[1] == "emb#0" and sh2[9] == (12293,)
    plan = BucketPlan(n2, nm2, sh2, compress_ratio=0.01)
    emb = [t for t, o in zip(plan.tensors, owner) if o == 1]
    for a, b in zip(emb[:-1], emb[1:]):
        assert a.elem_off + a.numel == b.elem_off                     # no padding between chunks: one gradient view spans them
    assert all(t.n_filter_words * 4 <= 88 * 1024 for t in emb)         # every chunk's filter fits the SMEM staging area
    whole = BucketPlan([31254528], compress_ratio=0.01).tensors[0]
    assert whole.n_filter_words * 4 > 227 * 1024                       # as one tensor it cannot
    assert split_large(numels, names, shapes, None)[0] == numels


def test_selfcheck_torch_decoder_matches_numpy_oracle():
    """utils/selfcheck.decode_slot_torch (the independent decoder bench.py uses for its multi-GPU check) agrees with
    the numpy slot decoder on every fp32-value mode, and declines value-coded plans."""
    import torch
    from deepreduce_b200.parallel import BucketPlan, engine_oracle
    from deepreduce_b200.parallel.engine import decode_slot_oracle
    from deepreduce_b200.utils.selfcheck import decode_slot_torch
    sizes = [64, 1001, 4097, 36864, 147456]
    gen = torch.Generator().manual_seed(3)
    for kw in (dict(index="bloom"), dict(index="bloom", hint=False), dict(index="bloom", policy="p0"), dict(index=None),
               dict(index="bloom", sparsifier="threshold", threshold=1.0, capacity_ratio=0.5),
               dict(index="bloom", policy="random", fpr=0.05), dict(index="bloom", policy="random", fpr=0.05, hint=False)):
        plan = BucketPlan(sizes, compress_ratio=0.01, **kw)
        g = torch.zeros(plan.total_elems)
        for v in plan.views(g):
            v.copy_(torch.randn(v.shape, generator=gen))
        out, _, slots = engine_oracle(plan, [g], [torch.zeros_like(g)])
        slot_t = torch.from_numpy(slots[0].view("int32").copy())
        dec = decode_slot_torch(plan, slot_t)
        assert torch.equal(dec, decode_slot_oracle(plan, slots[0])), kw
        assert torch.equal(dec, out), kw
    plan = BucketPlan(sizes, compress_ratio=0.01, index="bloom", value="qsgd")
    g = torch.randn(plan.total_elems)
    _, _, slots = engine_oracle(plan, [g], [torch.zeros_like(g)])
    assert decode_slot_torch(plan, torch.from_numpy(slots[0].view("int32").copy())) is None


def test_random_policy_is_a_seeded_draw_of_the_right_size():
    """Fused 'random' policy (P1, reference pytorch/deepreduce.py:484-490): the shipped set is a seeded Bernoulli draw
    of rate inserted/positives — about K coordinates, all of them filter positives, a different draw every step and
    every tensor, reproduced by the receiver from the header's acceptance threshold alone."""
    import numpy as np
    from deepreduce_b200.parallel import BucketPlan, decode_slot_oracle, engine_oracle
    from deepreduce_b200.parallel.plan import DYN_WORDS, SLOT_HEADER_WORDS
    d = 200000
    plan = BucketPlan([d, d], compress_ratio=0.01, index="bloom", policy="random", fpr=0.02, hint=False)
    g = torch.randn(plan.total_elems, generator=torch.Generator().manual_seed(0))
    sets = []
    for step in (1, 2):
        out, res, slots = engine_oracle(plan, [g], [torch.zeros_like(g)], epoch=step)
        assert torch.equal(decode_slot_oracle(plan, slots[0]), out)
        assert torch.equal(res[0] + out, g)                      # error feedback keeps what was not shipped
        for ti, t in enumerate(plan.tensors):
            n_sel, _, T, n_pos = (int(x) for x in slots[0][SLOT_HEADER_WORDS + DYN_WORDS * ti:][:4])
            assert n_pos > t.k * 1.5                               # fpr 2 % of the universe on top of K = 1 %
            assert T == (t.k << 32) // n_pos                       # the top-k select ships exactly K here (no 22-bit ties in randn)
            assert abs(n_sel - t.k) < 6 * np.sqrt(t.k) and n_sel <= t.k
            seg = out[t.elem_off:t.elem_off + t.numel]
            sets.append(set(torch.nonzero(seg).flatten().tolist()))
    assert sets[0] != sets[2] and sets[1] != sets[3]               # step 1 vs step 2: another draw
    top = set(torch.topk(g[:d].abs(), plan.tensors[0].k).indices.tolist())
    frac_true = len(sets[0] & top) / len(sets[0])
    assert 0.25 < frac_true < 0.55                                 # true elements and false positives are dropped alike (K / n_pos ~ 1/3)


def test_phase_cuts_cover_all_tiles_and_follow_speeds():
    """BucketPlan.phase_cuts: four monotone partitions of the tiles (one per phase class of the kernel); a CTA with
    relative speed s gets about s times the average cost."""
    import numpy as np
    from deepreduce_b200.parallel import BucketPlan
    plan = BucketPlan([100, 5000, 300000, 4097, 2000000, 64, 1200000], compress_ratio=0.01)
    G = 64
    c = plan.phase_cuts(G).numpy()
    assert c.shape == (4, G + 1) and (c[:, 0] == 0).all() and (c[:, -1] == plan.n_tiles).all() and (np.diff(c, axis=1) >= 0).all()
    assert not np.array_equal(c[0], c[1])                      # accumulate and insert weigh segment starts differently
    sp = np.ones((4, G)); sp[:, G // 2:] = 0.5
    c2 = plan.phase_cuts(G, sp).numpy()
    n_fast, n_slow = np.diff(c2[1])[:G // 2].sum(), np.diff(c2[1])[G // 2:].sum()
    assert 1.7 < n_fast / n_slow < 2.3
    tiny = BucketPlan([100, 200], compress_ratio=0.1)          # fewer tiles than CTAs: empty ranges are legal
    c3 = tiny.phase_cuts(296).numpy()
    assert (c3[:, -1] == tiny.n_tiles).all() and (np.diff(c3, axis=1) >= 0).all()


def test_partition_calibration_converges_on_a_two_speed_machine():
    """The speed update behind BucketEngine.calibrate_partition, on a model of a GPU running two CTAs per SM: half of the
    CTAs (the second-launched one of every SM) run a phase 15 % slower.  With shares proportional to the calibrated
    speeds the systematic gap is removed within two rounds, and the noise of a single round does not blow up."""
    import numpy as np
    from deepreduce_b200.parallel.plan import update_cta_speeds
    G = 264                                  # 2 CTAs x 132 SMs (H100)
    true = np.ones(G); true[G // 2:] = 0.85
    speeds = np.ones(G)
    rng = np.random.default_rng(0)
    spread = []
    for rnd in range(4):
        share = speeds / speeds.sum()
        dur = share / true * G * 80.0 * (1.0 + 0.03 * rng.standard_normal(G))      # ~80 us phase, 3 % timing noise
        spread.append(dur.max() / np.median(dur))
        speeds = update_cta_speeds(speeds, dur, 0.8)
    # the systematic 15 % is gone after two rounds; what is left is the per-launch noise itself (max of 296 draws)
    assert spread[0] > 1.18 and max(spread[2:]) < 1.15
    assert abs(speeds[G // 2:].mean() / speeds[:G // 2].mean() - 0.85) < 0.03
    assert abs(speeds.mean() - 1.0) < 1e-9 and speeds.min() >= 0.5 * 0.9 and speeds.max() <= 2.0 * 1.1


def test_phase_cuts_property_any_speeds_any_plan():
    """The kernel trusts the host-computed cuts blindly: for any plan, grid and speed vector every phase class must tile
    [0, n_tiles) with non-decreasing cut positions."""
    import numpy as np
    from hypothesis import given, settings, strategies as st
    from deepreduce_b200.parallel import BucketPlan

    @settings(max_examples=40, deadline=None)
    @given(st.lists(st.integers(1, 300000), min_size=1, max_size=12), st.sampled_from([2, 37, 132, 148, 264, 296]),
           st.integers(0, 2 ** 31 - 1))
    def check(numels, grid, seed):
        plan = BucketPlan(numels, compress_ratio=0.01)
        rng = np.random.default_rng(seed)
        sp = np.exp(rng.uniform(np.log(0.05), np.log(30.0), size=(4, grid)))
        c = plan.phase_cuts(grid, sp).numpy().astype(np.int64)
        assert c.shape == (4, grid + 1)
        assert (c[:, 0] == 0).all() and (c[:, -1] == plan.n_tiles).all() and (np.diff(c, axis=1) >= 0).all()
    check()
