"""The exchange half of the fused engine at W > 1, on one GPU: W engines in one process play W ranks.

Each engine is ``world=W, rank=r`` with its own arena, and every engine's ``arena_ptrs`` is the list of all W arenas,
so the kernel's "peer" stores and flag waits land in plain device buffers.  A step runs in waves: every engine runs a
range of phases as one launch, and all engines finish a wave before any engine starts the next.  So every flag wait
runs after the launches that release its flags have finished, and no kernel ever waits on one that cannot be
scheduled; a flag that is never released becomes status 2 after ``peer_timeout_ms``.  What the waves cannot see is
cross-GPU memory ordering (missing fences, NVLink stores racing a peer's reads): that stays with ``run_multigpu.py``.

Per step and rank the tests check the slot against ``engine_oracle``, that every arena holds every sender's slot word
for word, the aggregate against the decode of the slots actually shipped, that all ranks hold the same bits, and
(sharded) the stage-2 lists word by word."""
import numpy as np
import pytest
import torch

from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
from deepreduce_b200.parallel.engine import (PH_ACCUM, PH_END, PH_EXPAND, PH_PUSH, PH_PUSH2, PH_SIGNAL, PH_SIGNAL2,
                                             decode_slot_oracle)
from deepreduce_b200.parallel.plan import ARENA_HDR_WORDS, DYN_WORDS, MODE_BLOOM, MODE_RAW, MODE_RLE, SLOT_HEADER_WORDS
from test_gpu_engine import SIZES, _compare_slot, _fill

pytestmark = pytest.mark.gpu

BIG = SIZES + [2359296]                  # 772 tiles; plain pairs on both sides of phase_compact's n_sel <= 2048 branch
SMALL = [10, 64, 1001, 4097]             # 5 tiles: fewer tiles than ranks at W = 8 and 16
CTA_CAP = 4096                           # engine.cu kCtaCap: entries of phase_compact's CTA stage
U = 2.0 ** -24                           # unit roundoff of fp32


class _RankEngine(BucketEngine):
    """One rank of a W-rank group whose arenas are preallocated buffers on this GPU (no IPC, no collective)."""

    def __init__(self, plan, arenas, rank, **kw):
        self._arenas = arenas
        super().__init__(plan, device="cuda:0", world=len(arenas), rank=rank, transport="p2p", **kw)

    def _setup_arena(self):
        self.arena = self._arenas[self.rank]
        self.arena_ptrs = [a.data_ptr() for a in self._arenas]
        self._ipc = False
        self.multicast_ptr = 0


def _engines(plan, W, config, average):
    kw = dict(average=average, spin_limit=4_000_000, peer_timeout_ms=5000)
    if config == "nccl":                 # local arena; the test replays the all_gather of _step_nccl
        return [BucketEngine(plan, device="cuda:0", world=W, rank=r, transport="nccl", **kw) for r in range(W)]
    shard = config == "shard"
    arenas = [torch.zeros(plan.arena_words(W, shard), dtype=torch.int32, device="cuda:0") for _ in range(W)]
    return [_RankEngine(plan, arenas, r, shard=shard, **kw) for r in range(W)]


def _wave(engs, begin, end, epoch):
    for e in engs:
        e.run_phases(begin, end, epoch)
    torch.cuda.synchronize()
    for e in engs:
        e.check_status()


def _run_step(engs, config, epoch):
    if config == "shard":
        for b, e in ((PH_ACCUM, PH_SIGNAL), (PH_SIGNAL, PH_SIGNAL2), (PH_SIGNAL2, PH_END)):
            _wave(engs, b, e, epoch)
    elif config == "noshard":
        for b, e in ((PH_ACCUM, PH_SIGNAL), (PH_SIGNAL, PH_END)):
            _wave(engs, b, e, epoch)
    else:
        _wave(engs, PH_ACCUM, PH_PUSH, epoch)
        W, sw = len(engs), engs[0].plan.slot_words
        base = ARENA_HDR_WORDS + (epoch & 1) * W * sw
        for r, src in enumerate(engs):         # all_gather: rank r's slot lands at index r of every arena
            for dst in engs:
                if dst is not src:
                    dst.arena[base + r * sw:base + (r + 1) * sw].copy_(src.arena[base + r * sw:base + (r + 1) * sw])
        _wave(engs, PH_EXPAND, PH_PUSH2, epoch)


def _spans(n_tiles, W):
    """decode_span: the tiles [begin, end) that rank o owns in the sharded decode."""
    return [(n_tiles * o // W, n_tiles * (o + 1) // W) for o in range(W)]


def _tiles(plan):
    tt = plan.tile_table().numpy().view(np.uint32).reshape(-1, 4).astype(np.int64)
    return tt[:, 0], tt[:, 1], tt[:, 2] & 0xFFFF          # tensor, first element, elements


def _exact_tensor(t, W, average, ordered):
    """Whether the kernel's sum over senders for this tensor is determined bit for bit, so that torch's
    fp32 ``ref + dec * scale`` in rank order predicts it.  None: value codec (fp32 on the GPU vs fp64 fit)."""
    if t.vmode:
        return None
    pow2 = not average or (W & (W - 1)) == 0             # v * (1/W) is exact: an FMA contraction cannot change bits
    if t.mode == MODE_BLOOM:
        # ordered: one warp per tile walks the senders, `*o + v*scale` (contractible); fast: RED.ADD in any order,
        # which only W = 2 makes order-free (0 + a + b)
        return (ordered and pow2) or (not ordered and W == 2)
    if t.mode == MODE_RLE:
        return pow2                                      # SMEM `acc += v*scale` in rank order (contractible)
    return True                                          # plain pairs: SMEM atomicAdd of the rounded product, rank order


# (id, configuration, W, sizes, plan keyword arguments, DR_DETERMINISTIC, average, rank with an all-zero gradient,
#  properties the case asserts it has)
C = pytest.param
CASES = [
    # ---- sharded P2P: the full matrix
    C("shard", 2, BIG, dict(index="bloom"), False, True, None, {"raw"}, id="shard-bloom-W2-fast"),
    C("shard", 4, SIZES, dict(index="bloom", hint=False), True, True, None, {"nohint"}, id="shard-bloom-nohint-W4-det"),
    C("shard", 3, SIZES, dict(index="bloom", policy="p0"), True, False, None, {"split"}, id="shard-p0-W3-det-sum"),
    C("shard", 3, SIZES, dict(index="bloom", policy="random", fpr=0.02), False, True, None, {"random_T", "split"},
      id="shard-random-W3-fast"),
    C("shard", 3, BIG, dict(index=None), True, True, None, {"raw2048", "split"}, id="shard-raw-W3-det"),
    C("shard", 5, BIG, dict(index=None), False, False, None, {"raw2048", "split"}, id="shard-raw-W5-fast-sum"),
    C("shard", 8, SIZES, dict(index=None), False, True, None, {"raw"}, id="shard-raw-W8-fast"),
    C("shard", 5, SIZES, dict(index="bloom"), True, True, None, {"split"}, id="shard-bloom-W5-det"),
    C("shard", 8, SIZES, dict(index="bloom"), True, False, None, {"split"}, id="shard-bloom-W8-det-sum"),
    C("shard", 4, BIG, dict(index="rle"), False, True, None, {"rle"}, id="shard-rle-W4-fast"),
    C("shard", 3, SIZES, dict(index="rle"), True, True, None, {"rle", "split"}, id="shard-rle-W3-det"),
    C("shard", 2, SIZES, dict(index="bloom", value="polyfit", poly_min_k=300), False, True, None, {"polyfit"},
      id="shard-both-W2-fast"),
    C("shard", 3, SIZES, dict(index="bloom", value="qsgd"), True, True, None, {"qsgd8"}, id="shard-qsgd8-W3-det"),
    C("shard", 4, SIZES, dict(index="bloom", value="qsgd", quantum_num=1000), False, False, None, {"qsgd16"},
      id="shard-qsgd16-W4-fast-sum"),
    C("shard", 2, SIZES, dict(index=None, value="polyfit", poly_min_k=300), True, True, None, {"polyfit"},
      id="shard-valuepoly-W2-det"),
    C("shard", 2, BIG, dict(index="bloom", sparsifier="threshold", threshold=0.0, capacity_ratio=0.5), False, True, 0,
      {"cta_overflow"}, id="shard-dense-W2-fast"),
    C("shard", 4, SIZES, dict(index="bloom", sparsifier="threshold", threshold=1.0, capacity_ratio=0.2), True, True, 2,
      set(), id="shard-threshold-W4-det"),
    C("shard", 8, SMALL, dict(index="bloom"), False, True, None, {"empty"}, id="shard-small-W8-fast"),
    C("shard", 16, SMALL, dict(index="bloom"), True, True, None, {"empty"}, id="shard-small-W16-det"),
    C("shard", 16, SMALL, dict(index="rle"), False, True, None, {"empty", "rle"}, id="shard-small-rle-W16-fast"),
    # ---- unsharded P2P (DR_SHARD=0): every rank decodes every tile
    C("noshard", 3, SIZES, dict(index="bloom"), False, True, None, set(), id="noshard-bloom-W3-fast"),
    C("noshard", 4, SIZES, dict(index="rle"), False, True, None, {"rle"}, id="noshard-rle-W4-fast"),
    C("noshard", 3, SIZES, dict(index="bloom", value="polyfit", poly_min_k=300), False, True, None, {"polyfit"},
      id="noshard-both-W3-fast"),
    C("noshard", 3, SIZES, dict(index="bloom", sparsifier="threshold", threshold=1.0, capacity_ratio=0.2), False, False,
      1, set(), id="noshard-threshold-W3-fast-sum"),
    # ---- NCCL transport, its all_gather replayed by copies
    C("nccl", 4, SIZES, dict(index="bloom"), False, True, None, set(), id="nccl-bloom-W4-fast"),
    C("nccl", 3, SIZES, dict(index="rle"), True, True, None, {"rle"}, id="nccl-rle-W3-det"),
    C("nccl", 3, SIZES, dict(index="bloom", value="polyfit", poly_min_k=300), False, True, None, {"polyfit"},
      id="nccl-both-W3-fast"),
    C("nccl", 3, SIZES, dict(index="bloom", sparsifier="threshold", threshold=1.0, capacity_ratio=0.2), False, True, 0,
      set(), id="nccl-threshold-W3-fast"),
]


def _check_plan_claims(plan, W, claims):
    T = plan.tensors
    tensor_of_tile = _tiles(plan)[0]
    spans = _spans(plan.n_tiles, W)
    if "raw" in claims:
        assert any(t.mode == MODE_RAW for t in T)
    if "raw2048" in claims:                           # per-sender n_sel = K for top-k
        assert any(t.mode == MODE_RAW and t.k > 2048 for t in T) and any(t.mode == MODE_RAW and t.k <= 2048 for t in T)
    if "nohint" in claims:
        assert all(t.off_hint == 0 for t in T if t.mode == MODE_BLOOM) and any(t.mode == MODE_BLOOM for t in T)
    if "rle" in claims:
        assert any(t.mode == MODE_RLE for t in T)
    if "polyfit" in claims:
        assert any(t.vmode == 1 for t in T)
    if "qsgd8" in claims:
        assert any(t.vmode == 2 for t in T) and all(t.rank_u32 == 0 for t in T if t.vmode == 2)
    if "qsgd16" in claims:
        assert any(t.vmode == 2 for t in T) and all(t.rank_u32 == 1 for t in T if t.vmode == 2)
    if "empty" in claims:
        assert plan.n_tiles < W and any(b == e for b, e in spans)
    if "split" in claims:                             # a slice boundary falls inside a tensor
        assert plan.n_tiles % W and any(0 < b < plan.n_tiles and tensor_of_tile[b - 1] == tensor_of_tile[b]
                                        for b, _ in spans)


def _check_step_claims(plan, W, claims, slots, zero_rank, engs, outs, ordered):
    T = plan.tensors

    def dyn(r, ti, w):
        return int(slots[r][SLOT_HEADER_WORDS + DYN_WORDS * ti + w])
    if "random_T" in claims:                          # the senders' acceptance thresholds differ
        Ts = [{dyn(r, ti, 2) for r in range(W)} for ti, t in enumerate(T) if t.mode == MODE_BLOOM]
        assert any(len(s) > 1 and s != {0xFFFFFFFF} for s in Ts)
    if zero_rank is not None:                         # one sender ships nothing, another is at capacity
        assert all(dyn(zero_rank, ti, 0) == 0 for ti in range(len(T)))
        assert any(dyn(r, ti, 0) == t.val_cap for r in range(W) if r != zero_rank for ti, t in enumerate(T))
    if "cta_overflow" in claims:                      # some CTA's part of its slice holds more than its stage
        assert not ordered                             # the CTA stage exists only for RED.ADD sums
        _, base, n = _tiles(plan)
        nnz_tile = np.array([int((outs[0][b:b + k] != 0).sum()) for b, k in zip(base, n)])
        worst = 0
        for o, (sb, se) in enumerate(_spans(plan.n_tiles, W)):
            G, span = engs[o].grid(), se - sb
            for b in range(G):
                worst = max(worst, int(nnz_tile[sb + span * b // G:sb + span * (b + 1) // G].sum()))
        assert worst > CTA_CAP, worst


@pytest.mark.timeout(600)
@pytest.mark.parametrize("config,W,sizes,kw,deterministic,average,zero_rank,claims", CASES)
def test_engine_multirank_vs_oracle(monkeypatch, config, W, sizes, kw, deterministic, average, zero_rank, claims):
    monkeypatch.setenv("DR_DETERMINISTIC", "1" if deterministic else "0")
    monkeypatch.delenv("DR_S2_SLACK", raising=False)
    plan = BucketPlan(sizes, compress_ratio=0.01, **kw)
    _check_plan_claims(plan, W, claims)
    engs = _engines(plan, W, config, average)
    sharded = config == "shard"
    # unsharded engines at W > 2 take the rank-ordered sums whatever DR_DETERMINISTIC says (ranks must agree)
    ordered = deterministic or (not sharded and W > 2)
    scale = torch.tensor(1.0 / W if average else 1.0, dtype=torch.float32)    # the kernel's fp32 P.scale
    _, tbase, tn = _tiles(plan)
    exact = torch.ones(plan.total_elems, dtype=torch.bool)        # padding: must stay exactly zero
    coded = torch.zeros(plan.total_elems, dtype=torch.bool)
    for t in plan.tensors:
        how = _exact_tensor(t, W, average, ordered)
        seg = slice(t.elem_off, t.elem_off + t.numel)
        exact[seg] = bool(how)
        coded[seg] = how is None
    plain = ~exact & ~coded                                     # bits depend on order / contraction: explicit bound
    owner = torch.full((plan.total_elems,), -1, dtype=torch.int64)
    for o, (sb, se) in enumerate(_spans(plan.n_tiles, W)):
        for tile in range(sb, se):
            owner[tbase[tile]:tbase[tile] + tn[tile]] = o
    resid_refs = [torch.zeros(plan.total_elems) for _ in range(W)]
    value = kw.get("value")
    for step in range(3):                # step 0: no history; 1: history; 2: the first parity again, shrunk gradients
        epoch = step + 1
        grads = []
        for r in range(W):
            g = _fill(plan, torch.Generator().manual_seed(1000 * step + r)) * (0.2 if step == 2 else 1.0)
            grads.append(torch.zeros_like(g) if r == zero_rank else g)
        for e, g in zip(engs, grads):
            e.grad.copy_(g.cuda())
        _run_step(engs, config, epoch)
        outs = [e.grad.cpu() for e in engs]
        own = [e.slot().cpu() for e in engs]
        out_ref, new_res, slots = engine_oracle(plan, grads, resid_refs, average=average, epoch=epoch)
        tag = f"multirank_{config}_W{W}_s{step}"
        _check_step_claims(plan, W, claims, slots, zero_rank, engs, outs, ordered)
        # 1. every rank's slot against the oracle's, its residual against the oracle's
        for r, e in enumerate(engs):
            bad = _compare_slot(plan, own[r], slots[r], f"{tag}_r{r}")
            assert not bad, (r, bad[:4])
            if value is None:
                assert torch.equal(e.resid.cpu(), new_res[r]), (tag, r)
            else:
                sc = float(out_ref.abs().max())
                assert torch.allclose(e.resid.cpu(), new_res[r], atol=2e-3 * sc, rtol=1e-2), (tag, r)
        resid_refs = new_res if value is None else [e.resid.cpu().clone() for e in engs]
        # 2. delivery: every arena holds every sender's own slot, word for word
        for e in engs:
            for s in range(W):
                assert torch.equal(e.slot(s), engs[s].slot()), (tag, e.rank, s)
        # 3. the aggregate against the decode of the words shipped, summed in rank order (own rank included)
        decs = [decode_slot_oracle(plan, own[r]) for r in range(W)]
        ref = torch.zeros(plan.total_elems)
        ref64 = torch.zeros(plan.total_elems, dtype=torch.float64)
        mag = torch.zeros(plan.total_elems, dtype=torch.float64)
        for d in decs:
            ref = ref + d * scale                       # two fp32 roundings, as the kernel without contraction
            ref64 += d.double() * float(scale)
            mag += (d.double() * float(scale)).abs()
        for r, out in enumerate(outs):
            assert torch.equal(out[exact], ref[exact]), (tag, r, int((out[exact] != ref[exact]).sum()))
            err = (out[plain].double() - ref64[plain]).abs()
            assert bool((err <= (W + 1) * U * mag[plain]).all()), (tag, r, float(err.max()))
            if coded.any():
                sc = float(ref.abs().max())
                assert torch.allclose(out[coded], ref[coded], atol=2e-3 * sc, rtol=1e-2), (tag, r)
        # 4. every rank holds the same bits
        for r in range(1, W):
            assert torch.equal(outs[r].view(torch.int32), outs[0].view(torch.int32)), (tag, r)
        # 5. stage-2 lists: the owner's non-zeros of its slice, once each, with its bits, in every peer's arena
        if sharded:
            s2w = plan.stage2_layout(W)[1]
            s2_base = ARENA_HDR_WORDS + 2 * W * plan.slot_words + (epoch & 1) * W * s2w
            for o in range(W):
                mine = owner == o
                want = torch.nonzero(mine & (outs[o] != 0)).flatten()
                assert want.numel() == int((mine & (ref != 0)).sum()), (tag, o)
                assert engs[o].stage2_bytes() == 8 * want.numel() * (W - 1), (tag, o)
                for recv in range(W):
                    if recv == o:
                        continue
                    s2 = engs[recv].arena[s2_base + o * s2w:s2_base + (o + 1) * s2w].cpu()
                    n = int(s2[0])
                    assert n == want.numel() and int(s2[1]) == epoch, (tag, o, recv, n, want.numel(), int(s2[1]))
                    pairs = s2[4:4 + 2 * n].view(n, 2)
                    idx = pairs[:, 0].to(torch.int64)
                    assert torch.equal(torch.unique(idx), want), (tag, o, recv)      # unique sorts: no duplicates
                    assert idx.numel() == want.numel()
                    assert torch.equal(pairs[:, 1], outs[o].view(torch.int32)[idx]), (tag, o, recv)
        # 6. the sender-side oracle's aggregate
        # (sum of v) / W is exactly the sum of v / W when 1/W is a power of two
        same = exact if not average or (W & (W - 1)) == 0 else torch.zeros_like(exact)
        assert torch.equal(outs[0][same], out_ref[same]), (tag, int((outs[0][same] != out_ref[same]).sum()))
        rest = ~same & ~coded
        err = (outs[0][rest].double() - out_ref[rest].double()).abs()
        assert bool((err <= 2 * W * U * mag[rest]).all()), (tag, float(err.max()) if err.numel() else 0.0)
        if coded.any():
            sc = float(out_ref.abs().max())
            assert torch.allclose(outs[0][coded], out_ref[coded], atol=2e-3 * sc, rtol=1e-2), tag
    for e in engs:
        e.close()
