"""Multi-GPU correctness self-check of the fused exchange (used by ``bench.py`` at N > 1 and by the GPU tests).

SCALE-style benchmarks prove speed, not that W ranks end a step holding the same, right gradient.  ``multi_gpu_check``
runs ONE extra exchange step of a live engine on fresh per-rank random gradients and verifies, on the device:

1. every rank's aggregated gradient is bit-identical (all-reduce MIN/MAX of the raw bit patterns);
2. the slots that the in-kernel P2P pushes left in this rank's arena are bit-identical to the same slots gathered
   with a plain NCCL ``all_gather`` (the transport the reference uses, SURVEY C1);
3. the aggregate equals what an independent decoder makes of the NCCL-gathered slots — ``decode_slot_torch`` below,
   written with plain torch ops on the wire-format specification (``spec`` / ``codecs.bloom`` oracles), sharing no
   code with the CUDA kernels;
4. error feedback conserves the gradient: ``new_residual + own shipped contribution == beta*residual + gamma*grad``.

A bf16 engine gets the same check: its input is the bf16 rounding of the random gradient, the residual and the decode
stay fp32, and check 3 compares against the independent decode rounded once to bf16.

Reference semantics being checked: GRACE Allgather communicator = per-rank decode + sum + /W (reference README.md:37,
SURVEY Appendix A), Bloom.decompress (pytorch/deepreduce.py:536-555).
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from .. import spec
from ..codecs.bloom import bloom_query_oracle
from ..parallel.plan import DYN_WORDS, MODE_BLOOM, MODE_RAW, MODE_SHARED, SLOT_HEADER_WORDS, VMODE_FP32


def decode_slot_torch(plan, slot: torch.Tensor, seed: int = spec.DEFAULT_SEED):
    """One sender's dense contribution (flat fp32, unscaled) rebuilt from the words of its slot with torch ops on the
    slot's device.  Supports the fp32-value modes (bloom index with/without hint, plain pairs, the shared 'randomk'
    index); returns None if the plan uses a mode this decoder does not cover (value codecs, run-length) — callers then
    skip check 3."""
    dev = slot.device
    hdr = slot[:SLOT_HEADER_WORDS + DYN_WORDS * len(plan.tensors)].to(torch.int64).cpu() & 0xFFFFFFFF
    out = torch.zeros(plan.total_elems, dtype=torch.float32, device=dev)
    for ti, t in enumerate(plan.tensors):
        if t.vmode != VMODE_FP32 or t.mode not in (MODE_BLOOM, MODE_RAW, MODE_SHARED):
            return None
        d0 = SLOT_HEADER_WORDS + DYN_WORDS * ti
        n_sel, cutoff = int(hdr[d0]), int(hdr[d0 + 1])
        if n_sel == 0:
            continue
        if t.mode == MODE_BLOOM:
            words = slot[t.off_filter:t.off_filter + t.n_filter_words]
            pos = bloom_query_oracle(words, t.numel, t.n_hash, t.m_bits, seed)
            if t.off_hint:
                hint = slot[t.off_hint:t.off_hint + 4 * t.n_tiles].to(torch.int64) & 0xFFFFFFFF
                grp = pos // 32
                pos = pos[((hint[grp // 32] >> (grp % 32)) & 1).bool()]
            if plan.policy == "random":                    # header word 2 = acceptance threshold, word 1 of the slot = step
                T = int(hdr[d0 + 2])
                if T != 0xFFFFFFFF:
                    pos = pos[(spec.policy_hash(pos, spec.policy_seed(int(hdr[1]), t.salt)) <= T).to(pos.device)]
            if plan.policy == "conflict_sets":             # P2: keep the positives whose rank is set in the shipped pick
                head = pos[:t.pos_cap]
                q = torch.arange(head.numel(), device=head.device)
                pick = slot[t.off_pick:t.off_pick + (t.pos_cap + 31) // 32].to(torch.int64).to(head.device) & 0xFFFFFFFF
                pos = head[((pick[q >> 5] >> (q & 31)) & 1).bool()]
            if cutoff != 0xFFFFFFFF:
                pos = pos[pos <= cutoff]
            idx = pos[:n_sel]
        elif t.mode == MODE_SHARED:                        # no index on the wire: draw the set from the plan + the step
            from ..parallel.engine import select_randomk_oracle
            pos = select_randomk_oracle(t.numel, t.k, int(hdr[1]), t.salt)[0].to(dev)
            if cutoff != 0xFFFFFFFF:
                pos = pos[pos <= cutoff]
            idx = pos[:n_sel]
        else:
            idx = slot[t.off_idx:t.off_idx + n_sel].to(torch.int64) & 0xFFFFFFFF
        vals = slot[t.off_vals:t.off_vals + idx.numel()].view(torch.float32)
        out[t.elem_off:t.elem_off + t.numel].index_add_(0, idx, vals)
    return out


def _bits_equal_across_ranks(x: torch.Tensor, group=None) -> bool:
    bits = x.view(torch.int32)
    lo, hi = bits.clone(), bits.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=group)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=group)
    return bool(torch.equal(lo, hi))


@torch.no_grad()
def multi_gpu_check(engine, seed: int = 4242) -> dict:
    """Run one checked exchange step on ``engine`` (a live ``BucketEngine``; its residual / epoch advance by one
    step).  Returns ``{"status": "ok" | "FAILED: ...", ...details}``; collective — every rank must call it."""
    from ..parallel.engine import clip_oracle, decay_oracle
    W, rank, plan = engine.world, engine.rank, engine.plan
    dev = engine.device
    gen = torch.Generator(device=dev).manual_seed(seed + 1000 * rank)
    g = torch.zeros(plan.total_elems, device=dev)
    for v in plan.views(g):
        v.copy_(torch.randn(v.shape, device=dev, generator=gen) * 1e-2)
    g = g.to(engine.grad.dtype).float()         # bf16 engine: the widened bf16 gradient is what the engine accumulates
    if engine.mom is not None:                  # 'dgc': the momentum is compensated, then added to the residual
        c = clip_oracle(plan, g, engine.clip_thr, engine.owner) if engine.clip_thr is not None else g
        if engine.weight_decay != 0.0:
            d = c + (engine.weight_decay * engine.parameter_buffer())
        elif engine.reads_parameters:                # per-parameter factors ('weight_decay_exclude')
            d = decay_oracle(plan, c.cpu(), engine.parameter_buffer().cpu(), engine.decays).to(dev)
        else:
            d = c
        u = engine.momentum * engine.mom + d
        acc = engine.resid + ((d + (engine.momentum * u)) if engine.nesterov else u)
    else:
        acc = engine.beta * engine.resid + engine.gamma * g if engine.beta != 0.0 else engine.gamma * g
    engine.grad.copy_(g)
    engine.step()
    torch.cuda.synchronize(dev)
    engine.check_status()
    out = engine.grad.clone()
    res = {"world": W, "tensors": len(plan.tensors), "elements": int(plan.total_elems)}
    fails = []
    # 1. all ranks hold the same bits
    if W > 1 and not _bits_equal_across_ranks(out, engine.group):
        fails.append("ranks hold different aggregated gradients")
    # 2. P2P-delivered slots == NCCL-gathered slots
    mine = engine.slot(rank).clone()
    if W > 1:
        gathered = [torch.empty_like(mine) for _ in range(W)]
        dist.all_gather(gathered, mine, group=engine.group)
        p2p_same = all(torch.equal(engine.slot(r), gathered[r]) for r in range(W))
        if not p2p_same:
            fails.append("slots delivered by in-kernel P2P stores differ from the NCCL all_gather of the same slots")
    else:
        gathered = [mine]
    # 3. independent decode of the gathered slots
    scale = (1.0 / W) if engine.average else 1.0
    ref = torch.zeros_like(out)
    own = None
    covered = True
    for r in range(W):
        dec = decode_slot_torch(plan, gathered[r], seed=spec.DEFAULT_SEED)
        if dec is None:
            covered = False
            break
        if r == rank:
            own = dec
        ref += dec * scale              # same order as the kernel: rank-major, one multiply-add per sender
    if covered:
        ref_out = ref.to(out.dtype)     # bf16 engine: the fp32 aggregate rounded once
        diff = float((ref_out.float() - out.float()).abs().max())
        res["max_abs_diff_vs_independent_decode"] = diff
        if not torch.equal(ref_out, out):
            # the fp32 sums may differ in order (last ulps); in bf16 that can move the rounding by one bf16 ulp
            tol = 1e-6 * float(ref.abs().max()) + (2.0 ** -7 * ref.abs() if out.dtype == torch.bfloat16 else 0.0)
            if bool(((ref_out.float() - out.float()).abs() > tol).any()):
                fails.append(f"aggregate differs from the independent decode of the gathered slots (max abs {diff:.3e})")
        # 4. error feedback conserves the gradient (fp32 values on the wire: exact)
        if not torch.equal(engine.resid + own, acc):
            fails.append("residual + own shipped contribution != compensated gradient")
    else:
        res["note"] = "value-coded / run-length plan: independent torch decoder not applicable, checks 1-2 only"
    if W > 1:       # agree on the verdict
        flag = torch.tensor([1 if fails else 0], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=engine.group)
        if int(flag.item()) and not fails:
            fails.append("another rank reported a failure")
    res["status"] = "ok" if not fails else "FAILED: " + "; ".join(fails)
    return res
