"""Cost of the conflict-sets (P2) bloom policy in the fused exchange engine, on one GPU.

A ResNet-50-shaped bucket (every parameter of ``models.resnet50`` in reverse order, top-k 1 %, bloom index, residual
on), W = 1.  Arms, timed in alternating rounds with CUDA events around ``--steps`` back-to-back steps:

* fused ``leftmost``, ``random`` and ``conflict_sets`` (the pick shipped as a bitmask, ``'p2_pick_mask': True``);
* the per-tensor path that ``conflict_sets`` takes without the key, for the same gradients: per tensor, GRACE's
  top-k + residual, the bloom insert, the universe query, the P2 draw (``conflict_sets_pick_kernel``) and the
  receiver's repeat of the query and the draw.  At W = 1 there is no collective; at W > 1 it adds 2-3 all_gathers per
  tensor and one repeat of the query and the draw per sender.

Prints one JSON line with the card's name and power limit read in the same process, plus the wire bytes of every
fused arm and of the P2 arm at 0.1 / 1 / 3 / 10 %.

    python scripts/p2_fused.py --steps 20 --rounds 3 [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from bf16_buckets import card, time_ms  # noqa: E402


def resnet50_numels():
    from deepreduce_b200.models import resnet50
    return [p.numel() for p in reversed(list(resnet50().parameters()))]


def wire_table(numels):
    from deepreduce_b200.parallel import BucketPlan
    out = {}
    for ratio in (0.001, 0.01, 0.03, 0.1):
        row = {}
        for pol in ("leftmost", "conflict_sets"):
            row[pol] = BucketPlan(numels, compress_ratio=ratio, policy=pol).wire_bytes()
        row["p2_extra_bytes"] = row["conflict_sets"] - row["leftmost"]
        out[str(ratio)] = row
    return out


def per_tensor_p2(numels, g, resid):
    """One step of the per-tensor P2 path at W = 1, without collectives (GRACE residual + top-k, Bloom codec)."""
    from deepreduce_b200 import spec
    from deepreduce_b200.codecs.bloom import Bloom
    off = 0
    for i, d in enumerate(numels):
        x = g[off:off + d]
        r = resid[off:off + d]
        acc = r.add_(x)
        if d > spec.SMALL_TENSOR_NUMEL:
            k = spec.topk_k(d, 0.01)
            idx = torch.topk(acc.abs(), k, sorted=False).indices
            params = {'policy': 'conflict_sets', 'dense_tensor': acc, 'policy_seed': i}
            vals, words, shape = Bloom.compress((acc[idx], idx, acc.shape), params)
            v2, i2, _ = Bloom.decompress((vals, words, acc.shape), {'policy': 'conflict_sets', 'policy_seed': i})
            out = torch.zeros_like(acc)
            out.index_add_(0, i2, v2)
            acc[i2] = 0
            x.copy_(out)
        off += d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    from deepreduce_b200 import ops
    from deepreduce_b200.parallel import BucketEngine, BucketPlan
    ops.require()
    numels = resnet50_numels()
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    engs = {}
    for pol in ("leftmost", "random", "conflict_sets"):
        plan = BucketPlan(numels, compress_ratio=0.01, policy=pol)
        e = BucketEngine(plan, device="cuda:0", world=1, rank=0)
        e.grad.copy_(torch.randn(plan.total_elems, device="cuda:0", generator=gen) * 1e-2)
        for _ in range(5):
            e.step()
        e.check_status()
        engs[pol] = e
    total = sum(numels)
    g = torch.randn(total, device="cuda:0", generator=gen) * 1e-2
    resid = torch.zeros(total, device="cuda:0")
    for _ in range(2):
        per_tensor_p2(numels, g.clone(), resid)
    times = {k: [] for k in list(engs) + ["per_tensor_conflict_sets"]}
    for _ in range(a.rounds):
        for pol, e in engs.items():
            times[pol].append(round(time_ms(e.step, a.steps), 4))
        gg = g.clone()
        times["per_tensor_conflict_sets"].append(round(time_ms(lambda: per_tensor_p2(numels, gg, resid), max(1, a.steps // 4)), 3))
    for e in engs.values():
        e.check_status()
    st = engs["conflict_sets"].stats()["total"]
    out = {"card": card(), "elements": total, "ms_per_step": times,
           "p2_stats": {k: st[k] for k in ("k", "n_sel", "n_pos", "beyond_cap", "tensors_beyond_cap")},
           "wire_bytes": wire_table(numels)}
    for e in engs.values():
        e.close()
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "p2_fused.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
