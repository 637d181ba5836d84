"""Exchange time of double-exponential values in the fused engine ('fused_dexp') on ResNet-50's tensors.

One GPU, one fp32 bucket holding every ResNet-50 parameter (what ``bench.py``'s 128 MB bucket cap gives), seeded
gradients.  Per top-k ratio (1 % and 0.1 % by default) three arms:

* ``rle_dexp``    — fused engine, run-length index + double-exponential values (``'deepreduce': 'both'``,
  ``'fused_dexp': True``);
* ``rle_polyfit`` — fused engine, run-length index + polyfit values (``'fused_rle_values': True``);
* ``dexp_grace``  — the ``rle_dexp`` dict without the key, which runs the per-tensor path: one ``grc.step`` per
  parameter (torch sort, ``dexp_fit_kernel``, the GRACE allgather at W = 1).

The fused arms are timed with CUDA events over ``--launches`` exchange kernels per round, the per-tensor arm over one
step (every parameter once) per round, rounds alternating.  Prints one JSON line with ms per exchange, wire bytes per
step, and the card's name and power limit read in the same process.

    python scripts/dexp_fused_step.py --launches 200 --rounds 3 [--ratios 0.01,0.001] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from randomk_step import card, events_ms  # noqa: E402

TOPK = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather'}
RLE_DEXP = {**TOPK, 'deepreduce': 'both', 'index': 'rle', 'value': 'dexp'}


def arms(ratio):
    return {
        "rle_dexp": {**RLE_DEXP, 'compress_ratio': ratio, 'fused_dexp': True},
        "rle_polyfit": {**TOPK, 'compress_ratio': ratio, 'deepreduce': 'both', 'index': 'rle', 'value': 'polyfit',
                        'fused_rle_values': True},
        "dexp_grace": {**RLE_DEXP, 'compress_ratio': ratio},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200, help="exchange kernels per round (fused arms)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ratios", default="0.01,0.001")
    ap.add_argument("--out", default=None, help="directory for the JSON line (default: print only)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dexp_fused_step.py measures on a GPU; no CUDA device is visible")
    from deepreduce_b200 import models
    from deepreduce_b200.parallel import BucketEngine, BucketPlan
    from deepreduce_b200.parallel.ddp import fused_path, plan_kwargs_from_params
    from deepreduce_b200.wrappers import deepreduce_from_params
    torch.manual_seed(1234)
    named = [(n, p) for n, p in reversed(list(models.resnet50().named_parameters()))]
    numels = [p.numel() for _, p in named]
    gen = torch.Generator().manual_seed(77)
    grads = [(n, (torch.randn(p.numel(), generator=gen) * 1e-3).view(p.shape).cuda()) for n, p in named]
    res = {}
    for ratio in (float(r) for r in args.ratios.split(",")):
        table = arms(ratio)
        runners, row = {}, {}
        for a, params in table.items():
            assert fused_path(params) == (a != "dexp_grace"), a
            if a == "dexp_grace":
                grc = deepreduce_from_params(dict(params))
                runners[a] = (lambda i, grc=grc: [grc.step(g.clone(), n) for n, g in grads], 1)
                row[a] = {"params": params}
                continue
            plan = BucketPlan(numels, **plan_kwargs_from_params(params))
            eng = BucketEngine(plan, device="cuda:0", world=1, rank=0)
            flat = torch.zeros(plan.total_elems)
            for t, (_, g) in zip(plan.tensors, grads):
                flat[t.elem_off:t.elem_off + t.numel] = g.reshape(-1).cpu()
            eng.grad.copy_(flat.cuda())
            runners[a] = (lambda i, eng=eng: eng.step(), args.launches)
            row[a] = {"params": params, "wire_bytes_per_step": plan.wire_bytes(),
                      "coded_tensors": sum(t.vmode != 0 for t in plan.tensors), "engine": eng}
        for a, (fn, n) in runners.items():          # warm-up: modules, first launches, the per-tensor path's allocations
            for i in range(3):
                fn(i)
        torch.cuda.synchronize()
        names = list(runners)
        for a in names:
            row[a]["ms"] = []
        for rnd in range(args.rounds):
            for a in (names if rnd % 2 == 0 else list(reversed(names))):
                fn, n = runners[a]
                row[a]["ms"].append(events_ms(fn, n) / n)
        for a in names:
            eng = row[a].pop("engine", None)
            if eng is not None:
                eng.check_status()
                eng.close()
        res[str(ratio)] = row
    out = {"what": "ResNet-50 tensors in one fp32 bucket, W = 1: fused exchange kernel per launch (rle + dexp, rle + "
                   "polyfit) and one per-tensor dexp step (every parameter)", "card": card(), "ratios": res}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dexp_fused_step.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
