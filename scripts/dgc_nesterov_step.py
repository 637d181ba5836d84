"""Cost of Nesterov momentum ('nesterov') and weight-decay exclusions ('weight_decay_exclude') of the 'dgc' memory in
the exchange kernel, on ResNet-50 shapes.

One ``BucketEngine`` over every ResNet-50 parameter (top-k 1 %, bloom index, W = 1, 2 CTAs per SM), for fp32 and for
bf16 buckets, in five arms: 'dgc' with 'weight_decay'; the same + 'nesterov'; the same + 'weight_decay_exclude' on
every BatchNorm parameter and every bias; and the first and the last of these with 'clip_norm' (c = the median
parameter norm), which run the clipping kernels.  This project's ResNet-50 names its BatchNorms ``bn1`` .. ``bn3`` and,
on the shortcut, ``downsample.1``, so the patterns are ['*.bias', '*bn*', '*downsample.1.weight'] (107 of the 161
tensors): patterns match names, not layer types.  Nesterov adds two fp32 ops per element to phase 0; an excluded
tensor skips its parameter read.  Every arm exchanges the same gradients and reads the same parameters.  Arms alternate
round by round; ms per launch from CUDA events over ``--launches`` launches, with the gradient refill timed alone so
that it can be subtracted.

Prints one JSON line with the card's name and power limit read in the same process.

    python scripts/dgc_nesterov_step.py --launches 200 --rounds 3 [--out DIR]
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

DGC = {'compressor': 'topk', 'communicator': 'allgather', 'compress_ratio': 0.01, 'deepreduce': 'index',
       'index': 'bloom', 'calibrate_partition': False, 'memory': 'dgc', 'momentum': 0.9, 'weight_decay': 1e-4}
EXCLUDE = ['*.bias', '*bn*', '*downsample.1.weight']
ARMS = {"dgc": DGC, "nesterov": {**DGC, 'nesterov': True},
        "nesterov_exclude": {**DGC, 'nesterov': True, 'weight_decay_exclude': EXCLUDE},
        "clip": DGC, "clip_nesterov_exclude": {**DGC, 'nesterov': True, 'weight_decay_exclude': EXCLUDE}}


def exchange_kernel(launches, rounds):
    import torch
    from deepreduce_b200 import models
    from deepreduce_b200.parallel import BucketPlan
    from deepreduce_b200.parallel.ddp import make_engine, plan_kwargs_from_params
    named = list(reversed(list(models.resnet50().named_parameters())))
    names, numels = [n for n, _ in named], [p.numel() for _, p in named]
    gen = torch.Generator(device="cuda:0").manual_seed(7)
    g32 = torch.randn(sum(numels), device="cuda:0", generator=gen) * 1e-3
    w32 = torch.randn(sum(numels), device="cuda:0", generator=gen) * 1e-2
    norms = sorted(float(t.norm()) for t in torch.split(g32, numels))
    c = norms[len(norms) // 2]                 # the median parameter norm: about half of them are clipped
    engs, res = {}, {}
    for dtype in (torch.float32, torch.bfloat16):
        g = g32.to(dtype)
        params = [t.clone() for t in torch.split(w32.to(dtype), numels)]
        for arm, cfg in ARMS.items():
            cfg = {**cfg, 'clip_norm': c} if arm.startswith("clip") else cfg
            name = f"{str(dtype).split('.')[-1]}_{arm}"
            plan = BucketPlan(numels, names, **plan_kwargs_from_params(cfg))
            eng = make_engine(plan, cfg, device=torch.device("cuda:0"), group=None, use_history=True,
                              blocks_per_sm=2, grad_dtype=dtype, parameters=params, names=names)
            flat = torch.zeros(plan.total_elems, dtype=dtype, device="cuda:0")
            off = 0
            for v in plan.views(flat):
                v.copy_(g[off:off + v.numel()].view(v.shape))
                off += v.numel()
            engs[name] = (eng, flat)
            res[name] = {"elements": int(plan.total_elems), "nesterov": eng.nesterov, "clip_norm": eng.clip_norm,
                         "excluded_tensors": sum(d == 0.0 for d in eng.decays),
                         "excluded_elements": sum(t.numel for t, d in zip(plan.tensors, eng.decays) if d == 0.0),
                         "bucket_mb": round(plan.total_elems * flat.element_size() / 1e6, 1), "ms": []}

    def launch(name):
        eng, g = engs[name]
        return lambda i: (eng.grad.copy_(g), eng.step())

    for name in engs:                           # warm-up: module load, first launches, select history
        events_ms(launch(name), 5)
    refill = {n: [] for n in engs}
    for rnd in range(rounds):
        for name in (list(engs) if rnd % 2 == 0 else list(reversed(engs))):
            res[name]["ms"].append(round(events_ms(launch(name), launches) / launches, 4))
            eng, g = engs[name]
            refill[name].append(events_ms(lambda i: eng.grad.copy_(g), launches) / launches)
    for name, (eng, _) in engs.items():
        eng.check_status()
        eng.close()
        res[name]["refill_ms"] = round(min(refill[name]), 4)
        res[name]["kernel_ms_min"] = round(min(res[name]["ms"]) - res[name]["refill_ms"], 4)
    for dt in ("float32", "bfloat16"):
        base = res[f"{dt}_dgc"]["kernel_ms_min"]
        res[f"{dt}_nesterov_cost_ms"] = round(res[f"{dt}_nesterov"]["kernel_ms_min"] - base, 4)
        res[f"{dt}_nesterov_exclude_cost_ms"] = round(res[f"{dt}_nesterov_exclude"]["kernel_ms_min"] - base, 4)
        res[f"{dt}_clip_nesterov_exclude_cost_ms"] = round(res[f"{dt}_clip_nesterov_exclude"]["kernel_ms_min"]
                                                           - res[f"{dt}_clip"]["kernel_ms_min"], 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON line (default: print only)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dgc_nesterov_step.py measures on a GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    out = {"what": "ResNet-50 in one bucket, top-k 1 % + bloom index, W = 1, 2 CTAs/SM: 'dgc' memory with "
                   "'weight_decay', + 'nesterov', + 'weight_decay_exclude' " + json.dumps(EXCLUDE) + ", each of the "
                   "first and last also with 'clip_norm', fp32 and bf16 buckets",
           "card": card(), "exchange_kernel": exchange_kernel(args.launches, args.rounds)}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dgc_nesterov_step.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
