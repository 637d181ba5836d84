"""Cost of the 'dgc' memory (momentum correction + momentum factor masking) on ResNet-50, bf16 buckets, bloom at 1 %,
and of its weight decay.

Two measurements on one GPU, each alternating its three arms round by round:

* exchange kernel: one bf16 ``BucketEngine`` over every ResNet-50 parameter with the residual memory, the same
  engine with ``momentum=0.9`` (phase 0 also streams the fp32 momentum in and out: 8 B per element), and with
  ``momentum=0.9, weight_decay=1e-4`` (phase 0 also reads the bf16 parameters: 2 B more per element), once with
  random parameters and once with all-zero parameters ("w = 0": d = g exactly, so that arm computes what the plain
  'dgc' arm computes and differs from it only by the parameter read); every arm exchanges the same gradients;
  ms per launch from CUDA events over ``--launches`` launches;
* whole training step: ResNet-50 with bf16 conv / linear weights and fp32 BatchNorm (batch ``--batch``, 224 x 224,
  channels_last, so one bf16 and one fp32 bucket) under ``DeepReduceDDP`` with residual + SGD(momentum 0.9),
  dgc + SGD(momentum 0), and dgc with 'weight_decay' + SGD(momentum 0, weight_decay 0), img/s from CUDA events over
  ``--steps`` steps.

Prints one JSON line with the card's name and power limit read in the same process.

    python scripts/dgc_step.py --launches 200 --steps 30 --rounds 3 [--batch 64] [--out DIR]
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

BLOOM = {'compressor': 'topk', 'communicator': 'allgather', 'compress_ratio': 0.01, 'deepreduce': 'index',
         'index': 'bloom', 'calibrate_partition': False}
ARMS = {"residual": ({**BLOOM, 'memory': 'residual'}, 0.9),
        "dgc": ({**BLOOM, 'memory': 'dgc', 'momentum': 0.9}, 0.0),
        "dgc_weight_decay": ({**BLOOM, 'memory': 'dgc', 'momentum': 0.9, 'weight_decay': 1e-4}, 0.0)}


def exchange_kernel(launches, rounds):
    import torch
    from deepreduce_b200 import models
    from deepreduce_b200.parallel import BucketPlan
    from deepreduce_b200.parallel.ddp import make_engine, plan_kwargs_from_params
    numels = [p.numel() for p in reversed(list(models.resnet50().parameters()))]
    gen = torch.Generator(device="cuda:0").manual_seed(7)
    weights = [torch.randn(n, device="cuda:0", generator=gen).to(torch.bfloat16) for n in numels]
    g = (torch.randn(sum(numels), device="cuda:0", generator=gen) * 1e-3).to(torch.bfloat16)
    zeros = [torch.zeros_like(w) for w in weights]
    arms = {name: (params, weights) for name, (params, _) in ARMS.items()}
    arms["dgc_weight_decay_w0"] = (ARMS["dgc_weight_decay"][0], zeros)
    engs, res = {}, {}
    for name, (params, ws) in arms.items():
        plan = BucketPlan(numels, **plan_kwargs_from_params(params))
        eng = make_engine(plan, params, device=torch.device("cuda:0"), group=None, use_history=True, blocks_per_sm=2,
                          grad_dtype=torch.bfloat16, parameters=ws)
        flat = torch.zeros(plan.total_elems, dtype=torch.bfloat16, device="cuda:0")
        off = 0
        for v in plan.views(flat):       # every arm exchanges the same gradients: only the memory differs
            v.copy_(g[off:off + v.numel()].view(v.shape))
            off += v.numel()
        engs[name] = (eng, flat)
        res[name] = {"elements": int(plan.total_elems), "momentum_buffer": eng.mom is not None,
                     "weight_decay": eng.weight_decay, "ms": []}

    def launch(name):
        eng, g = engs[name]
        return lambda i: (eng.grad.copy_(g), eng.step())

    for name in engs:                       # warm-up: module load, first launches, select history
        events_ms(launch(name), 5)
    copy_ms = []
    for rnd in range(rounds):
        for name in (list(engs) if rnd % 2 == 0 else list(reversed(engs))):
            res[name]["ms"].append(round(events_ms(launch(name), launches) / launches, 4))
        eng, g = engs["residual"]         # the gradient refill alone, reported so that it can be subtracted
        copy_ms.append(events_ms(lambda i: eng.grad.copy_(g), launches) / launches)
    for name, (eng, _) in engs.items():
        eng.check_status()
        eng.close()
    res["refill_ms"] = round(min(copy_ms), 4)
    return res


def train_step(steps, rounds, batch):
    import torch
    from deepreduce_b200.models import resnet50
    from deepreduce_b200.parallel import DeepReduceDDP
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    x = torch.randn(batch, 3, 224, 224, device="cuda:0", generator=gen).to(torch.bfloat16)
    x = x.contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device="cuda:0", generator=gen)
    runs, res = {}, {}
    for name, (params, momentum) in ARMS.items():
        torch.manual_seed(0)
        model = resnet50().to(device="cuda:0", memory_format=torch.channels_last)
        for m in model.modules():       # bf16 weights (bf16 buckets); BatchNorm keeps fp32 parameters and statistics
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)):
                m.to(torch.bfloat16)
        ddp = DeepReduceDDP(model, params)
        opt = torch.optim.SGD(model.parameters(), lr=1e-3, momentum=momentum, fused=True)

        def step(i, model=model, ddp=ddp, opt=opt):
            ddp.zero_grad()
            torch.nn.functional.cross_entropy(model(x).float(), y).backward()
            ddp.finish()
            opt.step()
        events_ms(step, 3)
        ddp.check()
        runs[name] = (ddp, step)
        res[name] = {"buckets": len(ddp.flat), "bucket_dtypes": sorted({str(f.dtype) for f in ddp.flat}),
                     "optimizer_momentum": momentum, "img_per_s": []}
    for rnd in range(rounds):
        for name in (list(runs) if rnd % 2 == 0 else list(reversed(runs))):
            ddp, step = runs[name]
            ms = events_ms(step, steps) / steps
            res[name]["img_per_s"].append(round(batch / ms * 1e3, 1))
            ddp.check()
    for ddp, _ in runs.values():
        ddp.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", default=None, help="directory for the JSON line (default: print only)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("dgc_step.py measures on a GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    out = {"what": "ResNet-50, bf16 buckets, top-k 1 % + bloom index, W = 1: residual vs dgc memory vs dgc memory "
                   "with weight decay",
           "card": card(), "exchange_kernel": exchange_kernel(args.launches, args.rounds),
           "train_step": train_step(args.steps, args.rounds, args.batch)}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dgc_step.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
