"""Cost of the sparsity warm-up on ResNet-50 shapes: the exchange kernel at every stage's compress ratio, and one stage
switch.

One bucket over every ResNet-50 parameter (top-k, bloom index, residual memory, W = 1, fp32), chunked by the final
ratio (0.1 %) as ``DeepReduceDDP`` chunks it, with DGC's schedule 25 % / 6.25 % / 1.5625 % / 0.4 % ahead of it.

- exchange kernel: ms per launch of each stage's engine, from CUDA events over ``--launches`` launches, stages
  alternating round by round, the gradient refill timed alone and subtracted;
- stage switch: wall time of ``DeepReduceDDP._switch_stage``'s work for this bucket (stage plan already built, engine
  construction with the partition calibration, aggregate save and restore, residual carry, close of the old engine),
  host clock around work that ends in a device synchronise, min over ``--switches``.

Prints one JSON line with the card's name and power limit read in the same process.

    python scripts/warmup_step.py --launches 100 --rounds 3 --switches 3 [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from randomk_step import card, events_ms  # noqa: E402

PARAMS = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.001,
          'deepreduce': 'index', 'index': 'bloom', 'warmup_ratios': [0.25, 0.0625, 0.015625, 0.004],
          'warmup_steps': 1}


def _bucket():
    from deepreduce_b200 import models
    from deepreduce_b200.config import warmup_from_params
    from deepreduce_b200.parallel.ddp import engine_split_numel, stage_plans
    from deepreduce_b200.parallel.plan import split_large
    ps = list(reversed(list(models.resnet50().parameters())))
    numels = [p.numel() for p in ps]
    names = [f"p{i}" for i in range(len(ps))]
    shapes = [tuple(p.shape) for p in ps]
    numels, names, shapes, owner = split_large(numels, names, shapes, engine_split_numel(PARAMS, 2))
    t0 = time.perf_counter()
    plans = stage_plans(numels, names, shapes, PARAMS, warmup_from_params(PARAMS))
    return plans, (time.perf_counter() - t0) * 1e3


def _engine(plan, params, grad=None):
    import torch
    from deepreduce_b200.parallel.ddp import make_engine
    return make_engine(plan, params, device=torch.device("cuda:0"), group=None, use_history=True, blocks_per_sm=2,
                       grad_dtype=torch.float32, grad=grad)


def exchange_kernel(plans, launches, rounds):
    import torch
    static = {**PARAMS, 'calibrate_partition': False}
    gen = torch.Generator(device="cuda:0").manual_seed(7)
    g = torch.randn(plans[0].total_elems, device="cuda:0", generator=gen) * 1e-3
    engs = {p.compress_ratio: _engine(p, static) for p in plans}
    res = {r: {"wire_bytes": int(e.plan.wire_bytes()), "ms": []} for r, e in engs.items()}

    def launch(e):
        return lambda i: (e.grad.copy_(g), e.step())

    for e in engs.values():
        events_ms(launch(e), 5)
    refill = []
    for rnd in range(rounds):
        for r in (list(engs) if rnd % 2 == 0 else list(reversed(engs))):
            res[r]["ms"].append(round(events_ms(launch(engs[r]), launches) / launches, 4))
        e0 = next(iter(engs.values()))
        refill.append(events_ms(lambda i: e0.grad.copy_(g), launches) / launches)
    for r, e in engs.items():
        e.check_status()
        e.close()
        res[r]["kernel_ms_min"] = round(min(res[r]["ms"]) - min(refill), 4)
    return {"elements": int(plans[0].total_elems), "refill_ms": round(min(refill), 4),
            "stages": {str(r): v for r, v in res.items()}}


def stage_switch(plans, switches):
    import torch
    out = {}
    for calibrate in (False, True):
        params = {**PARAMS, 'calibrate_partition': calibrate}
        times = []
        for _ in range(switches):
            old = _engine(plans[0], params)
            old.grad.normal_()
            old.step()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            agg = old.grad.clone()
            new = _engine(plans[1], params, grad=old.grad)
            new.grad.copy_(agg)
            new.resid.copy_(old.resid)
            new.epoch = max(new.epoch, old.epoch)
            old.close()
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
            new.check_status()
            new.close()
        out["calibrated" if calibrate else "static_cut"] = {"ms": [round(t, 2) for t in times],
                                                           "ms_min": round(min(times), 2)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--switches", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JSON line (default: print only)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("warmup_step.py measures on a GPU; no CUDA device is visible")
    torch.cuda.set_device(0)
    plans, plan_ms = _bucket()
    out = {"what": "ResNet-50 in one fp32 bucket, top-k + bloom index, residual memory, W = 1: exchange kernel per "
                   "warm-up stage and one stage switch (25 % -> 6.25 %)",
           "card": card(), "stage_plans_ms": round(plan_ms, 1),
           "exchange_kernel": exchange_kernel(plans, args.launches, args.rounds),
           "stage_switch": stage_switch(plans, args.switches)}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "warmup_step.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
