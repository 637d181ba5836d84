"""fp32 against bf16 gradient buckets in the fused exchange engine, on one GPU.

1. Exchange kernel alone: a ResNet-50-shaped bucket (every parameter of ``models.resnet50`` in reverse order, top-k 1 %,
   bloom and run-length index, residual on), W = 1.  An fp32 engine and a bf16 engine on the same gradients (the bf16
   one gets them rounded) are timed in alternating rounds: CUDA events around ``--steps`` back-to-back ``step()``s.
2. A W = 1 BERT-large training step (``models.zoo.bert_large``, parameters in bf16, batch ``--batch`` x 128 tokens,
   plain SGD): ``DeepReduceDDP`` on the fused top-k 1 % path (bloom, run-length) against the dense bf16 baseline
   (``'compressor': 'none'``), timed in alternating rounds with CUDA events around whole steps.

Prints one JSON line with the card's name and power limit read in the same process.

    python scripts/bf16_buckets.py --steps 50 --rounds 3 [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e!r})"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def time_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def exchange_kernel(steps, rounds):
    from deepreduce_b200.models import resnet50
    from deepreduce_b200.parallel import BucketEngine, BucketPlan
    numels = [p.numel() for p in reversed(list(resnet50().parameters()))]
    res = {}
    for index in ("bloom", "rle"):
        plan = BucketPlan(numels, compress_ratio=0.01, index=index)
        engs = {dt: BucketEngine(plan, device="cuda:0", world=1, rank=0, grad_dtype=dt)
                for dt in (torch.float32, torch.bfloat16)}
        g = torch.randn(plan.total_elems, device="cuda:0", generator=torch.Generator(device="cuda:0").manual_seed(0)) * 1e-2
        for e in engs.values():
            e.grad.copy_(g)
            for _ in range(5):
                e.step()
            e.check_status()
        times = {str(dt).split(".")[1]: [] for dt in engs}
        for _ in range(rounds):
            for dt, e in engs.items():
                # the gradient is overwritten by the aggregate; the kernel's work depends on the select, not the values,
                # and the residual keeps it at the trained operating point
                times[str(dt).split(".")[1]].append(round(time_ms(e.step, steps), 4))
        for e in engs.values():
            e.check_status()
            e.close()
        res[index] = {"elements": int(plan.total_elems), "ms_per_step": times}
    return res


def bert_step(steps, rounds, batch):
    from deepreduce_b200.models.zoo import bert_large
    from deepreduce_b200.parallel import DeepReduceDDP
    arms = {
        "dense": {'compressor': 'none', 'communicator': 'allreduce'},
        "topk_bloom": {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
                       'deepreduce': 'index', 'index': 'bloom', 'calibrate_partition': False},
        "topk_rle": {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
                     'deepreduce': 'index', 'index': 'rle', 'calibrate_partition': False},
    }
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    tokens = torch.randint(0, 30522, (batch, 128), device="cuda:0", generator=gen)
    labels = torch.randint(0, 30522, (batch, 128), device="cuda:0", generator=gen)
    res = {}
    runs = {}
    for name, cfg in arms.items():
        torch.manual_seed(0)
        model = bert_large(seq_len=512).to(device="cuda:0", dtype=torch.bfloat16)
        ddp = DeepReduceDDP(model, cfg)
        opt = torch.optim.SGD(model.parameters(), lr=1e-4)

        def step(model=model, ddp=ddp, opt=opt):
            ddp.zero_grad()
            out = model(input_ids=tokens, labels=labels)
            out.loss.backward()
            ddp.finish()
            opt.step()
            return out.loss
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        if ddp.engines:
            ddp.check()
        runs[name] = (model, ddp, step)
        res[name] = {"buckets": len(ddp.flat), "bucket_dtypes": sorted({str(f.dtype) for f in ddp.flat}),
                     "wire_bytes": int(ddp.wire_bytes_per_step()), "dense_bytes": int(ddp.dense_bytes()), "ms_per_step": []}
    for _ in range(rounds):             # the three arms stay resident (~15 GB together) and take turns
        for name, (model, ddp, step) in runs.items():
            res[name]["ms_per_step"].append(round(time_ms(step, steps), 3))
            if ddp.engines:
                ddp.check()
            res[name]["loss"] = float(step().detach())
    for _, ddp, _ in runs.values():
        ddp.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--bert-steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    from deepreduce_b200 import ops
    ops.require()
    out = {"card": card(), "exchange_kernel_resnet50": exchange_kernel(a.steps, a.rounds),
           "bert_large_step": bert_step(a.bert_steps, a.rounds, a.batch)}
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bf16_buckets.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
