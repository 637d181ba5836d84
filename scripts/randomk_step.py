"""ResNet-50 training step with GRACE's 'randomk' sparsifier: the fused shared-index mode against the per-tensor path.

One GPU, batch 256, bf16 autocast, the ``Trainer`` arguments of ``bench.py --gpus 1`` and ``bench.reproducible_cudnn()``.
Four arms live in one process and are timed in alternating rounds:

* ``randomk``       — fused engine, shared-seed index: fp32 values only on the wire;
* ``randomk_qsgd``  — the same with QSGD int8 values (``'deepreduce': 'value', 'value': 'qsgd'``);
* ``randomk_grace`` — what this params dict ran before the fused mode existed: ``deepreduce_from_params(params).step``
  per parameter after backward (``DeepReduceDDP.finish`` with ``grc``), no buckets, no hooks, no overlap; its
  gradients come back contiguous, which torch's fused SGD does not take next to channels_last weights, so this arm
  steps with torch's foreach SGD (same hyperparameters);
* ``bloom``         — the benchmark's default fused top-k + bloom config, as context.

Per arm it prints images/s and ms/step (CUDA events around K steps, per round), the exchange's own ms/step (the fused
kernels, or the per-parameter ``grc.step`` calls, alone on the last gradients), wire bytes per step, and for the fused
randomk arms how many steps needed the select's fallback phase (``barrier[8]``; the draw does not depend on the data, so
a probe engine with the same plan replays the epochs of the run).  One JSON line per run, with the card's name and power
limit read in the same process.

    python scripts/randomk_step.py --steps 20 --warmup 5 --rounds 3 [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from unittest import mock

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

RANDOMK = {'compressor': 'randomk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
ARMS = {
    "randomk": dict(RANDOMK),
    "randomk_qsgd": {**RANDOMK, 'deepreduce': 'value', 'value': 'qsgd'},
    "randomk_grace": dict(RANDOMK),
    "bloom": dict(bench.CONFIGS["bloom"]),
}


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        f = [x.strip() for x in r.stdout.strip().split(",")]
        out["power_limit_w"], out["sm_max_mhz"] = float(f[0]), float(f[1])
    except Exception as e:  # noqa: BLE001
        out["power_limit_error"] = repr(e)
    return out


def build(arm, B):
    import torch
    from deepreduce_b200 import models
    from deepreduce_b200.trainer import Trainer
    torch.manual_seed(1234)
    model = models.resnet50().cuda()
    kw = dict(lr=0.05, amp_dtype=torch.bfloat16, channels_last=True, overlap=True, bucket_cap_mb=128.0,
              background_thread=True, blocks_per_sm=2, u8_input=True, loss_fn=None, overlap_grid=0)
    if arm == "randomk_grace":
        # grc.step hands back contiguous gradients, which torch's fused SGD rejects next to channels_last weights
        # (check_fast_path_restrictions): this arm steps with torch's default (foreach) SGD, same hyperparameters
        kw["optimizer"] = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)
        with mock.patch("deepreduce_b200.parallel.ddp.fused_path", lambda params: False):
            tr = Trainer(model, dict(ARMS[arm]), **kw)
        assert tr.ddp.grc is not None and not tr.ddp.fused
    else:
        tr = Trainer(model, dict(ARMS[arm]), **kw)
        assert tr.ddp.fused
    return tr


def events_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def exchange_ms(tr, n):
    """The exchange alone, on the gradients the last step left in place."""
    if tr.ddp.fused:
        def ex(i):
            for e in tr.ddp.engines:
                e.ctx.set_grid_cap(0)
                e.step()
    else:
        grads = [(name, p.grad.clone()) for name, p in tr.ddp.named if p.grad is not None]

        def ex(i):
            for name, g in grads:
                tr.ddp.grc.step(g, name)
    for i in range(2):
        ex(i)
    return events_ms(ex, n) / n


def fallback_steps(tr, epochs):
    """Steps (of ``epochs``) in which some tensor's static bound hid its threshold, and the tensors that did so in all:
    the select phases of a probe engine with the same plan, replayed epoch by epoch, read ``barrier[8]``."""
    from deepreduce_b200.parallel import BucketEngine
    from deepreduce_b200.parallel.engine import PH_ACCUM, PH_INSERT
    steps, tensors = 0, 0
    for e in tr.ddp.engines:
        probe = BucketEngine(e.plan, device=e.device, world=1, rank=0, beta=0.0)
        hit = []
        for ep in epochs:
            probe.hist.zero_(); probe.hist_total.zero_(); probe.barrier.zero_()
            probe.run_phases(PH_ACCUM, PH_INSERT, ep)
            hit.append(int(probe.barrier[8].item()))
        probe.check_status()
        probe.close()
        steps = max(steps, sum(1 for h in hit if h))
        tensors += sum(hit)
    return steps, tensors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--arms", default=",".join(ARMS))
    ap.add_argument("--out", default=None, help="directory for the JSON line (default: print only)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("randomk_step.py measures on a GPU; no CUDA device is visible")
    bench.reproducible_cudnn()
    B, K = args.batch, args.steps
    arms = args.arms.split(",")
    gen = torch.Generator().manual_seed(77)
    pool, tgt = bench.synth_batches("image224", B, 0, gen)
    xs = [tuple(t.cuda() for t in p) for p in pool]
    ys = [t.cuda() for t in tgt]
    trs = {a: build(a, B) for a in arms}
    for a, tr in trs.items():
        for i in range(args.warmup):
            tr.step(*xs[i & 1], target=ys[i & 1])
        tr.ddp.check()
    first_epoch = {a: [e.epoch + 1 for e in tr.ddp.engines] for a, tr in trs.items()}
    res = {a: {"ms_per_step": []} for a in arms}
    for rnd in range(args.rounds):
        order = arms if rnd % 2 == 0 else list(reversed(arms))
        for a in order:
            tr = trs[a]
            ms = events_ms(lambda i: tr.step(*xs[i & 1], target=ys[i & 1]), K)
            tr.ddp.check()
            res[a]["ms_per_step"].append(ms / K)
    for a, tr in trs.items():
        r = res[a]
        r["images_per_s"] = [B / (m / 1e3) for m in r["ms_per_step"]]
        r["wire_bytes_per_step"] = int(tr.ddp.wire_bytes_per_step())
        r["dense_bytes"] = int(tr.ddp.dense_bytes())
        if a.startswith("randomk") and tr.ddp.fused:
            last = [e.epoch for e in tr.ddp.engines]
            epochs = list(range(first_epoch[a][0], last[0] + 1))
            n_steps, n_tensors = fallback_steps(tr, epochs)
            r["fallback"] = {"steps_timed": len(epochs), "steps_with_phase1": n_steps, "tensor_hits": n_tensors}
        r["exchange_ms_per_step"] = exchange_ms(tr, K)
    out = {"what": "ResNet-50 training step, randomk arms, alternating rounds", "batch": B, "steps_per_round": K,
           "rounds": args.rounds, "dtype": "bf16 autocast", "card": card(), "arms": res}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "randomk_step.jsonl"), "a") as f:
            f.write(line + "\n")
    for tr in trs.values():
        tr.close()


if __name__ == "__main__":
    main()
