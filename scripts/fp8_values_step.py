"""ResNet-50 training step with fp8 values on the wire ('value': 'fp8') against fp32, QSGD int8 and sign values, per
index, and the coding error of each value codec on the step's own gradients.

One GPU, batch 256, bf16 autocast, the ``Trainer`` arguments of ``bench.py --gpus 1`` and ``bench.reproducible_cudnn()``.
The arms live in one process and are timed in alternating rounds, all at the same top-k ratio (1 % by default), over
four indices: ``ef`` (Elias-Fano), ``rle`` (run-length), ``bloom`` (leftmost policy, occupancy hint) and ``randomk``
(shared-seed random-k, values only).  Each index has four arms: ``<index>`` with fp32 values, ``<index>_qsgd`` with
QSGD int8 values (bucket 512; over rle with 'fused_rle_values'), ``<index>_sign`` with sign values and ``<index>_fp8``
with fp8 values.  All three code their values in the kernel's fix phase, one CTA per 512 values.

Per arm it prints images/s and ms/step (CUDA events around K steps, per round), the exchange's own ms/step (the fused
kernels alone on the last gradients) and the wire bytes per step.  For the coded arms it also prints the relative L2
error and the worst relative error of the decoded values against the fp32 values the sender shipped, read from the
last step's slots (the fp32 values stay in the slot's sender-local scratch).  One JSON line per run, with the card's
name and power limit read in the same process.  At W = 1 nothing crosses a wire, so the byte savings do not show as
time here.

    python scripts/fp8_values_step.py --steps 20 --warmup 5 --rounds 3 [--ratio 0.01] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench  # noqa: E402
from bf16_values_step import build  # noqa: E402
from randomk_step import card, events_ms, exchange_ms  # noqa: E402

TOPK = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather'}
RANDK = {'compressor': 'randomk', 'memory': 'residual', 'communicator': 'allgather'}
QSGD = {'value': 'qsgd', 'quantum_num': 127, 'bucket_size': 512}
ARMS = ",".join(f"{ix}{v}" for ix in ("ef", "rle", "bloom", "randomk") for v in ("", "_qsgd", "_sign", "_fp8"))


def arms(ratio):
    out = {}
    for name, ix in (("ef", {'index': 'elias_fano'}), ("rle", {'index': 'rle'}),
                     ("bloom", {'index': 'bloom', 'policy': 'leftmost'})):
        base = {**TOPK, 'compress_ratio': ratio, **ix}
        out[name] = {**base, 'deepreduce': 'index'}
        out[f"{name}_qsgd"] = {**base, 'deepreduce': 'both', **QSGD, **({'fused_rle_values': True} if name == "rle" else {})}
        out[f"{name}_sign"] = {**base, 'deepreduce': 'both', 'value': 'sign'}
        out[f"{name}_fp8"] = {**base, 'deepreduce': 'both', 'value': 'fp8'}
    out["randomk"] = {**RANDK, 'compress_ratio': ratio}
    out["randomk_qsgd"] = {**RANDK, 'compress_ratio': ratio, 'deepreduce': 'value', **QSGD}
    out["randomk_sign"] = {**RANDK, 'compress_ratio': ratio, 'deepreduce': 'value', 'value': 'sign'}
    out["randomk_fp8"] = {**RANDK, 'compress_ratio': ratio, 'deepreduce': 'value', 'value': 'fp8'}
    return out


def value_error(tr):
    """(relative L2 error, worst relative error, values) of the decoded values against the shipped fp32 values, over
    every coded tensor of the trainer's engines, from the last step's slots."""
    import numpy as np
    import torch
    from deepreduce_b200.parallel.engine import decode_slot_oracle, shipped_index_oracle
    num = den = worst = 0.0
    count = 0
    for eng in tr.ddp.engines:
        plan = eng.plan
        off = plan.slot_offset(eng.world, eng.epoch & 1, eng.rank)
        slot = eng.arena[off:off + plan.slot_words].cpu().numpy().view(np.uint32)
        dec = decode_slot_oracle(plan, slot[:plan.payload_words])
        for ti, t in enumerate(plan.tensors):
            if not t.coded:
                continue
            idx = shipped_index_oracle(plan, slot[:plan.payload_words], ti)
            n = int(idx.numel())
            if n == 0:
                continue
            v = torch.from_numpy(slot[t.off_vals:t.off_vals + n].view(np.float32).astype(np.float64))
            d = dec[t.elem_off + idx].double()
            num += float(((d - v) ** 2).sum())
            den += float((v ** 2).sum())
            nz = v != 0
            if bool(nz.any()):
                worst = max(worst, float(((d - v).abs()[nz] / v.abs()[nz]).max()))
            count += n
    return (num / den) ** 0.5 if den else 0.0, worst, count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--ratio", type=float, default=0.01, help="top-k ratio of every arm")
    ap.add_argument("--arms", default=ARMS)
    ap.add_argument("--out", default=None, help="directory for the JSON line (default: print only)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fp8_values_step.py measures on a GPU; no CUDA device is visible")
    bench.reproducible_cudnn()
    B, K = args.batch, args.steps
    table = arms(args.ratio)
    names = args.arms.split(",")
    gen = torch.Generator().manual_seed(77)
    pool, tgt = bench.synth_batches("image224", B, 0, gen)
    xs = [tuple(t.cuda() for t in p) for p in pool]
    ys = [t.cuda() for t in tgt]
    trs = {a: build(table[a]) for a in names}
    for a, tr in trs.items():
        for i in range(args.warmup):
            tr.step(*xs[i & 1], target=ys[i & 1])
        tr.ddp.check()
    res = {a: {"ms_per_step": []} for a in names}
    for rnd in range(args.rounds):
        order = names if rnd % 2 == 0 else list(reversed(names))
        for a in order:
            tr = trs[a]
            ms = events_ms(lambda i: tr.step(*xs[i & 1], target=ys[i & 1]), K)
            tr.ddp.check()
            res[a]["ms_per_step"].append(ms / K)
    for a, tr in trs.items():
        r = res[a]
        r["params"] = table[a]
        r["images_per_s"] = [B / (m / 1e3) for m in r["ms_per_step"]]
        r["wire_bytes_per_step"] = int(tr.ddp.wire_bytes_per_step())
        r["dense_bytes"] = int(tr.ddp.dense_bytes())
        if table[a].get("deepreduce") in ("value", "both"):
            torch.cuda.synchronize()
            r["value_rel_l2_error"], r["value_worst_rel_error"], r["values_checked"] = value_error(tr)
        r["exchange_ms_per_step"] = exchange_ms(tr, K)
    out = {"what": "ResNet-50 training step, fp32 / QSGD int8 / sign / fp8 wire values per index, alternating rounds",
           "batch": B, "steps_per_round": K, "rounds": args.rounds, "ratio": args.ratio, "dtype": "bf16 autocast",
           "card": card(), "arms": res}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_values_step.jsonl"), "a") as f:
            f.write(line + "\n")
    for tr in trs.values():
        tr.close()


if __name__ == "__main__":
    main()
