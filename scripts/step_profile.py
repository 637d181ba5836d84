#!/usr/bin/env python
"""Per-kernel-class profile of the headline ResNet-50 step (bench.py's default configuration: batch 256, bf16 autocast,
channels_last, top-k 1 % + bloom index, one 128 MB bucket, deterministic cuDNN by heuristics).

    python scripts/step_profile.py [--steps 3] [--warmup 3] [--out script_out/step_profile]

torch.profiler with CUDA activities, in a run of its own (tracing slows the host; take timings from bench.py).  Prints
and writes ``<out>/profile_fused<0|1>.json`` and a markdown table: per kernel class the GPU time per step, and for the
BatchNorm / ReLU / add classes the bytes per step computed from the activation shapes and the resulting GB/s.  The card
name and power limit are read in the same run.  ``DR_FUSED_BN`` selects the path as it does for the model.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (class, substrings of the kernel name); the first match wins
CLASSES = [
    ("exchange", ("dr_engine_kernel",)),
    ("stem bn + max pool (own)", ("bn_apply_pool_kernel",)),
    ("stem pool grad (own)", ("bn_pool_grad_kernel",)),
    ("bn fused apply (own)", ("bn_apply_kernel",)),
    ("bn stats (own)", ("bn_stats_kernel", "bn_stats_finalize_kernel")),
    ("bn bwd reduce (own)", ("bn_bwd_reduce_kernel", "bn_bwd_finalize_kernel")),
    ("bn bwd elemt (own)", ("bn_bwd_elemt_kernel",)),
    ("bn stats", ("batch_norm_collect_statistics",)),
    ("bn apply", ("batch_norm_transform_input",)),
    ("bn bwd reduce", ("batch_norm_backward_reduce",)),
    ("bn bwd elemt", ("batch_norm_backward_elemt",)),
    ("relu", ("clamp_scalar", "clamp_min")),
    ("max pool", ("max_pool",)),
    ("threshold_backward", ("threshold",)),
    ("add", ("AddFunctor", "CUDAFunctor_add", "add_kernel")),
    ("optimizer", ("sgd", "Sgd", "multi_tensor")),
    ("conv wgrad", ("wgrad",)),
    ("conv dgrad", ("dgrad",)),
    ("conv fprop", ("fprop", "implicit_gemm", "conv", "xmma", "cutlass", "cudnn")),
]


def classify(name: str) -> str:
    for cls, keys in CLASSES:
        if any(k in name for k in keys):
            return cls
    return "other"


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def shape_bytes(model, run_step):
    """Bytes of the bf16 BN inputs of one forward, by role: S = the stem (BN + ReLU + max pool), W = bn1/bn2 (BN + ReLU),
    T = bn3 (BN + add + ReLU), D = downsample BN, I = block inputs (where backward sums the skip and conv1 gradients),
    split by the producer of the block input: IS the stem, IT a tail with an identity skip, ID a tail with a downsample
    BN (I = IS + IT + ID)."""
    import torch.nn as nn
    from deepreduce_b200.models.resnet import _Bottleneck
    acc = collections.Counter()
    hooks = []
    add = lambda key, t: acc.__setitem__(key, acc[key] + t.numel() * t.element_size())      # noqa: E731
    for name, m in model.named_modules():
        if isinstance(m, nn.Conv2d):
            role = ("S" if name == "conv1" else "D" if name.endswith("downsample.0")
                    else "T" if name.endswith("conv3") else "W")
            hooks.append(m.register_forward_hook(lambda mod, i, o, r=role: add(r, o)))

    def block_input(mod, i, o, src):
        add("I", i[0])
        add(src, i[0])

    prev = None
    for m in model.modules():
        if isinstance(m, _Bottleneck):
            src = "IS" if prev is None else "IT" if prev.downsample is None else "ID"
            hooks.append(m.register_forward_hook(lambda mod, i, o, r=src: block_input(mod, i, o, r)))
            prev = m
    run_step()
    for h in hooks:
        h.remove()
    return dict(acc)


def pass_bytes(b, fused):
    """Minimum bytes each memory-bound class moves per step (reads + writes over the tensors it touches)."""
    S, W, T, D, I = b["S"], b["W"], b["T"], b["D"], b["I"]
    P = S / 4                  # the pooled stem output (kernel 3, stride 2: a quarter of the positions)
    out = {}
    if fused:
        # forward: bn_relu reads x, writes y; tails read x3 and idt (or xd), write o; each writes a 1/16-size ReLU mask.
        # The stem reads x and writes the pooled output and a code byte per pooled element (P / 2).
        # backward, per BN + ReLU kind (Ti = identity tails, D = downsample tails, T = Ti + D):
        #   stem pool grad: reads the pooled gradient and the codes, writes the masked g at x's size
        #   reduce: W and Ti read go, x, mask (Ti also writes g); D reads go, x, z, mask; the stem reads g, x
        #   elemt:  W reads go, x, mask, writes dx; Ti and the stem read g, x, write dx; D reads go, x, z, mask, writes
        #           dx, dz
        # A block input made by an identity tail is not summed by an add: the tail's reduce reads its two gradients.
        # The inputs made by the stem and by downsample tails are still summed by autograd's add (read, read, write).
        Ti, M = T - D, (W + T) / 16
        IS, IT, ID = b.get("IS", 0), b.get("IT", 0), b.get("ID", 0)
        out.update({"bn stats (own)": S + W + T + D, "stem bn + max pool (own)": S + 1.5 * P,
                    "stem pool grad (own)": 1.5 * P + S,
                    "bn fused apply (own)": 2 * W + 3 * T + M, "add": 3 * (IS + ID),
                    "bn bwd reduce (own)": 2 * S + 2 * W + 3 * Ti + 3 * D + M + IT,
                    "bn bwd elemt (own)": 3 * S + 3 * W + 3 * Ti + 5 * D + (W + D) / 16})
    else:          # apply: read x, write y; relu_ in place; forward add: 2 reads + 1 write; backward junction adds
        W += S
        # max pool: forward reads y, writes the output and int64 indices (4 P); backward zeroes dy, reads the gradient
        # and the indices, writes dy
        out.update({"bn stats": W + T + D, "bn apply": 2 * (W + T + D), "relu": 2 * (W + T), "add": 3 * T + 3 * I,
                    "bn bwd reduce": 2 * (W + T + D), "bn bwd elemt": 3 * (W + T + D), "threshold_backward": 3 * (W + T),
                    "max pool": 3 * S + 10 * P})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default=os.path.join(ROOT, "script_out", "step_profile"))
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from deepreduce_b200.models import fused_bn, resnet50
    from deepreduce_b200.trainer import Trainer
    assert torch.cuda.is_available(), "needs a GPU"
    torch.manual_seed(1234)
    bench.reproducible_cudnn()
    B = args.batch
    tr = Trainer(resnet50().cuda(), dict(bench.CONFIGS["bloom"]), lr=0.05, amp_dtype=torch.bfloat16, channels_last=True,
                 bucket_cap_mb=128.0, u8_input=True)
    gen = torch.Generator().manual_seed(77)
    x = torch.randint(0, 256, (B, 224, 224, 3), dtype=torch.uint8, generator=gen).cuda()
    y = torch.randint(0, 1000, (B,), generator=gen).cuda()
    step = lambda: tr.step(x, target=y)      # noqa: E731
    for _ in range(args.warmup):
        step()
    sizes = shape_bytes(tr.model, step)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    tr.close()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    per_cls, names = collections.Counter(), collections.defaultdict(collections.Counter)
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") == "kernel" and "dur" in ev:
            cls = classify(ev["name"])
            per_cls[cls] += ev["dur"] / args.steps
            names[cls][ev["name"][:140]] += ev["dur"] / args.steps
    fused = fused_bn.enabled()
    pb = pass_bytes(sizes, fused)
    total = sum(per_cls.values())
    rows = []
    for cls, us in sorted(per_cls.items(), key=lambda kv: -kv[1]):
        b = pb.get(cls)
        rows.append({"class": cls, "ms_per_step": us / 1e3, "share": us / total, "bytes_per_step": b,
                     "gbs": (b / (us * 1e-6) / 1e9) if b else None,
                     "top_kernels": [[n, t / 1e3] for n, t in names[cls].most_common(3)]})
    res = {"card": card(), "fused_bn": fused, "batch": B, "steps": args.steps, "kernel_ms_per_step": total / 1e3,
           "bn_input_bytes": sizes, "classes": rows}
    os.makedirs(args.out, exist_ok=True)
    tag = f"fused{int(fused)}"
    with open(os.path.join(args.out, f"profile_{tag}.json"), "w") as f:
        json.dump(res, f, indent=1)
    lines = [f"card: {res['card']}; DR_FUSED_BN={int(fused)}; batch {B}; GPU kernel time {total / 1e3:.2f} ms/step", "",
             "| class | ms/step | share | GB/step (from shapes) | GB/s |", "|---|---|---|---|---|"]
    for r in rows:
        gb = f"{r['bytes_per_step'] / 1e9:.2f}" if r["bytes_per_step"] else ""
        gbs = f"{r['gbs']:.0f}" if r["gbs"] else ""
        lines.append(f"| {r['class']} | {r['ms_per_step']:.2f} | {100 * r['share']:.1f} % | {gb} | {gbs} |")
    with open(os.path.join(args.out, f"profile_{tag}.md"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))
    for r in rows:
        print(r["class"], r["top_kernels"])


if __name__ == "__main__":
    main()
