"""Does a per-phase, per-CTA calibrated tile partition pay?  ResNet-50 gradient shapes, W = 1 (or torchrun for W > 1).
Prints the fused exchange time (median / min of N, L2 flushed) for: one cost prefix for all phases (DR_CUTS=0 behaviour),
per-phase-class weights, and 1..R calibration rounds (BucketEngine.calibrate_partition); plus the per-SM picture."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepreduce_b200.models import resnet50  # noqa: E402
from deepreduce_b200.parallel import BucketEngine, BucketPlan  # noqa: E402


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    world = int(os.environ.get("WORLD_SIZE", 1)); rank = int(os.environ.get("RANK", 0)); local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    named = list(reversed([(n, p) for n, p in resnet50().named_parameters()]))
    plan = BucketPlan([p.numel() for _, p in named], [n for n, _ in named], compress_ratio=0.01)
    eng = BucketEngine(plan, device=f"cuda:{local}") if world > 1 else BucketEngine(plan, device="cuda:0", world=1, rank=0)
    gen = torch.Generator(device="cuda").manual_seed(rank)
    grads = [torch.randn(plan.total_elems, device="cuda", generator=gen) * 0.01 for _ in range(4)]
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")

    def measure(tag):
        ts = []
        for i in range(steps + 5):
            eng.grad.copy_(grads[i % 4]); flush.zero_()
            if world > 1:
                dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); eng.step(); e1.record()
            torch.cuda.synchronize()
            if i >= 5:
                ts.append(e0.elapsed_time(e1))
        eng.check_status()
        t = torch.tensor([float(np.median(ts)), float(min(ts))], device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print(f"{tag:42s} fused median {t[0].item():.4f} ms  min {t[1].item():.4f} ms", flush=True)
        return t[0].item()

    out = {}
    eng.ctx.set_cuts(0, 0)
    out["single_prefix"] = measure("one cost prefix (6.0 / 2.0) for all phases")
    eng.cta_speeds = None; eng._set_cuts()
    out["phase_weights"] = measure("per-phase-class weights, uniform CTA speeds")
    for r in range(3):
        log = eng.calibrate_partition(steps=3, rounds=1, verbose=True)
        out[f"calibrated_{r + 1}"] = measure(f"calibrated, round {r + 1}")
    if rank == 0:
        sp = np.asarray(eng.cta_speeds)
        print("speeds accum  (every 8th CTA):", np.round(sp[0, ::8], 2).tolist())
        print("speeds query  (every 8th CTA):", np.round(sp[2, ::8], 2).tolist())
        G = eng.grid()
        dbg = torch.zeros(21 * G * 2, dtype=torch.int64, device="cuda")
        eng.ctx.set_debug_times(dbg.data_ptr())
        eng.grad.copy_(grads[0]); eng.step(); torch.cuda.synchronize()
        smid = dbg.cpu().numpy().reshape(21, G, 2)[20, :, 0]
        eng.ctx.set_debug_times(0)
        print("smid of CTA 0..15:", smid[:16].tolist(), " CTA 132..139:", smid[132:140].tolist())
        slow = sp[0] < np.median(sp[0]) * 0.97
        print("slow-in-accumulate CTAs:", int(slow.sum()), " distinct SMs among them:", len(set(smid[slow].tolist())),
              " SM id range:", int(smid[slow].min()) if slow.any() else None, int(smid[slow].max()) if slow.any() else None)
        os.makedirs(os.path.join(ROOT, "script_out"), exist_ok=True)
        json.dump({"world": world, "fused_ms_median": out, "speeds": sp.round(3).tolist(), "smid": smid.tolist()},
                  open(os.path.join(ROOT, "script_out", f"partition_experiment_n{world}.json"), "w"))
    elif world > 1:
        pass
    eng.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
