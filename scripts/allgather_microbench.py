"""Compressed-allgather microbenchmark (SURVEY §7.2 step 5): the in-kernel slot exchange of the fused engine
(push + flags, phases 12-13 alone) vs `dist.all_gather_into_tensor` of the same slots over NCCL, on W GPUs.

    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 scripts/allgather_microbench.py [iters]

Prints one JSON line on rank 0: per-variant device time (CUDA events, max over ranks) and bus bandwidth
(bytes a rank sends to its W-1 peers / time) against the H100's 450 GB/s per direction NVLink 4 data-sheet figure.
Variants: P2P stores (default arena), NVLS multicast (arena in symmetric memory), NCCL all_gather.
Not run on the H100."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, iters, world):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from deepreduce_b200.models import resnet50
    from deepreduce_b200.parallel import BucketEngine, BucketPlan
    from deepreduce_b200.parallel.engine import PH_ACCUM, PH_EXPAND, PH_PUSH
    named = list(reversed([(n, p) for n, p in resnet50().named_parameters()]))
    plan = BucketPlan([p.numel() for _, p in named], [n for n, _ in named], compress_ratio=0.01)
    out = {"world": world, "slot_bytes": plan.wire_bytes(), "iters": iters, "variants": {}}
    sent = (world - 1) * plan.wire_bytes()
    for name, env in (("p2p_stores", "0"), ("nvls_multicast", "1")):
        os.environ["DR_NVLS"] = env
        eng = BucketEngine(plan, device=f"cuda:{local}", shard=False)
        if name == "nvls_multicast" and not getattr(eng, "multicast_ptr", 0):
            out["variants"][name] = {"unavailable": getattr(eng, "_nvls_error", "no multicast pointer")}
            eng.close()
            continue
        eng.grad.normal_(generator=torch.Generator(device="cuda").manual_seed(rank))
        eng.epoch += 1
        eng.ctx.run(eng.epoch, PH_ACCUM, PH_PUSH)            # build a real slot once

        def push():                                          # push + flags of a fresh epoch (slot content is reused)
            eng.epoch += 2                                   # same parity -> same slot
            eng.ctx.run(eng.epoch, PH_PUSH, PH_EXPAND)
        ms = timed(push, iters, world)
        eng.check_status()
        out["variants"][name] = {"ms": ms, "bus_gbs": sent / (ms * 1e-3) / 1e9 if world > 1 else 0.0}
        eng.close()
    slot = torch.empty(plan.wire_bytes() // 4, dtype=torch.int32, device="cuda").random_()
    gathered = torch.empty(world * slot.numel(), dtype=torch.int32, device="cuda")
    ms = timed(lambda: dist.all_gather_into_tensor(gathered, slot), iters, world)
    out["variants"]["nccl_all_gather"] = {"ms": ms, "bus_gbs": sent / (ms * 1e-3) / 1e9 if world > 1 else 0.0}
    out["nvlink_gbs_per_dir"] = {"nominal": 450.0}
    if rank == 0:
        print(json.dumps(out), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
