"""Exchange-kernel microbenchmark on ResNet-50 gradient shapes at W GPUs (torchrun): device time of the fused kernel
per step (CUDA events, max over ranks), wire / stage-2 bytes, roofline fractions, compressed-allgather bus GB/s."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepreduce_b200.models import resnet50  # noqa: E402
from deepreduce_b200.parallel import BucketEngine, BucketPlan  # noqa: E402


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    index = sys.argv[2] if len(sys.argv) > 2 else "bloom"
    value = sys.argv[3] if len(sys.argv) > 3 else "none"
    index = None if index == "none" else index
    value = None if value == "none" else value
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    m = resnet50()
    named = list(reversed([(n, p) for n, p in m.named_parameters()]))
    plan = BucketPlan([p.numel() for _, p in named], [n for n, _ in named], compress_ratio=0.01, index=index, value=value)
    eng = BucketEngine(plan, device=f"cuda:{local}")
    if os.environ.get("DR_CALIBRATE", "1") != "0" and eng.cuts is not None:
        eng.calibrate_partition()
    gen = torch.Generator(device="cuda").manual_seed(rank)
    grads = [torch.randn(plan.total_elems, device="cuda", generator=gen) * 0.01 for _ in range(4)]
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")

    def one(i):
        eng.grad.copy_(grads[i % 4])
        flush.zero_()
        dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); eng.step(); e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for i in range(5):
        one(i)
    eng.check_status()
    ts = torch.tensor([one(i) for i in range(steps)], device="cuda", dtype=torch.float64)
    dist.all_reduce(ts, op=dist.ReduceOp.MAX)
    eng.check_status()
    med = float(ts.sort().values[steps // 2]); mn = float(ts.min())
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 3350.0)              # default: H100 SXM HBM3, data sheet
    d, wire, s2 = plan.dense_bytes(), plan.wire_bytes(), eng.stage2_bytes()
    nv = (world - 1) * wire + s2
    t_hbm = 4 * d / (hbm * 1e9) * 1e3
    t_nv = nv / 450e9 * 1e3                                  # H100 NVLink 4, data sheet, per direction
    if rank == 0:
        print(json.dumps({"kernel": "dr_engine_kernel (fused)", "world": world, "index": index, "value": value,
                          "fused_ms_median_max_over_ranks": med, "fused_ms_min": mn, "dense_bytes": d, "wire_bytes": wire,
                          "stage2_bytes": s2, "nvlink_bytes_out": nv, "hbm_bound_ms": t_hbm, "nvlink_bound_ms": t_nv,
                          "frac_of_roofline": max(t_hbm, t_nv) / med, "compressed_allgather_bus_gbs": nv / (med * 1e-3) / 1e9,
                          "grid": eng.grid(), "shard": eng.shard, "transport": eng.transport}), flush=True)
    eng.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
