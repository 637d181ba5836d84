"""The DDP communication hook on one GPU: the repack kernels, and a whole ResNet-50 step under three wrappers.

1. ``bucket_pack`` / ``bucket_unpack`` on the ResNet-50 layout (every parameter of ``models.resnet50``, back to back
   in reverse order as one DDP bucket, into the engine's padded layout), fp32 and bf16.  Two DDP-side bases: a 16-byte
   aligned one (most segments then take 16-byte accesses on both sides) and one shifted by one element (every DDP-side
   access is scalar), in alternating rounds, CUDA events around ``--reps`` back-to-back launches.  The bytes counted
   are the segments' elements read once and written once.
2. The W = 1 ResNet-50 training step, bf16 autocast, channels_last, batch ``--batch`` at 224^2, SGD with momentum,
   top-k 1 % + bloom index, in three arms taking turns (CUDA events around ``--steps`` whole steps per round):
   torch DDP + ``deepreduce_hook``; ``Trainer`` (``DeepReduceDDP``); torch DDP with its default all-reduce.

Prints one JSON line with the card's name, power limit and SM clock, read in the same process.

    python scripts/comm_hook_step.py --steps 20 --rounds 3 [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn.functional as F  # noqa: E402

CFG = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
       'deepreduce': 'index', 'index': 'bloom'}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
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


def repack(reps, rounds):
    from deepreduce_b200 import ops
    from deepreduce_b200.models import resnet50
    from deepreduce_b200.parallel import BucketPlan
    from deepreduce_b200.parallel.comm_hook import segment_table
    from deepreduce_b200.parallel.ddp import engine_split_numel
    from deepreduce_b200.parallel.plan import split_large
    numels = [p.numel() for p in reversed(list(resnet50().parameters()))]
    segs, off = [], 0
    for n in numels:
        segs.append((off, n))
        off += n
    n2, names, shapes, owner = split_large(numels, [f"p{i}" for i in range(len(numels))], [(n,) for n in numels],
                                           engine_split_numel(CFG, 2))
    plan = BucketPlan(n2, names, shapes, compress_ratio=0.01, index="bloom")
    table = segment_table(segs, plan, owner)
    res = {"parameters": len(numels), "elements": off, "engine_elements": plan.total_elems}
    for dt in (torch.float32, torch.bfloat16):
        raw = torch.randn(off + 1, device="cuda:0").to(dt)
        eng = torch.zeros(plan.total_elems, device="cuda:0", dtype=dt)
        rp = ops.cuda_module().Repack(table, off, plan.total_elems, eng)
        bufs = {"aligned": raw[:off], "shifted": raw[1:]}
        nbytes = 2 * off * raw.element_size()
        r = {k: {"pack_us": [], "unpack_us": []} for k in bufs}
        for b in bufs.values():
            for _ in range(10):
                rp.pack(b, eng)
                rp.unpack(eng, b)
        torch.cuda.synchronize()
        for _ in range(rounds):
            for k, b in bufs.items():
                r[k]["pack_us"].append(round(1e3 * time_ms(lambda: rp.pack(b, eng), reps), 2))
                r[k]["unpack_us"].append(round(1e3 * time_ms(lambda: rp.unpack(eng, b), reps), 2))
        for k in bufs:
            for d in ("pack", "unpack"):
                best = min(r[k][f"{d}_us"])
                r[k][f"{d}_GBps_best"] = round(nbytes / (best * 1e-6) / 1e9, 1)
        r["bytes_moved"] = nbytes
        res[str(dt).replace("torch.", "")] = r
    return res


def resnet_step(steps, rounds, batch):
    from torch.nn.parallel import DistributedDataParallel as DDP
    from deepreduce_b200.models import resnet50
    from deepreduce_b200.parallel import register_deepreduce_hook
    from deepreduce_b200.trainer import Trainer
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    x = torch.randn(batch, 3, 224, 224, device="cuda:0", generator=gen).to(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device="cuda:0", generator=gen)
    runs, res = {}, {}

    def ddp_arm(hooked):
        torch.manual_seed(0)
        model = resnet50().cuda().to(memory_format=torch.channels_last)
        ddp = DDP(model, device_ids=[0])
        st = register_deepreduce_hook(ddp, CFG) if hooked else None
        opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-4)

        def step():
            opt.zero_grad(set_to_none=False)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = ddp(x)
            loss = F.cross_entropy(out.float(), y)
            loss.backward()
            opt.step()
            return loss
        return step, st

    for name in ("ddp_hook", "trainer", "ddp_allreduce"):
        if name == "trainer":
            torch.manual_seed(0)
            tr = Trainer(resnet50().cuda(), dict(CFG), lr=0.05, amp_dtype=torch.bfloat16, channels_last=True)
            step, st = (lambda tr=tr: tr.step(x, target=y)), tr
        else:
            step, st = ddp_arm(name == "ddp_hook")
        for _ in range(5):
            step()
        torch.cuda.synchronize()
        runs[name] = (step, st)
        res[name] = {"ms_per_step": []}
        if name == "ddp_hook":
            res[name]["layouts"] = len(st.engines)
            res[name]["wire_bytes"] = int(st.wire_bytes_per_step())
    for _ in range(rounds):
        for name, (step, st) in runs.items():
            res[name]["ms_per_step"].append(round(time_ms(step, steps), 3))
            res[name]["loss"] = float(step().detach())
    for name, (step, st) in runs.items():
        if name == "ddp_hook":
            st.check()
            st.close()
        elif name == "trainer":
            st.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--skip-step", action="store_true", help="repack kernels only")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("comm_hook_step.py measures on a GPU; none found")
    torch.cuda.set_device(0)
    f = tempfile.NamedTemporaryFile(delete=False)
    f.close()
    os.unlink(f.name)
    dist.init_process_group("nccl", init_method=f"file://{f.name}", rank=0, world_size=1)
    out = {"card_before": card(), "repack": repack(a.reps, a.rounds)}
    if not a.skip_step:
        out["resnet50_step"] = resnet_step(a.steps, a.rounds, a.batch)
        out["resnet50_step"]["batch"] = a.batch
    out["card_after"] = card()
    dist.destroy_process_group()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "comm_hook_step.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
