"""torchrun script: torch DDP + ``deepreduce_hook`` at W > 1, one GPU per rank (``test_gpu_comm_hook``).

An MLP under DDP with small buckets (several layouts, and DDP's rebuild after the first iteration), top-k 1 % + bloom
index, a batch per rank, three steps.  Every step, on every rank:

1. the gradients DDP leaves in ``p.grad`` are bit-identical on all ranks;
2. they equal the oracle of the all-gathered local gradients: each bucket as DDP handed it to the hook (cloned
   before the exchange), through ``engine_oracle`` with W senders and the all-gathered residuals.  The decode adds
   the W senders in whatever order its work items finish, so the comparison allows a few fp32 ulps of the oracle's
   rank-ordered sum;
3. after the last step, ``multi_gpu_check`` passes on every engine the hook holds.
"""
import os
import sys
import traceback

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.nn.parallel import DistributedDataParallel as DDP

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

CFG = {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
       'deepreduce': 'index', 'index': 'bloom'}


def _gather(t, world):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    return [p.cpu() for p in parts]


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    from test_train_step_reference import ref_flat, unflatten
    from deepreduce_b200.parallel import DeepReduceHookState, engine_oracle
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    from deepreduce_b200.utils.selfcheck import multi_gpu_check
    torch.manual_seed(0)
    model = nn.Sequential(nn.Linear(64, 512), nn.ReLU(), nn.Linear(512, 512), nn.ReLU(), nn.Linear(512, 10)).cuda()
    ddp = DDP(model, device_ids=[local], bucket_cap_mb=0.5)
    st = DeepReduceHookState(CFG, model, overlap_grid=32)
    named = dict(model.named_parameters())
    by_id = {id(p): n for n, p in named.items()}
    captured = []

    def spy(state, bucket):
        captured.append((bucket.index(), bucket.buffer().clone(), bucket_segments(bucket),
                         [by_id[id(p)] for p in bucket.parameters()]))
        return deepreduce_hook(state, bucket)
    ddp.register_comm_hook(st, spy)
    failures = []
    resid = [{n: torch.zeros(p.numel()) for n, p in named.items()} for _ in range(world)]
    try:
        for step in range(3):
            captured.clear()
            g = torch.Generator(device="cuda").manual_seed(100 * step + rank)
            ddp(torch.randn(32, 64, device="cuda", generator=g)).pow(2).mean().backward()
            torch.cuda.synchronize()
            st.check()
            for n, p in named.items():
                parts = _gather(p.grad.view(-1).view(torch.int32), world)
                if not all(torch.equal(parts[0], q) for q in parts):
                    failures.append(f"step {step}: ranks hold different gradients for {n}")
            for idx, pre, segs, names in captured:
                lay = st._by_index[idx]
                pres = _gather(pre, world)
                params = {n: named[n] for n in names}
                flats, res_in = [], []
                for r in range(world):
                    grads = {n: pres[r][d:d + k].view(named[n].shape) for n, (d, k) in zip(names, segs)}
                    flats.append(ref_flat(lay.plan, params, grads))
                    rg = {n: resid[r][n].view(named[n].shape) for n in names}
                    res_in.append(ref_flat(lay.plan, params, rg))
                out, _, _ = engine_oracle(lay.plan, flats, res_in, epoch=lay.engine.epoch)
                want = unflatten(lay.plan, params, out)
                for n in names:
                    got, w = named[n].grad.cpu(), want[n].cpu()
                    scale = float(w.abs().max()) or 1.0
                    if not torch.allclose(got, w, rtol=1e-5, atol=1e-6 * scale):
                        failures.append(f"step {step}: {n} differs from the oracle by {float((got - w).abs().max())}")
                # the next step starts from the engines' residuals (the decode order only touches the aggregate)
                res_parts = _gather(lay.engine.resid, world)
                for r in range(world):
                    for t_name, t in zip(names, lay.params):
                        i = lay.slot[id(t)]
                        resid[r][t_name] = res_parts[r][lay.eng_off[i]:lay.eng_off[i] + lay.segments[i][1]].clone()
        for e in st.engines:
            res = multi_gpu_check(e)
            if res["status"] != "ok":
                failures.append(f"multi_gpu_check: {res['status']}")
        if len(st.engines) < 2:
            failures.append("expected several bucket layouts")
    except Exception:  # noqa: BLE001
        failures.append(traceback.format_exc())
    finally:
        st.close()
    flags = [None] * world
    dist.all_gather_object(flags, failures)
    dist.destroy_process_group()
    bad = [f for fl in flags for f in fl]
    if rank == 0:
        for f in bad:
            print(f, flush=True)
        if not bad:
            print("COMM_HOOK_MULTIGPU_OK", flush=True)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
