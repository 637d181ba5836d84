"""torchrun script: the benchmark's training step at W > 1 against the plain reference step of
``tests/test_train_step_reference.py``.

The benchmark's N > 1 layout: ResNet-50 at 224^2, ``bloom``, one bucket launched after backward, a batch per rank seeded
``77 + rank``.  Every rank builds its reference bucket from plain-torch gradients, all-gathers the W reference buckets
and residuals, runs ``engine_oracle`` with W senders and checks its own exchanged bucket, residual, parameters and
momentum.  The parameters must also be identical on every rank.  The decode adds the W senders' values in whatever
order its work items finish, so the bucket is compared within a few fp32 ulps of the oracle's rank-ordered sum; the
optimizer then reads the rank's own bucket, and everything after that is compared bit for bit.
"""
import os
import sys
import traceback

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


class _Env:
    """The one method of pytest's ``monkeypatch`` the reference step uses."""

    @staticmethod
    def setenv(name, value):
        os.environ[name] = value


def _gather_cpu(t, world):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    return [p.cpu() for p in parts]


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    torch.set_num_threads(max(1, (os.cpu_count() or 1) // world))       # W CPU oracles run side by side
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    import test_train_step_reference as T
    from deepreduce_b200.parallel import engine_oracle
    env = _Env()
    failures = []

    def check(what, fn):
        try:
            fn()
        except AssertionError as e:
            failures.append(f"[rank {rank}] {what}: {e}")
            print(failures[-1], flush=True)

    gen = torch.Generator().manual_seed(77 + rank)
    batches = [(tuple(x.cuda() for x in xs), y.cuda()) for xs, y in T.make_batches("image", 16, 224, gen)]
    with T.reproducible_cudnn():
        model, ref = T.build_models("image")
        env.setenv("DR_FUSED_BN", "1")
        tr = T.make_trainer(model, "image", "bloom", bucket_cap_mb=1e9)
        try:
            assert len(tr.ddp.engines) == 1 and tr.ddp.engines[0].cta_speeds is not None
            with torch.no_grad():                # the wrapper broadcasts rank 0's weights; the reference starts there too
                for p, q in zip(tr.model.parameters(), ref.parameters()):
                    q.copy_(p)
                for a, b in zip(tr.model.buffers(), ref.buffers()):
                    b.copy_(a)
            ref_named = dict(ref.named_parameters())
            ref_opt = torch.optim.SGD(ref.parameters(), lr=T.LR, momentum=T.MOMENTUM, weight_decay=T.WEIGHT_DECAY,
                                      fused=True)
            eng = tr.ddp.engines[0]
            plan = eng.plan
            params = {n: ref_named[n] for n, _ in tr.ddp.buckets[0]}
            resid_ref = [torch.zeros(plan.total_elems) for _ in range(world)]
            captured = T.capture_exchanged(tr)
            for step in range(T.STEPS):
                tag = f"step {step}"
                micro = [batches[step & 1]]
                ref_losses = (T.ref_backward_checked if step == 0 else T.ref_backward)(ref, "image", micro, env)
                env.setenv("DR_FUSED_BN", "1")
                loss = tr.step(*micro[0][0], target=micro[0][1])
                torch.cuda.synchronize()
                tr.ddp.check()
                check(f"{tag} loss", lambda: T.compare_bucket(tag, loss, ref_losses[0], False))

                grads = {n: q.grad for n, q in params.items()}
                flats = _gather_cpu(T.ref_flat(plan, params, grads).cuda(), world)
                out, new_res, _ = engine_oracle(plan, flats, resid_ref, epoch=eng.epoch)
                got = captured[step][0].cpu()
                scale = float(out.abs().max())

                def bucket():
                    assert torch.allclose(got, out, rtol=1e-6, atol=1e-6 * scale), \
                        f"{tag} bucket: max |diff| {float((got - out).abs().max())} (scale {scale})"
                check(f"{tag} bucket", bucket)
                check(f"{tag} residual", lambda: T.compare_bucket(f"{tag} residual", eng.resid.cpu(), new_res[rank], False))

                exchanged = T.unflatten(plan, params, got)
                for n, q in ref_named.items():
                    q.grad = exchanged[n]
                ref_opt.step()
                check(f"{tag} parameters", lambda: T.check_after_step(tag, tr, ref, ref_opt))
                mine = torch.cat([p.detach().reshape(-1) for p in tr.model.parameters()])
                rank0 = mine.clone()
                dist.broadcast(rank0, 0)

                def same_on_all_ranks():
                    assert torch.equal(mine, rank0), f"{tag}: parameters differ from rank 0's: {T.first_diff(mine, rank0)}"
                check(f"{tag} replicas", same_on_all_ranks)
                T.sync_reference(tr, ref, ref_opt)
                resid_ref = _gather_cpu(eng.resid, world)
        except Exception:                            # noqa: BLE001
            # the peers may be inside a collective this rank will never join: leave now, torch.distributed.run then
            # stops the other workers
            print(f"[rank {rank}] {traceback.format_exc()}", flush=True)
            os._exit(1)
        tr.close()
    flag = torch.tensor([0 if failures else 1], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0 and int(flag.item()) == 1:
        print("TRAIN_STEP_MULTIGPU_OK", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
