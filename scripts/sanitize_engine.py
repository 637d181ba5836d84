"""Small engine run for compute-sanitizer (memcheck / racecheck / synccheck): 2 steps in every fused mode, both
phase-0 copy engines (TMA bulk ring / per-thread cp.async ring) and the threshold / value-only recipes.
SAN_CASES=<n> limits the number of cases (racecheck is ~100x slower than memcheck)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle  # noqa: E402

# (index codec, value codec, plan kwargs, use_tma)
CASES = [
    ("bloom", None, {}, True),
    ("bloom", "polyfit", {}, True),
    ("bloom", "qsgd", {}, False),
    ("rle", None, {}, True),
    (None, None, {}, False),
    ("bloom", None, dict(sparsifier="threshold", threshold=1.0, capacity_ratio=0.5), True),
    (None, "polyfit", {}, True),
    ("bloom", "qsgd", dict(quantum_num=1000), True),
    ("bloom", None, dict(policy="random", fpr=0.02), True),          # not yet run under the sanitizer
    ("bloom", None, dict(policy="conflict_sets"), True),             # fused P2 (ops/csrc/p2.cu); not yet run under the sanitizer
]
CASES = CASES[:int(os.environ.get("SAN_CASES", len(CASES)))]
for index, value, kw, tma in CASES:
    plan = BucketPlan([5000, 300, 40000, 9000], compress_ratio=0.02, index=index, value=value, poly_min_k=100, **kw)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=200_000_000, use_tma=tma)
    gen = torch.Generator().manual_seed(0)
    res = torch.zeros(plan.total_elems)
    for step in range(2):
        g = torch.zeros(plan.total_elems)
        for v in plan.views(g):
            v.copy_(torch.randn(v.shape, generator=gen))
        eng.grad.copy_(g.cuda())
        eng.step()
        torch.cuda.synchronize()
        eng.check_status()
        out, new_res, _ = engine_oracle(plan, [g], [res], epoch=eng.epoch)
        if value == "qsgd":      # a reduction-order difference may flip a rounding decision: allow a few level flips
            ok = float(((eng.grad.cpu() - out).abs() > 1e-3 * float(out.abs().max())).float().mean()) < 2e-3
        else:
            ok = torch.allclose(eng.grad.cpu(), out, atol=1e-2 if value else 0, rtol=1e-2 if value else 0)
        print(f"index={index} value={value} kw={kw} tma={tma} step={step} matches_oracle={ok}", flush=True)
        res = eng.resid.cpu().clone() if value else new_res[0]
    eng.close()
print("SANITIZE_RUN_DONE")
