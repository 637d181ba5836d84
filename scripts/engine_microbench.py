"""Exchange-kernel microbenchmark on ResNet-50 gradient shapes (1 GPU): device time of the fused
kernel per step, per-phase times (unfused chain), bytes and roofline fractions vs MEASURED_PEAKS.json."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepreduce_b200.models import resnet50  # noqa: E402
from deepreduce_b200.parallel import BucketEngine, BucketPlan  # noqa: E402

PHASES = ["accum+hist1", "fallback", "hist2", "insert", "query", "emit", "rank_hist", "rank_scan", "rank_scatter", "rank_exact",
          "fit", "fix", "push", "signal", "expand", "decode", "compact", "push2", "signal2", "scatter"]


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    bps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    use_tma = bool(int(sys.argv[3])) if len(sys.argv) > 3 else True
    hist_shift = int(sys.argv[4]) if len(sys.argv) > 4 else 23
    hint = bool(int(sys.argv[5])) if len(sys.argv) > 5 else True
    value = (sys.argv[6] if len(sys.argv) > 6 else 'none')
    value = None if value == 'none' else value
    shape = sys.argv[7] if len(sys.argv) > 7 else 'resnet50'
    if shape == 'resnet50':
        m = resnet50()
        named = list(reversed([(n, p) for n, p in m.named_parameters()]))
        plan = BucketPlan([p.numel() for _, p in named], [n for n, _ in named], compress_ratio=0.01, hint=hint, value=value)
    else:            # 'uniformN': N equal tensors with ResNet-50's total size (isolates the per-tensor overheads)
        n = int(shape.replace('uniform', ''))
        plan = BucketPlan([25557032 // n] * n, compress_ratio=0.01, hint=hint, value=value)
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, blocks_per_sm=bps, use_tma=use_tma, hist_shift=hist_shift)
    calibrate = bool(int(sys.argv[8])) if len(sys.argv) > 8 else True
    if calibrate and eng.cuts is not None:
        eng.calibrate_partition()
    gen = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(plan.total_elems, device="cuda", generator=gen) * 0.01 for _ in range(4)]
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")

    def one(i, fused=True):
        eng.grad.copy_(grads[i % 4])
        flush.zero_()                       # L2 flush between timed iterations
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        if fused:
            eng.step()
        else:
            eng.run_unfused()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for i in range(5):
        one(i)
    eng.check_status()
    fused = sorted(one(i) for i in range(steps))
    # per-phase (separate launches)
    per = [0.0] * len(PHASES)
    for i in range(5):
        eng.grad.copy_(grads[i % 4])
        flush.zero_()
        eng.epoch += 1
        for ph in range(len(PHASES)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.ctx.run(eng.epoch, ph, ph + 1)
            e1.record()
            torch.cuda.synchronize()
            per[ph] += e0.elapsed_time(e1) / 5
    eng.check_status()
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 3350.0)              # default: H100 SXM HBM3, data sheet
    d = plan.dense_bytes()
    # algorithmic HBM bytes: read g + read r + write r (accum), write dense out (decode); other passes re-read r (L2/HBM)
    min_bytes = 4 * d
    med = fused[len(fused) // 2]
    out = {"kernel": "dr_engine_kernel (fused, W=1)", "model": f"{shape} grads", "dense_bytes": d,
           "wire_bytes": plan.wire_bytes(), "grid": eng.grid(), "blocks_per_sm": bps, "use_tma": use_tma, "hist_shift": hist_shift, "calibrated_partition": calibrate, "hint": hint, "value": value,
           "fused_ms_median": med, "fused_ms_min": fused[0],
           "phase_ms_unfused": dict(zip(PHASES, [round(x, 4) for x in per])),
           "algorithmic_min_bytes": min_bytes, "achieved_gbs_vs_min_bytes": min_bytes / med / 1e6,
           "frac_of_measured_hbm": min_bytes / med / 1e6 / hbm, "hbm_gbs_measured": hbm,
           "all_pass_bytes": 8 * d, "achieved_gbs_all_passes": 8 * d / med / 1e6}
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
