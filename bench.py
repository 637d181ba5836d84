#!/usr/bin/env python
"""Headline benchmark (BASELINE.json): ResNet-50 images/sec (whole job, device-timed,
max over ranks) with top-k 1 % + bloom-index + residual gradient exchange, synthetic
224² data, random-init weights, bf16 autocast.

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # unmodified reference file + GRACE/cupy shims (baseline/)

Prints ONE JSON line on rank 0.
"""
from __future__ import annotations

import argparse
import json
import os
import socket
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CONFIGS = {
    # BASELINE.json config 2 (default) and 3; plus context rows
    "bloom": {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
              'deepreduce': 'index', 'index': 'bloom'},
    "bloom_p0": {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
                 'deepreduce': 'index', 'index': 'bloom', 'policy': 'p0'},
    "both": {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01,
             'deepreduce': 'both', 'index': 'bloom', 'value': 'polyfit'},
    "topk": {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01},
    # BASELINE.json config 4: NCF top-k 0.1 % + run-length index
    "rle": {'compressor': 'topk', 'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.001,
            'deepreduce': 'index', 'index': 'rle'},
    "dense": {'compressor': 'none', 'memory': 'none', 'communicator': 'allreduce'},
}


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="bloom", choices=sorted(CONFIGS))
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--batch", type=int, default=None, help="per-GPU batch (weak scaling); default 256 (resnet50), 8 (bert_large), 65536 (ncf)")
    ap.add_argument("--seq", type=int, default=128, help="sequence length for bert_large")
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--no-overlap", action="store_true")
    ap.add_argument("--no-thread", action="store_true")
    ap.add_argument("--bucket-mb", type=float, default=None,
                    help="flat bucket size; default 128 MB on 1 GPU (ResNet-50 = one bucket; BERT-large = 11, overlapped with "
                         "backward) and ONE bucket launched after backward on N > 1 GPUs (a persistent exchange kernel that "
                         "waits for its peers must not sit on SMs backward needs)")
    ap.add_argument("--blocks-per-sm", type=int, default=2)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--breakdown", action="store_true", help="(kept for compatibility: the exchange-kernel timing is always reported)")
    ap.add_argument("--overlap-grid", type=int, default=0,
                    help="CTAs for exchange kernels launched while backward is still running (0 = whole GPU)")
    ap.add_argument("--no-dense-context", action="store_true", help="skip the dense NCCL all-reduce context measurement")
    ap.add_argument("--no-check", action="store_true", help="skip the multi-GPU correctness self-check (N > 1)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step returned to the caller (loss, exchanged "
                         "gradients, updated parameters; a fixed seeded sample of the large ones) as DIR/<name>.npy")
    return ap.parse_args()


def exchange_roofline(exchange_ms, dense_bytes, wire_bytes, world, stage2_bytes=None):
    """Achieved fraction of the exchange kernel's roofline = the slower of (a) its unavoidable HBM traffic at the
    copy bandwidth (read g, read r, write r, write the dense result: 4 x dense bytes) and (b) the bytes it
    sends over NVLink at link bandwidth (the slot to W-1 peers, plus about as much again for the decoded slices of
    the sharded decode).  Denominators: MEASURED_PEAKS.json when present, else the H100 SXM data-sheet figures
    (3 350 GB/s HBM3, 450 GB/s per direction of NVLink 4); data-sheet peaks are not reached in practice."""
    hbm = 3350.0
    try:
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "MEASURED_PEAKS.json")) as f:
            hbm = float(json.load(f).get("hbm_gbs", hbm))
    except Exception:
        pass
    nvlink = 450.0
    t_hbm = 4.0 * dense_bytes / (hbm * 1e9) * 1e3
    # bytes this rank puts on NVLink: its slot to W-1 peers + its decoded slice lists (live count, or ~ as much again)
    nv_bytes = (world - 1) * wire_bytes + (stage2_bytes if stage2_bytes is not None else (world - 1) * wire_bytes)
    t_nv = nv_bytes / (nvlink * 1e9) * 1e3
    return {"hbm_min_bytes": int(4 * dense_bytes), "hbm_gbs_measured": hbm, "hbm_bound_ms": t_hbm,
            "nvlink_bytes_out": int(nv_bytes), "nvlink_gbs_per_dir": nvlink, "nvlink_bound_ms": t_nv,
            "bound": "hbm" if t_hbm >= t_nv else "nvlink", "frac_of_roofline": max(t_hbm, t_nv) / exchange_ms,
            "compressed_allgather_bus_gbs": nv_bytes / (exchange_ms * 1e-3) / 1e9}


class ClockSampler:
    """nvidia-smi clocks/throttle reasons DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.proc = None
        self.lines = []
        self.gpu_index = gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "200", "-i", str(self.gpu_index)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=3)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for l in self.lines:
            f = [x.strip() for x in l.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for n, v in zip(names, f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def init_dist(args):
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    need = world > 1 or args.impl == "reference"
    if need:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", str(free_port()))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{local}"))
    return rank, world, local


def build_model(name):
    import torch
    if name == "resnet50":
        from deepreduce_b200.models import resnet50
        return resnet50()
    if name == "resnet20":
        from deepreduce_b200.models import resnet20
        return resnet20()
    raise ValueError(name)


def max_over_ranks(x, world):
    import torch
    import torch.distributed as dist
    if world == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def barrier(world):
    import torch
    import torch.distributed as dist
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


def timed(fn, steps, world):
    """K steps bracketed by barrier + synchronize, CUDA events on the launching stream."""
    import torch
    barrier(world)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for i in range(steps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    barrier(world)
    return max_over_ranks(e0.elapsed_time(e1), world), max_over_ranks(wall, world)


MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def bench_config(args, kind, B, world, cfg):
    """The `config` object of the JSON line — IDENTICAL in the `ours` and `reference` arms (same model architecture,
    batch, dtype, optimizer, input pipeline, step counts); everything implementation-specific goes to `harness`."""
    return {"model": args.model, "global_batch": B * world, "per_gpu_batch": B,
            "seq_len": args.seq if kind == "bert" else None, "parallelism": f"dp{world}",
            "gradient_exchange": args.config,
            "params": {k: v for k, v in cfg.items() if isinstance(v, (str, int, float, bool, type(None)))},
            "optimizer": "SGD(momentum=0.9, weight_decay=1e-4, fused=True)" if kind != "bert" else "SGD(momentum=0.9, weight_decay=1e-4, fused=True, lr=1e-4)",
            "input": ("uint8 NHWC batch in pinned host memory -> H2D -> normalise -> bf16 channels_last" if kind.startswith("image")
                      else "int64 ids in pinned host memory -> H2D"),
            "e2e": "H2D of the step's batch (prefetched one step ahead on a copy stream) + loss read back to the host, every step",
            "e2e_steps": args.steps,
            "l2": "working set (activations + fp32 gradients + residual) exceeds the 50 MB L2 every step",
            "cudnn": "deterministic algorithms chosen by heuristics (benchmark=False): same arguments, same outputs"}


def reproducible_cudnn():
    """Same arguments, same outputs: cuDNN may only use deterministic algorithms, and picks them by its heuristics
    instead of by timing (``benchmark=True`` lets the fastest measured algorithm win, which changes from run to run and
    changes the gradients in the last bits; the top-k selection then turns that into different selected sets)."""
    import torch
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True


def synth_batches(kind, B, seq, gen):
    import torch
    if kind.startswith("image"):
        hw = 224 if kind == "image224" else 32
        ncls = 1000 if kind == "image224" else 10
        pool = [(torch.randint(0, 256, (B, hw, hw, 3), dtype=torch.uint8, generator=gen),) for _ in range(2)]
        tgt = [torch.randint(0, ncls, (B,), generator=gen) for _ in range(2)]
    elif kind == "bert":
        pool = [(torch.randint(0, 30522, (B, seq), generator=gen),) for _ in range(2)]
        tgt = [p[0].clone() for p in pool]
    else:   # ncf
        pool = [(torch.randint(0, 138493, (B,), generator=gen), torch.randint(0, 26744, (B,), generator=gen)) for _ in range(2)]
        tgt = [torch.randint(0, 2, (B,), generator=gen).float() for _ in range(2)]
    return pool, tgt


def loss_for(kind):
    import torch
    if kind == "bert":
        return lambda out, y: torch.nn.functional.cross_entropy(
            (out.logits if hasattr(out, "logits") else out).reshape(-1, 30522).float(), y.reshape(-1))
    if kind == "ncf":
        return torch.nn.functional.binary_cross_entropy_with_logits
    return None


def model_spec(args):
    """(model, kind, default per-GPU batch, metric unit)"""
    from deepreduce_b200 import models as M
    if args.model == "resnet50":
        return M.resnet50(), "image224", 256, "images/s"
    if args.model == "resnet20":
        return M.resnet20(), "image32", 256, "images/s"
    if args.model == "bert_large":
        return M.bert_large(seq_len=max(args.seq, 128)), "bert", 8, "sequences/s"
    if args.model == "ncf":
        return M.NeuMF(), "ncf", 65536, "samples/s"
    raise ValueError(args.model)


DUMP_SAMPLE = 2 << 20          # elements kept of a flattened output larger than this (8 MB in float32)


def dump_outputs(out_dir, loss, model):
    """What the last timed step handed back to its caller: the loss, the exchanged gradients and the parameters after
    the optimizer step, each flattened in ``model.parameters()`` order.  Arrays longer than DUMP_SAMPLE are cut to a
    fixed seeded sample of positions (saved as ``sample_index``), so two builds can be compared output for output."""
    import numpy as np
    import torch
    params = [p for p in model.parameters()]
    grad = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).detach().float().reshape(-1) for p in params])
    weight = torch.cat([p.detach().float().reshape(-1) for p in params])
    arrays = {"loss": loss.detach().float().reshape(1)}
    if grad.numel() > DUMP_SAMPLE:
        g = torch.Generator().manual_seed(2024)
        idx = torch.randperm(grad.numel(), generator=g)[:DUMP_SAMPLE].sort().values
        arrays["sample_index"] = idx.double()
        idx = idx.to(grad.device)
        grad, weight = grad[idx], weight[idx]
    arrays["grad"], arrays["params"] = grad, weight
    os.makedirs(out_dir, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, f"{name}.npy"), t.cpu().numpy())


def measure_dense_context(args, kind, B, world, pool, tgt):
    """Dense NCCL all-reduce data parallelism on the same box, same model / batch / optimizer (context row: on NVLink
    it is the strongest baseline; the compressed path is expected to match it, not beat it)."""
    import torch
    from deepreduce_b200.trainer import Trainer
    model, _, _, _ = model_spec(args)
    model = model.cuda()
    amp = torch.bfloat16 if args.dtype == "bf16" else None
    tr = Trainer(model, dict(CONFIGS["dense"]), lr=0.05 if kind != "bert" else 1e-4, amp_dtype=amp,
                 channels_last=kind.startswith("image"), bucket_cap_mb=args.bucket_mb if args.bucket_mb else 128.0,
                 u8_input=kind.startswith("image"),
                 loss_fn=loss_for(kind))
    dev_x = [tuple(t.cuda() for t in p) for p in pool]
    dev_y = [t.cuda() for t in tgt]

    def step(i):
        tr.step(*dev_x[i & 1], target=dev_y[i & 1])

    for i in range(args.warmup):
        step(i)
    ms, _ = timed(step, args.steps, world)
    tr.close()
    del tr, model
    torch.cuda.empty_cache()
    return {"value": world * B * args.steps / (ms / 1e3), "ms_per_step": ms / args.steps,
            "what": "dense NCCL all-reduce DDP, same model/batch/optimizer, device-timed, same process"}


def run_ours(args, rank, world, local):
    import torch
    from deepreduce_b200 import ops
    from deepreduce_b200.trainer import Trainer
    torch.manual_seed(1234)
    reproducible_cudnn()
    model, kind, default_b, unit = model_spec(args)
    model = model.cuda()
    B = args.batch or default_b
    cfg = dict(CONFIGS[args.config])
    amp = torch.bfloat16 if args.dtype == "bf16" else None
    gen = torch.Generator().manual_seed(77 + rank)
    pool, tgt = synth_batches(kind, B, args.seq, gen)
    bucket_mb = args.bucket_mb if args.bucket_mb else (128.0 if world == 1 else 1e9)      # see --bucket-mb
    tr = Trainer(model, cfg, lr=0.05 if kind != "bert" else 1e-4, amp_dtype=amp, channels_last=kind.startswith("image"),
                 overlap=not args.no_overlap, bucket_cap_mb=bucket_mb, background_thread=not args.no_thread,
                 blocks_per_sm=args.blocks_per_sm, u8_input=kind.startswith("image"), loss_fn=loss_for(kind),
                 overlap_grid=args.overlap_grid)
    dev_x = [tuple(t.cuda() for t in p) for p in pool]
    dev_y = [t.cuda() for t in tgt]
    last = {}

    def step(i):
        last["loss"] = tr.step(*dev_x[i & 1], target=dev_y[i & 1])

    for i in range(args.warmup):
        step(i)
    tr.ddp.check()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    l0 = ops.launch_count()
    ms, wall = timed(step, args.steps, world)
    launches = ops.launch_count() - l0
    clocks = sampler.stop() if rank == 0 else None
    tr.ddp.check()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last["loss"], tr.model)
    value = world * B * args.steps / (ms / 1e3)

    e2e = None
    if not args.no_e2e:
        host_x = [tuple(t.pin_memory() for t in p) for p in pool]
        host_y = [t.pin_memory() for t in tgt]

        def step_e2e(i):
            nxt = (host_x[(i + 1) & 1], host_y[(i + 1) & 1])
            tr.step_host(host_x[i & 1], host_y[i & 1], next_batch=nxt)

        for i in range(2):
            step_e2e(i)
        _, wall_e = timed(step_e2e, args.steps, world)
        e2e = {"value": world * B * args.steps / (wall_e / 1e3), "unit": unit,
               "h2d_bytes_per_step": int(tr.h2d_bytes), "d2h_bytes_per_step": int(tr.d2h_bytes)}

    extra = {}
    wire = tr.ddp.wire_bytes_per_step()
    dense = tr.ddp.dense_bytes()
    if tr.ddp.engines:
        def ex(i):       # the exchange kernels alone, on the last gradients (all buckets back to back)
            for e in tr.ddp.engines:
                e.ctx.set_grid_cap(0)
                e.step()
        for i in range(3):
            ex(i)
        ms_ex, _ = timed(ex, args.steps, world)
        stage2 = tr.ddp.stage2_bytes_per_step()
        extra["exchange_ms_per_step"] = ms_ex / args.steps
        extra["engine_grid"] = tr.ddp.engines[0].grid()
        extra["stage2_bytes_per_step_per_rank"] = int(stage2)
        extra["nvlink_bytes_out_per_step_per_rank"] = int((world - 1) * wire + stage2)
        extra["roofline"] = exchange_roofline(extra["exchange_ms_per_step"], dense, wire, world, stage2)
        extra["compressed_allgather_bus_gbs"] = extra["roofline"]["compressed_allgather_bus_gbs"]
        if world > 1 and not args.no_check:
            from deepreduce_b200.utils.selfcheck import multi_gpu_check
            chk = multi_gpu_check(tr.ddp.engines[0])
            extra["multi_gpu_check"] = chk["status"]
            extra["multi_gpu_check_detail"] = {k: v for k, v in chk.items() if k != "status"}
        tr.ddp.check()
    names = {"resnet50": "ResNet-50 images/sec (whole job, device-timed, max over ranks)",
             "bert_large": "BERT-large sequences/sec (whole job, device-timed, max over ranks)",
             "ncf": "NCF (MovieLens-20M shapes) samples/sec (whole job, device-timed, max over ranks)"}
    out = {
        "metric": names.get(args.model, f"{args.model} {unit}"),
        "value": value, "unit": unit, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": args.dtype, "data": "synthetic (shapes of the named benchmark, random-init weights)", "impl": "ours",
        "config": bench_config(args, kind, B, world, cfg),
        "harness": {"model_impl": "deepreduce_b200.models", "exchange": "fused bucket engine (one persistent kernel per bucket, in-kernel P2P)",
                    "overlap": not args.no_overlap, "buckets": len(tr.ddp.flat), "bucket_mb": bucket_mb if bucket_mb < 1e8 else "one bucket",
                    "overlap_grid": args.overlap_grid, "input_kernel": "u8_to_nhwc_norm (own)"},
        "clocks": clocks, "e2e": e2e, "gpu_launches": int(launches),
        "wire_bytes_per_step_per_rank": int(wire), "dense_bytes": int(dense),
        "relative_volume": wire / dense, "wall_ms_per_step": wall / args.steps,
    }
    out.update(extra)
    tr.close()
    del tr, model
    torch.cuda.empty_cache()
    if args.config != "dense" and not args.no_dense_context:
        out["dense_allreduce_context"] = measure_dense_context(args, kind, B, world, pool, tgt)
        out["dense_allreduce_context"]["ours_over_dense"] = out["value"] / out["dense_allreduce_context"]["value"]
    return out


class _RefNeuMF:
    """Plain-torch NeuMF of the MovieLens-20M shapes for the REFERENCE arm (the reference's NCF trainer is the external
    grace-benchmarks ``ncf_grace.py``; nothing of deepreduce_b200 may run on that path)."""

    @staticmethod
    def build():
        import torch
        import torch.nn as nn
        import torch.nn.functional as F

        class NeuMF(nn.Module):
            def __init__(self, n_users=138493, n_items=26744, mf_dim=64, mlp_layers=(256, 256, 128, 64)):
                super().__init__()
                self.mf_user = nn.Embedding(n_users, mf_dim); self.mf_item = nn.Embedding(n_items, mf_dim)
                self.mlp_user = nn.Embedding(n_users, mlp_layers[0] // 2); self.mlp_item = nn.Embedding(n_items, mlp_layers[0] // 2)
                self.mlp = nn.ModuleList(nn.Linear(a, b) for a, b in zip(mlp_layers[:-1], mlp_layers[1:]))
                self.out = nn.Linear(mf_dim + mlp_layers[-1], 1)
                for e in (self.mf_user, self.mf_item, self.mlp_user, self.mlp_item):
                    nn.init.normal_(e.weight, 0.0, 0.01)

            def forward(self, user, item):
                mf = self.mf_user(user) * self.mf_item(item)
                x = torch.cat([self.mlp_user(user), self.mlp_item(item)], dim=1)
                for l in self.mlp:
                    x = F.relu(l(x))
                return self.out(torch.cat([mf, x], dim=1)).squeeze(-1)
        return NeuMF()


def run_reference(args, rank, world, local):
    """UNMODIFIED reference pytorch/deepreduce.py through its documented API (README.md:36-48):
    grace_from_params + Value/Index/DeepReduce wrapper, grc.step(grad, name) per tensor after backward.  Same model
    architecture, batch, dtype, optimizer, input pipeline (uint8 NHWC pinned -> H2D -> normalise -> bf16
    channels_last, prefetched one step ahead) and step counts as the `ours` arm; nothing of deepreduce_b200 is
    imported on this path."""
    import numpy as np
    import torch
    ref_file = os.path.join(ROOT, "oracle", "_ref", "deepreduce_ref", "deepreduce.py")
    if not os.path.exists(ref_file):        # build() makes the copy; the benchmark never writes into the tree
        return {"impl": "reference", "unavailable": "reference copy absent: build() found no checkout of the reference (DEEPREDUCE_REFERENCE, else BASELINE.json reference_path)"}
    sys.path.insert(0, os.path.join(ROOT, "baseline", "shims"))
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    if not hasattr(np, "RankWarning"):
        np.RankWarning = np.exceptions.RankWarning        # numpy>=2 moved it; the reference reads np.RankWarning
    from deepreduce_ref import deepreduce as R
    from grace_dl.dist.helper import grace_from_params

    torch.manual_seed(1234)
    reproducible_cudnn()
    if args.model == "resnet50":
        import torchvision
        model, kind, default_b, unit = torchvision.models.resnet50(weights=None), "image224", 256, "images/s"
    elif args.model == "bert_large":
        from transformers import BertConfig, BertForMaskedLM
        model = BertForMaskedLM(BertConfig(vocab_size=30522, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                                           intermediate_size=4096, max_position_embeddings=max(args.seq, 128)))
        kind, default_b, unit = "bert", 8, "sequences/s"
    elif args.model == "ncf":
        model, kind, default_b, unit = _RefNeuMF.build(), "ncf", 65536, "samples/s"
    else:
        return {"impl": "reference", "unavailable": f"no reference arm for model {args.model}"}
    model = model.cuda()
    if kind.startswith("image"):
        model = model.to(memory_format=torch.channels_last)
    cfg = dict(CONFIGS[args.config])
    cfg["world_size"] = world
    grc = grace_from_params(cfg)
    if cfg.get("deepreduce"):
        d_max = max(p.numel() for p in model.parameters())
        g = torch.Generator(device="cuda").manual_seed(18)
        cfg["hash_table"] = torch.randint(0, 2 ** 31 - 1, (d_max, 16), dtype=torch.int32, device="cuda", generator=g)
        wrapper = {'value': R.ValueCompressor, 'index': R.IndexCompressor, 'both': R.DeepReduce}[cfg["deepreduce"]]
        grc.compressor = wrapper(grc.compressor, cfg)
    opt = torch.optim.SGD(model.parameters(), lr=0.05 if kind != "bert" else 1e-4, momentum=0.9, weight_decay=1e-4, fused=True)
    B = args.batch or default_b
    gen = torch.Generator().manual_seed(77 + rank)
    pool, tgt = synth_batches(kind, B, args.seq, gen)
    amp = args.dtype == "bf16"
    named = [(n, p) for n, p in model.named_parameters()]
    loss_fn = loss_for(kind) or torch.nn.functional.cross_entropy
    mean = torch.tensor(MEAN, device="cuda").view(1, 1, 1, 3)
    inv_std = (1.0 / torch.tensor(STD, device="cuda")).view(1, 1, 1, 3)

    def prep(xs):
        if kind.startswith("image"):          # uint8 NHWC -> normalised bf16, NCHW view of the NHWC storage (= channels_last)
            x = xs[0]
            return (((x.float() * (1.0 / 255.0) - mean) * inv_std).to(torch.bfloat16).permute(0, 3, 1, 2),)
        return xs

    def train(xs, y):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            out = model(*prep(xs))
        loss = loss_fn(out.float() if torch.is_tensor(out) else out, y)
        loss.backward()
        for n, p in named:
            if p.grad is not None:
                g = grc.step(p.grad, n).view(p.shape).to(p.dtype)
                if g.stride() != p.stride():           # channels_last conv weights: the fused optimizer wants matching layouts
                    g = torch.empty_like(p).copy_(g)
                p.grad = g
        opt.step()
        return loss

    dev_x = [tuple(t.cuda() for t in p) for p in pool]
    dev_y = [t.cuda() for t in tgt]

    last = {}

    def step(i):
        last["loss"] = train(dev_x[i & 1], dev_y[i & 1])

    for i in range(args.warmup):
        step(i)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    ms, wall = timed(step, args.steps, world)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last["loss"], model)     # p.grad holds what grc.step returned
    value = world * B * args.steps / (ms / 1e3)
    e2e = None
    if not args.no_e2e:
        host_x = [tuple(t.pin_memory() for t in p) for p in pool]
        host_y = [t.pin_memory() for t in tgt]
        copy_stream = torch.cuda.Stream()
        loss_host = torch.zeros(1).pin_memory()
        staged = {}

        def stage(i):
            with torch.cuda.stream(copy_stream):
                xs = tuple(t.cuda(non_blocking=True) for t in host_x[i & 1])
                y = host_y[i & 1].cuda(non_blocking=True)
                ev = torch.cuda.Event(); ev.record(copy_stream)
            staged["cur"] = (xs, y, ev)

        def step_e2e(i):
            if "cur" not in staged:
                stage(i)
            xs, y, ev = staged.pop("cur")
            torch.cuda.current_stream().wait_event(ev)
            stage(i + 1)                                   # prefetch the next batch while this step computes
            loss = train(xs, y)
            loss_host.copy_(loss.detach().reshape(1), non_blocking=True)
            torch.cuda.current_stream().synchronize()
            for t in xs:
                t.record_stream(torch.cuda.current_stream())
            return float(loss_host[0])

        for i in range(2):
            step_e2e(i)
        _, wall_e = timed(step_e2e, args.steps, world)
        h2d = sum(t.numel() * t.element_size() for t in host_x[0]) + host_y[0].numel() * host_y[0].element_size()
        e2e = {"value": world * B * args.steps / (wall_e / 1e3), "unit": unit,
               "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": 4}
    names = {"resnet50": "ResNet-50 images/sec (whole job, device-timed, max over ranks)",
             "bert_large": "BERT-large sequences/sec (whole job, device-timed, max over ranks)",
             "ncf": "NCF (MovieLens-20M shapes) samples/sec (whole job, device-timed, max over ranks)"}
    pub_cfg = {k: v for k, v in CONFIGS[args.config].items()}
    return {
        "metric": names.get(args.model, f"{args.model} {unit}"),
        "value": value, "unit": unit, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": args.dtype, "data": "synthetic (shapes of the named benchmark, random-init weights)", "impl": "reference",
        "config": bench_config(args, kind, B, world, pub_cfg),
        "harness": {"model_impl": "torchvision / transformers / plain torch (bench.py)",
                    "exchange": "unmodified reference pytorch/deepreduce.py + GRACE/cupy shims (baseline/), per-tensor grc.step after backward",
                    "input_kernel": "torch ops"},
        "clocks": clocks, "e2e": e2e, "gpu_launches": 0, "wall_ms_per_step": wall / args.steps,
    }


def main():
    args = parse()
    # stdout carries exactly ONE line (the JSON): keep a private handle to it and point fd 1 at stderr so that
    # library banners (e.g. "NCCL version ...") and stray prints cannot end up next to the result
    sys.stdout.flush()
    result_out = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"impl": args.impl, "unavailable": "no CUDA device on this box"}), file=result_out, flush=True)
        return 0
    rank, world, local = init_dist(args)
    if world != args.gpus and rank == 0:
        print(f"[bench] warning: --gpus {args.gpus} but WORLD_SIZE={world}; using {world}", file=sys.stderr)
    if args.impl == "ours":
        out = run_ours(args, rank, world, local)
    else:
        try:
            out = run_reference(args, rank, world, local)
        except Exception as e:      # the unmodified reference can fail on its own (e.g. its CPU 6x6 inverse on a singular segment)
            import traceback
            traceback.print_exc()
            last = (traceback.extract_tb(e.__traceback__) or [None])[-1]
            where = f"{os.path.basename(last.filename)}:{last.lineno}" if last else "?"
            out = {"impl": "reference", "unavailable": f"reference raised {type(e).__name__} at {where}: {str(e).splitlines()[0][:160]}",
                   "config": {"model": args.model, "gradient_exchange": args.config}}
    if rank == 0:
        print(json.dumps(out), file=result_out, flush=True)
    import torch.distributed as dist
    if dist.is_initialized():
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
