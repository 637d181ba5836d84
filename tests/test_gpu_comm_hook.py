"""The DDP communication hook on the GPU: ``bucket_pack`` / ``bucket_unpack`` against torch indexing, and DDP (nccl,
world 1) + ``deepreduce_hook`` against the CPU oracle of the exchange for steps 0-3, across DDP's bucket rebuild.

The oracle of a step is built from what DDP handed the hook (the bucket buffer, cloned before the exchange), the
hook's own plan for that layout and the residual the test carries itself: ``ref_flat`` -> ``engine_oracle`` ->
``unflatten`` (``test_train_step_reference``).  Every ``p.grad`` must equal it bit for bit; the value-coded 'both'
configuration compares within the fp32-vs-fp64 tolerances of ``test_gpu_engine``.  When DDP rebuilds its buckets,
the residual each parameter finds in its new engine must be the one it left in the old."""
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.nn as nn
from torch.nn.parallel import DistributedDataParallel as DDP

from test_train_step_reference import chunk_offsets, compare_bucket, first_diff, ref_flat, unflatten

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 4


# ---------------------------------------------------------------------------
# pack / unpack against torch indexing
# ---------------------------------------------------------------------------
def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _check_repack(numels, dtype, base_shift=0, gaps=False, seed=0):
    from deepreduce_b200 import ops
    from deepreduce_b200.parallel import BucketPlan
    from deepreduce_b200.parallel.comm_hook import pack_reference, segment_table, unpack_reference
    gen = torch.Generator(device="cuda").manual_seed(seed)
    segs, off = [], 0
    for i, n in enumerate(numels):
        off += (i % 3) if gaps else 0
        segs.append((off, n))
        off += n
    plan = BucketPlan(numels, index=None)
    table = segment_table(segs, plan, list(range(len(numels))))
    rp = ops.cuda_module().Repack(table, off, plan.total_elems, torch.empty(1, dtype=dtype, device="cuda"))
    # DDP side: a slice whose base is `base_shift` elements past an allocation (not 16-byte aligned for shift > 0)
    raw = torch.randn(off + base_shift, device="cuda", generator=gen).to(dtype)
    ddp = raw[base_shift:]
    assert (ddp.data_ptr() % 16 != 0) == (base_shift * ddp.element_size() % 16 != 0)
    sentinel = torch.randn(plan.total_elems, device="cuda", generator=gen).to(dtype)
    eng, want = sentinel.clone(), sentinel.clone()
    rp.pack(ddp, eng)
    pack_reference(ddp, want, table)
    assert torch.equal(_bits(eng), _bits(want)), "pack"
    eng_in = torch.randn(plan.total_elems, device="cuda", generator=gen).to(dtype)
    out_raw, want_ddp = raw.clone(), raw[base_shift:].clone()
    out = out_raw[base_shift:]
    rp.unpack(eng_in, out)
    unpack_reference(eng_in, want_ddp, table)
    assert torch.equal(_bits(out), _bits(want_ddp)), "unpack"
    assert torch.equal(_bits(out_raw[:base_shift]), _bits(raw[:base_shift]))
    torch.cuda.synchronize()


DTYPES = [torch.float32, torch.bfloat16]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shift", [0, 1, 3])
def test_repack_odd_offsets_and_single_elements(dtype, shift):
    _check_repack([1, 1, 3, 7, 1, 33, 5, 1, 64, 2], dtype, base_shift=shift, gaps=True)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shift", [0, 1])
def test_repack_4097(dtype, shift):
    _check_repack([4097, 1, 4097, 4096, 4095, 8193], dtype, base_shift=shift)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shift", [0, 5])
def test_repack_resnet50_parameter_list(dtype, shift):
    from deepreduce_b200.models import resnet50
    numels = [p.numel() for p in reversed(list(resnet50().parameters()))]
    assert len(numels) > 150 and min(numels) <= 64 and max(numels) >= 2359296
    _check_repack(numels, dtype, base_shift=shift, seed=1)


@pytest.mark.gpu
def test_repack_checks():
    from deepreduce_b200 import ops
    R = ops.cuda_module().Repack
    like = torch.empty(1, device="cuda")
    with pytest.raises(RuntimeError, match="outside the DDP buffer"):
        R(torch.tensor([[5, 0, 10]]), 12, 64, like)
    with pytest.raises(RuntimeError, match="16-byte vector"):
        R(torch.tensor([[0, 2, 10]]), 12, 64, like)
    with pytest.raises(RuntimeError, match="outside the engine buffer"):
        R(torch.tensor([[0, 32, 33]]), 40, 64, like)
    with pytest.raises(RuntimeError, match="overlap"):
        R(torch.tensor([[0, 0, 10], [5, 32, 10]]), 20, 64, like)
    with pytest.raises(RuntimeError, match="fp32 or bf16"):
        R(torch.tensor([[0, 0, 10]]), 20, 64, torch.empty(1, device="cuda", dtype=torch.float16))
    rp = R(torch.tensor([[0, 0, 10]]), 20, 64, like)
    with pytest.raises(RuntimeError, match="built for"):
        rp.pack(torch.zeros(20, device="cuda", dtype=torch.bfloat16), torch.zeros(64, device="cuda", dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="the table needs"):
        rp.pack(torch.zeros(19, device="cuda"), torch.zeros(64, device="cuda"))


# ---------------------------------------------------------------------------
# DDP + hook against the oracle
# ---------------------------------------------------------------------------
@pytest.fixture
def nccl_world1():
    f = tempfile.NamedTemporaryFile(delete=False)
    f.close()
    os.unlink(f.name)
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method=f"file://{f.name}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


BASE = {'memory': 'residual', 'communicator': 'allgather', 'compress_ratio': 0.01}
CONFIGS = {
    "topk": {'compressor': 'topk', **BASE},
    "bloom_leftmost": {'compressor': 'topk', **BASE, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'leftmost'},
    "bloom_random": {'compressor': 'topk', **BASE, 'deepreduce': 'index', 'index': 'bloom', 'policy': 'random'},
    "rle": {'compressor': 'topk', **BASE, 'deepreduce': 'index', 'index': 'rle'},
    "threshold": {'compressor': 'threshold', **BASE, 'threshold': 0.002},
    "randomk": {'compressor': 'randomk', **BASE},
    "both": {'compressor': 'topk', **BASE, 'deepreduce': 'both', 'index': 'bloom', 'value': 'polyfit'},
}


class MLP(nn.Module):
    def __init__(self, unused=False):
        super().__init__()
        self.a, self.b, self.c = nn.Linear(64, 512), nn.Linear(512, 512), nn.Linear(512, 10)
        self.spare = nn.Linear(512, 7) if unused else None      # never called: DDP marks it ready unused

    def forward(self, x):
        return self.c(torch.relu(self.b(torch.relu(self.a(x)))))


def _model(kind, dtype, unused):
    torch.manual_seed(0)
    if kind == "resnet20":
        from deepreduce_b200.models import resnet20
        m = resnet20()
    else:
        m = MLP(unused)
    return m.cuda().to(dtype)


def _inputs(kind, step, micro, dtype):
    g = torch.Generator(device="cuda").manual_seed(100 * step + micro)
    if kind == "resnet20":
        return torch.randn(8, 3, 32, 32, device="cuda", generator=g).to(dtype)
    return torch.randn(32, 64, device="cuda", generator=g).to(dtype)


def _to_flat(plan, names, per_param):
    """fp32 flat buffer of the plan from per-parameter flat fp32 vectors (storage order)."""
    rows, _ = chunk_offsets(plan, names)
    flat = torch.zeros(plan.total_elems)
    for t, n, off in rows:
        flat[t.elem_off:t.elem_off + t.numel] = per_param[n][off:off + t.numel]
    return flat


def _from_flat(plan, names, flat):
    rows, seen = chunk_offsets(plan, names)
    out = {n: torch.empty(seen[n]) for n in seen}
    for t, n, off in rows:
        out[n][off:off + t.numel] = flat[t.elem_off:t.elem_off + t.numel]
    return out


def run_ddp_case(cfg_name, kind="mlp", dtype=torch.float32, accum=1, unused=False, as_view=False, bucket_cap_mb=0.5):
    from deepreduce_b200.parallel import DeepReduceHookState, engine_oracle
    from deepreduce_b200.parallel.comm_hook import bucket_segments, deepreduce_hook
    cfg = dict(CONFIGS[cfg_name])
    value_coded = cfg.get("deepreduce") in ("value", "both")
    model = _model(kind, dtype, unused)
    ddp = DDP(model, device_ids=[0], bucket_cap_mb=bucket_cap_mb, find_unused_parameters=unused,
              gradient_as_bucket_view=as_view)
    st = DeepReduceHookState(cfg, model, overlap_grid=32)
    named = dict(model.named_parameters())
    by_id = {id(p): n for n, p in named.items()}
    captured, carried, spans = [], [], []

    def spy_hook(state, bucket):
        buf = bucket.buffer()
        captured.append((bucket.index(), buf.clone(), bucket_segments(bucket),
                         [by_id[id(p)] for p in bucket.parameters()]))
        spans.append((buf.data_ptr(), buf.data_ptr() + buf.numel() * buf.element_size()))
        return deepreduce_hook(state, bucket)
    ddp.register_comm_hook(st, spy_hook)

    new_layout = st._new_layout

    def spy_layout(*a, **k):
        lay = new_layout(*a, **k)
        torch.cuda.synchronize()
        carried.append({n: lay.resid_of(p).cpu().clone() for p, n in zip(lay.params, lay.names)})
        return lay
    st._new_layout = spy_layout

    resid = {n: torch.zeros(p.numel()) for n, p in named.items()}
    layouts = []
    try:
        for step in range(STEPS):
            captured.clear()
            n_layouts = len(carried)
            for p in model.parameters():
                p.grad = None
            for j in range(accum):
                x = _inputs(kind, step, j, dtype)
                if j < accum - 1:
                    with ddp.no_sync():
                        ddp(x).float().pow(2).mean().backward()
                else:
                    ddp(x).float().pow(2).mean().backward()
            torch.cuda.synchronize()
            st.check()
            # a new layout starts from the residual its parameters left behind (zero at step 0)
            for c in carried[n_layouts:]:
                for n, r in c.items():
                    assert torch.equal(r, resid[n]), f"step {step}: carried residual of {n}: {first_diff(r, resid[n])}"
            layouts.append(sorted((i, tuple(names)) for i, _, _, names in captured))
            for idx, pre, segs, names in captured:
                lay = st._by_index[idx]
                assert lay.names == names
                params = {n: named[n] for n in names}
                grads = {n: pre[d:d + k].view(named[n].shape) for n, (d, k) in zip(names, segs)}
                flat = ref_flat(lay.plan, params, grads)
                out, new_res, _ = engine_oracle(lay.plan, [flat], [_to_flat(lay.plan, params, resid)],
                                                epoch=lay.engine.epoch)
                want = unflatten(lay.plan, params, out)
                for n in names:
                    p = named[n]
                    if p.grad is None:
                        assert unused and n.startswith("spare"), n
                        continue
                    tag = f"{cfg_name} step {step} {n}"
                    if value_coded:
                        compare_bucket(tag, p.grad.float().cpu(), want[n].float().cpu(), True)
                    else:
                        assert torch.equal(p.grad.cpu(), want[n].cpu()), f"{tag}: {first_diff(p.grad.cpu(), want[n].cpu())}"
                got_res = _from_flat(lay.plan, params, lay.engine.resid.cpu())
                want_res = _from_flat(lay.plan, params, new_res[0])
                for n in names:
                    compare_bucket(f"{cfg_name} step {step} residual {n}", got_res[n], want_res[n], value_coded)
                    # a value-coded step is only close: carry the engine's own residual on (test_train_step_reference)
                    resid[n] = got_res[n] if value_coded else want_res[n]
            if as_view:       # DDP's gradients are views into the buckets the hook wrote
                for n, p in named.items():
                    assert p.grad is None or any(a <= p.grad.data_ptr() < b for a, b in spans), n
            spans.clear()
        assert len(carried) >= 2, "DDP's bucket rebuild was not met"
        assert layouts[1] == layouts[2] == layouts[3]
        assert st.step_count == STEPS
    finally:
        st.close()
    return st


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("kind", ["mlp", "resnet20"])
def test_ddp_hook_vs_oracle(nccl_world1, cfg, kind):
    run_ddp_case(cfg, kind)


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("cfg", ["topk", "bloom_leftmost"])
def test_ddp_hook_bf16_model(nccl_world1, cfg):
    run_ddp_case(cfg, "mlp", dtype=torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ddp_hook_no_sync_accumulation(nccl_world1):
    run_ddp_case("bloom_leftmost", "mlp", accum=2)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ddp_hook_find_unused_parameters(nccl_world1):
    run_ddp_case("bloom_leftmost", "mlp", unused=True)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ddp_hook_gradient_as_bucket_view(nccl_world1):
    run_ddp_case("topk", "resnet20", as_view=True)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ddp_hook_state_dict_into_other_bucket_cap(nccl_world1):
    """Fused checkpoint keyed by parameter name: two steps at one bucket size, resumed at another; the third step's
    gradients and residuals equal those of the run that kept going."""
    from deepreduce_b200.parallel import register_deepreduce_hook
    cfg = CONFIGS["bloom_leftmost"]

    def make(cap):
        m = _model("mlp", torch.float32, False)
        d = DDP(m, device_ids=[0], bucket_cap_mb=cap)
        return m, d, register_deepreduce_hook(d, cfg)

    def step(m, d, s):
        for p in m.parameters():
            p.grad = None
        d(_inputs("mlp", s, 0, torch.float32)).pow(2).mean().backward()
        torch.cuda.synchronize()
        return {n: p.grad.clone() for n, p in m.named_parameters()}

    ma, da, sa = make(0.01)
    mb, db, sb = make(25.0)
    try:
        for s in range(2):
            step(ma, da, s)
        ckpt = sa.state_dict()
        assert set(ckpt["residuals"]) == set(dict(ma.named_parameters()))
        sb.load_state_dict(ckpt)
        # the resumed run's engines are built at its first step; their epoch continues the saved one, so the random
        # policy / random-k draws would also continue
        ga, gb = step(ma, da, 2), step(mb, db, 2)
        for n in ga:
            assert torch.equal(ga[n], gb[n]), f"{n}: {first_diff(ga[n], gb[n])}"
        ra, rb = sa.state_dict()["residuals"], sb.state_dict()["residuals"]
        for n in ra:
            assert torch.equal(ra[n], rb[n]), n
        assert len(sb.engines) < len(sa.engines)
    finally:
        sa.close()
        sb.close()


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_status_checks_name_front_end_and_status(nccl_world1):
    """``check()`` and ``check_async()`` of ``DeepReduceDDP`` and of the hook turn a non-zero engine status word into
    an error with the front end's rank / bucket label and the status name: ``check()`` at once, ``check_async()`` on
    the call after the one that enqueued the copy.  The word is written from the host between steps."""
    from deepreduce_b200.parallel import DeepReduceDDP, register_deepreduce_hook
    cfg = dict(CONFIGS["topk"], calibrate_partition=False)

    def linear():
        torch.manual_seed(0)
        return nn.Linear(64, 64).cuda()

    ours = DeepReduceDDP(linear(), cfg)
    model = linear()
    ddp = DDP(model, device_ids=[0])
    hook = register_deepreduce_hook(ddp, cfg)
    ddp(torch.randn(8, 64, device="cuda")).pow(2).mean().backward()
    torch.cuda.synchronize()
    fronts = ((ours, "[rank 0/1] bucket 0"), (hook, "[rank 0/1] DDP bucket 0"))
    try:
        for st, label in fronts:
            assert len(st.engines) == 1
            st.check()
            st.check_async()
            torch.cuda.synchronize()
            st.engines[0].status.copy_(torch.tensor([2, 7, 0, 0, 0, 0, 0, 0], dtype=torch.int32))
            err = "deepreduce engine error: peer flag watchdog (aux=7)"
            with pytest.raises(RuntimeError, match=re.escape(f"{label} (2 tensors, step {st.step_count}): {err}")):
                st.check()
            st.check_async()                 # reads the clean copy, enqueues the failed word
            torch.cuda.synchronize()
            with pytest.raises(RuntimeError, match=re.escape(f"{label} (step {st.step_count}): {err}")):
                st.check_async()
    finally:
        for e in ours.engines + hook.engines:
            e.status.copy_(torch.zeros(8, dtype=torch.int32))
        hook.close()
        ours.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_ddp_hook_multigpu():
    """W = min(GPUs, 8) ranks, one GPU each: ``tests/run_comm_hook_multigpu.py`` under ``torch.distributed.run``."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    import bench
    W = min(n, 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={W}",
           "--master-addr", "127.0.0.1", "--master-port", str(bench.free_port()),
           os.path.join(ROOT, "tests", "run_comm_hook_multigpu.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=850)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "COMM_HOOK_MULTIGPU_OK" in r.stdout
