"""The training step ``bench.py`` times, against a plain reference step; and the uint8 input kernel against fp64.

Every kernel family has its own test against its own reference.  This file checks what those pieces compute together,
in the configuration the benchmark runs: parameter gradients that are strided views into the flat fp32 buckets,
post-accumulate hooks that launch the exchange during backward (on the launch thread's side stream with a capped grid,
the last bucket inline), the partition calibration at construction, tile-aligned splits of large tensors, real bf16
gradients (massive ties at the top-k threshold, exact zeros, a residual that grows from step 2 on) and the fused
optimizer reading the exchanged views.

The reference step is plain torch plus the CPU oracle of the exchange:

1. the input goes through ``ops.u8_to_nhwc_norm`` (checked against fp64 on its own below);
2. forward / backward of the unfused BatchNorm graph (``DR_FUSED_BN=0``) under bf16 autocast;
3. per bucket, a flat buffer built from the gradients without ``parallel/ddp.py`` (zeros + storage-order gradient at
   the plan's offsets), then ``engine_oracle``, mapped back to per-parameter gradients;
4. ``torch.optim.SGD(fused=True)`` with the benchmark's hyperparameters.

The comparison is ``torch.equal``: loss, every bucket after ``finish()``, every residual, every parameter, momentum
buffer and BatchNorm buffer.  Only the value-coded configuration ('both', polyfit) compares bucket and residual with
the fp32-vs-fp64 tolerances of ``test_gpu_engine._run_vs_oracle``.
"""
import contextlib
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import bench

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the benchmark's optimizer for the image and NCF models, written out rather than read from Trainer
LR, MOMENTUM, WEIGHT_DECAY = 0.05, 0.9, 1e-4
STEPS = 3


# ---------------------------------------------------------------------------
# reference step
# ---------------------------------------------------------------------------
@contextlib.contextmanager
def reproducible_cudnn():
    """``bench.reproducible_cudnn()`` for the duration of a case, restored afterwards."""
    det, bm = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    bench.reproducible_cudnn()
    try:
        yield
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = det, bm


def make_batches(kind, B, hw, gen):
    """Two host batches ((inputs...), target) of the benchmark's types: uint8 NHWC images, or NCF user / item ids."""
    if kind == "image":
        return [((torch.randint(0, 256, (B, hw, hw, 3), dtype=torch.uint8, generator=gen),),
                 torch.randint(0, 1000, (B,), generator=gen)) for _ in range(2)]
    pool, tgt = bench.synth_batches("ncf", B, 0, gen)
    return list(zip(pool, tgt))


def loss_fn(kind):
    return bench.loss_for("ncf") if kind == "ncf" else F.cross_entropy


def ref_backward(model, kind, micro, monkeypatch):
    """Plain torch forward / backward of the unfused graph over the micro-batches of one optimisation step, gradients
    accumulated by autograd from ``p.grad = None``.  Returns the losses (the undivided loss of every micro-batch)."""
    from deepreduce_b200 import ops
    monkeypatch.setenv("DR_FUSED_BN", "0")
    for q in model.parameters():
        q.grad = None
    losses = []
    for xs, y in micro:
        if kind == "image":
            xs = (ops.u8_to_nhwc_norm(xs[0]).permute(0, 3, 1, 2),)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(*xs)
        loss = loss_fn(kind)(out.float(), y)
        (loss / len(micro) if len(micro) > 1 else loss).backward()
        losses.append(loss.detach())
    return losses


def ref_backward_checked(model, kind, micro, monkeypatch):
    """``ref_backward`` run twice on the same weights and batch: the gradients (and losses) must be bit-identical, or
    the reference itself is not a fixed point to compare against.  BatchNorm buffers are restored in between, so they
    move once."""
    buffers = [b.clone() for b in model.buffers()]
    l0 = ref_backward(model, kind, micro, monkeypatch)
    g0 = [q.grad.clone() for q in model.parameters()]
    with torch.no_grad():
        for b, s in zip(model.buffers(), buffers):
            b.copy_(s)
    l1 = ref_backward(model, kind, micro, monkeypatch)
    assert all(torch.equal(a, b) for a, b in zip(l0, l1)), "reference loss is not reproducible"
    for (n, q), g in zip(model.named_parameters(), g0):
        assert torch.equal(q.grad, g), f"reference gradient of {n} is not reproducible"
    return l1


def storage_order(q, g):
    """Gradient ``g`` of parameter ``q`` as a flat vector in the storage order of ``q``'s own dense layout."""
    buf = torch.empty_like(q)
    buf.copy_(g)
    return buf.as_strided((q.numel(),), (1,))


def chunk_offsets(plan, names):
    """(plan tensor, parameter name, element offset inside that parameter) for every tensor of the plan; a split
    parameter enters the plan as chunks ``name#0``, ``name#1``, ... in order."""
    seen, rows = {}, []
    for t in plan.tensors:
        n = t.name if t.name in names else t.name.rsplit("#", 1)[0]
        assert n in names, t.name
        rows.append((t, n, seen.get(n, 0)))
        seen[n] = seen.get(n, 0) + t.numel
    return rows, seen


def ref_flat(plan, params, grads):
    """The bucket the exchange should see, built without ``ddp.py``: zeros + every gradient in its parameter's storage
    order at the plan's offsets (the bucket is zeroed and accumulated into, so ``-0.0`` becomes ``+0.0``)."""
    rows, seen = chunk_offsets(plan, params)
    for n, q in params.items():
        assert seen.get(n) == q.numel(), n
    flat = torch.zeros(plan.total_elems)
    store = {n: storage_order(q, grads[n]).cpu() for n, q in params.items()}
    for t, n, off in rows:
        flat[t.elem_off:t.elem_off + t.numel] += store[n][off:off + t.numel]
    return flat


def unflatten(plan, params, flat):
    """Inverse of ``ref_flat``: per-parameter gradients (in each parameter's own layout) from an exchanged bucket."""
    rows, _ = chunk_offsets(plan, params)
    store = {n: torch.empty(q.numel()) for n, q in params.items()}
    for t, n, off in rows:
        store[n][off:off + t.numel] = flat[t.elem_off:t.elem_off + t.numel]
    out = {}
    for n, q in params.items():
        g = torch.empty_like(q)
        g.as_strided((q.numel(),), (1,)).copy_(store[n].to(q.device))
        out[n] = g
    return out


def first_diff(a, b):
    bad = (a != b) & ~(torch.isnan(a) & torch.isnan(b))
    n = int(bad.sum())
    if n == 0:
        return "equal"
    i = int(bad.flatten().nonzero()[0])
    return f"{n} of {a.numel()} differ, first at {i}: {a.flatten()[i].item()!r} vs {b.flatten()[i].item()!r}"


def compare_bucket(tag, got, want, value_coded):
    if value_coded:       # fp32 Gram sums on the GPU vs fp64 in the oracle (test_gpu_engine._run_vs_oracle)
        scale = float(want.abs().max())
        assert torch.allclose(got, want, atol=2e-3 * scale, rtol=1e-2), f"{tag}: max |diff| {float((got - want).abs().max())}"
    else:
        assert torch.equal(got, want), f"{tag}: {first_diff(got, want)}"


def capture_exchanged(tr):
    """Wrap ``tr.opt.step`` so that every bucket is cloned after ``finish()``, before the optimizer reads it."""
    captured = []
    step = tr.opt.step

    def wrapped(*a, **k):
        captured.append([e.grad.clone() for e in tr.ddp.engines])
        return step(*a, **k)
    tr.opt.step = wrapped
    return captured


def sync_reference(tr, ref, ref_opt):
    """Load the Trainer's parameters, BatchNorm buffers and momentum into the reference (the next step then compares
    like with like even where a value-coded exchange is only close)."""
    with torch.no_grad():
        for p, q in zip(tr.model.parameters(), ref.parameters()):
            q.copy_(p)
            ref_opt.state[q]["momentum_buffer"].copy_(tr.opt.state[p]["momentum_buffer"])
        for a, b in zip(tr.model.buffers(), ref.buffers()):
            b.copy_(a)


def check_after_step(tag, tr, ref, ref_opt):
    for (n, p), q in zip(tr.model.named_parameters(), ref.parameters()):
        assert torch.equal(p, q), f"{tag} parameter {n}: {first_diff(p, q)}"
        mp, mq = tr.opt.state[p]["momentum_buffer"], ref_opt.state[q]["momentum_buffer"]
        assert torch.equal(mp, mq), f"{tag} momentum of {n}: {first_diff(mp, mq)}"
    for (n, a), b in zip(tr.model.named_buffers(), ref.buffers()):
        assert torch.equal(a, b), f"{tag} buffer {n}: {first_diff(a, b)}"


def make_trainer(model, kind, cfg, **kw):
    """``Trainer`` with the arguments ``bench.py --gpus 1`` passes (``kw`` overrides the bucket layout)."""
    from deepreduce_b200.trainer import Trainer
    image = kind == "image"
    args = dict(lr=LR, amp_dtype=torch.bfloat16, channels_last=image, overlap=True, bucket_cap_mb=128.0,
                background_thread=True, u8_input=image, loss_fn=bench.loss_for("ncf") if kind == "ncf" else None,
                overlap_grid=0)
    args.update(kw)
    return Trainer(model, dict(bench.CONFIGS[cfg]), **args)


def build_models(kind):
    from deepreduce_b200 import models
    torch.manual_seed(1234)
    model = (models.resnet50() if kind == "image" else models.NeuMF()).cuda()
    ref = copy.deepcopy(model)
    if kind == "image":
        ref = ref.to(memory_format=torch.channels_last)
    return model, ref


def run_case(monkeypatch, kind, cfg, B, hw=224, accum=1, host=False, check=None, on_flat=None, **tr_kw):
    from deepreduce_b200.parallel import engine_oracle
    value_coded = bench.CONFIGS[cfg].get("deepreduce") in ("value", "both")
    gen = torch.Generator().manual_seed(77)
    batches = make_batches(kind, B, hw, gen)
    dev = [(tuple(x.cuda() for x in xs), y.cuda()) for xs, y in batches]
    pinned = [(tuple(x.pin_memory() for x in xs), y.pin_memory()) for xs, y in batches]
    with reproducible_cudnn():
        model, ref = build_models(kind)
        monkeypatch.setenv("DR_FUSED_BN", "1")
        tr = make_trainer(model, kind, cfg, accum_steps=accum, **tr_kw)
        try:
            if check is not None:
                check(tr)
            ref_named = dict(ref.named_parameters())
            ref_opt = torch.optim.SGD(ref.parameters(), lr=LR, momentum=MOMENTUM, weight_decay=WEIGHT_DECAY, fused=True)
            resid_ref = [torch.zeros(e.plan.total_elems) for e in tr.ddp.engines]
            captured = capture_exchanged(tr)
            for step in range(STEPS):
                tag = f"{cfg} step {step}"
                micro = [dev[(step * accum + j) & 1] for j in range(accum)]
                ref_losses = (ref_backward_checked if step == 0 else ref_backward)(ref, kind, micro, monkeypatch)

                monkeypatch.setenv("DR_FUSED_BN", "1")
                epochs = [e.epoch for e in tr.ddp.engines]
                for j in range(accum):
                    i = step * accum + j
                    if host:
                        loss = tr.step_host(*pinned[i & 1], next_batch=pinned[(i + 1) & 1])
                        assert loss == float(ref_losses[j]), f"{tag}: loss {loss!r} vs {float(ref_losses[j])!r}"
                    else:
                        loss = tr.step(*micro[j][0], target=micro[j][1])
                        assert torch.equal(loss, ref_losses[j]), f"{tag}: loss {loss.item()!r} vs {ref_losses[j].item()!r}"
                    if j < accum - 1:       # accumulation micro-step: no exchange, no optimizer step
                        assert [e.epoch for e in tr.ddp.engines] == epochs and len(captured) == step, tag
                torch.cuda.synchronize()
                tr.ddp.check()
                # the exchange ran exactly once per bucket for this optimisation step
                assert [e.epoch for e in tr.ddp.engines] == [x + 1 for x in epochs], tag
                assert len(captured) == step + 1, tag

                ref_grads = {n: q.grad if q.grad is not None else torch.zeros_like(q) for n, q in ref_named.items()}
                exchanged = {}
                for b, items in enumerate(tr.ddp.buckets):
                    eng = tr.ddp.engines[b]
                    params = {n: ref_named[n] for n, _ in items}
                    flat = ref_flat(eng.plan, params, ref_grads)
                    if on_flat is not None:
                        on_flat(eng.plan, flat)
                    out, new_res, _ = engine_oracle(eng.plan, [flat], [resid_ref[b]], epoch=eng.epoch)
                    got = captured[step][b].cpu()
                    compare_bucket(f"{tag} bucket {b}", got, out, value_coded)
                    compare_bucket(f"{tag} residual {b}", eng.resid.cpu(), new_res[0], value_coded)
                    # a value-coded exchange is only close to the oracle: the reference optimizer then reads the
                    # Trainer's own exchanged bucket, so that parameters and momentum still compare bit for bit
                    exchanged.update(unflatten(eng.plan, params, got if value_coded else out))
                    resid_ref[b] = eng.resid.cpu().clone()
                for n, q in ref_named.items():
                    q.grad = exchanged[n]
                ref_opt.step()
                check_after_step(tag, tr, ref, ref_opt)
                sync_reference(tr, ref, ref_opt)
        finally:
            tr.close()


# ---------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------
def _one_bucket_calibrated(tr):
    assert len(tr.ddp.engines) == 1, len(tr.ddp.engines)
    assert tr.ddp.sched is not None                          # overlap + launch thread on
    assert all(e.cta_speeds is not None for e in tr.ddp.engines), "partition calibration did not run"


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_resnet50_bloom_one_bucket(monkeypatch):
    """Case 1, the headline: one 128 MB bucket, calibrated partition, overlap and launch thread on."""
    run_case(monkeypatch, "image", "bloom", 16, check=_one_bucket_calibrated)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_resnet50_bloom_overlapped_buckets(monkeypatch):
    """Case 2: 16 MB buckets; all but the last launch from the launch thread during backward with a 32-CTA grid."""
    def check(tr):
        assert len(tr.ddp.engines) > 1 and tr.ddp.sched is not None and tr.ddp.overlap_grid_cap == 32
    run_case(monkeypatch, "image", "bloom", 16, bucket_cap_mb=16, overlap_grid=32, check=check)


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("cfg", ["topk", "bloom_p0"])
def test_resnet50_other_index_configs(monkeypatch, cfg):
    """Case 3: plain top-k pairs, and the bloom index with the p0 policy."""
    run_case(monkeypatch, "image", cfg, 16, check=_one_bucket_calibrated)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_resnet50_both_polyfit(monkeypatch):
    """Case 4: bloom index + polyfit values (value-coded: bucket and residual within the fp32-vs-fp64 tolerances)."""
    def check(tr):
        _one_bucket_calibrated(tr)
        assert any(t.vmode == 1 for t in tr.ddp.engines[0].plan.tensors), "no tensor takes the polynomial fit"
    run_case(monkeypatch, "image", "both", 16, check=check)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_resnet50_bloom_accumulated(monkeypatch):
    """Case 5: two micro-steps per exchange; the reference runs two backward passes of loss / 2."""
    run_case(monkeypatch, "image", "bloom", 16, accum=2, check=_one_bucket_calibrated)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_resnet50_bloom_step_host(monkeypatch):
    """Case 6: ``step_host`` with pinned batches, the next one prefetched on the copy stream, two batches alternating."""
    run_case(monkeypatch, "image", "bloom", 16, host=True, check=_one_bucket_calibrated)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_resnet50_bloom_smoke_shape(monkeypatch):
    """Case 7: the ``smoke()`` shape, 64x64 at batch 8 (layer4 is 2x2: BatchNorm reduces 32 rows)."""
    run_case(monkeypatch, "image", "bloom", 8, hw=64, check=_one_bucket_calibrated)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ncf_bloom_split_embeddings(monkeypatch):
    """Case 8: NCF under the bloom index: the embedding tables are split into tile-aligned chunks, and embedding rows
    outside the batch leave chunks with fewer non-zeros than K."""
    def check(tr):
        _one_bucket_calibrated(tr)
        assert any("#" in t.name for t in tr.ddp.engines[0].plan.tensors), "no tensor was split"

    sparse = []

    def on_flat(plan, f):
        sparse.extend(t.name for t in plan.tensors if int(torch.count_nonzero(f[t.elem_off:t.elem_off + t.numel])) < t.k)
    run_case(monkeypatch, "ncf", "bloom", 1024, check=check, on_flat=on_flat)
    assert sparse, "no tensor had fewer non-zeros than K"


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ncf_rle(monkeypatch):
    """Case 9: NCF, top-k 0.1 % + run-length index (BASELINE config 4)."""
    from deepreduce_b200.parallel.plan import MODE_RLE

    def check(tr):
        _one_bucket_calibrated(tr)
        assert any(t.mode == MODE_RLE for t in tr.ddp.engines[0].plan.tensors)
    run_case(monkeypatch, "ncf", "rle", 4096, check=check)


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_train_step_multigpu():
    """Case 1 at W = min(GPUs, 8) with the benchmark's N > 1 layout (one bucket, launched after backward), a batch
    per rank: ``tests/run_train_step_multigpu.py`` under ``torch.distributed.run``."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    W = min(n, 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={W}",
           "--master-addr", "127.0.0.1", "--master-port", str(bench.free_port()),
           os.path.join(ROOT, "tests", "run_train_step_multigpu.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1100)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "TRAIN_STEP_MULTIGPU_OK" in r.stdout


# ---------------------------------------------------------------------------
# B. u8_to_nhwc_norm against fp64
# ---------------------------------------------------------------------------
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
# every mean sits halfway between two multiples of 1/255, so |b/255 - mean| >= 1/510: no cancellation to zero, and
# the fp32 evaluation (contracted to an FMA or not) rounds to the same bf16 as fp64 for all 768 inputs
CUSTOM_MEAN, CUSTOM_STD = (0.1, 0.7, 0.9), (0.01, 3.0, 0.2)


def fp64_table(mean, std):
    """[3, 256] fp64 value of every (channel, byte) and its bf16 rounding: ``(b / 255 - mean) / std``."""
    b = torch.arange(256, dtype=torch.float64)
    v = torch.stack([(b / 255 - m) / s for m, s in zip(mean, std)])
    return v, v.to(torch.bfloat16)


def all_bytes_image():
    """One 16x16 image holding every byte 0..255 in each of the 3 channels (a different pixel order per channel)."""
    b = torch.arange(256, dtype=torch.uint8)
    return torch.stack([b, b.flip(0), b.roll(85)], dim=-1).view(1, 16, 16, 3)


def expected(x, table):
    """The fp64 table looked up for an NHWC uint8 batch (on x's device)."""
    t = table.to(x.device)
    return torch.stack([t[c][x[..., c].long()] for c in range(3)], dim=-1)


def near_midpoint(v):
    """True where fp64 ``v`` lies within 2^-20 (relative) of a midpoint between two neighbouring bf16 values."""
    a = v.abs()
    _, e = torch.frexp(a)                               # a = m * 2^e, m in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(a), e - 8)        # bf16 keeps 8 significant bits
    f = a / ulp
    return ((f - f.floor() - 0.5).abs() * ulp) <= a * 2.0 ** -20


def bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.gpu
def test_u8_norm_all_bytes_exact():
    from deepreduce_b200 import ops
    x = all_bytes_image()
    _, want = fp64_table(MEAN, STD)
    got = ops.u8_to_nhwc_norm(x.cuda()).cpu()
    assert got.dtype == torch.bfloat16 and got.shape == x.shape
    assert torch.equal(bits(got), bits(expected(x, want))), first_diff(bits(got), bits(expected(x, want)))


@pytest.mark.gpu
def test_u8_norm_all_bytes_custom_mean_std():
    """Another mean / std: at most one bf16 ulp apart, and only where the fp64 value is within 2^-20 of a rounding
    midpoint (where fp32 evaluation may round either way)."""
    from deepreduce_b200 import ops
    x = all_bytes_image()
    v, want = fp64_table(CUSTOM_MEAN, CUSTOM_STD)
    got = ops.u8_to_nhwc_norm(x.cuda(), CUSTOM_MEAN, CUSTOM_STD).cpu()
    g, w = bits(got).int(), bits(expected(x, want)).int()
    ulps = (g - w).abs()
    assert int(ulps.max()) <= 1, int(ulps.max())
    ok = (ulps == 0) | near_midpoint(expected(x, v))
    assert bool(ok.all()), f"{int((~ok).sum())} values off by one ulp away from a rounding midpoint"


# pixel counts = 0, 1, 2, 3 (mod 4): the 4-pixel loop, its tail, and the tail alone (1, 2 and 3 pixels in all);
# 256 x 224 x 224 is the benchmark's batch and exceeds one pass of the capped grid (16 CTAs / SM x 256 threads x 4 px)
SHAPES = [(1, 1, 1), (1, 1, 2), (1, 1, 3), (1, 2, 2), (1, 3, 3), (2, 5, 5), (3, 7, 7), (5, 33, 31), (256, 224, 224)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w", SHAPES)
def test_u8_norm_shapes(n, h, w):
    from deepreduce_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n * 1000 + h * 10 + w)
    x = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
    _, want = fp64_table(MEAN, STD)
    one_pass = 16 * torch.cuda.get_device_properties(0).multi_processor_count * 256 * 4
    assert (n * h * w > one_pass) == (n == 256)        # only the benchmark batch makes the grid-stride loop wrap
    got = ops.u8_to_nhwc_norm(x)
    assert torch.equal(bits(got), bits(expected(x, want)))


@pytest.mark.gpu
@pytest.mark.parametrize("start", [1, 2, 3])
def test_u8_norm_misaligned_batch_slice(start):
    """A batch slice of images with an odd byte count (5 x 5 x 3 = 75 B) starts off a 4-byte boundary; the kernel
    reads 32-bit words, so the binding hands it an aligned copy."""
    from deepreduce_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(start)
    base = torch.randint(0, 256, (8, 5, 5, 3), dtype=torch.uint8, device="cuda", generator=g)
    x = base[start:]
    assert x.data_ptr() % 4 != 0 and x.is_contiguous()
    _, want = fp64_table(MEAN, STD)
    got = ops.u8_to_nhwc_norm(x)
    assert torch.equal(bits(got), bits(expected(x, want)))
    torch.cuda.synchronize()
