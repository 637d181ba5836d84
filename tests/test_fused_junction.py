"""Block inputs with two consumers: a forked producer (``fork=True`` of bn_add_relu, bn_bn_add_relu, bn_relu_maxpool)
returns its output twice, and bn_backward adds the two gradients as it loads them (``go2``).  The reference is the
unfused graph with autograd's own accumulation: ``torch.autograd.backward([o, o], [ga, gb])``.  Bit patterns are
compared for the output, every gradient and the saved and running statistics.

Covered: every junction shape of ResNet-50 at batch 256 (tails at C = 256, 512, 1024, 2048 and the stem); small and odd
batches whose reduction tree has block_y 4, 8, 16 and grid_y > 1; gradient pairs whose bf16 sum rounds to even, signed
zeros, inf + -inf, NaN on either side and finite sums that overflow, at masked and unmasked positions; only one of the
two outputs used, in both orders; stem inputs that win two or four windows.
"""
import pytest
import torch
import torch.nn as nn

from deepreduce_b200.models import fused_bn, resnet50
from deepreduce_b200.models.resnet import _Bottleneck

# (n, C, H = W): rows 98, 196, 1568 give block_y 4, 8, 16 with one block; 6272 gives block_y 16, grid_y 25
TAILS_SMALL = [(2, 512, 7), (1, 256, 14), (2, 256, 28), (8, 256, 28)]
TAILS_R50 = [(256, 256, 56), (256, 512, 28), (256, 1024, 14), (256, 2048, 7)]
STEM_SMALL = [(2, 64, 15), (3, 64, 14), (8, 64, 30)]
STEM_R50 = (256, 64, 112)
USES = ["both", "first", "second"]

# (a, b) pairs whose bf16 sum is an edge case: ties that round to even (1 + 2^-8 halfway, either way), signed zeros,
# inf + -inf, NaN on either side, finite sums past the bf16 maximum
_PAIRS = [(1.0, 2.0 ** -8), (1.0 + 2.0 ** -7, 2.0 ** -8), (-0.0, -0.0), (0.0, -0.0), (-0.0, 0.0),
          (float("inf"), float("-inf")), (float("nan"), 1.0), (1.0, float("nan")), (3.0e38, 3.0e38),
          (-3.0e38, -3.0e38)]


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm2d(c)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.2)
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn.cuda().train()


def _act(n, c, hw, seed, multi_win=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, hw, hw, c, device="cuda", generator=g) * 1.7 + 0.3          # NHWC storage
    if multi_win:
        # spikes at odd (h, w) win the four pool windows that overlap there; at odd h, even w the two above / below
        x[:, 1::4, 1::4, :] += 20.0
        x[:, 3::4, 2::4, :] += 20.0
    return x.to(torch.bfloat16).permute(0, 3, 1, 2)                               # channels_last NCHW view


def _grads(out, seed, special):
    """Two gradients of out's shape; with ``special``, _PAIRS placed where out == 0 (masked) and where out != 0."""
    n, c, h, w = out.shape
    ga, gb = _act(n, c, h, seed), _act(n, c, h, seed + 1)
    ga, gb = ga.clone(memory_format=torch.channels_last), gb.clone(memory_format=torch.channels_last)
    if special:
        g = torch.Generator(device="cuda").manual_seed(seed + 2)
        fa, fb = ga.permute(0, 2, 3, 1).reshape(-1), gb.permute(0, 2, 3, 1).reshape(-1)     # NHWC storage order
        zero = out.permute(0, 2, 3, 1).reshape(-1) == 0
        pa = torch.tensor([a for a, _ in _PAIRS], device="cuda").to(torch.bfloat16)
        pb = torch.tensor([b for _, b in _PAIRS], device="cuda").to(torch.bfloat16)
        reps = 8
        for where in (zero, ~zero):
            # a stem whose every window holds a spike (multi_win) has no masked winner
            idx = where.nonzero().flatten()
            k = min(reps * len(_PAIRS), idx.numel())
            pick = idx[torch.randperm(idx.numel(), device="cuda", generator=g)[:k]]
            fa[pick], fb[pick] = pa.repeat(reps)[:k], pb.repeat(reps)[:k]
        assert (~zero).sum() >= reps * len(_PAIRS)
    return ga, gb


def _backward(fused, outs, ga, gb, use):
    # fused: the two outputs of the forked producer; unfused: the one output, whose gradients autograd sums
    o1, o2 = outs if fused else (outs, outs)
    if use == "both":
        torch.autograd.backward([o1, o2], [ga, gb])
    elif use == "first":
        torch.autograd.backward([o1], [ga])
    else:
        torch.autograd.backward([o2], [gb])


def _record_stats(monkeypatch, saved):
    stats = fused_bn._stats

    def record(x_, bn_):
        i = len(saved) // 2
        saved[f"save_mean{i}"], saved[f"save_invstd{i}"] = stats(x_, bn_)
        return saved[f"save_mean{i}"], saved[f"save_invstd{i}"]
    monkeypatch.setattr(fused_bn, "_stats", record)


def _run_tail(monkeypatch, fused, kind, n, c, hw, special, use):
    monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
    bn, bnd = _bn(c, 1), _bn(c, 2)
    x, z = _act(n, c, hw, 3).requires_grad_(), _act(n, c, hw, 4).requires_grad_()
    assert fused_bn.eligible(x, bn) == fused
    saved = {}
    if fused:
        _record_stats(monkeypatch, saved)
    else:
        # the unfused graph's saved statistics, in the fused path's order (downsample BN first)
        for i, (t, b) in enumerate([(z, bnd), (x, bn)] if kind == "bnadd" else [(x, bn)]):
            _, saved[f"save_mean{i}"], saved[f"save_invstd{i}"] = torch.native_batch_norm(
                t.detach(), b.weight, b.bias, b.running_mean.clone(), b.running_var.clone(), True, b.momentum, b.eps)
    if kind == "add":
        outs = fused_bn.bn_add_relu(x, bn, z, fork=fused)
    else:
        outs = fused_bn.bn_bn_add_relu(x, bn, z, bnd, fork=fused)
    out = (outs[0] if fused else outs).detach()
    ga, gb = _grads(out, 5, special)
    _backward(fused, outs, ga, gb, use)
    torch.cuda.synchronize()
    monkeypatch.undo()
    res = {"out": out, "dx": x.grad, "dz": z.grad, "dw": bn.weight.grad, "db": bn.bias.grad,
           "dw_z": bnd.weight.grad, "db_z": bnd.bias.grad, "running_mean": bn.running_mean,
           "running_var": bn.running_var, **saved}
    if kind == "bnadd":
        res.update(running_mean_z=bnd.running_mean, running_var_z=bnd.running_var)
    return {k: v for k, v in res.items() if v is not None}


def _run_stem(monkeypatch, fused, n, c, hw, special, use, multi_win):
    monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
    bn, pool = _bn(c, 1), nn.MaxPool2d(3, 2, 1)
    if special:
        with torch.no_grad():
            bn.bias -= 1.0          # many windows all <= 0, so that the edge pairs also land on masked winners
    x = _act(n, c, hw, 2, multi_win).requires_grad_()
    assert fused_bn.eligible(x, bn) == fused
    saved = {}
    if fused:
        _record_stats(monkeypatch, saved)
    else:
        _, saved["save_mean0"], saved["save_invstd0"] = torch.native_batch_norm(
            x.detach(), bn.weight, bn.bias, bn.running_mean.clone(), bn.running_var.clone(), True, bn.momentum, bn.eps)
    outs = fused_bn.bn_relu_maxpool(x, bn, pool, fork=fused)
    out = (outs[0] if fused else outs).detach()
    ga, gb = _grads(out, 7, special)
    _backward(fused, outs, ga, gb, use)
    torch.cuda.synchronize()
    monkeypatch.undo()
    return {"out": out, "dx": x.grad, "dw": bn.weight.grad, "db": bn.bias.grad, "running_mean": bn.running_mean,
            "running_var": bn.running_var, **saved}


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _compare(ref, new, what):
    assert ref.keys() == new.keys(), what
    for k in ref:
        a, b = ref[k], new[k]
        assert a.dtype == b.dtype and a.shape == b.shape, (what, k)
        diff = (_bits(a) != _bits(b)).sum().item()
        assert diff == 0, f"{what} {k}: {diff} entries differ in their bits"


@pytest.mark.gpu
@pytest.mark.parametrize("use", USES)
@pytest.mark.parametrize("special", [False, True], ids=["finite", "edge_pairs"])
@pytest.mark.parametrize("n,c,hw", TAILS_SMALL)
@pytest.mark.parametrize("kind", ["add", "bnadd"])
def test_forked_tail_bits(monkeypatch, kind, n, c, hw, special, use):
    ref = _run_tail(monkeypatch, False, kind, n, c, hw, special, use)
    new = _run_tail(monkeypatch, True, kind, n, c, hw, special, use)
    _compare(ref, new, f"{kind} {n}x{c}x{hw}x{hw} {use}")
    if special and use == "both":
        assert ref["dx"].isnan().any()


@pytest.mark.gpu
@pytest.mark.parametrize("n,c,hw", TAILS_R50, ids=lambda v: str(v))
@pytest.mark.parametrize("kind", ["add", "bnadd"])
def test_forked_tail_bits_resnet50_shapes(monkeypatch, kind, n, c, hw):
    ref = _run_tail(monkeypatch, False, kind, n, c, hw, False, "both")
    new = _run_tail(monkeypatch, True, kind, n, c, hw, False, "both")
    _compare(ref, new, f"{kind} {n}x{c}x{hw}x{hw}")


@pytest.mark.gpu
@pytest.mark.parametrize("use", USES)
@pytest.mark.parametrize("special", [False, True], ids=["finite", "edge_pairs"])
@pytest.mark.parametrize("multi_win", [False, True], ids=["random", "multi_win"])
@pytest.mark.parametrize("n,c,hw", STEM_SMALL)
def test_forked_stem_bits(monkeypatch, n, c, hw, multi_win, special, use):
    ref = _run_stem(monkeypatch, False, n, c, hw, special, use, multi_win)
    new = _run_stem(monkeypatch, True, n, c, hw, special, use, multi_win)
    _compare(ref, new, f"stem {n}x{c}x{hw}x{hw} {use}")


@pytest.mark.gpu
def test_forked_stem_bits_resnet50_shape(monkeypatch):
    n, c, hw = STEM_R50
    ref = _run_stem(monkeypatch, False, n, c, hw, False, "both", False)
    new = _run_stem(monkeypatch, True, n, c, hw, False, "both", False)
    _compare(ref, new, "stem")


@pytest.mark.gpu
def test_junction_runs_no_add_kernel():
    # the backward of a block pair: the junction between them (an identity tail's output, 256 x 56 x 56 at batch 32,
    # as layer1.1's) is summed inside bn.cu, so no elementwise add kernel runs
    from torch.profiler import ProfilerActivity, profile
    torch.manual_seed(0)
    blk0 = _Bottleneck(256, 64, 1, downsample=False).cuda().to(memory_format=torch.channels_last).train()
    blk1 = _Bottleneck(256, 64, 1, downsample=False).cuda().to(memory_format=torch.channels_last).train()
    x = _act(32, 256, 56, 1)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        h, skip = blk0(x, fork=True)
        out = blk1(h, skip)
    g = torch.ones_like(out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out.backward(g)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("bn_bwd_reduce_kernel" in k for k in names)
    adds = [k for k in names if any(s in k for s in ("AddFunctor", "CUDAFunctor_add", "add_kernel"))]
    assert not adds, adds


def test_forked_helpers_fall_back_to_a_pair():
    # on the CPU the composites run, and fork=True returns the one output twice
    torch.manual_seed(0)
    x, z = torch.randn(2, 16, 5, 5), torch.randn(2, 16, 5, 5)
    bn, bnd = nn.BatchNorm2d(16).train(), nn.BatchNorm2d(16).train()
    for outs in (fused_bn.bn_add_relu(x, bn, z, fork=True), fused_bn.bn_bn_add_relu(x, bn, z, bnd, fork=True),
                 fused_bn.bn_relu_maxpool(x, bn, nn.MaxPool2d(3, 2, 1), fork=True)):
        assert isinstance(outs, tuple) and len(outs) == 2 and outs[0] is outs[1]
    assert torch.is_tensor(fused_bn.bn_add_relu(x, bn, z))


def test_bottleneck_fork_matches_single_output():
    # an identity tail forks (here the CPU composite: one tensor twice); a downsample tail returns (output, None)
    torch.manual_seed(0)
    for blk, inp in ((_Bottleneck(64, 16, 1, downsample=False).train(), 64),
                     (_Bottleneck(64, 16, 2, downsample=True).train(), 64)):
        x = torch.randn(2, inp, 6, 6)
        one = blk(x)
        pair = blk(x, x, fork=True)
        assert torch.is_tensor(one) and len(pair) == 2 and torch.equal(pair[0], one)
        assert pair[1] is (pair[0] if blk.downsample is None else None)


def test_resnet50_state_dict_keys_unchanged():
    bn_keys = ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")
    want = ["conv1.weight"] + [f"bn1.{k}" for k in bn_keys]
    i = 0
    for n in (3, 4, 6, 3):
        for j in range(n):
            for k in (1, 2, 3):
                want += [f"layers.{i}.conv{k}.weight"] + [f"layers.{i}.bn{k}.{b}" for b in bn_keys]
            if j == 0:
                want += [f"layers.{i}.downsample.0.weight"] + [f"layers.{i}.downsample.1.{b}" for b in bn_keys]
            i += 1
    want += ["fc.weight", "fc.bias"]
    assert list(resnet50().state_dict().keys()) == want
