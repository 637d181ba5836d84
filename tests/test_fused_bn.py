"""Fused BatchNorm (+ ReLU, + residual add) of models/fused_bn.py against the unfused graph it replaces.

The acceptance bar is bitwise equality (torch.equal), not a tolerance: outputs, saved statistics, running statistics and
every gradient, at every distinct BN shape of ResNet-50 at batch 256 and at a small batch, and for a whole ResNet-50
training step.
"""
import copy

import pytest
import torch
import torch.nn as nn

from deepreduce_b200.models import fused_bn
from deepreduce_b200.models.resnet import _Bottleneck, resnet50

# (channels, H = W) of the BN inputs of ResNet-50 at 224^2
RELU_SHAPES = [(64, 112), (64, 56), (128, 56), (128, 28), (256, 28), (256, 14), (512, 14), (512, 7)]
TAIL_SHAPES = [(256, 56), (512, 28), (1024, 14), (2048, 7)]


def test_cpu_runs_the_unfused_graph():
    torch.manual_seed(0)
    blk = _Bottleneck(16, 8, 2, downsample=True).train()
    ref = copy.deepcopy(blk)
    x = torch.randn(2, 16, 8, 8)
    assert not fused_bn.eligible(x, blk.bn1)
    out = blk(x)
    idt = ref.downsample(x)
    y = torch.relu(ref.bn1(ref.conv1(x)))
    y = torch.relu(ref.bn2(ref.conv2(y)))
    assert torch.equal(out, torch.relu(ref.bn3(ref.conv3(y)) + idt))
    for a, b in zip(blk.buffers(), ref.buffers()):
        assert torch.equal(a, b)


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm2d(c)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.2)
        bn.running_mean.copy_(torch.randn(c, generator=g))
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn.cuda().train()


def _act(n, c, hw, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, hw, hw, c, device="cuda", generator=g) * 1.7 + 0.3
    return x.to(torch.bfloat16).permute(0, 3, 1, 2).requires_grad_()      # channels_last NCHW view


def _run(monkeypatch, fused, kind, n, c, hw):
    monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
    bn, bnd = _bn(c, 1), _bn(c, 2)
    x, z = _act(n, c, hw, 3), _act(n, c, hw, 4)
    assert fused_bn.eligible(x, bn) == fused
    if kind == "relu":
        out = fused_bn.bn_relu(x, bn)
    elif kind == "add":
        out = fused_bn.bn_add_relu(x, bn, z)
    else:
        out = fused_bn.bn_bn_add_relu(x, bn, z, bnd)
    gy = _act(n, c, hw, 5).detach()
    out.backward(gy)
    res = {"out": out.detach(), "dx": x.grad, "dz": z.grad}
    for name, m in (("bn", bn), ("bnd", bnd)):
        res.update({f"{name}.{k}": v for k, v in m.state_dict().items()})
        res[f"{name}.dw"], res[f"{name}.db"] = m.weight.grad, m.bias.grad
    torch.cuda.synchronize()
    return res


def _assert_same(a, b):
    for k in a:
        if a[k] is None:
            assert b[k] is None, k
            continue
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert torch.equal(a[k], b[k]), f"{k}: {(a[k].float() != b[k].float()).sum().item()} entries differ"


CASES = ([("relu", 256, c, hw) for c, hw in RELU_SHAPES] + [(k, 256, c, hw) for k in ("add", "bnadd") for c, hw in TAIL_SHAPES]
         + [("relu", 2, 64, 56), ("add", 2, 256, 56), ("bnadd", 3, 512, 7)])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,c,hw", CASES)
def test_fused_bn_is_bitwise_unfused(monkeypatch, kind, n, c, hw):
    ref = _run(monkeypatch, False, kind, n, c, hw)
    new = _run(monkeypatch, True, kind, n, c, hw)
    _assert_same(ref, new)


@pytest.mark.gpu
@pytest.mark.parametrize("c,hw", [(64, 112), (2048, 7)])
def test_saved_stats_are_native_batch_norm(c, hw):
    from deepreduce_b200 import ops
    bn = _bn(c, 1)
    x = _act(256, c, hw, 3).detach()
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    _, save_mean, save_invstd = torch.ops.aten.native_batch_norm(x, bn.weight, bn.bias, rm, rv, True, 0.1, 1e-5)
    mean, invstd = ops.cuda_module().bn_stats(x, bn.running_mean, bn.running_var, 0.1, 1e-5)
    assert torch.equal(mean, save_mean) and torch.equal(invstd, save_invstd)
    assert torch.equal(bn.running_mean, rm) and torch.equal(bn.running_var, rv)


def _train_step(monkeypatch, fused, batch):
    monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
    torch.manual_seed(1234)
    model = resnet50().cuda().to(memory_format=torch.channels_last).train()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(batch, 3, 224, 224, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device="cuda", generator=g)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = model(x)
    loss = torch.nn.functional.cross_entropy(out.float(), y)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), model


@pytest.mark.gpu
def test_resnet50_step_is_bitwise_unfused(monkeypatch):
    det, bench = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        l0, m0 = _train_step(monkeypatch, False, 32)
        l1, m1 = _train_step(monkeypatch, True, 32)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = det, bench
    assert torch.equal(l0, l1)
    for (name, p0), p1 in zip(m0.named_parameters(), m1.parameters()):
        assert torch.equal(p0.grad, p1.grad), name
    for (name, b0), b1 in zip(m0.named_buffers(), m1.buffers()):
        assert torch.equal(b0, b1), name
