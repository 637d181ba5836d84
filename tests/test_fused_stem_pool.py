"""The fused stem, maxpool(relu(bn(x))) with a one-byte winner code per pooled element (ops/csrc/bn.cu:
bn_apply_pool_kernel, and mode 3 of the backward kernels), against the unfused graph (native BN -> relu_ ->
max_pool2d_with_indices and its backward), bit for bit.

Covered: the real stem shape at batch 256; odd and even H and W, where the bottom and right windows clip; windows full
of ties after the ReLU; inputs that win two or four overlapping windows (their gradient is an fp32 sum rounded once);
NaN and +-inf in x; NaN, +-inf and -0.0 in the pooled gradient at masked and unmasked winners.
"""
import pytest
import torch
import torch.nn as nn

from deepreduce_b200.models import fused_bn

# (n, c, h, w)
SMALL = [(2, 64, 15, 15), (1, 64, 16, 17), (3, 128, 7, 7), (2, 64, 14, 14)]
KINDS = ["random", "ties", "multi_win", "x_special", "g_special"]


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm2d(c)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.2)
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn.cuda().train()


def _input(n, c, h, w, kind, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, h, w, c, device="cuda", generator=g) * 1.7 + 0.3          # NHWC storage
    if kind == "ties":
        # 90 % zeros, which BN maps below 0, and three positive levels: many windows are all +0 after the ReLU, and
        # the rest tie often
        lvl = torch.randint(1, 4, (n, h, w, c), device="cuda", generator=g).float() * 0.75
        x = torch.where(torch.rand(n, h, w, c, device="cuda", generator=g) < 0.1, lvl, torch.zeros_like(lvl))
    elif kind == "multi_win":
        # spikes at odd (h, w) win the four windows that overlap there; at odd h, even w the two windows above/below
        x[:, 1::4, 1::4, :] += 20.0
        x[:, 3::4, 2::4, :] += 20.0
    elif kind == "x_special":
        x[0, 1, 2, 3] = float("nan")
        x[-1, h - 1, w - 1, 9] = float("inf")
        x[0, h // 2, 0, 17] = float("-inf")
    return x.to(torch.bfloat16).permute(0, 3, 1, 2)                           # channels_last NCHW view


def _grad(out, kind, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, c, ho, wo = out.shape
    gy = (torch.randn(n, ho, wo, c, device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
    if kind == "g_special":
        flat, o = gy.reshape(-1), out.permute(0, 2, 3, 1).reshape(-1)
        specials = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0], device="cuda", dtype=torch.bfloat16)
        for where in (o == 0, o != 0):          # masked and unmasked winners
            idx = where.nonzero().flatten()
            assert idx.numel() >= 16
            pick = idx[torch.randperm(idx.numel(), device="cuda", generator=g)[:max(16, idx.numel() // 4)]]
            flat[pick] = specials.repeat(pick.numel() // 4 + 1)[:pick.numel()]
    return gy.permute(0, 3, 1, 2)


def _run(monkeypatch, fused, shape, kind):
    monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
    n, c, h, w = shape
    bn, pool = _bn(c, 1), nn.MaxPool2d(3, 2, 1)
    x = _input(n, c, h, w, kind, 2).requires_grad_()
    assert fused_bn.eligible(x, bn) == fused
    saved = {}
    if fused:
        stats = fused_bn._stats

        def record(x_, bn_):
            saved["save_mean"], saved["save_invstd"] = stats(x_, bn_)
            return saved["save_mean"], saved["save_invstd"]
        monkeypatch.setattr(fused_bn, "_stats", record)
    else:
        _, saved["save_mean"], saved["save_invstd"] = torch.native_batch_norm(
            x.detach(), bn.weight, bn.bias, bn.running_mean.clone(), bn.running_var.clone(), True, bn.momentum, bn.eps)
    out = fused_bn.bn_relu_maxpool(x, bn, pool)
    out.backward(_grad(out.detach(), kind, 3))
    torch.cuda.synchronize()
    monkeypatch.undo()
    return {"out": out.detach(), "dx": x.grad, "dw": bn.weight.grad, "db": bn.bias.grad,
            "running_mean": bn.running_mean, "running_var": bn.running_var, **saved}


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _compare(monkeypatch, shape, kind):
    ref = _run(monkeypatch, False, shape, kind)
    new = _run(monkeypatch, True, shape, kind)
    assert ref.keys() == new.keys()
    for k in ref:
        a, b = ref[k], new[k]
        assert a.dtype == b.dtype and a.shape == b.shape, k
        diff = (_bits(a) != _bits(b)).sum().item()
        assert diff == 0, f"{kind} {shape} {k}: {diff} entries differ in their bits"
    return ref


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", SMALL, ids=lambda s: "x".join(map(str, s)))
def test_stem_pool_bits(monkeypatch, shape, kind):
    ref = _compare(monkeypatch, shape, kind)
    if kind == "ties":
        assert (ref["out"] == 0).float().mean() > 0.2
    if kind == "g_special":
        assert ref["dx"].isnan().any()


@pytest.mark.gpu
def test_stem_pool_bits_resnet50_shape(monkeypatch):
    _compare(monkeypatch, (256, 64, 112, 112), "random")


@pytest.mark.gpu
def test_bn_apply_pool_rejects_other_pools():
    from deepreduce_b200 import ops
    mod = ops.cuda_module()
    x = torch.randn(2, 64, 8, 8, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    p = [torch.zeros(64, device="cuda"), torch.ones(64, device="cuda"), torch.ones(64, device="cuda"),
         torch.zeros(64, device="cuda")]
    out, codes = mod.bn_apply_pool(x, p)
    assert out.shape == (2, 64, 4, 4) and codes.shape == (2 * 4 * 4, 64) and codes.dtype == torch.uint8
    for kw in ({"kernel_size": 2}, {"stride": 1}, {"padding": 0}, {"dilation": 2}, {"ceil_mode": True}):
        with pytest.raises(RuntimeError, match="bn_apply_pool"):
            mod.bn_apply_pool(x, p, **kw)


@pytest.mark.parametrize("pool", [nn.MaxPool2d(3, 2, 1), nn.MaxPool2d(2, 2), nn.MaxPool2d(3, 2, 1, ceil_mode=True)])
def test_bn_relu_maxpool_falls_back(pool):
    # on the CPU, and for any other pool, the module composite runs unchanged
    torch.manual_seed(0)
    bn = nn.BatchNorm2d(16).train()
    x = torch.randn(2, 16, 9, 9)
    ref_bn = nn.BatchNorm2d(16).train()
    ref = pool(torch.relu(ref_bn(x)))
    out = fused_bn.bn_relu_maxpool(x, bn, pool)
    assert torch.equal(out, ref)
    assert torch.equal(bn.running_mean, ref_bn.running_mean) and torch.equal(bn.running_var, ref_bn.running_var)
    assert not fused_bn._stem_pool(nn.MaxPool2d(3, 2, 1, return_indices=True))
    assert fused_bn._stem_pool(nn.MaxPool2d(3, 2, 1)) and fused_bn._stem_pool(nn.MaxPool2d((3, 3), (2, 2), (1, 1)))
