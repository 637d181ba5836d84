"""The fused BatchNorm backward (ReLU mask + torch's reduction tree, ops/csrc/bn.cu) against the unfused graph, bit for
bit, where tests/test_fused_bn.py does not look: small row counts, whose reduction tree has 4, 8 or 16 threads per
column and a single block, and output gradients holding NaN, +-inf and -0.0 at masked and unmasked positions.

Bit patterns are compared (int16 / int32 views), so NaN results must match too: a NaN gradient where the ReLU output
is 0 must give +0, as threshold_backward does.
"""
import pytest
import torch
import torch.nn as nn

from deepreduce_b200.models import fused_bn

# (n, channels, H = W): rows = n * H * W = 98, 196 and 1568 give torch's channels-last backward reduce
# block_y = 4, 8 and 16, each with grid_y = 1
SMALL = [(2, 512, 7), (1, 256, 14), (2, 128, 28)]
KINDS = ["relu", "add", "bnadd"]


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm2d(c)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.2)
    return bn.cuda().train()


def _act(n, c, hw, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, hw, hw, c, device="cuda", generator=g) * 1.7 + 0.3
    return x.to(torch.bfloat16).permute(0, 3, 1, 2)      # channels_last NCHW view


def _special_grad(out, seed):
    """A random gradient with NaN, +inf, -inf and -0.0 placed both where out == 0 (masked) and where out > 0."""
    gy = _act(*out.shape[:2], out.shape[2], seed).clone(memory_format=torch.channels_last)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    flat = gy.permute(0, 2, 3, 1).reshape(-1)            # NHWC storage order
    zero = (out.permute(0, 2, 3, 1).reshape(-1) == 0)
    specials = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0], device="cuda", dtype=torch.bfloat16)
    for where in (zero, ~zero):
        idx = where.nonzero().flatten()
        assert idx.numel() >= 64
        pick = idx[torch.randperm(idx.numel(), device="cuda", generator=g)[:4 * 16]]
        flat[pick] = specials.repeat(16)
    return gy


def _run(monkeypatch, fused, kind, n, c, hw, special):
    monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
    bn, bnd = _bn(c, 1), _bn(c, 2)
    x, z = _act(n, c, hw, 3).requires_grad_(), _act(n, c, hw, 4).requires_grad_()
    assert fused_bn.eligible(x, bn) == fused
    if kind == "relu":
        out = fused_bn.bn_relu(x, bn)
    elif kind == "add":
        out = fused_bn.bn_add_relu(x, bn, z)
    else:
        out = fused_bn.bn_bn_add_relu(x, bn, z, bnd)
    gy = _special_grad(out.detach(), 5) if special else _act(n, c, hw, 5)
    out.backward(gy)
    torch.cuda.synchronize()
    res = {"out": out.detach(), "dx": x.grad, "dz": z.grad, "dw": bn.weight.grad, "db": bn.bias.grad,
           "dw_z": bnd.weight.grad, "db_z": bnd.bias.grad}
    return {k: v for k, v in res.items() if v is not None}


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("special", [False, True], ids=["finite", "nan_inf_negzero"])
@pytest.mark.parametrize("n,c,hw", SMALL)
@pytest.mark.parametrize("kind", KINDS)
def test_fused_bn_backward_bits(monkeypatch, kind, n, c, hw, special):
    ref = _run(monkeypatch, False, kind, n, c, hw, special)
    new = _run(monkeypatch, True, kind, n, c, hw, special)
    assert ref.keys() == new.keys()
    for k in ref:
        a, b = ref[k], new[k]
        assert a.dtype == b.dtype and a.shape == b.shape, k
        diff = (_bits(a) != _bits(b)).sum().item()
        assert diff == 0, f"{kind} {n}x{c}x{hw}x{hw} {k}: {diff} entries differ in their bits"
    if kind == "add":
        # the gradient of the identity skip is threshold_backward's: +0 (bits 0) wherever the output is 0
        assert (_bits(new["dz"])[new["out"] == 0] == 0).all()
