"""Training BatchNorm fused with the ReLU and the residual add of ResNet-50, on channels_last bf16 activations.

Forward runs the sm_90a kernels of ``ops/csrc/bn.cu``: a statistics pass that reproduces torch's channels-last Welford
reduction tree and updates the running stats, then one vectorised pass that applies BN, adds the skip branch and applies
the ReLU, and saves a one-bit-per-element ReLU mask.
The unfused graph writes and re-reads the BN output, the sum and the ReLU output instead.  Backward runs two more
kernels of ``bn.cu`` on the output gradient and the mask: the per-channel sums in torch's reduction tree, then the
elementwise input gradient(s).  They replace ``threshold_backward`` and ``native_batch_norm_backward``, which write and
re-read a masked copy of the gradient.
The stem's BN + ReLU is fused with the max pool that follows it (``bn_relu_maxpool``): its forward writes the pooled
output and a one-byte winner code per pooled element instead of the ReLU output and max pool's int64 indices, and its
backward gathers the pooled gradient back through the codes, already masked, before the two backward kernels.

Every fused result is bitwise that of the unfused graph: same reductions, same fp32 expressions, same bf16 rounding
points.  ``eligible()`` decides per call; anything it rejects (CPU, eval mode, fp32, another memory layout) runs the
unfused modules unchanged.  ``DR_FUSED_BN=0`` selects the unfused graph everywhere, for A/B comparisons.
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn
import torch.nn.functional as F


def enabled() -> bool:
    return os.environ.get("DR_FUSED_BN", "1") != "0"


def _eligible_x(x: torch.Tensor) -> bool:
    # the layout the native training path runs its channels-last kernels on (and that the fused kernels assume)
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.stride(1) == 1
            and x.is_contiguous(memory_format=torch.channels_last) and x.size(1) % 8 == 0 and x.size(1) <= 8192
            and x.numel() < 2 ** 31 - 1 and x.numel() // x.size(1) > 1)


def _eligible_bn(bn: nn.BatchNorm2d) -> bool:
    return (bn.training and bn.track_running_stats and bn.running_mean is not None and bn.momentum is not None
            and bn.affine)


def eligible(x: torch.Tensor, bn: nn.BatchNorm2d) -> bool:
    return enabled() and _eligible_x(x) and _eligible_bn(bn)


def _stats(x, bn):
    """(save_mean, save_invstd) of a training step; updates the running stats and counter as nn.BatchNorm2d does."""
    from .. import ops
    bn.num_batches_tracked.add_(1)
    return ops.cuda_module().bn_stats(x, bn.running_mean, bn.running_var, float(bn.momentum), float(bn.eps))


def _grad(go):
    # the gradient reaching the fused op; the backward kernels read it in x's channels_last layout
    return go.contiguous(memory_format=torch.channels_last)


class _BNReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, mean, invstd):
        from .. import ops
        y, mask = ops.cuda_module().bn_apply(0, x, [mean, invstd, weight, bias])
        ctx.save_for_backward(x, weight, mean, invstd, mask)
        return y

    @staticmethod
    def backward(ctx, gy):
        from .. import ops
        x, weight, mean, invstd, mask = ctx.saved_tensors
        dx, dw, db = ops.cuda_module().bn_backward(0, _grad(gy), mask, x, [mean, invstd, weight])
        return dx, dw, db, None, None


class _BNAddReLU(torch.autograd.Function):
    """relu(bn(x) + z) for an identity skip, relu(bn(x) + bn_z(z)) for a downsample skip (``wz`` given)."""

    @staticmethod
    def forward(ctx, x, weight, bias, mean, invstd, z, wz, bz, mz, iz):
        from .. import ops
        mod = ops.cuda_module()
        if wz is None:
            o, mask = mod.bn_apply(1, x, [mean, invstd, weight, bias], z)
            ctx.save_for_backward(x, weight, mean, invstd, mask)
        else:
            o, mask = mod.bn_apply(2, x, [mean, invstd, weight, bias], z, [mz, iz, wz, bz])
            ctx.save_for_backward(x, weight, mean, invstd, mask, z, wz, mz, iz)
        ctx.has_bn_z = wz is not None
        return o

    @staticmethod
    def backward(ctx, go):
        from .. import ops
        mod = ops.cuda_module()
        saved = ctx.saved_tensors
        x, weight, mean, invstd, mask = saved[:5]
        if not ctx.has_bn_z:
            dx, dw, db, g = mod.bn_backward(1, _grad(go), mask, x, [mean, invstd, weight])
            return dx, dw, db, None, None, g, None, None, None, None
        z, wz, mz, iz = saved[5:]
        dx, dw, db, dz, dwz, dbz = mod.bn_backward(2, _grad(go), mask, x, [mean, invstd, weight], z, [mz, iz, wz])
        return dx, dw, db, None, None, dz, dwz, dbz, None, None


class _BNReLUMaxPool(torch.autograd.Function):
    """maxpool(relu(bn(x))) for the stem's pool (kernel 3, stride 2, padding 1).  The ReLU output is never stored: the
    forward pass writes the pooled output and one code byte per pooled element (winner slot + its ReLU mask), and
    backward gathers the pooled gradient back onto x's positions from the codes."""

    @staticmethod
    def forward(ctx, x, weight, bias, mean, invstd):
        from .. import ops
        out, codes = ops.cuda_module().bn_apply_pool(x, [mean, invstd, weight, bias])
        ctx.save_for_backward(x, weight, mean, invstd, codes)
        return out

    @staticmethod
    def backward(ctx, go):
        from .. import ops
        x, weight, mean, invstd, codes = ctx.saved_tensors
        dx, dw, db = ops.cuda_module().bn_backward(3, _grad(go), codes, x, [mean, invstd, weight])
        return dx, dw, db, None, None


def _stem_pool(pool: nn.Module) -> bool:
    # the only pool bn_apply_pool implements
    if type(pool) is not nn.MaxPool2d:
        return False
    pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)      # noqa: E731
    return (pair(pool.kernel_size) == (3, 3) and pair(pool.stride) == (2, 2) and pair(pool.padding) == (1, 1)
            and pair(pool.dilation) == (1, 1) and not pool.ceil_mode and not pool.return_indices)


def bn_relu_maxpool(x: torch.Tensor, bn: nn.BatchNorm2d, pool: nn.MaxPool2d) -> torch.Tensor:
    """``pool(F.relu(bn(x), inplace=True))``."""
    if not (eligible(x, bn) and _stem_pool(pool)):
        return pool(F.relu(bn(x), inplace=True))
    mean, invstd = _stats(x, bn)
    return _BNReLUMaxPool.apply(x, bn.weight, bn.bias, mean, invstd)


def bn_relu(x: torch.Tensor, bn: nn.BatchNorm2d) -> torch.Tensor:
    """``F.relu(bn(x), inplace=True)``."""
    if not eligible(x, bn):
        return F.relu(bn(x), inplace=True)
    mean, invstd = _stats(x, bn)
    return _BNReLU.apply(x, bn.weight, bn.bias, mean, invstd)


def bn_add_relu(x: torch.Tensor, bn: nn.BatchNorm2d, idt: torch.Tensor) -> torch.Tensor:
    """``F.relu(bn(x) + idt, inplace=True)``."""
    if not (eligible(x, bn) and idt.dtype == x.dtype and idt.shape == x.shape and idt.stride() == x.stride()):
        return F.relu(bn(x) + idt, inplace=True)
    mean, invstd = _stats(x, bn)
    return _BNAddReLU.apply(x, bn.weight, bn.bias, mean, invstd, idt, None, None, None, None)


def bn_bn_add_relu(x: torch.Tensor, bn: nn.BatchNorm2d, xd: torch.Tensor, bnd: nn.BatchNorm2d) -> torch.Tensor:
    """``F.relu(bn(x) + bnd(xd), inplace=True)``: the tail of a bottleneck with a downsample branch."""
    if not (eligible(x, bn) and eligible(xd, bnd) and xd.shape == x.shape and xd.stride() == x.stride()):
        return F.relu(bn(x) + bnd(xd), inplace=True)
    md, id_ = _stats(xd, bnd)
    mean, invstd = _stats(x, bn)
    return _BNAddReLU.apply(x, bn.weight, bn.bias, mean, invstd, xd, bnd.weight, bnd.bias, md, id_)
