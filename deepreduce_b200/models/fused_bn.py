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
A block input of ResNet-50 feeds two consumers (conv1 and the skip path).  With ``fork=True`` its producer (the stem, or
the previous block's tail) returns the output twice, as two autograd outputs sharing one storage, so backward receives
the two gradients separately and the kernels add them as they load them, instead of autograd writing their sum with an
elementwise add that the backward passes then read again.

Every fused result is bitwise that of the unfused graph: same reductions, same fp32 expressions, same bf16 rounding
points.  ``eligible()`` decides per call.  It accepts a channels_last bf16 CUDA input with C % 8 == 0, C <= 2048
(``kBnMaxChannels`` of ``ops/csrc/ops.h``: the row-walking kernels hold one row's C / 8 threads in a 256-thread CTA),
fewer than 2^31 - 1 elements and more than one row, paired with a training, affine BatchNorm with eps > 0 that tracks
running stats, and whose weight, bias, running_mean and running_var are fp32 on the input's device.  Anything it
rejects (CPU, eval mode, fp32 or NCHW input, more channels, a bf16 BatchNorm, eps <= 0) runs the unfused modules
unchanged.  ``DR_FUSED_BN=0`` selects the
unfused graph everywhere, for A/B comparisons.
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
            and x.is_contiguous(memory_format=torch.channels_last) and x.size(1) % 8 == 0 and x.size(1) <= 2048
            and x.numel() < 2 ** 31 - 1 and x.numel() // x.size(1) > 1)


def _eligible_bn(bn: nn.BatchNorm2d, device: torch.device) -> bool:
    # the kernels read fp32 per-channel parameters and statistics (binding.cpp: check_chan); F.batch_norm refuses
    # eps <= 0, so such a module runs unfused and raises there
    return (bn.training and bn.track_running_stats and bn.running_mean is not None and bn.momentum is not None
            and bn.affine and bn.eps > 0 and all(t.dtype == torch.float32 and t.device == device
                                  for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var)))


def eligible(x: torch.Tensor, bn: nn.BatchNorm2d) -> bool:
    return enabled() and _eligible_x(x) and _eligible_bn(bn, x.device)


def _stats(x, bn):
    """(save_mean, save_invstd) of a training step; updates the running stats and counter as nn.BatchNorm2d does."""
    from .. import ops
    bn.num_batches_tracked.add_(1)
    return ops.cuda_module().bn_stats(x, bn.running_mean, bn.running_var, float(bn.momentum), float(bn.eps))


def _grad(go):
    # the gradient reaching the fused op; the backward kernels read it in x's channels_last layout
    return go.contiguous(memory_format=torch.channels_last)


def _fork(ctx, o, fork):
    """o, or for a forked producer (o, alias of o): two autograd outputs, so their gradients reach backward apart."""
    if not fork:
        return o
    ctx.set_materialize_grads(False)       # an unused output's gradient arrives as None, not as a zeros tensor
    return o, o.detach()


def _grads(grads):
    """(go, go2) for bn_backward from the gradients of a producer's outputs: go2 is None unless both were used."""
    gs = [_grad(g) for g in grads if g is not None]
    return (gs + [None, None])[:2]


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
    def forward(ctx, x, weight, bias, mean, invstd, z, wz, bz, mz, iz, fork):
        from .. import ops
        mod = ops.cuda_module()
        if wz is None:
            o, mask = mod.bn_apply(1, x, [mean, invstd, weight, bias], z)
            ctx.save_for_backward(x, weight, mean, invstd, mask)
        else:
            o, mask = mod.bn_apply(2, x, [mean, invstd, weight, bias], z, [mz, iz, wz, bz])
            ctx.save_for_backward(x, weight, mean, invstd, mask, z, wz, mz, iz)
        ctx.has_bn_z = wz is not None
        return _fork(ctx, o, fork)

    @staticmethod
    def backward(ctx, *grads):
        from .. import ops
        mod = ops.cuda_module()
        go, go2 = _grads(grads)
        if go is None:
            return (None,) * 11
        saved = ctx.saved_tensors
        x, weight, mean, invstd, mask = saved[:5]
        if not ctx.has_bn_z:
            dx, dw, db, g = mod.bn_backward(1, go, mask, x, [mean, invstd, weight], go2=go2)
            return dx, dw, db, None, None, g, None, None, None, None, None
        z, wz, mz, iz = saved[5:]
        dx, dw, db, dz, dwz, dbz = mod.bn_backward(2, go, mask, x, [mean, invstd, weight], z, [mz, iz, wz], go2=go2)
        return dx, dw, db, None, None, dz, dwz, dbz, None, None, None


class _BNReLUMaxPool(torch.autograd.Function):
    """maxpool(relu(bn(x))) for the stem's pool (kernel 3, stride 2, padding 1).  The ReLU output is never stored: the
    forward pass writes the pooled output and one code byte per pooled element (winner slot + its ReLU mask), and
    backward gathers the pooled gradient back onto x's positions from the codes."""

    @staticmethod
    def forward(ctx, x, weight, bias, mean, invstd, fork):
        from .. import ops
        out, codes = ops.cuda_module().bn_apply_pool(x, [mean, invstd, weight, bias])
        ctx.save_for_backward(x, weight, mean, invstd, codes)
        return _fork(ctx, out, fork)

    @staticmethod
    def backward(ctx, *grads):
        from .. import ops
        go, go2 = _grads(grads)
        if go is None:
            return (None,) * 6
        x, weight, mean, invstd, codes = ctx.saved_tensors
        dx, dw, db = ops.cuda_module().bn_backward(3, go, codes, x, [mean, invstd, weight], go2=go2)
        return dx, dw, db, None, None, None


def _stem_pool(pool: nn.Module) -> bool:
    # the only pool bn_apply_pool implements
    if type(pool) is not nn.MaxPool2d:
        return False
    pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)      # noqa: E731
    return (pair(pool.kernel_size) == (3, 3) and pair(pool.stride) == (2, 2) and pair(pool.padding) == (1, 1)
            and pair(pool.dilation) == (1, 1) and not pool.ceil_mode and not pool.return_indices)


def _pair(o, fork):
    # the unfused composite's output for fork=True: one tensor twice, whose gradients autograd adds
    return (o, o) if fork else o


def bn_relu_maxpool(x: torch.Tensor, bn: nn.BatchNorm2d, pool: nn.MaxPool2d, fork: bool = False):
    """``pool(F.relu(bn(x), inplace=True))``; with ``fork`` a pair of it, one per consumer (module docstring)."""
    if not (eligible(x, bn) and _stem_pool(pool)):
        return _pair(pool(F.relu(bn(x), inplace=True)), fork)
    mean, invstd = _stats(x, bn)
    return _BNReLUMaxPool.apply(x, bn.weight, bn.bias, mean, invstd, fork)


def bn_relu(x: torch.Tensor, bn: nn.BatchNorm2d) -> torch.Tensor:
    """``F.relu(bn(x), inplace=True)``."""
    if not eligible(x, bn):
        return F.relu(bn(x), inplace=True)
    mean, invstd = _stats(x, bn)
    return _BNReLU.apply(x, bn.weight, bn.bias, mean, invstd)


def bn_add_relu(x: torch.Tensor, bn: nn.BatchNorm2d, idt: torch.Tensor, fork: bool = False):
    """``F.relu(bn(x) + idt, inplace=True)``; with ``fork`` a pair of it, one per consumer (module docstring)."""
    if not (eligible(x, bn) and idt.dtype == x.dtype and idt.shape == x.shape and idt.stride() == x.stride()):
        return _pair(F.relu(bn(x) + idt, inplace=True), fork)
    mean, invstd = _stats(x, bn)
    return _BNAddReLU.apply(x, bn.weight, bn.bias, mean, invstd, idt, None, None, None, None, fork)


def bn_bn_add_relu(x: torch.Tensor, bn: nn.BatchNorm2d, xd: torch.Tensor, bnd: nn.BatchNorm2d, fork: bool = False):
    """``F.relu(bn(x) + bnd(xd), inplace=True)``: the tail of a bottleneck with a downsample branch; with ``fork`` a
    pair of it, one per consumer (module docstring)."""
    if not (eligible(x, bn) and eligible(xd, bnd) and xd.shape == x.shape and xd.stride() == x.stride()):
        return _pair(F.relu(bn(x) + bnd(xd), inplace=True), fork)
    md, id_ = _stats(xd, bnd)
    mean, invstd = _stats(x, bn)
    return _BNAddReLU.apply(x, bn.weight, bn.bias, mean, invstd, xd, bnd.weight, bnd.bias, md, id_, fork)
