"""The BatchNorm statistics pass of ops/csrc/bn.cu against native_batch_norm(training=True), bit for bit.

bn_stats mirrors the reduction tree of torch's channels-last Welford kernel (flexible_launch_configs' block_y and
grid_y, four accumulators per virtual thread, the vertical merge tree, the cross-block merge) in a different thread
layout, so every case here picks a tree shape: block_y 4, 8, 16, 32 and 64, grid_y 1, 8, 25, 49 and 128, last
iterations with rows past the end, and channel counts that are not a multiple of the kernel's channel tile.  The saved
mean and invstd and the updated running stats are compared as int32 bit patterns, so NaN results must match too.
"""
import pytest
import torch

# (channels, H = W) of the BN inputs of ResNet-50 at 224^2, as in tests/test_fused_bn.py
RELU_SHAPES = [(64, 112), (64, 56), (128, 56), (128, 28), (256, 28), (256, 14), (512, 14), (512, 7)]
TAIL_SHAPES = [(256, 56), (512, 28), (1024, 14), (2048, 7)]
RESNET = [(256, c, hw, hw) for c, hw in RELU_SHAPES + TAIL_SHAPES]

# (n, c, h, w): rows = n * h * w; comments give torch's (block_y, grid_y) and the last iteration
TREES = [
    (2, 512, 7, 7),       # rows 98: (4, 1)
    (1, 256, 14, 14),     # rows 196: (8, 1)
    (2, 128, 28, 28),     # rows 1568: (16, 1)
    (8, 64, 16, 16),      # rows 2048: (16, 8), full
    (5, 64, 20, 20),      # rows 2000: (16, 8), rows past the end in the last iteration
    (2, 8, 56, 56),       # rows 6272, C = 8: (64, 1)
    (16, 24, 28, 28),     # rows 12544, C = 24: (32, 25)
    (4, 520, 14, 14),     # rows 784, C = 520: (16, 1)
    (8, 520, 28, 28),     # rows 6272, C = 520: (16, 25)
    (3, 40, 5, 5),        # rows 75, C = 40: (4, 1), rows past the end in the last iteration
]


def _x(rows_nhwc, n, h, w):
    c = rows_nhwc.shape[1]
    return rows_nhwc.to(torch.bfloat16).reshape(n, h, w, c).permute(0, 3, 1, 2)     # channels_last NCHW view


def _randn(n, c, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n * h * w, c, device="cuda", generator=g) * 1.7 + 0.3


def _running(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(c, device="cuda", generator=g) * 0.1, torch.rand(c, device="cuda", generator=g) + 0.5


def _bits(t):
    return t.contiguous().view(torch.int32)


def _compare(x, momentum=0.1, eps=1e-5, torch_kernel=False):
    from deepreduce_b200 import ops
    c = x.size(1)
    weight, bias = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    rm, rv = _running(c, 9)
    rm2, rv2 = rm.clone(), rv.clone()
    _, ref_mean, ref_invstd = torch.ops.aten.native_batch_norm(x, weight, bias, rm, rv, True, momentum, eps)
    mean, invstd = ops.cuda_module().bn_stats(x, rm2, rv2, momentum, eps, torch_kernel=torch_kernel)
    torch.cuda.synchronize()
    for name, a, b in (("save_mean", ref_mean, mean), ("save_invstd", ref_invstd, invstd),
                       ("running_mean", rm, rm2), ("running_var", rv, rv2)):
        assert a.dtype == b.dtype == torch.float32 and a.shape == b.shape, name
        diff = (_bits(a) != _bits(b)).nonzero().flatten()
        assert diff.numel() == 0, f"{tuple(x.shape)} {name}: channels {diff[:8].tolist()} differ in their bits"
    return mean, invstd


@pytest.mark.gpu
@pytest.mark.parametrize("n,c,h,w", RESNET + TREES)
def test_bn_stats_bits(n, c, h, w):
    _compare(_x(_randn(n, c, h, w, 3), n, h, w))


@pytest.mark.gpu
@pytest.mark.parametrize("n,c,h,w", [(5, 64, 20, 20), (256, 512, 28, 28)])
def test_bn_stats_hard_channels(n, c, h, w):
    """Channels far from zero (cancellation), constant channels (variance 0) and NaN, +-inf, -0.0."""
    a = _randn(n, c, h, w, 4)
    g = torch.Generator(device="cuda").manual_seed(5)
    rows = a.shape[0]
    a[:, 0] = 300 + torch.randn(rows, device="cuda", generator=g)
    a[:, 1] = -1000 + 0.01 * torch.randn(rows, device="cuda", generator=g)
    a[:, 2] = 2.5
    a[:, 3] = 0.0
    a[:, 4] = -0.0
    a[:, 5][rows // 3] = float("nan")
    a[:, 6][rows // 2] = float("inf")
    a[:, 7][7] = float("-inf")
    a[:, 8][11] = -0.0
    a[:, 8][12] = 0.0
    a[:, 9][3] = float("inf")
    a[:, 9][rows - 1] = float("-inf")
    # rows 2000 (tree (16, 8), S = 128): accumulator j = 3 of virtual thread 100 takes rows 100 + (4i + 3) * 128, the
    # last valid one at i = 2 and a row past the end at i = 3; an inf there leaves mean = inf, which that row's
    # (0 - mean) * 0 turns into NaN
    if rows == 2000:
        a[:, 10][100 + 11 * 128] = float("inf")
        a[:, 11][100] = float("-inf")
        a[:, 12][10] = float("inf")              # virtual thread 10 has no rows past the end
    mean, invstd = _compare(_x(a, n, h, w))
    assert torch.isnan(mean[5]) and torch.isnan(invstd[6])


@pytest.mark.gpu
@pytest.mark.parametrize("n,c,h,w", [(5, 64, 20, 20), (256, 2048, 7, 7)])
def test_bn_stats_torch_kernel(n, c, h, w):
    """The torch-kernel path of bn_stats (A/B comparisons, trees the mirror does not cover) gives the same bits."""
    x = _x(_randn(n, c, h, w, 6), n, h, w)
    own = _compare(x)
    ref = _compare(x, torch_kernel=True)
    for a, b in zip(own, ref):
        assert torch.equal(_bits(a), _bits(b))
