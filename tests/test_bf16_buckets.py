"""bf16 gradient buckets, host side: how ``DeepReduceDDP`` groups parameters into flat buckets by dtype, and the
``grad_dtype`` argument of ``BucketEngine``."""
import pytest
import torch

from deepreduce_b200.parallel import BucketEngine, BucketPlan
from deepreduce_b200.parallel.ddp import group_buckets


def _named(specs):
    return [(f"p{i}", torch.zeros(n, dtype=dt)) for i, (n, dt) in enumerate(specs)]


def _fp32_buckets_before(named, cap_mb):
    """The fp32-only bucketing ``DeepReduceDDP`` always did: reverse order, cut at cap_mb MiB of fp32."""
    cap = int(cap_mb * 1024 * 1024 / 4)
    buckets, cur, cur_n = [], [], 0
    for n, p in reversed(named):
        if cur and cur_n + p.numel() > cap:
            buckets.append(cur)
            cur, cur_n = [], 0
        cur.append((n, p))
        cur_n += p.numel()
    if cur:
        buckets.append(cur)
    return buckets


def _names(buckets):
    return [[n for n, _ in b] for b in buckets]


@pytest.mark.parametrize("cap_mb", [1e9, 1.0, 0.25, 0.01, 1e-6])
def test_all_fp32_gives_the_same_buckets(cap_mb):
    named = _named([(n, torch.float32) for n in (300_000, 10, 65_536, 1_000, 70_000, 4097, 262_144, 1)])
    got = group_buckets(named, cap_mb)
    want = _fp32_buckets_before(named, cap_mb)
    assert _names(got) == _names(want)
    assert all(a is b for gb, wb in zip(got, want) for (_, a), (_, b) in zip(gb, wb))


def test_mixed_dtypes_get_their_own_buckets_in_reverse_order():
    bf, f32 = torch.bfloat16, torch.float32
    named = _named([(100_000, bf), (1_000, f32), (200_000, bf), (300_000, bf), (50, f32), (400_000, bf)])
    # 1 MiB holds 262 144 fp32 or 524 288 bf16 elements
    got = group_buckets(named, 1.0)
    assert _names(got) == [["p5"], ["p3", "p2"], ["p0"], ["p4", "p1"]]
    for b in got:
        dts = {p.dtype for _, p in b}
        assert len(dts) == 1
        dt = dts.pop()
        cap = 1024 * 1024 // (2 if dt == bf else 4)
        assert len(b) == 1 or sum(p.numel() for _, p in b) <= cap
    # fp32 first in reverse order -> fp32 buckets come first
    named2 = _named([(10, bf), (20, f32)])
    assert _names(group_buckets(named2, 1e9)) == [["p1"], ["p0"]]


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64])
def test_other_dtypes_raise(dtype):
    named = _named([(10, torch.float32), (20, dtype)])
    with pytest.raises(ValueError, match="fp32 or bf16"):
        group_buckets(named, 1e9)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64, torch.int32])
def test_engine_grad_dtype_is_validated(dtype):
    plan = BucketPlan([4096, 10], compress_ratio=0.01, index="bloom")
    with pytest.raises(ValueError, match="grad_dtype"):
        BucketEngine(plan, device="cpu", world=1, rank=0, grad_dtype=dtype)
