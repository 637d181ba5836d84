"""The fused BatchNorm of ops/csrc/bn.cu over the whole domain models/fused_bn.py::eligible() accepts, not only
ResNet-50's shapes: channel counts whose C / 8 channel groups do not divide a 256-thread CTA (down to one group), row
counts at every corner of torch's channels-last reduction tree, tiny pools with clipped windows, momentum and eps
away from their defaults, and one input just under 2^31 elements.

Shapes are chosen from the launch geometry.  ``row_tree`` mirrors bn.cu's row_tree (torch's flexible_launch_configs):
block_x = min(lastPow2(C), 32), block_y = min(lastPow2(ceil(rows / 16)), 512 / block_x), grid_y = min(ceil(rows /
(16 block_y)), 128), 1 when below 8.  Each row class of MATRIX claims a tree (the smallest row counts, each side of the
grid_y 1 -> 8 jump and of the 128 cap, a last iteration exactly full or partial), and a CPU test holds it to that.

Two checks at every shape:
  1. fused == unfused (DR_FUSED_BN=0) bit for bit: outputs, saved mean / invstd, running stats, the batch counter and
     every gradient.
  2. the fused results against an fp64 BatchNorm computed here from the bf16 input, independent of torch's kernels
     (``check_stats``, ``check_apply``, ``check_sums``, ``check_dx``, ``pool_ref``).  Sums are bounded by (fp32
     roundings on the longest path of the kernel's tree) * 2^-24 * sum |terms|; a bf16 output must be the rounding of
     a value within a few fp32 roundings of the fp64 one, computed from the kernel's own statistics and sums; the pool
     output and its winner gradient are exact.  The CPU tests at the end feed each check a planted defect of the size
     a real bug causes and assert that it is rejected.

Outside the domain: C > 2048 and a bf16 BatchNorm run the unfused modules and give their bits, and eps = 0 raises
as F.batch_norm does.
"""
import math

import pytest
import torch
import torch.nn as nn

from deepreduce_b200.models import fused_bn

U = 2.0 ** -24          # fp32 unit roundoff
LOADS = 4               # accumulators per virtual thread of the tree (torch's ELEMENTS_PER_ITER)
POOL = (3, 2, 1)        # the stem's max pool: kernel, stride, padding


# ---------------------------------------------------------------------------------------------------------------------
# the reduction tree
# ---------------------------------------------------------------------------------------------------------------------
def last_pow2(n):
    return 1 << (max(int(n), 1).bit_length() - 1)


def row_tree(rows, c):
    """(block_y, grid_y) of torch's channels-last reduction tree for rows x C, as bn.cu's row_tree computes it."""
    block_x = min(last_pow2(c), 32)
    block_y = min(last_pow2(-(-rows // 16)), 512 // block_x)
    grid_y = min(-(-rows // (16 * block_y)), 128)
    return block_y, (1 if grid_y < 8 else grid_y)


def tree_path(rows, c):
    """(chain, merges) on the longest path of the tree: `chain` rows into one accumulator, then `merges` pairwise
    combinations (the 4-way merge of the accumulators, the tree over y, and for grid_y > 1 the cross-block chain and
    its tree over y)."""
    by, gy = row_tree(rows, c)
    chain = 1 + (rows - 1) // (by * gy * LOADS)
    lg = by.bit_length() - 1
    merges = LOADS - 1 + lg + ((-(-gy // by) + lg) if gy > 1 else 0)
    return chain, merges


# (class, rows for a C): block_x = 8, 16, 32 give block_y at most ymax = 64, 32, 16
def _ymax(c):
    return 512 // min(last_pow2(c), 32)


ROW_CLASSES = {
    "jump_lo": lambda c: 7 * 16 * _ymax(c),           # ceil(rows / (16 block_y)) = 7: grid_y 1
    "jump_hi": lambda c: 7 * 16 * _ymax(c) + 1,       # = 8: grid_y 8
    "cap_exact": lambda c: 128 * 16 * _ymax(c),       # = 128
    "cap_over": lambda c: 128 * 16 * _ymax(c) + 1,    # = 129: the cap binds
    "full": lambda c: 8 * 16 * _ymax(c),              # grid_y 8, four iterations, the last one full
    "partial": lambda c: 8 * 16 * _ymax(c) - 48,      # grid_y 8, rows past the end in the last iteration
}
TINY = [2, 3, 15, 16, 17]         # block_y 1 or 2, most of the last iteration past the end
CHANNELS = [8, 16, 24, 40, 72, 136, 520, 1000, 2040, 2048]     # C / 8 = 1, 2, 3, 5, 9, 17, 65, 125, 255, 256
MID_ROWS = 6272                   # every C: 2 x 56 x 56


def _claims(cls, rows, c):
    by, gy = row_tree(rows, c)
    full_rows = -(-rows // (16 * by))
    if cls == "tiny":
        return by <= 2 and gy == 1
    if cls == "jump_lo":
        return gy == 1 and full_rows == 7
    if cls == "jump_hi":
        return gy == 8 and full_rows == 8
    if cls == "cap_exact":
        return gy == 128 and full_rows == 128
    if cls == "cap_over":
        return gy == 128 and full_rows > 128
    if cls == "full":
        return gy > 1 and rows % (by * gy * LOADS) == 0
    if cls == "partial":
        return gy > 1 and rows % (by * gy * LOADS) != 0
    return True


def _shape(rows, c):
    """(n, c, h, w) with n * h * w = rows."""
    n = next((k for k in (4, 3, 2) if rows % k == 0 and rows // k > 1), 1)
    hw = rows // n
    h = max(d for d in range(1, math.isqrt(hw) + 1) if hw % d == 0)
    return n, c, h, hw // h


def _matrix():
    cases = []
    extra = iter([16, 40, 72, 136, 520])
    for rows in TINY:
        for c in (8, 24, 2048, next(extra)):
            cases.append(("tiny", rows, c))
    extra = iter([1000, 2040, 16, 40, 72, 136])
    for cls, f in ROW_CLASSES.items():
        for c in (8, 24, 2048, next(extra)):
            cases.append((cls, f(c), c))
    cases += [("mid", MID_ROWS, c) for c in CHANNELS]
    return cases


MATRIX = _matrix()
KINDS = [("relu", None)] + [(k, u) for k in ("add", "bnadd") for u in (None, "both", "first", "second")]

# bn_relu_maxpool: H, W in 1..5 (every window clipped), odd and even, N in {1, 3}; then trees with block_y 16 and
# grid_y > 1
POOL_SHAPES = [(1, 8, 1, 2), (3, 8, 1, 1), (3, 8, 2, 5), (1, 24, 5, 4), (3, 24, 2, 3), (3, 64, 3, 3), (1, 64, 4, 5),
               (3, 64, 5, 2), (1, 520, 2, 2), (3, 520, 5, 5), (3, 2048, 4, 1), (1, 2048, 3, 5),
               (3, 64, 15, 17), (4, 8, 45, 41), (2, 64, 45, 46), (2, 24, 33, 40)]


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference checks (plain functions on tensors of any device; rows x C, NHWC order)
# ---------------------------------------------------------------------------------------------------------------------
def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _within(name, got, want, bound):
    got = got.double()
    fin = torch.isfinite(want)
    bad = ~fin & (got != want)
    bad |= fin & ~((got - want).abs() <= bound)
    idx = bad.nonzero().flatten()
    assert idx.numel() == 0, (f"{name}: {idx.numel()} entries out of bound, first {idx[:6].tolist()}: got "
                              f"{got[idx[:6]].tolist()}, fp64 {want[idx[:6]].tolist()}, "
                              f"bound {bound[idx[:6]].tolist()}")


def moments(x, chunk=1 << 22):
    """fp64 moments of x (rows x C, bf16) for check_stats, in chunks of rows."""
    R = x.shape[0]
    s = sum(x[i:i + chunk].double().sum(0) for i in range(0, R, chunk))
    m = s / R
    ax = sum(x[i:i + chunk].double().abs().sum(0) for i in range(0, R, chunk)) / R
    var, tv = 0, 0
    for i in range(0, R, chunk):
        xd = x[i:i + chunk].double()
        d = xd - m
        var = var + (d * d).sum(0)
        tv = tv + (d.abs() + xd.abs()).pow(2).sum(0)
    return {"rows": R, "C": x.shape[1], "mean": m, "var": var / R, "abs": ax, "var_terms": tv / R}


def check_stats(mo, mean, invstd, rm, rv, rm0, rv0, momentum, eps):
    """The statistics pass against fp64: mean, invstd = 1 / sqrt(var + eps) and the running stats, which take the
    unbiased variance.  Welford's update costs 3 roundings per row of the chain and 4 per merge for the mean, 4 and 7
    for m2n (whose terms, bounded by (|x - mean| + |x|)^2, carry the running means' errors too)."""
    R, C = mo["rows"], mo["C"]
    chain, merges = tree_path(R, C)
    bm = (3 * chain + 4 * merges) * U * mo["abs"]
    _within("mean", mean, mo["mean"], bm)
    bv = (4 * chain + 7 * merges + 1) * U * mo["var_terms"]
    ve = mo["var"] + _f32(eps)
    inv64 = ve.rsqrt()
    # rsqrtf: 2 ulps
    _within("invstd", invstd, inv64, inv64 * (0.5 * (bv + U * ve) / ve + 6 * U))
    mom = _f32(momentum)
    keep = float(torch.tensor(1.0, dtype=torch.float32) - torch.tensor(mom, dtype=torch.float32))
    bessel = _f32(R / (R - 1))
    rm0, rv0 = rm0.double(), rv0.double()
    rm64 = rm0 * keep + mom * mo["mean"]
    _within("running_mean", rm, rm64, mom * bm + 2 * U * ((rm0 * keep).abs() + mom * mo["mean"].abs()))
    rv64 = rv0 * keep + mom * bessel * mo["var"]
    _within("running_var", rv, rv64, mom * bessel * bv + 3 * U * ((rv0 * keep).abs() + mom * bessel * mo["var"]))


def _rn_range(lo, hi):
    """The bf16 roundings of every value in [lo, hi] (fp64) lie in [rn(lo), rn(hi)]; widened by one fp32 ulp."""
    lo32 = torch.nextafter(lo.float(), torch.tensor(-math.inf, device=lo.device))
    hi32 = torch.nextafter(hi.float(), torch.tensor(math.inf, device=hi.device))
    return lo32.bfloat16(), hi32.bfloat16()


def _in_range(name, out, lo, hi):
    o = out.float()
    bad = ~((o >= lo.float()) & (o <= hi.float()))
    idx = bad.nonzero()
    assert idx.shape[0] == 0, (f"{name}: {idx.shape[0]} outputs outside their rounding range, first at "
                               f"{idx[:4].tolist()}: got {o[bad][:4].tolist()}, range {lo.float()[bad][:4].tolist()}"
                               f" .. {hi.float()[bad][:4].tolist()}")


def _bn_range(x, mean, invstd, w, b):
    # fma(w * (x - mean), invstd, b): three roundings of at most |w (x - mean) invstd|, one of |y|
    p = w.double() * (x.double() - mean.double()) * invstd.double()
    y = p + b.double()
    d = 3 * U * (p.abs() + y.abs())
    return _rn_range(y - d, y + d)


def check_apply(out, x, mean, invstd, w, b, z=None, pz=None):
    """The apply output: relu(bn(x)) (z None), relu(bn(x) + z) (pz None) or relu(bn(x) + bn_z(z)), from the kernel's
    own fp32 statistics.  Every step after the fp64 BN value is monotone, so out must lie between the results of the
    two ends of bn's rounding range: equal to bf16(y64) wherever y64 is not within a few fp32 ulps of a bf16 rounding
    boundary."""
    lo, hi = _bn_range(x, mean, invstd, w, b)
    if z is not None:
        zlo, zhi = (z, z) if pz is None else _bn_range(z, *pz)
        lo = (lo.float() + zlo.float()).bfloat16()
        hi = (hi.float() + zhi.float()).bfloat16()
    _in_range("out", out, lo.clamp_min(0), hi.clamp_min(0))


def check_sums(g, x, mean, invstd, db, dw, name=""):
    """db = sum g and dw = sum g (x - mean) * invstd, with g the masked gradient and the kernel's own mean / invstd."""
    R, C = g.shape
    chain, merges = tree_path(R, C)
    P = chain + merges + 1                   # + the rounding of x - mean in each term
    gd = g.double()
    t = gd * (x.double() - mean.double())
    inv = invstd.double()
    _within("db" + name, db, gd.sum(0), P * U * gd.abs().sum(0))
    s1 = t.sum(0) * inv
    _within("dw" + name, dw, s1, (P + 1) * U * t.abs().sum(0) * inv + U * s1.abs())


def check_dx(dx, g, x, mean, invstd, w, db, dw, name="dx"):
    """dx = w invstd (g - sum_dy / R - (x - mean) invstd^2 sum_dy_xmu / R) in fp64 from the kernel's own sums: sum_dy
    is db, sum_dy_xmu is dw / invstd (within the one rounding of dw).  The kernel's expression rounds at most 10 times
    in fp32 before the bf16 rounding."""
    R = g.shape[0]
    gd, d, inv = g.double(), x.double() - mean.double(), invstd.double()
    f2 = w.double() * inv
    sdy = db.double()
    sx = dw.double() / inv
    f1d = d * inv * inv * sx / R
    y = f2 * (gd - sdy / R - f1d)
    delta = 10 * U * f2.abs() * (gd.abs() + sdy.abs() / R + f1d.abs()) + 2 * U * f2.abs() * f1d.abs()
    _in_range(name, dx, *_rn_range(y - delta, y + delta))


def pool_ref(y, gp):
    """The stem's max pool (3, 2, 1) of y (N, H, W, C bf16: the fused ReLU output) and its gradient, exactly:
    -> (out (N, Ho, Wo, C), g (N, H, W, C), the masked gradient of y).  Each window is scanned row by row from -inf and
    taken by v > best or a NaN, so the first of equal maxima and the last NaN win.  A position covered by one window
    gets that window's gradient where it won it (the bf16 value, -0.0 kept); a position covered by more gets the fp32
    sum from +0 of the gradients of the windows it won, in (oh, ow) order, rounded to bf16.  g is then +0 where
    y <= 0."""
    N, H, W, C = y.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    yp = torch.full((N, 2 * Ho + 1, 2 * Wo + 1, C), -math.inf, device=y.device)
    yp[:, 1:H + 1, 1:W + 1] = y.float()
    best = torch.full((N, Ho, Wo, C), -math.inf, device=y.device)
    slot = torch.zeros((N, Ho, Wo, C), dtype=torch.long, device=y.device)
    for k in range(9):
        kh, kw = divmod(k, 3)
        v = yp[:, kh:kh + 2 * Ho - 1:2, kw:kw + 2 * Wo - 1:2]
        take = (v > best) | v.isnan()
        best, slot = torch.where(take, v, best), torch.where(take, k, slot)
    h = torch.arange(H, device=y.device).view(1, H, 1, 1)
    w = torch.arange(W, device=y.device).view(1, 1, W, 1)
    ph, pw = h // 2, w // 2
    nh = torch.clamp((h + 1) // 2 + 1, max=Ho) - ph          # windows covering row h: ph, ph + 1 if odd and in range
    nw = torch.clamp((w + 1) // 2 + 1, max=Wo) - pw
    acc = torch.zeros((N, H, W, C), device=y.device)
    one = torch.zeros((N, H, W, C), dtype=torch.bfloat16, device=y.device)
    won = torch.zeros((N, H, W, C), dtype=torch.bool, device=y.device)
    nidx = torch.arange(N, device=y.device).view(N, 1, 1, 1)
    cidx = torch.arange(C, device=y.device).view(1, 1, 1, C)
    for a, b in ((0, 0), (0, 1), (1, 0), (1, 1)):
        oh, ow = torch.clamp(ph + a, max=Ho - 1), torch.clamp(pw + b, max=Wo - 1)
        s = slot[nidx, oh, ow, cidx]
        gk = gp[nidx, oh, ow, cidx]
        hit = (a < nh) & (b < nw) & (s == (h - 2 * (ph + a) + 1) * 3 + (w - 2 * (pw + b) + 1))
        acc = torch.where(hit, acc + gk.float(), acc)
        one = torch.where(hit, gk, one)
        won |= hit
    g = torch.where((nh == 1) & (nw == 1), one, acc.bfloat16())
    g = torch.where(won & ~(y.float() <= 0), g, torch.zeros_like(g))
    return best.bfloat16(), g


# ---------------------------------------------------------------------------------------------------------------------
# runs
# ---------------------------------------------------------------------------------------------------------------------
def _bn(c, seed, momentum=0.1, eps=1e-5, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm2d(c, eps=eps, momentum=momentum)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.2)
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn.cuda().to(dtype).train()


def _hard(a, c):
    """test_bn_stats.py's hard channels (folded onto C channels): far from zero, constant, NaN, +-inf, -0.0."""
    rows = a.shape[0]
    g = torch.Generator(device="cuda").manual_seed(5)
    a[:, 0 % c] = 300 + torch.randn(rows, device="cuda", generator=g)
    a[:, 1 % c] = -1000 + 0.01 * torch.randn(rows, device="cuda", generator=g)
    a[:, 2 % c] = 2.5
    a[:, 3 % c] = 0.0
    a[:, 4 % c] = -0.0
    a[rows // 3, 5 % c] = float("nan")
    a[rows // 2, 6 % c] = float("inf")
    a[rows - 1, 7 % c] = float("-inf")
    if c > 8:
        a[0, 8] = -0.0
        a[rows - 1, 9] = float("inf")
        a[0, 9] = float("-inf")
    return a


def _act(n, c, h, w, seed, hard=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(n * h * w, c, device="cuda", generator=g) * 1.7 + 0.3
    if hard:
        a = _hard(a, c)
    return a.to(torch.bfloat16).reshape(n, h, w, c).permute(0, 3, 1, 2)      # channels_last NCHW view


def _special(gy, out, seed):
    """test_fused_bn_backward.py's gradient: NaN, +inf, -inf and -0.0 where out == 0 (masked) and where it is not."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    flat = gy.permute(0, 2, 3, 1).reshape(-1)
    zero = out.permute(0, 2, 3, 1).reshape(-1) == 0
    specials = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0], device="cuda", dtype=torch.bfloat16)
    for where in (zero, ~zero):
        idx = where.nonzero().flatten()
        k = min(64, idx.numel() // 4 * 4)
        pick = idx[torch.randperm(idx.numel(), device="cuda", generator=g)[:k]]
        flat[pick] = specials.repeat(k // 4)
    return gy


def _grads(out, seed, special):
    n, c, h, w = out.shape
    ga = _act(n, c, h, w, seed).clone(memory_format=torch.channels_last)
    gb = _act(n, c, h, w, seed + 1).clone(memory_format=torch.channels_last)
    if special:
        ga, gb = _special(ga, out, seed + 2), _special(gb, out, seed + 3)
    return ga, gb


def _rows(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _run(monkeypatch, fused, kind, shape, use=None, momentum=0.1, eps=1e-5, special=False, expect=None,
         dtype=torch.float32):
    """One forward + backward of a fused_bn helper; -> (results to compare bitwise, inputs for the fp64 checks)."""
    monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
    expect = fused if expect is None else expect
    n, c, h, w = shape
    bn, bnd = _bn(c, 1, momentum, eps, dtype), _bn(c, 2, momentum, eps, dtype)
    x = _act(n, c, h, w, 3, special).requires_grad_()
    z = _act(n, c, h, w, 4).requires_grad_()
    assert fused_bn.eligible(x, bn) == expect
    ctx = {"x": x.detach(), "z": z.detach(), "w": bn.weight.detach().clone(), "b": bn.bias.detach().clone(),
           "rm0": bn.running_mean.clone(), "rv0": bn.running_var.clone(), "wz": bnd.weight.detach().clone(),
           "bz": bnd.bias.detach().clone(), "rmz0": bnd.running_mean.clone(), "rvz0": bnd.running_var.clone()}
    saved = {}
    if expect:
        stats = fused_bn._stats

        def record(x_, bn_):
            i = len(saved) // 2
            saved[f"save_mean{i}"], saved[f"save_invstd{i}"] = stats(x_, bn_)
            return saved[f"save_mean{i}"], saved[f"save_invstd{i}"]
        monkeypatch.setattr(fused_bn, "_stats", record)
    else:
        # the unfused graph's saved statistics, in the fused path's order (downsample BN first)
        for i, (t, b) in enumerate([(z, bnd), (x, bn)] if kind == "bnadd" else [(x, bn)]):
            _, saved[f"save_mean{i}"], saved[f"save_invstd{i}"] = torch.native_batch_norm(
                t.detach(), b.weight, b.bias, b.running_mean.clone(), b.running_var.clone(), True, b.momentum, b.eps)
    # with the fused path enabled a forked helper returns a pair (an alias, or the unfused output twice)
    fork = use is not None and fused
    if kind == "relu":
        outs = fused_bn.bn_relu(x, bn)
    elif kind == "add":
        outs = fused_bn.bn_add_relu(x, bn, z, fork=fork)
    elif kind == "bnadd":
        outs = fused_bn.bn_bn_add_relu(x, bn, z, bnd, fork=fork)
    else:
        outs = fused_bn.bn_relu_maxpool(x, bn, nn.MaxPool2d(*POOL), fork=fork)
    out = (outs[0] if fork else outs).detach()
    ga, gb = _grads(out, 5, special)
    if use is None:
        outs.backward(ga)
    else:
        o1, o2 = outs if fork else (outs, outs)
        if use == "both":
            torch.autograd.backward([o1, o2], [ga, gb])
        elif use == "first":
            torch.autograd.backward([o1], [ga])
        else:
            torch.autograd.backward([o2], [gb])
    torch.cuda.synchronize()
    monkeypatch.undo()
    res = {"out": out, "dx": x.grad, "dw": bn.weight.grad, "db": bn.bias.grad, "running_mean": bn.running_mean,
           "running_var": bn.running_var, "num_batches_tracked": bn.num_batches_tracked, **saved}
    if kind in ("add", "bnadd"):
        res["dz"] = z.grad
    if kind == "bnadd":
        res.update(dw_z=bnd.weight.grad, db_z=bnd.bias.grad, running_mean_z=bnd.running_mean,
                   running_var_z=bnd.running_var, num_batches_tracked_z=bnd.num_batches_tracked)
    ctx["go"] = ga
    return {k: v for k, v in res.items() if v is not None}, ctx


def _bits(t):
    return t.contiguous().view({torch.bfloat16: torch.int16, torch.float32: torch.int32}.get(t.dtype, t.dtype))


def _compare(ref, new, what):
    assert ref.keys() == new.keys(), (what, sorted(ref.keys() ^ new.keys()))
    for k in ref:
        a, b = ref[k], new[k]
        assert a.dtype == b.dtype and a.shape == b.shape, (what, k)
        diff = (_bits(a) != _bits(b)).sum().item()
        assert diff == 0, f"{what} {k}: {diff} entries differ in their bits"


def _check_fp64(kind, res, ctx, momentum, eps):
    """Check 2 on a fused run without fork: every result against the fp64 BatchNorm."""
    from deepreduce_b200 import ops
    x, z = _rows(ctx["x"]), _rows(ctx["z"])
    i = 1 if kind == "bnadd" else 0
    mean, inv = res[f"save_mean{i}"], res[f"save_invstd{i}"]
    check_stats(moments(x), mean, inv, res["running_mean"], res["running_var"], ctx["rm0"], ctx["rv0"], momentum, eps)
    pz = None
    if kind == "bnadd":
        pz = (res["save_mean0"], res["save_invstd0"], ctx["wz"], ctx["bz"])
        check_stats(moments(z), pz[0], pz[1], res["running_mean_z"], res["running_var_z"], ctx["rmz0"], ctx["rvz0"],
                    momentum, eps)
    if kind == "stem":
        y = ops.cuda_module().bn_apply(0, ctx["x"], [mean, inv, ctx["w"], ctx["b"]])[0]
        check_apply(_rows(y), x, mean, inv, ctx["w"], ctx["b"])
        y_nhwc = y.permute(0, 2, 3, 1)
        out_ref, g = pool_ref(y_nhwc, ctx["go"].permute(0, 2, 3, 1))
        assert torch.equal(_bits(res["out"].permute(0, 2, 3, 1)), _bits(out_ref)), "pool output"
        g = g.reshape(-1, x.shape[1])
    else:
        out = _rows(res["out"])
        check_apply(out, x, mean, inv, ctx["w"], ctx["b"], None if kind == "relu" else z, pz)
        go = _rows(ctx["go"])
        g = torch.where(~(out <= 0), go, torch.zeros_like(go))      # the ReLU mask: a NaN output passes
    check_sums(g, x, mean, inv, res["db"], res["dw"])
    check_dx(_rows(res["dx"]), g, x, mean, inv, ctx["w"], res["db"], res["dw"])
    if kind == "add":
        assert torch.equal(_bits(_rows(res["dz"])), _bits(g)), "dz of the identity skip is the masked gradient"
    if kind == "bnadd":
        assert torch.equal(_bits(res["db_z"]), _bits(res["db"]))
        check_sums(g, z, pz[0], pz[1], res["db_z"], res["dw_z"], name="_z")
        check_dx(_rows(res["dz"]), g, z, pz[0], pz[1], ctx["wz"], res["db"], res["dw_z"], name="dz")


def _case(monkeypatch, kind, shape, use=None, momentum=0.1, eps=1e-5, special=False):
    ref, _ = _run(monkeypatch, False, kind, shape, use, momentum, eps, special)
    new, ctx = _run(monkeypatch, True, kind, shape, use, momentum, eps, special)
    _compare(ref, new, f"{kind} {use} {shape} momentum {momentum} eps {eps}")
    if use is None and not special:
        _check_fp64(kind, new, ctx, momentum, eps)
    return new


# ---------------------------------------------------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,use", KINDS, ids=[f"{k}-{u}" for k, u in KINDS])
@pytest.mark.parametrize("cls,rows,c", MATRIX, ids=[f"{cls}-{rows}x{c}" for cls, rows, c in MATRIX])
def test_domain_matrix(monkeypatch, cls, rows, c, kind, use):
    _case(monkeypatch, kind, _shape(rows, c), use)


@pytest.mark.gpu
@pytest.mark.parametrize("use", [None, "both"])
@pytest.mark.parametrize("shape", POOL_SHAPES, ids=["x".join(map(str, s)) for s in POOL_SHAPES])
def test_domain_stem_pool(monkeypatch, shape, use):
    _case(monkeypatch, "stem", shape, use)


# (rows, C): grid_y 1 with one group, grid_y 8 at C = 24, a full last iteration at C = 2048
KNOB_SHAPES = [(17, 8), (ROW_CLASSES["jump_hi"](24), 24), (ROW_CLASSES["full"](2048), 2048)]


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [0.0, 1e-12, 1e-5, 1e-3])
@pytest.mark.parametrize("momentum", [0.0, 0.01, 0.1, 1.0])
@pytest.mark.parametrize("rows,c", KNOB_SHAPES)
def test_domain_momentum_eps(monkeypatch, rows, c, momentum, eps):
    if eps == 0:
        # F.batch_norm refuses eps <= 0; eligible() refuses it too, so the helpers raise as the modules do
        for fused in (False, True):
            with pytest.raises(ValueError, match="eps must be positive"):
                _run(monkeypatch, fused, "bnadd", _shape(rows, c), None, momentum, eps, expect=False)
            monkeypatch.undo()
        return
    _case(monkeypatch, "bnadd", _shape(rows, c), None, momentum, eps)


SPECIAL_SHAPES = [(17, 24), (ROW_CLASSES["partial"](8), 8), (ROW_CLASSES["jump_hi"](520), 520), (MID_ROWS, 2040)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,use", [("relu", None), ("add", None), ("bnadd", None), ("bnadd", "both")])
@pytest.mark.parametrize("rows,c", SPECIAL_SHAPES)
def test_domain_nan_inf_negzero(monkeypatch, rows, c, kind, use):
    new = _case(monkeypatch, kind, _shape(rows, c), use, special=True)
    assert new["dx"].isnan().any() and new["save_mean1" if kind == "bnadd" else "save_mean0"].isnan().any()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 24, 5, 4), (4, 8, 45, 41), (2, 64, 15, 17)], ids=lambda s: "x".join(map(str, s)))
def test_domain_stem_nan_inf_negzero(monkeypatch, shape):
    _case(monkeypatch, "stem", shape, None, special=True)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [2056, 4096, 8192])
@pytest.mark.parametrize("kind", ["relu", "add", "bnadd", "stem"])
def test_wide_channels_run_unfused(monkeypatch, kind, c):
    """C > 2048 is outside what the row-walking kernels can launch: eligible() refuses it and the helpers give the
    unfused graph's bits; the kernels' entry points refuse it with a clear message."""
    from deepreduce_b200 import ops
    shape = (2, c, 3, 3)
    ref, _ = _run(monkeypatch, False, kind, shape, "both" if kind != "relu" else None)
    new, _ = _run(monkeypatch, True, kind, shape, "both" if kind != "relu" else None, expect=False)
    _compare(ref, new, f"{kind} C = {c}")
    mod = ops.cuda_module()
    x = _act(*shape, 1)
    p = [torch.zeros(c, device="cuda"), torch.ones(c, device="cuda"), torch.ones(c, device="cuda"),
         torch.zeros(c, device="cuda")]
    for call in (lambda: mod.bn_apply(0, x, p), lambda: mod.bn_apply_pool(x, p),
                 lambda: mod.bn_stats(x, p[0].clone(), p[1].clone(), 0.1, 1e-5),
                 lambda: mod.bn_backward(0, x, torch.zeros(18, c // 8, dtype=torch.uint8, device="cuda"), x, p[:3])):
        with pytest.raises(RuntimeError, match="at most 2048"):
            call()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["relu", "add", "bnadd", "stem"])
def test_bf16_batchnorm_runs_unfused(monkeypatch, kind):
    """A BatchNorm converted to bf16 (model.bfloat16()) is refused by eligible(), since the kernels read fp32
    parameters and running stats, and runs the unfused modules."""
    shape = (2, 64, 5, 5)
    ref, _ = _run(monkeypatch, False, kind, shape, dtype=torch.bfloat16)
    new, _ = _run(monkeypatch, True, kind, shape, expect=False, dtype=torch.bfloat16)
    _compare(ref, new, f"{kind} bf16 BatchNorm")
    assert ref["running_mean"].dtype == torch.bfloat16


@pytest.mark.gpu
def test_largest_tensor(monkeypatch):
    """numel = 2^31 - 130 944, the most rows eligible() accepts at C = 8: the 32-bit row arithmetic of the statistics
    pass and of the backward reduce (rr * C + c, rr * mgroups + group) at its largest."""
    n, c, h, w = 1, 8, 16384, 16383
    assert n * c * h * w < 2 ** 31 - 1 and row_tree(h * w, c) == (64, 128)
    free, _ = torch.cuda.mem_get_info()
    if free < 36 * 2 ** 30:
        pytest.skip(f"needs 36 GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    g = torch.Generator(device="cuda").manual_seed(11)
    x = (torch.randn(n * h * w, c, device="cuda", generator=g, dtype=torch.bfloat16) * 1.7 + 0.3)
    x = x.reshape(n, h, w, c).permute(0, 3, 1, 2)
    gy = torch.randn(n * h * w, c, device="cuda", generator=g, dtype=torch.bfloat16).reshape(n, h, w, c)
    gy = gy.permute(0, 3, 1, 2)
    res = []
    for fused in (False, True):
        monkeypatch.setenv("DR_FUSED_BN", "1" if fused else "0")
        bn = _bn(c, 1)
        rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
        xi = x.detach().requires_grad_()
        assert fused_bn.eligible(xi, bn) == fused
        saved = {}
        if fused:
            stats = fused_bn._stats

            def record(x_, bn_):
                saved["mean"], saved["invstd"] = stats(x_, bn_)
                return saved["mean"], saved["invstd"]
            monkeypatch.setattr(fused_bn, "_stats", record)
        out = fused_bn.bn_relu(xi, bn)
        out.backward(gy)
        torch.cuda.synchronize()
        monkeypatch.undo()
        res.append({"out": out.detach(), "dx": xi.grad, "dw": bn.weight.grad, "db": bn.bias.grad,
                    "running_mean": bn.running_mean, "running_var": bn.running_var,
                    "num_batches_tracked": bn.num_batches_tracked})
        del out, xi                        # the unfused graph is gone before the fused run; its results stay
    for k in res[0]:
        assert torch.equal(_bits(res[0][k]), _bits(res[1][k])), k
    del res[0]
    check_stats(moments(_rows(x)), saved["mean"], saved["invstd"], res[0]["running_mean"], res[0]["running_var"],
                rm0, rv0, 0.1, 1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests: the tree claims, the export, and the checks' teeth
# ---------------------------------------------------------------------------------------------------------------------
def test_matrix_reaches_its_trees():
    for cls, rows, c in MATRIX:
        assert _claims(cls, rows, c), (cls, rows, c, row_tree(rows, c))
        n, c_, h, w = _shape(rows, c)
        assert n * h * w == rows and c_ == c
    by_class = {}
    for cls, rows, c in MATRIX:
        by_class.setdefault(cls, set()).add(c)
    for cls, cs in by_class.items():
        assert {8, 24, 2048} <= cs and len(cs) >= 3, cls
    assert by_class["mid"] == set(CHANNELS)
    assert {rows for cls, rows, _ in MATRIX if cls == "tiny"} == set(TINY)
    # the classes reach each side of every step of the tree for every block_x (8, 16, 32)
    for c in (8, 24, 2048):
        assert row_tree(ROW_CLASSES["jump_lo"](c), c)[1] == 1 and row_tree(ROW_CLASSES["jump_hi"](c), c)[1] == 8
    assert {c // 8 for c in CHANNELS} == {1, 2, 3, 5, 9, 17, 65, 125, 255, 256}
    for s in POOL_SHAPES:
        assert s[0] * s[2] * s[3] > 1 and s[1] % 8 == 0


def test_row_tree_export_matches_mirror():
    from deepreduce_b200 import ops
    if not ops.has_cuda_native():
        pytest.skip("CUDA extension not built")
    mod = ops.cuda_module()
    cases = {(rows, c) for _, rows, c in MATRIX} | {(s[0] * s[2] * s[3], s[1]) for s in POOL_SHAPES}
    cases |= {(r, c) for r in list(range(2, 4200, 7)) + [2 ** 28, 16384 * 16383] for c in (8, 16, 24, 32, 2048)}
    for rows, c in sorted(cases):
        assert tuple(mod.bn_row_tree(rows, c)) == row_tree(rows, c), (rows, c)


def _teeth_data(rows=2000, c=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(rows, c, generator=g) * 1.7 + 0.3).bfloat16()
    go = torch.randn(rows, c, generator=g).bfloat16()
    w = torch.rand(c, generator=g) + 0.5
    b = torch.randn(c, generator=g) * 0.2
    rm0, rv0 = torch.randn(c, generator=g) * 0.1, torch.rand(c, generator=g) + 0.5
    return x, go, w, b, rm0, rv0


def _fp32_stats(xs, rm0, rv0, momentum, eps, bessel_rows):
    """Statistics as an fp32 kernel computes them (torch's CPU reductions stand in for the tree)."""
    xf = xs.float()
    mean, var = xf.mean(0), xf.var(0, unbiased=False)
    keep = 1 - torch.tensor(momentum, dtype=torch.float32)
    bessel = bessel_rows / (bessel_rows - 1) if bessel_rows else 1.0
    return (mean, torch.rsqrt(var + eps), mean * momentum + rm0 * keep,
            (var * torch.tensor(bessel, dtype=torch.float32)) * momentum + rv0 * keep)


def test_teeth_stats():
    x, _, _, _, rm0, rv0 = _teeth_data()
    R = x.shape[0]
    mo = moments(x)
    check_stats(mo, *_fp32_stats(x, rm0, rv0, 0.1, 1e-5, R), rm0, rv0, 0.1, 1e-5)        # a correct pass passes
    for planted in (_fp32_stats(x[1:], rm0, rv0, 0.1, 1e-5, R),                          # one row dropped
                    _fp32_stats(torch.cat([x, x[R // 2:R // 2 + 1]]), rm0, rv0, 0.1, 1e-5, R),    # a row twice
                    _fp32_stats(x, rm0, rv0, 0.1, 1e-5, None)):                          # biased running_var
        with pytest.raises(AssertionError):
            check_stats(mo, *planted, rm0, rv0, 0.1, 1e-5)


def _fp32_sums(g, x, mean, inv):
    gf = g.float()
    return gf.sum(0), (gf * (x.float() - mean)).sum(0) * inv


def test_teeth_sums():
    x, go, _, _, rm0, rv0 = _teeth_data()
    mean, inv = _fp32_stats(x, rm0, rv0, 0.1, 1e-5, x.shape[0])[:2]
    check_sums(go, x, mean, inv, *_fp32_sums(go, x, mean, inv))
    for planted in (_fp32_sums(go[1:], x[1:], mean, inv),                                 # one row dropped
                    _fp32_sums(torch.cat([go, go[7:8]]), torch.cat([x, x[7:8]]), mean, inv)):     # a row twice
        with pytest.raises(AssertionError):
            check_sums(go, x, mean, inv, *planted)


def _fp32_apply(x, mean, inv, w, b):
    return ((w * (x.float() - mean)) * inv + b).bfloat16().clamp_min(0)


def test_teeth_apply_one_ulp():
    x, _, w, b, rm0, rv0 = _teeth_data()
    mean, inv = _fp32_stats(x, rm0, rv0, 0.1, 1e-5, x.shape[0])[:2]
    out = _fp32_apply(x, mean, inv, w, b)
    check_apply(out, x, mean, inv, w, b)
    # one positive output whose rounding range is a single bf16 value, moved by one ulp
    lo, hi = _bn_range(x, mean, inv, w, b)
    i = ((lo == hi) & (out > 0)).flatten().nonzero()[0].item()
    for step in (1, -1):
        bad = out.clone()
        bad.view(-1).view(torch.int16)[i] += step
        with pytest.raises(AssertionError):
            check_apply(bad, x, mean, inv, w, b)


def _fp32_dx(g, x, mean, inv, w, db, dw):
    R = g.shape[0]
    norm = torch.tensor(1.0 / R, dtype=torch.float32)
    f1 = inv * inv * (dw / inv) * norm
    return ((g.float() - db * norm - (x.float() - mean) * f1) * (w * inv)).bfloat16()


def test_teeth_pool_wrong_winner():
    """A tied window whose gradient goes to the second of its equal maxima instead of the first."""
    g = torch.Generator().manual_seed(3)
    n, c, h, w = 1, 8, 5, 5
    y = (torch.rand(n, h, w, c, generator=g) * 2).bfloat16()
    y[0, 1, 1] = y[0, 2, 2] = 5.0          # window (1, 1): slot 0 and slot 4 tie; (2, 2) is in no other window
    gp = (torch.rand(n, 3, 3, c, generator=g) + 0.5).bfloat16()
    out, gref = pool_ref(y, gp)
    assert torch.equal(out[0, 1, 1], y[0, 1, 1]) and torch.equal(gref[0, 2, 2], torch.zeros(c, dtype=torch.bfloat16))
    # the planted winner: (2, 2) takes window (1, 1)'s gradient, (1, 1) keeps only those of windows (0, 0) - (1, 0)
    planted = gref.clone()
    planted[0, 2, 2] = gp[0, 1, 1]
    planted[0, 1, 1] = (gp[0, 0, 0].float() + gp[0, 0, 1].float() + gp[0, 1, 0].float()).bfloat16()
    x = y.reshape(-1, c)                   # y stands in for x, with mean 0, invstd 1, weight 1
    mean, inv, wt = torch.zeros(c), torch.ones(c), torch.ones(c)
    for gk, ok in ((gref, True), (planted, False)):
        gk = gk.reshape(-1, c)
        db, dw = _fp32_sums(gk, x, mean, inv)
        dx = _fp32_dx(gk, x, mean, inv, wt, db, dw)
        if ok:
            check_dx(dx, gref.reshape(-1, c), x, mean, inv, wt, db, dw)
        else:
            with pytest.raises(AssertionError):
                check_dx(dx, gref.reshape(-1, c), x, mean, inv, wt, db, dw)


def test_pool_ref_rules():
    """pool_ref's own rules on hand-made windows: the first of equal maxima wins, a NaN wins, and a position that wins
    several windows gets their fp32 sum in (oh, ow) order."""
    # a 3 x 3 input has four windows: (0, 0) rows 0-1 cols 0-1, (0, 1) rows 0-1 cols 1-2, (1, 0), (1, 1)
    y = torch.zeros(1, 3, 3, 8, dtype=torch.bfloat16)
    y[0, 1, 1, 0] = 1.0                    # channel 0: (1, 1) wins all four windows
    y[0, 0, 0, 1] = y[0, 2, 2, 1] = 2.0    # channel 1: (0, 0) wins window (0, 0), (2, 2) window (1, 1)
    y[0, 2, 0, 2] = float("nan")           # channel 2: the NaN wins window (1, 0)
    y[0, 1, 1, 3] = y[0, 1, 2, 3] = 3.0    # channel 3: (1, 1) and (1, 2) tie in windows (0, 1) and (1, 1)
    gp = torch.tensor([1.0, 2.0 ** -9, 2.0 ** -9, 2.0 ** -9]).bfloat16().reshape(1, 2, 2, 1).expand(1, 2, 2, 8)
    out, g = pool_ref(y, gp.contiguous())
    assert out[0, :, :, 0].float().eq(1.0).all()
    four = (torch.tensor(1.0) + 3 * 2.0 ** -9).bfloat16().item()      # fp32 sum of the four, rounded once
    assert g[0, 1, 1, 0].item() == four and g[0, 1, 1, 3].item() == four and g[0, 1, 2, 3].item() == 0
    assert g[0, 0, 0, 1].item() == 1.0 and g[0, 2, 2, 1].item() == 2.0 ** -9
    assert out[0, 1, 0, 2].isnan() and g[0, 2, 0, 2].item() == 2.0 ** -9
    # channel 1's window (0, 1) is all +0 after the ReLU: its first position wins, and the ReLU mask zeroes its gradient
    assert out[0, 0, 1, 1].item() == 0 and g[0, 0, 1, 1].view(torch.int16).item() == 0
