"""The fused engine's value codecs (ops/csrc/engine.cu: phase_rank_hist / scan / scatter / exact, phase_fit, phase_fix,
phase_expand) against exact and fp64 references built by the test itself, not against engine_oracle.

Every case runs one step of a BucketEngine and reads the shipped index back from the slot (shipped_index_oracle); the
values are acc[idx] with acc = beta * resid + grad as the test holds them.  Then:

* polyfit: the rank map equals the stable descending fp64 sort permutation, word for word; the header tail holds the
  positives and the count; each segment's curve is within fused_poly_tol of the fp64 least-squares curve
  (test_fused_value_bounds); the output within eval_tol of the fp64 evaluation of the shipped coefficients; the
  residual is v - output to the bit (so phase_fix and phase_expand evaluate the same curve).
* QSGD: each bucket's norm within the fp32 summation bound of the fp64 norm; every level bitwise the kernel formula
  on the shipped norm; the output norm / q * level and the residual v - output to the bit.
* Unshipped coordinates: output exactly 0, residual exactly acc.

The unfused phase chain must give the fused launch's bits.  Further: an unbiasedness check of the stochastic
rounding over 4096 epochs, a NaN / inf / -0.0 tensor that must not disturb its bucket mates, and W = 2 and 4 through
the one-GPU W-rank harness of test_engine_multirank."""
import zlib

import numpy as np
import pytest
import torch

import test_engine_multirank as multirank
from deepreduce_b200.codecs.polyfit import MAX_SEGMENTS, get_segments, gram_basis
from deepreduce_b200.parallel import BucketEngine, BucketPlan
from deepreduce_b200.parallel.engine import shipped_index_oracle
from deepreduce_b200.parallel.plan import MODE_BLOOM, MODE_RAW, MODE_RLE, MODE_SHARED
from test_fused_value_bounds import U32, check_segment, eval_tol
from test_gpu_codec_kernels import _dominant_value, _qsgd_levels_f32, _seed_rounding_up

pytestmark = pytest.mark.gpu
F = np.float32
FLT_MAX = float(np.finfo(np.float32).max)
INDEX = {None: MODE_RAW, "bloom": MODE_BLOOM, "rle": MODE_RLE}


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


# ---------------------------------------------------------------------------
# inputs: exactly K non-zeros, num_pos of them positive
# ---------------------------------------------------------------------------
def _magnitudes(kind, K, rng):
    if kind == "randn":
        return np.abs(rng.standard_normal(K)) + 1e-3
    if kind == "offset":
        return 1000.0 + 0.01 * rng.standard_normal(K)
    if kind == "heavy":                          # ~60 octaves: the coarse rank bins above 4T and their clamps
        return np.exp2(rng.uniform(-30, 30, K))
    if kind == "equal":
        return np.full(K, 0.37)
    if kind == "denormal":
        return rng.uniform(1.0, 2.0, K) * 1e-40
    if kind == "huge":                           # sum of squares of a 512-bucket about FLT_MAX / 3
        return rng.uniform(0.9, 1.0, K) * np.sqrt(FLT_MAX / 1536)
    raise ValueError(kind)


def _grad(plan, d, K, num_pos, kind, key, signed_zeros=False, off=0):
    """Flat gradient: tensor 0 (numel d at element `off`) holds exactly K non-zeros at random positions, num_pos of
    them positive; every other element is +0.0, or +-0.0 at random with signed_zeros."""
    rng = _rng("grad", key)
    g = np.zeros(plan.total_elems, F)
    if signed_zeros:
        g[:] = np.where(rng.random(plan.total_elems) < 0.5, F(-0.0), F(0.0))
    pos = rng.choice(d, K, replace=False)
    sign = np.full(K, -1.0)
    sign[rng.choice(K, num_pos, replace=False)] = 1.0
    g[off + pos] = (sign * _magnitudes(kind, K, rng)).astype(F)
    return torch.from_numpy(g)


# ---------------------------------------------------------------------------
# one step, fused and unfused
# ---------------------------------------------------------------------------
def _run(eng, g, epoch, unfused=False):
    eng.resid.zero_()
    eng.grad.copy_(g.to(eng.grad.dtype).cuda())
    (eng.run_unfused if unfused else eng.step)(epoch)
    torch.cuda.synchronize()
    eng.check_status()
    return (eng.slot().cpu().numpy().view(np.uint32).copy(), eng.grad.float().cpu().numpy().copy(),
            eng.resid.cpu().numpy().copy())


def _step_both(plan, g, epoch=1, check_unfused=True, **kw):
    """The fused step, and (check_unfused) the unfused chain on the same input, bit for bit."""
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, spin_limit=2_000_000, **kw)
    try:
        got = _run(eng, g, epoch)
        if check_unfused:
            again = _run(eng, g, epoch, unfused=True)
            for a, b, what in zip(got, again, ("slot", "output", "residual")):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), what
    finally:
        eng.close()
    return got


def _acc(g, beta):
    """What phase 0 accumulates from a zero residual: gamma * g, or 0 + g (which turns -0.0 into +0.0)."""
    g = g.float().numpy()
    return g.copy() if beta == 0.0 else (np.zeros_like(g) + g).astype(F)


# ---------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------
def _shipped(plan, a, ti, acc):
    t = plan.tensors[ti]
    idx = shipped_index_oracle(plan, a, ti).numpy()
    return t, idx, acc[t.elem_off + idx]


def _unshipped_untouched(t, idx, acc, out, res):
    seg = slice(t.elem_off, t.elem_off + t.numel)
    mask = np.ones(t.numel, bool)
    mask[idx] = False
    assert not out[seg][mask].any()
    assert np.array_equal(res[seg][mask].view(np.uint32), acc[seg][mask].view(np.uint32))


def _rank_map(a, t, n):
    if t.rank_u32:
        return a[t.off_rankmap:t.off_rankmap + n].astype(np.int64)
    return a[t.off_rankmap:t.off_rankmap + (n + 1) // 2].view(np.uint16)[:n].astype(np.int64)


def check_polyfit(plan, ti, a, acc, out, res, bf16=False):
    t, idx, v = _shipped(plan, a, ti, acc)
    n, deg = idx.size, t.poly_degree
    assert t.vmode == 1 and n > 0
    nc = MAX_SEGMENTS * (deg + 1)
    C = a[t.off_coef:t.off_coef + nc].view(np.float32).reshape(MAX_SEGMENTS, deg + 1)
    num_pos, n_hdr = int(a[t.off_coef + nc]), int(a[t.off_coef + nc + 1])
    assert (num_pos, n_hdr) == (int((v > 0).sum()), n)
    # rank map: the stable descending sort of the values (+0.0 == -0.0: ties by position), every entry
    v64 = v.astype(np.float64)
    order = torch.sort(torch.from_numpy(v64), descending=True, stable=True).indices.numpy()
    want = np.empty(n, np.int64)
    want[order] = np.arange(n)
    rank = _rank_map(a, t, n)
    bad = np.flatnonzero(rank != want)
    assert bad.size == 0, (t.name, n, bad.size, bad[:5], rank[bad[:5]], want[bad[:5]], v[bad[:5]])
    # per segment: the curve against fp64 least squares, and the fp64 evaluation of the shipped coefficients
    ys = v64[order]
    curve, etol = np.empty(n), np.empty(n)
    start = 0
    for s, ln in enumerate(get_segments(n, num_pos)):
        if ln == 0:
            continue
        c = C[s]
        de = min(deg, ln - 1)
        assert not np.any(c[de + 1:]), (t.name, s, ln, c)
        fs = gram_basis(ln, deg).numpy() @ c.astype(np.float64)
        err, tol, dr, rtol = check_segment(ys[start:start + ln], fs, c, deg)
        assert err <= tol, (t.name, s, ln, err, tol)
        assert dr <= rtol, (t.name, s, ln, dr, rtol)
        curve[start:start + ln] = fs
        etol[start:start + ln] = eval_tol(ln, c[:de + 1])
        start += ln
    assert start == n
    o = out[t.elem_off + idx].astype(np.float64)
    f64 = curve[rank]
    slack = etol[rank] + U32 * np.abs(f64) + (np.abs(f64) * 2.0 ** -8 if bf16 else 0.0)
    bad = np.flatnonzero(np.abs(o - f64) > slack)
    assert bad.size == 0, (t.name, bad[:5], o[bad[:5]], f64[bad[:5]], slack[bad[:5]])
    r = res[t.elem_off + idx]
    if bf16:
        # the bf16 output is rounded from the fitted value the residual was taken from: v - r is that value
        fit = (v.astype(np.float64) - r.astype(np.float64))
        assert np.all(np.abs(fit - f64) <= etol[rank] + 4 * U32 * (np.abs(f64) + np.abs(v)))
    else:
        # phase_fix and phase_expand evaluate the same curve: the residual is v - output to the bit (+-0 equal)
        bad = np.flatnonzero(r != (v - out[t.elem_off + idx]).astype(F))
        assert bad.size == 0, (t.name, bad[:5], r[bad[:5]], v[bad[:5]], out[t.elem_off + idx][bad[:5]])
    _unshipped_untouched(t, idx, acc, out, res)
    return v, rank


def _norm_bound(v64, n):
    """|fp32 norm - fp64 norm| for phase_fix's order: squares (one rounding, or fused), a 5-level shuffle tree, then
    8 sequential warp partials: 14 roundings deep.  Squares below 2^-150 underflow (2^-150 each at most)."""
    nb = (n + 511) // 512
    x = np.zeros(nb * 512)
    x[:n] = v64
    ss = (x.reshape(nb, 512) ** 2).sum(axis=1)
    gam = 14 * U32 / (1 - 14 * U32)
    return np.sqrt(ss), (gam / 2 + U32) * np.sqrt(ss) + np.sqrt(512 * 2.0 ** -150)


def check_qsgd(plan, ti, a, acc, out, res, epoch, bf16=False):
    t, idx, v = _shipped(plan, a, ti, acc)
    n, q = idx.size, int(t.poly_degree)
    assert t.vmode == 2 and n > 0
    nb = (n + 511) // 512
    norms = a[t.off_coef:t.off_coef + nb].view(np.float32)
    ref, bound = _norm_bound(v.astype(np.float64), n)
    assert np.all(np.abs(norms.astype(np.float64) - ref) <= bound), (t.name, norms, ref)
    if t.rank_u32:
        lvl = a[t.off_rankmap:t.off_rankmap + (n + 1) // 2].view(np.int16)[:n].astype(np.float32)
    else:
        lvl = a[t.off_rankmap:t.off_rankmap + (n + 3) // 4].view(np.int8)[:n].astype(np.float32)
    want = _qsgd_levels_f32(v, norms, q, 512, 0x51ED + epoch)
    bad = np.flatnonzero(lvl != want)
    assert bad.size == 0, (t.name, bad[:5], lvl[bad[:5]], want[bad[:5]])
    assert np.abs(lvl).max() <= q
    assert np.all((lvl == 0) | (np.sign(lvl) == np.sign(v)))
    step = (norms / F(q)).astype(F)[np.arange(n) // 512]
    dec = (step * lvl).astype(F)
    o = out[t.elem_off + idx]
    if bf16:
        assert torch.equal(torch.from_numpy(o), torch.from_numpy(dec).bfloat16().float())
    else:
        assert np.array_equal(o, dec), (t.name, np.flatnonzero(o != dec)[:5])
    # the residual of the level shipped, v - norm/q * level with or without the multiply-add contracted
    r = res[t.elem_off + idx]
    plain = (v - dec).astype(F)
    fused = (v.astype(np.float64) - step.astype(np.float64) * lvl.astype(np.float64)).astype(F)
    bad = np.flatnonzero((r != plain) & (r != fused))
    assert bad.size == 0, (t.name, bad[:5], r[bad[:5]], plain[bad[:5]])
    _unshipped_untouched(t, idx, acc, out, res)
    return v, lvl, norms


# ---------------------------------------------------------------------------
# polyfit
# ---------------------------------------------------------------------------
# (id, n, num_pos, degree, values, index, bf16).  num_pos 1 and n - 2: segments of length 1 and 2; 154 / 155: the
# first fine segment appears (int(155 / 5) > 30); 65 536 / 65 537: u16 / u32 rank map; 131 072: MAX_POLY_K
P = pytest.param
POLY_CASES = [
    P(512, 0, 5, "randn", None, False, id="512-neg-d5-raw"),
    P(513, 1, 1, "randn", None, False, id="513-pos1-d1-raw"),
    P(512, 510, 7, "heavy", "rle", False, id="512-neg2-d7-rle"),
    P(65_535, 154, 7, "heavy", None, False, id="65535-154-d7-raw"),
    P(65_536, 155, 2, "offset", "rle", False, id="65536-155-d2-rle"),
    P(65_537, 65_537, 5, "randn", None, False, id="65537-allpos-d5-raw"),
    P(131_072, 155, 7, "heavy", "bloom", False, id="131072-155-d7-bloom"),
    P(8192, 0, 1, "equal", None, False, id="8192-equal-d1-raw"),
    P(4097, 0, 5, "equal", "rle", True, id="4097-equal-d5-rle-bf16"),
    P(1025, 1, 2, "offset", "bloom", True, id="1025-offset-d2-bloom-bf16"),
    P(70_001, 35_000, 5, "randn", "bloom", True, id="70001-half-d5-bloom-bf16"),
]


def _poly_plan(d, n, deg, index, **kw):
    return BucketPlan([d], ks=[n], index=index, value="polyfit", poly_degree=deg, poly_min_k=min(512, n), **kw)


@pytest.mark.parametrize("n,num_pos,deg,kind,index,bf16", POLY_CASES)
def test_polyfit_vs_fp64(n, num_pos, deg, kind, index, bf16):
    d = max(4 * n, 8192)
    plan = _poly_plan(d, n, deg, index)
    t = plan.tensors[0]
    assert t.vmode == 1 and t.mode == INDEX[index] and t.rank_u32 == int(n > 65536)
    g = _grad(plan, d, n, num_pos, kind, ("poly", n, num_pos, deg, kind, index))
    if bf16:
        g = g.bfloat16().float()                    # the engine widens the bf16 gradient exactly
    a, out, res = _step_both(plan, g, grad_dtype=torch.bfloat16 if bf16 else torch.float32)
    v, _ = check_polyfit(plan, 0, a, _acc(g, 1.0), out, res, bf16)
    if index != "bloom":
        assert v.size == n and int((v > 0).sum()) == num_pos


@pytest.mark.parametrize("opt", [dict(use_tma=False), dict(blocks_per_sm=1)])
@pytest.mark.parametrize("case", ["513-pos1-d1-raw", "131072-155-d7-bloom", "65536-155-d2-rle"])
def test_polyfit_kernel_variants(case, opt):
    """TMA off (the cp.async ring) and one CTA per SM (the other register variant): the same references hold."""
    n, num_pos, deg, kind, index, _ = next(c.values for c in POLY_CASES if c.id == case)
    d = max(4 * n, 8192)
    plan = _poly_plan(d, n, deg, index)
    g = _grad(plan, d, n, num_pos, kind, ("poly", n, num_pos, deg, kind, index))
    a, out, res = _step_both(plan, g, check_unfused=False, **opt)
    check_polyfit(plan, 0, a, _acc(g, 1.0), out, res)


@pytest.mark.parametrize("deg", [1, 5])
def test_polyfit_signed_zeros_rank_as_equals(deg):
    """beta = 0 keeps the gradient's -0.0, and the bloom filter's false positives ship exact zeros of both signs.  The
    specification ranks +0.0 and -0.0 as equals, by position; the rank map, the fit and the residual must agree."""
    d, K = 200_000, 3000
    plan = BucketPlan([d], ks=[K], index="bloom", value="polyfit", poly_degree=deg, fpr=0.05)
    g = _grad(plan, d, K, K // 2, "randn", ("pm0", deg), signed_zeros=True)
    a, out, res = _step_both(plan, g, beta=0.0)
    v, rank = check_polyfit(plan, 0, a, _acc(g, 0.0), out, res)
    z = v == 0
    neg0 = z & (np.signbit(v))
    assert neg0.sum() >= 10 and (z & ~neg0).sum() >= 10, (int(neg0.sum()), int(z.sum()))
    # somewhere a -0.0 precedes a +0.0: the order main's rank bins got wrong
    first_neg = np.flatnonzero(neg0)[0]
    assert np.any(z[first_neg:] & ~np.signbit(v[first_neg:]))


# ---------------------------------------------------------------------------
# QSGD
# ---------------------------------------------------------------------------
# (id, n, q, values, index, plan keywords, bf16)
QSGD_CASES = [
    P(1, 127, "randn", None, {}, False, id="1-q127-raw"),
    P(511, 1, "randn", "rle", {}, False, id="511-q1-rle"),
    P(512, 128, "heavy", "bloom", {}, False, id="512-q128-bloom"),
    P(513, 32767, "randn", None, {}, False, id="513-q32767-raw"),
    P(1025, 127, "equal", "rle", {}, False, id="1025-q127-equal-rle"),
    P(1025, 127, "denormal", None, {}, False, id="1025-q127-denormal-raw"),
    P(1025, 32767, "huge", None, {}, False, id="1025-q32767-huge-raw"),
    P(1025, 128, "randn", "rle", {}, True, id="1025-q128-rle-bf16"),
    P(1025, 127, "heavy", "bloom", {}, True, id="1025-q127-bloom-bf16"),
]


@pytest.mark.parametrize("n,q,kind,index,kw,bf16", QSGD_CASES)
def test_qsgd_vs_formula(n, q, kind, index, kw, bf16):
    d = max(4 * n, 8192)
    plan = BucketPlan([d], ks=[n], index=index, value="qsgd", quantum_num=q, **kw)
    t = plan.tensors[0]
    assert t.vmode == 2 and t.mode == INDEX[index] and t.rank_u32 == int(q >= 128)
    g = _grad(plan, d, n, n // 3, kind, ("qsgd", n, q, kind, index))
    if bf16:
        g = g.bfloat16().float()
    epoch = 3
    a, out, res = _step_both(plan, g, epoch, grad_dtype=torch.bfloat16 if bf16 else torch.float32)
    v, lvl, norms = check_qsgd(plan, 0, a, _acc(g, 1.0), out, res, epoch, bf16)
    if index != "bloom":
        assert v.size == n
    if kind == "denormal":                         # the squares underflow: norm 0, every level 0
        assert not norms.any() and not lvl.any()
    if kind == "huge":
        assert np.isfinite(norms).all() and float((v.astype(np.float64)[:512] ** 2).sum()) > FLT_MAX / 4


@pytest.mark.parametrize("n", [1, 513])
def test_qsgd_dominated_bucket_is_clamped(n):
    """A bucket holding one value (n = 1, or the tail bucket of n = 513): its norm is |v|, lf rounds to q (1 + 2^-23)
    and the epoch is chosen so that the stochastic rounding goes up.  The formula clamps the level to q; so must the
    kernel, or the int8 level wraps to the opposite sign."""
    q = 127
    v, frac = _dominant_value(q)
    epoch = _seed_rounding_up(n - 1, frac, first=0x51ED + 1) - 0x51ED
    d = 8192
    plan = BucketPlan([d], ks=[n], index=None, value="qsgd", quantum_num=q)
    g = _grad(plan, d, n, n // 2, "randn", ("dominated", n))
    last = int(torch.nonzero(g).max())                 # the last shipped value: alone in its bucket
    g[last] = -float(v)
    a, out, res = _step_both(plan, g, epoch)
    _, lvl, norms = check_qsgd(plan, 0, a, _acc(g, 1.0), out, res, epoch)
    assert norms[-1] == v and lvl[-1] == -q


def test_qsgd_zero_buckets_and_signed_zeros():
    """p0 ships every positive of the filter in index order; with the true non-zeros in the first tenth of the tensor
    the tail is false positives only, so whole 512-buckets are zeros (+0.0 and -0.0: beta = 0): norm 0, levels 0,
    output 0, residual the zero itself."""
    d, K = 100_000, 1000
    plan = BucketPlan([d], ks=[K], index="bloom", policy="p0", value="qsgd", fpr=0.05, hint=False)
    rng = _rng("zero_buckets")
    g = np.where(rng.random(plan.total_elems) < 0.5, F(-0.0), F(0.0))
    g[rng.choice(d // 10, K, replace=False)] = rng.standard_normal(K).astype(F)
    g = torch.from_numpy(g)
    a, out, res = _step_both(plan, g, 2, beta=0.0)
    v, lvl, norms = check_qsgd(plan, 0, a, _acc(g, 0.0), out, res, 2)
    zero_buckets = [b for b in range(norms.size - 1) if not v[512 * b:512 * (b + 1)].any()]
    assert zero_buckets and all(norms[b] == 0 for b in zero_buckets)
    assert np.signbit(v[v == 0]).any()


@pytest.mark.parametrize("what", ["randomk", "threshold"])
def test_qsgd_other_sparsifiers(what):
    d = 300_000
    if what == "randomk":
        plan = BucketPlan([d], compress_ratio=0.01, index=None, value="qsgd", sparsifier="randomk")
        assert plan.tensors[0].mode == MODE_SHARED
    else:
        plan = BucketPlan([d], index="bloom", value="qsgd", sparsifier="threshold", threshold=1.0, capacity_ratio=0.5)
    g = torch.from_numpy(_rng("sparsifier", what).standard_normal(plan.total_elems).astype(F))
    g[d:] = 0
    a, out, res = _step_both(plan, g, 5)
    v, _, _ = check_qsgd(plan, 0, a, _acc(g, 1.0), out, res, 5)
    assert v.size > 1024


def test_qsgd_unbiased_over_epochs():
    """beta = 0 and one fixed gradient for E = 4096 epochs (seed 0x51ED + epoch): the mean decoded value of each
    coordinate is within 5 sigma of v, sigma <= norm / (2 q sqrt(E)) (a level is floor or floor + 1 of lf), plus the
    fp32 rounding of lf."""
    d, K, q, E = 8192, 1025, 127, 4096
    plan = BucketPlan([d], ks=[K], index=None, value="qsgd", quantum_num=q)
    g = _grad(plan, d, K, K // 2, "randn", ("unbiased",))
    eng = BucketEngine(plan, device="cuda:0", world=1, rank=0, beta=0.0)
    try:
        gd = g.cuda()
        total = torch.zeros(plan.total_elems, dtype=torch.float64, device="cuda")
        for e in range(1, E + 1):
            eng.grad.copy_(gd)
            eng.step(e)
            total += eng.grad.double()
        torch.cuda.synchronize()
        eng.check_status()
        a = eng.slot().cpu().numpy().view(np.uint32)
    finally:
        eng.close()
    idx = shipped_index_oracle(plan, a, 0).numpy()
    v = g.numpy()[idx].astype(np.float64)
    norms = a[plan.tensors[0].off_coef:plan.tensors[0].off_coef + 3].view(np.float32).astype(np.float64)
    nrm = norms[np.arange(K) // 512]
    mean = total.cpu().numpy()[idx] / E
    sigma = nrm / (2 * q * np.sqrt(E))
    bad = np.flatnonzero(np.abs(mean - v) > 5 * sigma + 8 * U32 * nrm)
    assert bad.size == 0, (bad[:5], mean[bad[:5]], v[bad[:5]], sigma[bad[:5]])


# ---------------------------------------------------------------------------
# a non-finite tensor stays in its own tensor
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("value", ["polyfit", "qsgd"])
def test_nonfinite_tensor_is_isolated(value):
    """NaN, +-inf and -0.0 among tensor 0's values: the step finishes with a clean status, tensors 1 and 2 get the
    bits they get next to a finite tensor 0, and tensor 0's rank map is still a permutation."""
    sizes, ks = [20_000, 30_000, 40_000], [600, 700, 800]
    plan = BucketPlan(sizes, ks=ks, index="bloom", value=value, poly_min_k=512)
    assert all(t.vmode for t in plan.tensors)
    rnd = torch.from_numpy(_rng("iso", value).standard_normal(plan.total_elems).astype(F))
    g = torch.zeros(plan.total_elems)
    for t in plan.tensors:
        g[t.elem_off:t.elem_off + t.numel] = rnd[t.elem_off:t.elem_off + t.numel]
    bad = g.clone()
    t0 = plan.tensors[0]
    bad[t0.elem_off + torch.tensor([5, 77, 900, 4000, 4001])] = torch.tensor([float("nan"), float("inf"), -float("inf"),
                                                                               float("nan"), -0.0])
    _, out_ok, res_ok = _step_both(plan, g, check_unfused=False, beta=0.0)
    a, out_bad, res_bad = _step_both(plan, bad, check_unfused=False, beta=0.0)
    for t in plan.tensors[1:]:
        seg = slice(t.elem_off, t.elem_off + t.numel)
        assert np.array_equal(out_ok[seg].view(np.uint32), out_bad[seg].view(np.uint32)), t.name
        assert np.array_equal(res_ok[seg].view(np.uint32), res_bad[seg].view(np.uint32)), t.name
    idx = shipped_index_oracle(plan, a, 0).numpy()
    assert {5, 77, 900, 4000} <= set(idx.tolist())
    if value == "polyfit":
        assert np.array_equal(np.sort(_rank_map(a, t0, idx.size)), np.arange(idx.size))


# ---------------------------------------------------------------------------
# W > 1: the aggregate against the fp64 decode of every rank's shipped coefficients / levels
# ---------------------------------------------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("value", ["polyfit", "qsgd"])
@pytest.mark.parametrize("W", [2, 4])
def test_multirank_aggregate(W, value):
    plan = BucketPlan([50_000, 200_000], compress_ratio=0.01, index="bloom", value=value, poly_min_k=300)
    assert all(t.vmode for t in plan.tensors)
    engs = multirank._engines(plan, W, "shard", True)
    epoch = 1
    try:
        grads = [torch.from_numpy(_rng("mr", W, value, r).standard_normal(plan.total_elems).astype(F))
                 for r in range(W)]
        for e, g in zip(engs, grads):
            e.grad.copy_(g.cuda())
        multirank._run_step(engs, "shard", epoch)
        outs = [e.grad.cpu().numpy().copy() for e in engs]
        slots = [e.slot().cpu().numpy().view(np.uint32).copy() for e in engs]
        resids = [e.resid.cpu().numpy() for e in engs]
    finally:
        for e in engs:
            e.close()
    scale = 1.0 / W
    for ti, t in enumerate(plan.tensors):
        ref = np.zeros(t.numel)
        tol = np.zeros(t.numel)
        mag = np.zeros(t.numel)
        for r in range(W):
            acc = _acc(grads[r], 1.0)
            idx = shipped_index_oracle(plan, slots[r], ti).numpy()
            n = idx.size
            if value == "polyfit":
                deg = t.poly_degree
                nc = MAX_SEGMENTS * (deg + 1)
                C = slots[r][t.off_coef:t.off_coef + nc].view(np.float32).reshape(MAX_SEGMENTS, deg + 1)
                num_pos = int(slots[r][t.off_coef + nc])
                curve, etol, start = np.empty(n), np.empty(n), 0
                for s, ln in enumerate(get_segments(n, num_pos)):
                    if ln:
                        curve[start:start + ln] = gram_basis(ln, deg).numpy() @ C[s].astype(np.float64)
                        etol[start:start + ln] = eval_tol(ln, C[s][:min(deg, ln - 1) + 1])
                        start += ln
                rank = _rank_map(slots[r], t, n)
                val, vt = curve[rank], etol[rank]
            else:
                v = acc[t.elem_off + idx]
                nb = (n + 511) // 512
                norms = slots[r][t.off_coef:t.off_coef + nb].view(np.float32)
                q = int(t.poly_degree)
                lvl = _qsgd_levels_f32(v, norms, q, 512, 0x51ED + epoch)
                got = (slots[r][t.off_rankmap:t.off_rankmap + (n + 3) // 4].view(np.int8)[:n]).astype(np.float32)
                assert np.array_equal(got, lvl), (r, t.name)
                val = ((norms / F(q)).astype(F)[np.arange(n) // 512] * lvl).astype(F).astype(np.float64)
                vt = np.zeros(n)
            ref[idx] += val * scale
            tol[idx] += vt * scale
            mag[idx] += np.abs(val) * scale
        bound = tol + (W + 1) * U32 * mag
        for r in range(W):
            o = outs[r][t.elem_off:t.elem_off + t.numel].astype(np.float64)
            bad = np.flatnonzero(np.abs(o - ref) > bound)
            assert bad.size == 0, (W, value, t.name, r, bad[:5], o[bad[:5]], ref[bad[:5]], bound[bad[:5]])
    assert all(np.isfinite(x).all() for x in resids)
