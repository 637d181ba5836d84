"""The stand-alone per-tensor kernels of ops/csrc/ops.cu (the GRACE-compatible codec path), each pinned to an exact
or fp64 reference at the shapes where the kernel branches: multi-chunk scan carries, strided loops, integer-width
switches, word-straddling bit fields, degenerate segments and buckets.

Integer outputs are compared bit for bit.  Float outputs are compared with an fp64 computation, within a tolerance
derived from the kernel's fp32 arithmetic (stated next to each comparison).  One check compares a kernel with the
formula it implements: the QSGD levels, recomputed in numpy float32 from the kernel's own norms, because a stochastic
rounding decision cannot be checked against fp64 without a tolerance that would hide a wrong level.

Tests that need a GPU are marked ``gpu``; the CPU-only checks of the QSGD oracle are at the end."""
import math
import zlib

import numpy as np
import pytest
import torch

from deepreduce_b200 import spec
from deepreduce_b200.codecs import bitpack, dexp, polyfit, qsgd, rle
from deepreduce_b200.codecs import bloom as B

U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)


def _ops():
    from deepreduce_b200 import ops
    ops.require()
    return ops


def _gen(*key):
    """A generator seeded from the case's key (crc32: stable across processes, unlike hash())."""
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


# ---------------------------------------------------------------------------
# bloom: bloom_insert_kernel, bloom_query_kernel (+ scan_counts_kernel), policies
# ---------------------------------------------------------------------------
# 4096 * 1024 + 1 is 1 025 tiles of 4 096: scan_counts_kernel carries across its 1 024-entry chunks
BLOOM_D = [1, 4095, 4096, 4097, 300_000, 4096 * 1024 + 1, 6_000_007]


def _bloom_cases():
    for d in BLOOM_D:
        ks = {0, 1, max(1, d // 100), d} if d <= 300_000 else {1, d // 100}
        for K in sorted(ks):
            yield d, K


def _check_select(w, d, K, k, m_bits, seed, pos):
    """Every selection of the CUDA path against the oracle's positives `pos` (bitwise)."""
    ops = _ops()
    assert torch.equal(ops.bloom_select(w, d, K, k, m_bits, "p0", seed=seed).cpu(), pos)
    assert torch.equal(ops.bloom_select(w, d, K, k, m_bits, "leftmost", seed=seed).cpu(),
                       B.apply_policy_oracle(pos, K, "leftmost"))
    assert torch.equal(ops.bloom_select(w, d, K, k, m_bits, "random", 9, seed=seed).cpu(),
                       B.apply_policy_oracle(pos, K, "random", 9))
    n_pos = int(pos.numel())
    for limit in sorted({0, 1, n_pos // 2, max(0, n_pos - 1), n_pos, n_pos + 5}):     # below, at and above the count
        got = ops.cuda_module().bloom_select(w, d, limit, k, m_bits, seed)
        assert torch.equal(got.cpu(), pos[:limit]), (limit, n_pos)


@pytest.mark.gpu
@pytest.mark.parametrize("d,K", list(_bloom_cases()))
def test_bloom_insert_and_select_vs_oracle(d, K):
    """Filter words bitwise bloom_insert_oracle; positives bitwise bloom_query_oracle; leftmost / random / p0 and
    explicit limits bitwise apply_policy_oracle."""
    ops = _ops()
    idx = torch.randperm(d, generator=_gen("bloom", d, K))[:K].sort().values
    k, m_bits, _ = spec.bloom_layout(K, d)
    w_ref = B.bloom_insert_oracle(idx, k, m_bits)
    w = ops.bloom_insert(idx.cuda(), k, m_bits)
    assert torch.equal(w.cpu(), w_ref)
    pos = B.bloom_query_oracle(w_ref, d, k, m_bits)
    assert torch.all(torch.isin(idx, pos))                     # no false negatives
    _check_select(w, d, K, k, m_bits, spec.DEFAULT_SEED, pos)


@pytest.mark.gpu
@pytest.mark.parametrize("n_hash,m_bits", [(1, 1000), (1, 4097), (3, 999), (16, 33)])
def test_bloom_single_hash_and_partial_word_filters(n_hash, m_bits):
    """A filter whose bit count is not a multiple of 32 (the last word is partly unused) and a single hash; another
    seed than the default.  Bitwise against the oracle."""
    ops = _ops()
    d, K, seed = 20_000, 300, 0x1234567
    idx = torch.randperm(d, generator=_gen("bloom_odd", n_hash, m_bits))[:K].sort().values
    w_ref = B.bloom_insert_oracle(idx, n_hash, m_bits, seed)
    w = ops.bloom_insert(idx.cuda(), n_hash, m_bits, seed)
    assert torch.equal(w.cpu(), w_ref)
    pos = B.bloom_query_oracle(w_ref, d, n_hash, m_bits, seed)
    _check_select(w, d, K, n_hash, m_bits, seed, pos)


# ---------------------------------------------------------------------------
# QSGD: qsgd_encode_kernel / qsgd_decode_kernel
# ---------------------------------------------------------------------------
QSGD_K = [1, 511, 512, 513, 2 ** 20 + 3]
QSGD_BUCKETS = [1, 7, 256, 257, 512, 4096]         # the kernel runs 256 threads: > 256 takes the strided loop
QSGD_Q = [1, 127, 128, 32767]                      # int8 levels below 128, int16 from 128


def _policy_u(pos, seed):
    """f32(policy_hash(pos, seed) / 2^32): the kernel's uniform draw, elementwise over pos and/or seed."""
    h = spec.policy_hash(torch.as_tensor(pos, dtype=torch.int64), seed)
    return (h.numpy().astype(np.float64) / 4294967296.0).astype(np.float32)


def _qsgd_levels_f32(x, norms, q, bucket, seed):
    """The level formula of qsgd_encode_kernel (and of engine.cu::phase_fix) evaluated in numpy float32 with the
    kernel's own norms: scale = f32(q) / norm, lf = scale * |x|, prev = floor(lf), l = prev + (u < lf - prev),
    l = min(l, q), signed.  Every step is one correctly rounded fp32 operation; the sm_90a code is FMUL, FRND.FLOOR
    and FADD with no contraction, and the division is the IEEE one (nvcc's default -prec-div=true)."""
    x = np.asarray(x, dtype=np.float32)
    nrm = np.asarray(norms, dtype=np.float32)[np.arange(x.size) // bucket]
    safe = np.where(nrm > 0, nrm, np.float32(1))
    scale = np.where(nrm > 0, np.float32(q) / safe, np.float32(0)).astype(np.float32)
    lf = (scale * np.abs(x)).astype(np.float32)
    prev = np.floor(lf)
    l = prev + (_policy_u(np.arange(x.size), seed) < (lf - prev)).astype(np.float32)
    l = np.minimum(l, np.float32(q))
    return np.where(x > 0, l, np.where(x < 0, -l, np.float32(0))).astype(np.float32)


def _qsgd_input(K, bucket, g):
    x = torch.randn(K, generator=g) * 3
    x[torch.rand(K, generator=g) < 0.05] = 0.0
    if K > bucket:
        x[bucket:2 * bucket] = 0.0                  # one all-zero bucket: norm 0, every level 0, decode 0
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("q", QSGD_Q)
@pytest.mark.parametrize("K", QSGD_K)
def test_qsgd_encode_decode(K, q):
    """Norms against fp64; levels bitwise against the kernel's formula in numpy float32; decode bitwise against
    qsgd_decode_oracle and within one quantum (norm / q) of the input in fp64."""
    ops = _ops()
    for bucket in QSGD_BUCKETS:
        g = _gen("qsgd", K, q, bucket)
        x = _qsgd_input(K, bucket, g)
        seed = 1000 + bucket
        lvl, nrm = ops.qsgd_encode(x.cuda(), q, bucket, seed)
        assert lvl.dtype == (torch.int16 if q >= 128 else torch.int8)
        nb = (K + bucket - 1) // bucket
        n_in = np.minimum(bucket, K - bucket * np.arange(nb))            # values per bucket
        x64 = np.zeros(nb * bucket)
        x64[:K] = x.double().numpy()
        ref = np.sqrt((x64.reshape(nb, bucket) ** 2).sum(axis=1))
        got = nrm.cpu().double().numpy()
        # n squares summed in any order in fp32: relative error <= gamma_n = n u / (1 - n u) (each square or FMA
        # rounds once, each add once); the square root halves it and rounds once more
        gam = n_in * U32 / (1 - n_in * U32)
        assert np.all(np.abs(got - ref) <= (gam / 2 + U32) * ref), (bucket, float(np.max(np.abs(got - ref) / ref)))
        assert np.all((got == 0) == (ref == 0))
        lvl_c = lvl.cpu()
        want = _qsgd_levels_f32(x.numpy(), nrm.cpu().numpy(), q, bucket, seed)
        bad = np.flatnonzero(lvl_c.numpy().astype(np.float32) != want)
        assert bad.size == 0, (bucket, bad[:5], lvl_c.numpy()[bad[:5]], want[bad[:5]])
        assert int(lvl_c.abs().max()) <= q
        if K > bucket:
            assert not lvl_c[bucket:2 * bucket].any() and float(nrm[1]) == 0.0
        dec = ops.qsgd_decode(lvl, nrm, q, bucket).cpu()
        assert torch.equal(dec, qsgd.qsgd_decode_oracle(lvl_c, nrm.cpu(), q, bucket))
        # |x| <= norm, and the level is floor(lf) or floor(lf) + 1: |dec - x| <= norm / q, up to the relative error
        # of lf (two fp32 roundings and the norm's) carried over q + 1 quanta
        nq = got[np.arange(K) // bucket] / q
        slack = (q + 1) * (4 * U32 + gam[np.arange(K) // bucket])
        assert np.all(np.abs(dec.double().numpy() - x.double().numpy()) <= nq * (1 + slack))
        if K > bucket:
            assert not dec[bucket:2 * bucket].any()


def _dominant_value(q, like=None):
    """A float32 v > 0 whose bucket norm is v itself and whose level rounds above q: f32(f32(q) / v) * v > q in
    fp32 (kernel formula), or, with like='oracle', (q * (1 / v)) * v > q (qsgd_encode_oracle's torch formula).
    Returns (v, lf - q): the stochastic round-up happens when u < lf - q."""
    rng = np.random.default_rng(q)
    for _ in range(10_000):
        v = np.float32(rng.uniform(0.25, 8.0))
        if like == "oracle":
            lf = np.float32(float(((q / torch.tensor([v])) * torch.tensor([v]))[0]))
        else:
            lf = np.float32(np.float32(q) / v) * v
        if lf > q:
            return v, np.float32(lf - np.float32(q))
    raise AssertionError("no dominated value found")


def _seed_rounding_up(pos, frac, first=0):
    """The smallest seed >= first with f32(policy_hash(pos, seed) / 2^32) < frac."""
    n = 1 << 22
    for lo in range(first, first + (1 << 27), n):
        s = torch.arange(lo, lo + n, dtype=torch.int64)
        u = (spec.policy_hash(torch.full_like(s, pos), s).numpy().astype(np.float64) / 4294967296.0).astype(np.float32)
        hit = np.flatnonzero(u < frac)
        if hit.size:
            return lo + int(hit[0])
    raise AssertionError("no seed found")


@pytest.mark.gpu
@pytest.mark.parametrize("q", [127, 32767])
@pytest.mark.parametrize("layout", ["single", "tail"])
def test_qsgd_dominated_bucket_keeps_its_sign(q, layout):
    """A bucket whose norm is |v| (one value, or a tail bucket of one value): lf rounds to q(1 + 2^-23) and the
    seed is chosen so the stochastic rounding goes up.  The level must be +-q with the sign of v (q + 1 would wrap
    the int8 / int16 wire type to the opposite sign), and the decode within one quantum of v.  (A power-of-two q
    such as 128 cannot round above q: f32(q / v) * v is then q times f32(1 / v) * v, which never exceeds 1.)"""
    ops = _ops()
    v, frac = _dominant_value(q)
    K, bucket, p = (1, 1, 0) if layout == "single" else (513, 512, 512)
    seed = _seed_rounding_up(p, frac)
    for sign in (1.0, -1.0):
        x = torch.randn(K, generator=_gen("dom", q, layout))
        x[p] = sign * float(v)
        lvl, nrm = ops.qsgd_encode(x.cuda(), q, bucket, seed)
        assert float(nrm[p // bucket]) == float(v)              # sqrt(fl(v^2)) == |v| in fp32
        assert int(lvl[p]) == int(sign) * q, (int(lvl[p]), sign, q)
        want = _qsgd_levels_f32(x.numpy(), nrm.cpu().numpy(), q, bucket, seed)
        assert np.array_equal(lvl.cpu().numpy().astype(np.float32), want)
        dec = float(ops.qsgd_decode(lvl, nrm, q, bucket)[p])
        assert math.copysign(1.0, dec) == sign and abs(dec - sign * float(v)) <= float(v) / q


@pytest.mark.gpu
@pytest.mark.parametrize("q", [127, 32767])
def test_fused_qsgd_dominated_bucket_keeps_its_sign(q):
    """The fused engine's QSGD (engine.cu::phase_fix, value-only mode, W = 1).  Exactly K entries are non-zero, one of
    them dominates its 512-value bucket, and the step's epoch (seed 0x51ED + epoch) makes its rounding go up.  The
    slot level must be +-q with the right sign, the residual v - norm/q * level of the level shipped, and the output
    gradient of the right sign.  Every other level bitwise against the kernel formula; the dominant coordinate
    against engine_oracle."""
    from deepreduce_b200.parallel import BucketEngine, BucketPlan, engine_oracle
    from deepreduce_b200.parallel.plan import SLOT_HEADER_WORDS
    _ops()
    d, K, p = 8192, 64, 37                           # p: rank of the dominant value among the K (ascending index)
    plan = BucketPlan([d], ks=[K], index=None, value="qsgd", quantum_num=q)
    tp = plan.tensors[0]
    assert tp.vmode == 2 and tp.val_cap == K
    v, frac = _dominant_value(q)
    epoch = _seed_rounding_up(p, frac, first=0x51ED + 1) - 0x51ED
    g = _gen("fused_dom", q)
    idx = torch.randperm(d, generator=g)[:K].sort().values
    tiny = (torch.rand(K, generator=g) + 0.5) * 1e-6 * float(v)      # squares far below half an ulp of v^2
    tiny[torch.rand(K, generator=g) < 0.5] *= -1
    for sign in (1.0, -1.0):
        vals = tiny.clone()
        vals[p] = sign * float(v)
        grad = torch.zeros(plan.total_elems)
        grad[idx] = vals
        eng = BucketEngine(plan, device="cuda:0", world=1, rank=0)
        try:
            eng.grad.copy_(grad.cuda())
            eng.step(epoch=epoch)
            torch.cuda.synchronize()
            eng.check_status()
            a = eng.slot().cpu().numpy().view(np.uint32)
            assert int(a[SLOT_HEADER_WORDS]) == K
            norm = a[tp.off_coef:tp.off_coef + 1].view(np.float32)[0]
            assert norm == v                                          # the bucket's norm is |v| exactly
            if tp.rank_u32:
                lvl = a[tp.off_rankmap:tp.off_rankmap + (K + 1) // 2].view(np.int16)[:K]
            else:
                lvl = a[tp.off_rankmap:tp.off_rankmap + (K + 3) // 4].view(np.int8)[:K]
            assert int(lvl[p]) == int(sign) * q, (int(lvl[p]), sign, q)
            assert np.array_equal(lvl.astype(np.float32), _qsgd_levels_f32(vals.numpy(), [norm], q, 512, 0x51ED + epoch))
            # residual of the shipped level: fl(v - fl(norm/q) * l) with or without the multiply-add contracted
            step = np.float32(norm / np.float32(q))
            l = np.float32(sign * q)
            sv = np.float32(sign * v)
            allowed = {float(np.float32(sv - np.float32(step * l))), float(np.float32(np.float64(sv) - np.float64(step) * np.float64(l)))}
            r = float(eng.resid[idx[p]])
            assert r in allowed, (r, allowed)
            out = float(eng.grad[idx[p]])
            assert math.copysign(1.0, out) == sign and abs(out - float(sv)) <= float(norm) / q
            # the oracle clamps the same way (its lf uses q * (1 / norm), so only the dominant level is compared)
            out_ref, new_res, slots = engine_oracle(plan, [grad], [torch.zeros_like(grad)], epoch=epoch)
            s = slots[0]
            if tp.rank_u32:
                lref = s[tp.off_rankmap:tp.off_rankmap + (K + 1) // 2].view(np.int16)[:K]
            else:
                lref = s[tp.off_rankmap:tp.off_rankmap + (K + 3) // 4].view(np.int8)[:K]
            assert int(lref[p]) == int(sign) * q
            assert math.copysign(1.0, float(out_ref[idx[p]])) == sign
            assert abs(float(new_res[0][idx[p]])) <= float(norm) / q * 1e-3
        finally:
            eng.close()


# ---------------------------------------------------------------------------
# bit packing: pack_bits_kernel / unpack_bits_kernel
# ---------------------------------------------------------------------------
PACK_N = [1, 31, 32, 33, 1000, 100_003]


def _pack_inputs(bits, n):
    """All-max, and a pattern of 0 / 2^bits - 1 / random in runs of 32 values, so that within a run every value
    starts at every bit offset (i * bits mod 32) the width reaches; plus all-random."""
    top = (1 << bits) - 1
    rng = np.random.default_rng(bits * 1_000_003 + n)
    rnd = rng.integers(0, top, size=n, dtype=np.uint64, endpoint=True).astype(np.int64)
    cls = (np.arange(n) // 32) % 3
    pat = np.where(cls == 0, top, np.where(cls == 1, 0, rnd)).astype(np.int64)
    return [torch.full((n,), top, dtype=torch.int64), torch.from_numpy(pat), torch.from_numpy(rnd)]


@pytest.mark.gpu
@pytest.mark.parametrize("bits", range(1, 64))
def test_pack_unpack_bits_every_width(bits):
    """pack_bits bitwise pack_bits_oracle; unpack_bits of it returns the input exactly and agrees with
    unpack_bits_oracle; bitpack.pack / unpack round-trip on the device."""
    ops = _ops()
    for n in PACK_N:
        for vals in _pack_inputs(bits, n):
            ref = bitpack.pack_bits_oracle(vals, bits)
            buf = ops.pack_bits(vals.cuda(), bits)
            assert torch.equal(buf.cpu(), ref), (bits, n)
            back = ops.unpack_bits(buf, n, bits).cpu()
            bad = torch.nonzero(back != vals).flatten()
            assert bad.numel() == 0, (bits, n, bad[:4].tolist(), back[bad[:4]].tolist(), vals[bad[:4]].tolist())
            assert torch.equal(ops.unpack_bits(ref.cuda(), n, bits).cpu(), bitpack.unpack_bits_oracle(ref, n, bits))
    vals = _pack_inputs(bits, 1000)[1]
    assert torch.equal(bitpack.unpack(bitpack.pack(vals.cuda())).cpu(), vals)


# ---------------------------------------------------------------------------
# polyfit: polyfit_fit_kernel / polyfit_eval_kernel
# ---------------------------------------------------------------------------
POLY_N = [1, 2, 7, 22, 23, 300, 23_592, 131_072, 1_000_000]


def _poly_y(kind, N):
    g = _gen("poly", kind, N)
    if kind == "randn":
        y = torch.randn(N, generator=g)
    elif kind == "const":
        y = torch.full((N,), 0.7)
    else:                                           # large mean, small spread: cancellation in fp32 sums
        y = 1000.0 + 0.01 * torch.randn(N, generator=g)
    return torch.sort(y, descending=True).values


def _lstsq_curve(y64, deg):
    """fp64 least squares in the Legendre basis on x scaled to [-1, 1] (not the Gram basis the kernel uses)."""
    n = y64.size
    x = np.linspace(-1.0, 1.0, n) if n > 1 else np.zeros(1)
    V = np.polynomial.legendre.legvander(x, deg)
    c = np.linalg.lstsq(V, y64, rcond=None)[0]
    return V @ c


def _gram_err(N, deg):
    """First-order bound of |fl(p_k(x)) - p_k(x)| on the grid for common.cuh::gram_eval in fp32.  p_{k+1} =
    (a_k (N - 2x) p_k - b_k p_{k-1}) / D_k with |p| <= 1: the error of step k+1 is the two inherited errors scaled by
    |a_k (N - 2x)| / D_k <= (2k+1) N / D_k and b_k / D_k = k (N+k+1) / D_k, plus about four roundings (two products,
    the difference, the division) of terms of those sizes; 6u per term is used."""
    e = [0.0, 3 * U32]
    for k in range(1, deg):
        D = (k + 1) * (N - k)
        a, b = (2 * k + 1) * N / D, k * (N + k + 1) / D
        e.append(a * e[k] + b * e[k - 1] + 6 * U32 * (a + b))
    return e[:deg + 1]


def _gram_den(N, k):
    """sum_x p_k(x)^2 over x = 0..N for the Gram polynomials with p_k(0) = 1: (N+k+1)! (N-k)! / ((2k+1) N!^2)."""
    return math.exp(math.lgamma(N + k + 2) + math.lgamma(N - k + 1) - 2 * math.lgamma(N + 1)) / (2 * k + 1)


def _poly_tol(y64, c):
    """Bound of |GPU curve - exact least-squares curve| for one segment, from the kernel's fp32 arithmetic.
    Fit (one CTA of 256 threads): num_k = sum p_k y and den_k = sum p_k^2 are summed over at most m = ceil(n/256) + 13
    terms per path (strided per thread, 5 shuffle levels, 8 warp partials), so each carries gamma_m = m u / (1 - m u)
    times the sum of the magnitudes, <= sqrt(den_k) ||y||_2 for num_k; the basis values themselves err by e_k
    (_gram_err), which moves num_k by <= e_k sum|y| and den_k by 2 e_k sqrt(den_k) sqrt(n).  c_k = num_k / den_k
    rounds once more.  Eval: sum_k c_k p_k(x) errs by e_k |c_k| per term, plus (deg + 1) u sum|c_k| of accumulation
    and u |f| for the stored result."""
    n = y64.size
    deg = c.size - 1
    N = n - 1
    m = -(-n // 256) + 13
    gam = m * U32 / (1 - m * U32)
    e = _gram_err(N, deg) if deg >= 1 else [0.0]
    ynorm, ysum = float(np.linalg.norm(y64)), float(np.abs(y64).sum())
    tol = 0.0
    for k in range(deg + 1):
        den = _gram_den(N, k)
        dnum = gam * math.sqrt(den) * ynorm + e[k] * ysum
        dden = gam * den + 2 * e[k] * math.sqrt(den * n)
        dc = dnum / den + abs(c[k]) * (dden / den + U32)
        tol += dc + abs(c[k]) * e[k]
    fmax = float(np.abs(y64).max()) + tol
    return tol + (deg + 2) * U32 * float(np.abs(c).sum()) + U32 * fmax


def _poly_run(kind, N, deg):
    ops = _ops()
    y = _poly_y(kind, N)
    num_pos = int((y > 0).sum())
    segs = polyfit.get_segments(N, num_pos)
    coef = ops.polyfit_fit(y.cuda(), segs, deg)
    fit = ops.polyfit_eval(coef, segs, deg, N).cpu().double().numpy()
    C = coef.cpu().double().numpy().reshape(polyfit.MAX_SEGMENTS, deg + 1)
    return y.double().numpy(), segs, C, fit


def _poly_check(y64, segs, C, fit, deg, perturb=None):
    """Per segment: |GPU curve - fp64 curve| <= _poly_tol, and the GPU residual norm within that distance of the
    fp64 optimum.  perturb = (segment, k): evaluate with c_k of that segment scaled by 1.01 instead (self-check)."""
    off = 0
    worst = []
    for s, n in enumerate(segs):
        if n == 0:
            continue
        ys, fs = y64[off:off + n], fit[off:off + n]
        de = min(deg, n - 1)
        assert not np.any(C[s, de + 1:]), (s, n, C[s])          # degree clamps to n - 1: higher coefficients are 0
        if perturb is not None and perturb[0] == s:
            k = perturb[1]
            pk = polyfit.gram_basis(n, k).numpy()[:, k]         # the basis the coefficients are in (for the shift only)
            fs = fs + 0.01 * C[s, k] * pk
        ref = _lstsq_curve(ys, de)
        tol = _poly_tol(ys, C[s, :de + 1])
        err = float(np.abs(fs - ref).max())
        # residual norm: within ||f_gpu - f_opt||_2 <= sqrt(n) tol of the fp64 optimum, on either side (the fp32
        # values are not exactly a polynomial, so they may undercut the optimum by their rounding)
        r_gpu, r_opt = float(np.linalg.norm(ys - fs)), float(np.linalg.norm(ys - ref))
        worst.append((err, tol, s, n, abs(r_gpu - r_opt), math.sqrt(n) * tol))
        off += n
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["randn", "const", "offset"])
@pytest.mark.parametrize("N", POLY_N)
def test_polyfit_curve_vs_fp64_lstsq(N, kind):
    """Every segment of get_segments(N, num_pos) (lengths 0, 1, 2 included), degree 1..7: the GPU curve against an
    fp64 Legendre least-squares fit within the fp32 bound of _poly_tol, and its residual norm against the optimum."""
    for deg in range(1, polyfit.MAX_DEGREE + 1):
        y64, segs, C, fit = _poly_run(kind, N, deg)
        for err, tol, s, n, dr, rtol in _poly_check(y64, segs, C, fit, deg):
            assert err <= tol, (deg, s, n, err, tol)
            assert dr <= rtol, (deg, s, n, dr, rtol)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,N,deg", [("offset", 23_592, 5), ("randn", 23_592, 2), ("randn", 300, 1),
                                        ("offset", 1_000_000, 3)])
def test_polyfit_tolerance_has_teeth(kind, N, deg):
    """Scaling the largest coefficient of the largest segment by 1.01 must break _poly_tol: the bound is tight
    enough to see a 1 % error in the fit."""
    y64, segs, C, fit = _poly_run(kind, N, deg)
    s = int(np.argmax(segs))
    k = int(np.argmax(np.abs(C[s])))
    hit = [w for w in _poly_check(y64, segs, C, fit, deg, perturb=(s, k)) if w[2] == s]
    err, tol = hit[0][0], hit[0][1]
    assert err > tol, (err, tol, C[s])


# ---------------------------------------------------------------------------
# delta + bp128: bp128_width / pack / header_scan / unpack kernels
# ---------------------------------------------------------------------------
def _bp128_cases(n):
    g = _gen("bp128", n)
    gaps = torch.randint(1, 50, (n,), generator=g)
    yield "random gaps, first 0", torch.cumsum(gaps, 0) - gaps[0]
    yield "all gaps 1, first 5", torch.arange(5, 5 + n)
    if n == 1:
        yield "first index >= 2^31", torch.tensor([2 ** 31 + 3])
    else:
        idx = torch.arange(n) + 2 ** 31 + 7
        idx[0] = 0                                   # delta 2^31 + 7: a 32-bit wide block
        yield "one gap >= 2^31", idx


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 128, 129, 256, 2 ** 20 + 1])
def test_delta_bp128_vs_host_codec(n):
    """Wire bitwise the host C++ int_encode(deltas, 'bp128'); decode exact."""
    from deepreduce_b200.codecs.integer import int_encode
    ops = _ops()
    for what, idx in _bp128_cases(n):
        enc = ops.delta_bp128_encode(idx.cuda())
        deltas = np.diff(idx.numpy(), prepend=0).astype(np.uint32)
        ref = int_encode(deltas, "bp128")
        assert np.array_equal(enc.cpu().numpy().view(np.uint32), ref), what
        assert torch.equal(ops.delta_bp128_decode(enc, n).cpu(), idx), what


# ---------------------------------------------------------------------------
# run-length: rle_count / rle_mark (+ scan_counts_kernel) / rle_runs / rle_expand kernels
# ---------------------------------------------------------------------------
def _rle_cases():
    g = _gen("rle")
    d = 50_000
    yield "empty", torch.empty(0, dtype=torch.int64), d
    yield "[0]", torch.tensor([0]), d
    yield "[d-1]", torch.tensor([d - 1]), d
    yield "all of 0..d-1", torch.arange(d), d
    yield "every other index", torch.arange(0, d, 2), d
    yield "every other index, tail", torch.arange(1, d - 5, 2), d
    # a run over positions 1000..1100 of idx crosses rle_mark's 1 024-index blocks
    head = torch.arange(1000) * 3
    run = head[-1] + 2 + torch.arange(101)
    rest = run[-1] + 2 + torch.cumsum(torch.randint(1, 4, (2000,), generator=g), 0)
    cross = torch.cat([head, run, rest])
    yield "run across a block edge", cross, int(cross[-1]) + 1
    yield "run across a block edge, tail", cross, int(cross[-1]) + 17
    # more than 1 024 * 1 024 indices: scan_counts_kernel carries over its 1 024-entry chunks
    big = torch.cumsum(torch.randint(1, 3, (1024 * 1024 + 5000,), generator=g), 0)
    yield "n > 1024^2", big, int(big[-1]) + 1
    yield "n > 1024^2, tail", big, int(big[-1]) + 1000


@pytest.mark.gpu
def test_rle_runs_and_indices_vs_oracle():
    """Runs bitwise runs_from_sorted_oracle; indices bitwise indices_from_runs_oracle and the input."""
    ops = _ops()
    for what, idx, d in _rle_cases():
        runs_ref = rle.runs_from_sorted_oracle(idx, d)
        runs = ops.rle_runs(idx.cuda(), d)
        assert torch.equal(runs.cpu(), runs_ref), (what, runs.cpu()[:8], runs_ref[:8])
        back = ops.rle_indices(runs, idx.numel()).cpu()
        assert torch.equal(back, rle.indices_from_runs_oracle(runs_ref)), what
        assert torch.equal(back, idx), what


# ---------------------------------------------------------------------------
# double-exponential fit: dexp_fit_kernel
# ---------------------------------------------------------------------------
def _dexp_curve(c, K):
    a, b, p, q = (float(t) for t in c)
    x = np.arange(1, K + 1, dtype=np.float64) / K
    return a * np.exp(p * x) + b * np.exp(q * x)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 1023, 1024, 1025, 2049, 1_000_000])
def test_dexp_fit_vs_fp64_oracle(K):
    """The kernel (fp64, one CTA, scans chunked by 1 024) against double_exponential_fit_oracle (fp64 torch).
    Random data: both sides are fp64 and differ only in summation order, but the 4x4 normal system of (SS, S, x, 1)
    is nearly singular, so a, b, p, q can move far more than the curve: the curves are compared, to 1e-3 relative
    and 1e-4 of max|y|, and the kernel's curve must fit the data as well as the oracle's (residual norm within
    1e-6 relative).  An exact double exponential: both recover it, to 1e-5 of max|y| (fp32 input rounding, 6e-8,
    and the trapezoid rule's O(K^-2) bias, 3e-7 at K = 1 023 for this curve in the oracle)."""
    ops = _ops()
    y = torch.sort(torch.randn(K, generator=_gen("dexp", K)).abs()).values
    got = ops.dexp_fit(y.cuda()).cpu()
    ref = torch.stack(dexp.double_exponential_fit_oracle(y))
    assert torch.isfinite(got).all()
    if K == 2:
        # two points for the four unknowns of y ~ A SS + B S + C x + D: the system is underdetermined, and the
        # kernel's pivoted elimination and the oracle's ridge solve pick different solutions.  Known difference: the
        # oracle's p, q reproduce both points; the kernel's come out (nearly) equal, its 2x2 solve for a, b is then
        # ill-conditioned, and its curve does not.  Only finiteness is required at K = 2.
        return
    fg, fr = _dexp_curve(got, K), _dexp_curve(ref, K)
    y64 = y.double().numpy()
    assert np.allclose(fg, fr, rtol=1e-3, atol=1e-4 * float(y64.max())), (got, ref)
    assert np.linalg.norm(y64 - fg) <= np.linalg.norm(y64 - fr) * (1 + 1e-6) + 1e-12
    x = np.arange(1, K + 1, dtype=np.float64) / K
    true = 2.0 * np.exp(3.0 * x) - 0.5 * np.exp(-1.0 * x)
    yt = torch.from_numpy(true).float()
    got = ops.dexp_fit(yt.cuda()).cpu()
    for c in (got, torch.stack(dexp.double_exponential_fit_oracle(yt))):
        assert np.abs(_dexp_curve(c, K) - true).max() <= 1e-5 * true.max(), c


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["K=1", "constant", "zeros"])
def test_dexp_fit_degenerate_inputs(case):
    """K = 1, a constant y and all zeros: the normal system is singular.  The outputs are finite and give the same
    curve as the oracle (both fall back to p = q = 0 and a = mean of y, b = 0)."""
    ops = _ops()
    y = {"K=1": torch.tensor([0.37]), "constant": torch.full((3000,), 0.37), "zeros": torch.zeros(3000)}[case]
    K = y.numel()
    got = ops.dexp_fit(y.cuda()).cpu()
    ref = torch.stack(dexp.double_exponential_fit_oracle(y))
    assert torch.isfinite(got).all() and torch.isfinite(ref).all(), (got, ref)
    # y is exactly representable and the fit is y itself: the curves agree to a few ulps of max|y| (fp64 sums)
    tol = 1e-12 * max(1.0, float(y.abs().max()))
    assert np.abs(_dexp_curve(got, K) - _dexp_curve(ref, K)).max() <= tol, (got, ref)
    assert np.abs(_dexp_curve(got, K) - y.double().numpy()).max() <= tol, got


# ---------------------------------------------------------------------------
# conflict sets (P2): conflict_sets_pick_kernel
# ---------------------------------------------------------------------------
def _conflict_sets_reaches_fallback(positives, K, k, m_bits, seed, pseed):
    """conflict_sets_oracle's pure-Python walk, reporting whether a full pass picked nothing (the termination
    fallback to the leftmost unchosen positives)."""
    P = positives.tolist()
    sets = {}
    for x in P:
        for pos in spec.bloom_positions_int(x, k, m_bits, seed):
            s = sets.setdefault(pos, [])
            if not s or s[-1] != x:
                s.append(x)
    ordered = [list(v) for _, v in sorted(sets.items(), key=lambda kv: (len(kv[1]), kv[0]))]
    chosen, left, draw = set(), min(K, len(P)), 0
    while left > 0:
        picked = False
        for cset in ordered:
            if left == 0:
                break
            before = len(cset)
            cset[:] = [x for x in cset if x not in chosen]
            if len(cset) == before and cset:
                chosen.add(cset.pop(spec.policy_hash_int(draw, pseed) % len(cset)))
                draw += 1
                left -= 1
                picked = True
        if not picked:
            return True
    return False


def _conflict_cases():
    """(what, positives, K, n_hash, m_bits, policy seeds)"""
    g = _gen("p2")
    d = 100_000
    pos = torch.randperm(d, generator=g)[:3000].sort().values
    yield "long sets (small filter)", pos, 400, 2, 64, (7, 99991)          # ~90 members per set
    yield "K = 1", pos, 1, 3, 4096, (7, 99991)
    yield "K >= positives", pos[:500], 800, 3, 2048, (7, 99991)
    # found by a random search over small inputs (about 1 in 3 000 reaches it); asserted below with the Python walk
    few = torch.tensor([34, 728, 1304, 1992, 2718, 2816, 2867, 3495, 3588, 3872, 4082, 4212, 4214, 4389, 4489, 4502])
    assert _conflict_sets_reaches_fallback(few, 16, 2, 3, spec.DEFAULT_SEED, 7)
    yield "termination fallback", few, 16, 2, 3, (7,)


@pytest.mark.gpu
def test_conflict_sets_pick_vs_host():
    """The device draw bitwise the host routine (native_cpu.cpp::conflict_sets_impl)."""
    ops = _ops()
    for what, pos, K, k, m_bits, pseeds in _conflict_cases():
        for pseed in pseeds:
            ref = ops.cpu.conflict_sets(pos, K, k, m_bits, spec.DEFAULT_SEED, pseed)
            got = B.conflict_sets_cuda(pos.cuda(), K, k, m_bits, spec.DEFAULT_SEED, pseed)
            assert got is not None and torch.equal(got.cpu(), ref), (what, pseed)
            assert ref.numel() == min(K, pos.numel()), what


# ---------------------------------------------------------------------------
# top-k: ops.topk_select (the engine's radix select)
# ---------------------------------------------------------------------------
def _topk_ref(x, k):
    """Stable fp64 sort of |x|, descending: the k largest, ties to the smaller index; ascending indices."""
    order = torch.sort(x.double().abs(), descending=True, stable=True).indices[:k]
    return torch.sort(order).values


def _topk_inputs(d):
    g = _gen("topk", d)
    yield "randn", torch.randn(d, generator=g)
    x = torch.randint(-3, 4, (d,), generator=g).float()          # few distinct magnitudes: ties everywhere
    yield "small integers", x
    sub = torch.zeros(d)                                           # subnormal ties (+-1e-40) above +-0.0 ties
    r = torch.rand(d, generator=g)
    sub[r < 0.6] = 1e-40
    sub[r < 0.3] = -1e-40
    sub[r < 0.1] = torch.randn(int((r < 0.1).sum()), generator=g)
    sub[(r >= 0.6) & (r < 0.8)] = -0.0
    yield "subnormal and signed-zero ties", sub
    tiny = torch.zeros(d)                                          # subnormals below 2^-140 (a 22-bit key prefix of 0)
    tiny[r < 0.5] = 1e-44
    tiny[r < 0.02] = 3.0
    yield "tiny subnormals", tiny


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 4095, 4097, 2 ** 22 + 1])
def test_topk_select_vs_stable_fp64_sort(d):
    """Exact top-k by |x| with ties to the smaller index, against a stable fp64 sort.  Fewer than k non-zeros: the
    non-zeros, then (index 0, 0.0) padding (the documented contract)."""
    ops = _ops()
    for what, x in _topk_inputs(d):
        nnz = int((x != 0).sum())
        for k in sorted({1, max(1, d // 2), d}):
            v, i = ops.topk_select(x.cuda(), k)
            v, i = v.cpu(), i.cpu()
            assert v.numel() == k and i.numel() == k, (what, k)
            if nnz >= k:
                ref = _topk_ref(x, k)
                assert torch.equal(i, ref), (what, k, d)
                assert torch.equal(v.view(torch.int32), x[ref].view(torch.int32)), (what, k)
            else:
                ref = _topk_ref(x, nnz)
                assert torch.equal(i[:nnz], ref) and torch.equal(v[:nnz], x[ref]), (what, k, d)
                assert not i[nnz:].any() and not v[nnz:].any(), (what, k)


# ---------------------------------------------------------------------------
# GRACE codecs end to end: a CUDA tensor and the same CPU tensor give byte-identical wires
# ---------------------------------------------------------------------------
def _wire_bytes(t):
    return t.detach().cpu().contiguous().view(torch.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("codec", ["bloom", "rle", "integer", "bitpack"])
def test_grace_exact_codec_wires_cpu_equals_cuda(codec):
    from deepreduce_b200.codecs.base import compressor
    _ops()
    d = 147_456
    g = _gen("grace", codec)
    idx = torch.randperm(d, generator=g)[:1474]
    vals = torch.randn(1474, generator=g)
    shape = torch.Size([d])
    if codec == "bitpack":
        m = torch.randint(0, 2 ** 40, (5001,), generator=g)
        assert torch.equal(_wire_bytes(bitpack.pack(m.cuda())), _wire_bytes(bitpack.pack(m)))
        return
    params = {"bloom": {}, "rle": {}, "integer": {"code": "bp128"}}[codec]
    cls = compressor[codec]
    wc = cls.compress((vals, idx, shape), dict(params))
    wg = cls.compress((vals.cuda(), idx.cuda(), shape), dict(params))
    for a, b in zip(wc[:2], wg[:2]):
        assert torch.equal(_wire_bytes(b), _wire_bytes(a)), codec
    back_c = cls.decompress(wc, dict(params))
    back_g = cls.decompress(wg, dict(params))
    assert torch.equal(back_g[1].cpu(), back_c[1]) and torch.equal(back_g[0].cpu(), back_c[0])


# ---------------------------------------------------------------------------
# CPU: the QSGD oracle and the CPU GRACE codec on a dominated bucket
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("q", [127, 32767])
def test_qsgd_oracle_dominated_bucket_is_clamped(q):
    """qsgd_encode_oracle on a one-value bucket whose level rounds above q: |level| <= q with the sign of v.  (With
    the oracle's q * (1 / v), a power-of-two q such as 128 never rounds above q.)"""
    v, frac = _dominant_value(q, like="oracle")
    seed = _seed_rounding_up(0, frac)
    for sign in (1.0, -1.0):
        lvl, norm = qsgd.qsgd_encode_oracle(torch.tensor([sign * float(v)]), q, 1, seed)
        assert float(norm[0]) == float(v)
        assert float(lvl[0]) == sign * q, (float(lvl[0]), sign, q)


@pytest.mark.parametrize("q", [127, 32767])
def test_qsgd_cpu_codec_wire_keeps_the_sign(q):
    """The CPU QSGD codec ships int8 / int16 levels; a dominated tail bucket must decode to the sign of its value."""
    v, frac = _dominant_value(q, like="oracle")
    K, bucket = 513, 512
    seed = _seed_rounding_up(K - 1, frac)
    for sign in (1.0, -1.0):
        vals = torch.randn(K, generator=_gen("cpu_qsgd", q))
        vals[-1] = sign * float(v)
        idxs = torch.arange(K)
        params = {"quantum_num": q, "bucket_size": bucket, "qsgd_seed": seed}
        wire = qsgd.QSGD.compress((vals, idxs, torch.Size([K])), params)
        assert wire[0].dtype == (torch.int16 if q >= 128 else torch.int8)
        dec, _, _ = qsgd.QSGD.decompress(wire, params)
        assert math.copysign(1.0, float(dec[-1])) == sign and abs(float(dec[-1]) - sign * float(v)) <= float(v) / q
