"""The fused engine's value coders (ops/csrc/engine.cu), checked on the CPU.

1. The polynomial fit of ``phase_fit`` (one warp per segment: lane-strided fp32 sums over x = lane + 32 j, the ra / rb
   recurrence, a 5-level xor-shuffle tree, num / den) and the curve evaluation of ``common.cuh::gram_eval`` +
   ``poly_value``, emulated in numpy float32 in the kernels' order of operations.  ``fused_poly_tol`` bounds the
   distance of that fp32 curve from the exact least-squares curve; the emulation must stay within it, and a 1 % error
   in the largest coefficient must break it.  The GPU tests (test_gpu_fused_values.py) hold the kernel to the same
   bounds.
2. The rank bins of ``rank_bin`` / ``order_key``, compiled for the host from engine.cu's own source: bins must be
   monotone in the value and equal values (+0.0 and -0.0 included) must share a bin, or the exact rank cannot match
   the stable descending sort of the specification (engine_oracle's ``torch.sort(stable=True)``)."""
import ctypes
import math
import os
import re
import subprocess
import zlib

import numpy as np
import pytest

from deepreduce_b200.codecs import polyfit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINE_CU = os.path.join(ROOT, "deepreduce_b200", "ops", "csrc", "engine.cu")
U32 = 2.0 ** -24              # unit roundoff of fp32
F = np.float32
MAX_DEG = 7                   # engine.cu kMaxDeg
POLY_N = [1, 2, 7, 22, 23, 300, 23_592, 131_072, 1_000_000]


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


# ---------------------------------------------------------------------------
# fp32 emulation of phase_fit, gram_eval and poly_value
# ---------------------------------------------------------------------------
def fit_emulated(y, deg):
    """Coefficients of one segment as ``phase_fit`` computes them (every operation one fp32 rounding as written)."""
    y = np.asarray(y, dtype=F)
    n = y.size
    de = min(deg, n - 1)
    N = F(n - 1)
    invN = F(1) / N if n > 1 else F(0)
    ra, rb = np.zeros(MAX_DEG, F), np.zeros(MAX_DEG, F)
    for k in range(1, MAX_DEG):
        dnm = F(k + 1) * F(N - F(k))
        if k < de:
            ra[k] = F(2 * k + 1) / dnm
            rb[k] = F(F(k) * F(F(N + F(k)) + F(1))) / dnm
    J = -(-n // 32)
    x = np.arange(J * 32)
    inside = x < n
    yv = np.zeros(J * 32, F)
    yv[:n] = y
    uu = (N - F(2) * x.astype(F)).astype(F)
    p = [np.ones(J * 32, F), (uu * invN).astype(F) if de >= 1 else np.zeros(J * 32, F)]
    for k in range(1, MAX_DEG):
        p.append(((ra[k] * uu).astype(F) * p[k] - rb[k] * p[k - 1]).astype(F) if k < de else np.zeros(J * 32, F))
    coef = np.zeros(deg + 1, F)
    for k in range(deg + 1):
        pk = np.where(inside, p[k], F(0))
        # per lane: sequential sums over x = lane, lane + 32, ... (the 8-deep unroll keeps that order)
        num = np.cumsum((pk * yv).astype(F).reshape(J, 32), axis=0, dtype=F)[-1]
        den = np.cumsum((pk * pk).astype(F).reshape(J, 32), axis=0, dtype=F)[-1]
        for o in (16, 8, 4, 2, 1):                 # __shfl_xor_sync tree: every lane adds its partner's partial
            num = (num + num[np.arange(32) ^ o]).astype(F)
            den = (den + den[np.arange(32) ^ o]).astype(F)
        if k <= de and den[k] > 0:                 # lane k writes coefficient k
            coef[k] = num[k] / den[k]
    return coef


def gram_eval_emulated(x, n, deg):
    """``common.cuh::gram_eval`` for x (fp32 grid points) of a segment of n values: [deg + 1, len(x)] basis values."""
    x = np.asarray(x, dtype=F)
    N = F(n - 1)
    de = min(deg, n - 1)
    p = [np.ones_like(x)] + [np.zeros_like(x) for _ in range(deg)]
    if de >= 1:
        u = (N - F(2) * x).astype(F)
        p[1] = (u / N).astype(F)
        for k in range(1, deg):
            if k < de:
                a = (F(F(2 * k) + F(1)) * u).astype(F) * p[k]
                b = F(F(k) * F(F(N + F(k)) + F(1))) * p[k - 1]
                p[k + 1] = ((a.astype(F) - b.astype(F)).astype(F) / F(F(k + 1) * F(N - F(k)))).astype(F)
    return p


def eval_emulated(c, n, deg):
    """``poly_value`` over a whole segment: acc += c_k * p_k, k = 0..deg, in fp32."""
    p = gram_eval_emulated(np.arange(n, dtype=F), n, deg)
    acc = np.zeros(n, F)
    for k in range(deg + 1):
        acc = (acc + (F(c[k]) * p[k]).astype(F)).astype(F)
    return acc


# ---------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------
def _basis_err(N, deg, e1, per_term):
    """First-order bound of |fl(p_k(x)) - p_k(x)| on the grid for a three-term recurrence p_{k+1} = (a_k (N - 2x) p_k -
    b_k p_{k-1}) / D_k with |p| <= 1: step k+1 inherits the two errors scaled by (2k+1) N / D_k and k (N+k+1) / D_k,
    plus `per_term` roundings of terms of those sizes.  e1: the error of p_1."""
    e = [0.0, e1]
    for k in range(1, deg):
        D = (k + 1) * (N - k)
        a, b = (2 * k + 1) * N / D, k * (N + k + 1) / D
        e.append(a * e[k] + b * e[k - 1] + per_term * U32 * (a + b))
    return e[:deg + 1]


def fit_basis_err(N, deg):
    """phase_fit's basis: p_1 = (N - 2x) * fl(1/N) (two roundings); ra_k = fl((2k+1) / D_k) and rb_k = fl(k (N+k+1)
    / D_k) carry up to three and five roundings, and each step rounds ra*u, *p_k, rb*p_{k-1} and the difference."""
    return _basis_err(N, deg, 2 * U32, 9)


def eval_basis_err(N, deg):
    """gram_eval's basis: p_1 = (N - 2x) / N (one rounding); each step rounds two products per term, the difference
    and the division (the constants are exact integers in fp32 below 2^24)."""
    return _basis_err(N, deg, 3 * U32, 6)


def _gram_den(N, k):
    """sum_x p_k(x)^2 over x = 0..N for the Gram polynomials with p_k(0) = 1: (N+k+1)! (N-k)! / ((2k+1) N!^2)."""
    return math.exp(math.lgamma(N + k + 2) + math.lgamma(N - k + 1) - 2 * math.lgamma(N + 1)) / (2 * k + 1)


def eval_tol(n, c):
    """Bound of |fp32 poly_value - the fp64 evaluation of the same coefficients c| over a segment of n values:
    e_k |c_k| per basis value (gram_eval_err), (deg + 2) u sum|c_k| for the products and the sequential sum."""
    deg = c.size - 1
    e = eval_basis_err(n - 1, deg) if deg >= 1 and n > 1 else [0.0] * (deg + 1)
    ac = np.abs(np.asarray(c, dtype=np.float64))
    return float(sum(ac[k] * e[k] for k in range(deg + 1)) + (deg + 2) * U32 * ac.sum())


def fused_poly_tol(y64, c):
    """Bound of |fp32 fitted curve - exact least-squares curve| for one segment (y64: the segment's values in fp64,
    c: its fp32 coefficients, degree already clamped to n - 1).  Fit: num_k = sum p_k y and den_k = sum p_k^2 are
    summed over at most m = ceil(n / 32) + 5 terms per path (lane-strided sequential sums, then 5 shuffle levels), so
    each errs by gamma_m = m u / (1 - m u) times its sum of magnitudes (<= sqrt(den_k) ||y||_2 for num_k, den_k for
    den_k); the fit's basis errs by e_k (fit_basis_err), which moves num_k by <= e_k sum|y| and den_k by <= 2 e_k
    sqrt(den_k n); c_k = num_k / den_k rounds once more.  The curve is then evaluated in a different basis rounding
    (gram_eval), bounded separately by eval_tol; the two are added."""
    n = y64.size
    deg = c.size - 1
    N = n - 1
    m = -(-n // 32) + 5
    gam = m * U32 / (1 - m * U32)
    e = fit_basis_err(N, deg) if deg >= 1 else [0.0]
    ynorm, ysum = float(np.linalg.norm(y64)), float(np.abs(y64).sum())
    tol = 0.0
    for k in range(deg + 1):
        den = _gram_den(N, k)
        dnum = gam * math.sqrt(den) * ynorm + e[k] * ysum
        dden = gam * den + 2 * e[k] * math.sqrt(den * n)
        tol += dnum / den + abs(float(c[k])) * (dden / den + U32)
    fmax = float(np.abs(y64).max()) + tol
    return tol + eval_tol(n, c) + U32 * fmax


def lstsq_curve(y64, deg):
    """fp64 least squares in the Legendre basis on x scaled to [-1, 1] (not the Gram basis of the kernels)."""
    n = y64.size
    x = np.linspace(-1.0, 1.0, n) if n > 1 else np.zeros(1)
    V = np.polynomial.legendre.legvander(x, deg)
    return V @ np.linalg.lstsq(V, y64, rcond=None)[0]


def check_segment(ys64, fs64, c, deg):
    """(|curve - fp64 optimum|_inf, bound, ||y - curve|| - ||y - optimum||, sqrt(n) bound) for one segment."""
    n = ys64.size
    de = min(deg, n - 1)
    ref = lstsq_curve(ys64, de)
    tol = fused_poly_tol(ys64, np.asarray(c[:de + 1]))
    err = float(np.abs(fs64 - ref).max())
    dr = abs(float(np.linalg.norm(ys64 - fs64)) - float(np.linalg.norm(ys64 - ref)))
    return err, tol, dr, math.sqrt(n) * tol


def poly_values(kind, n, rng):
    """Descending fp32 values of one tensor: randn, const, offset (large mean, small spread: cancellation in the fp32
    sums), heavy (magnitudes spread over 60 octaves, both signs)."""
    if kind == "randn":
        y = rng.standard_normal(n)
    elif kind == "const":
        y = np.full(n, 0.7)
    elif kind == "offset":
        y = 1000.0 + 0.01 * rng.standard_normal(n)
    else:
        y = np.exp2(rng.uniform(-30, 30, n)) * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    return np.sort(y.astype(F))[::-1].copy()


def _fit_all(y, deg):
    """Emulated coefficients and curve of every segment of get_segments(n, num_pos)."""
    n = y.size
    segs = polyfit.get_segments(n, int((y > 0).sum()))
    out, off = [], 0
    for s, ln in enumerate(segs):
        if ln:
            c = fit_emulated(y[off:off + ln], deg)
            out.append((s, off, ln, c, eval_emulated(c, ln, deg)))
        off += ln
    return out


@pytest.mark.parametrize("kind", ["randn", "const", "offset", "heavy"])
@pytest.mark.parametrize("n", POLY_N)
def test_emulated_fit_within_fused_poly_tol(n, kind):
    """Every segment (lengths 1 and 2 included), degrees 1..7: the fp32 emulation of phase_fit + gram_eval against the
    fp64 Legendre least-squares curve within fused_poly_tol, its residual norm within sqrt(n) tol of the optimum,
    coefficients above the clamped degree exactly 0."""
    y = poly_values(kind, n, _rng("fit", kind, n))
    y64 = y.astype(np.float64)
    for deg in range(1, MAX_DEG + 1):
        for s, off, ln, c, f in _fit_all(y, deg):
            assert not np.any(c[min(deg, ln - 1) + 1:]), (deg, s, ln, c)
            err, tol, dr, rtol = check_segment(y64[off:off + ln], f.astype(np.float64), c, deg)
            assert err <= tol, (deg, s, ln, err, tol)
            assert dr <= rtol, (deg, s, ln, dr, rtol)


@pytest.mark.parametrize("kind,n,deg", [("offset", 23_592, 5), ("randn", 23_592, 2), ("randn", 300, 1),
                                        ("heavy", 131_072, 7), ("const", 131_072, 3), ("offset", 131_072, 3)])
def test_fused_poly_tol_has_teeth(kind, n, deg):
    """Scaling the largest coefficient of the largest segment by 1.01 must break fused_poly_tol."""
    y = poly_values(kind, n, _rng("fit", kind, n))
    s, off, ln, c, _ = max(_fit_all(y, deg), key=lambda t: t[2])
    k = int(np.argmax(np.abs(c)))
    c2 = c.copy()
    c2[k] = F(c2[k] * F(1.01))
    f = eval_emulated(c2, ln, deg).astype(np.float64)
    err, tol, _, _ = check_segment(y[off:off + ln].astype(np.float64), f, c, deg)
    assert err > tol, (err, tol, c)


def test_eval_tol_holds_for_gram_eval():
    """eval_tol against an fp64 evaluation of the same coefficients, at the fused engine's segment lengths."""
    rng = _rng("eval")
    for n in (1, 2, 3, 31, 32, 1000, 65_537, 131_072):
        for deg in range(1, MAX_DEG + 1):
            de = min(deg, n - 1)
            c = np.zeros(deg + 1, F)
            c[:de + 1] = (rng.standard_normal(de + 1) * np.exp2(rng.uniform(-8, 8, de + 1))).astype(F)
            got = eval_emulated(c, n, deg).astype(np.float64)
            want = polyfit.gram_basis(n, deg).numpy() @ c.astype(np.float64)
            assert float(np.abs(got - want).max()) <= eval_tol(n, c[:de + 1]), (n, deg)


# ---------------------------------------------------------------------------
# rank_bin / order_key, compiled from engine.cu
# ---------------------------------------------------------------------------
_PRELUDE = r"""
#include <cstdint>
#include <cstring>
#include <algorithm>
#define DR_D static inline
using std::min;
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
"""
_WRAP = r"""
#ifdef HAS_ORDER_KEY
#define BIN(v, T) rank_bin(order_key(v), T)
#else
#define BIN(v, T) rank_bin(v, T)
#endif
extern "C" void bins(const float* v, const uint32_t* T, uint32_t* out, long n) {
  for (long i = 0; i < n; ++i) out[i] = BIN(v[i], T[i]);
}
"""


def _function(src, name):
    m = re.search(r"^DR_D uint32_t " + name + r"\(.*?^}\n", src, re.S | re.M)
    return m.group(0) if m else None


@pytest.fixture(scope="module")
def kernel_bins(tmp_path_factory):
    """engine.cu's rank_bin (and order_key, when the source has one) built for the host; returns bins(v, T)."""
    src = open(ENGINE_CU).read()
    rb, ok = _function(src, "rank_bin"), _function(src, "order_key")
    assert rb is not None, "rank_bin not found in engine.cu"
    d = str(tmp_path_factory.mktemp("rank_bin"))
    cpp, so = os.path.join(d, "rank_bin.cpp"), os.path.join(d, "rank_bin.so")
    with open(cpp, "w") as f:
        f.write(_PRELUDE + (ok or "") + rb + ("#define HAS_ORDER_KEY\n" if ok else "") + _WRAP)
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", cpp, "-o", so], check=True, capture_output=True)
    lib = ctypes.CDLL(so)
    fp = np.ctypeslib.ndpointer(dtype=np.float32, flags="C")
    up = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C")
    lib.bins.argtypes = [fp, up, up, ctypes.c_long]

    def bins(v, T):
        v = np.ascontiguousarray(v, dtype=np.float32)
        Ts = np.ascontiguousarray(np.broadcast_to(np.uint32(T), v.shape), dtype=np.uint32)
        out = np.empty(v.shape, np.uint32)
        lib.bins(v, Ts, out, v.size)
        return out
    return bins


def _f(bits):
    return np.asarray(bits, dtype=np.uint32).view(np.float32)


# selection thresholds (31-bit magnitude keys): the smallest top-k threshold, a denormal, small, 1.0, large, FLT_MAX
THRESHOLDS = [1 << 9, 0x0000_1000, int(np.float32(1e-20).view(np.uint32)), int(np.float32(1e-3).view(np.uint32)),
              int(np.float32(1.0).view(np.uint32)), int(np.float32(3e30).view(np.uint32)), 0x7F7F_FFFF]


def _probe_values(T):
    """+-0, denormals, values just above and below T, around 4T (T + 2^24 in the key) and at the coarse clamps, +-1,
    +-FLT_MAX, +-inf, and random values over the whole range: every one with both signs."""
    keys = {0, 1, 2, 0x7F_FFFF, 0x80_0000, 0x3F80_0000, 0x7F7F_FFFF, 0x7F80_0000}
    for base in (T, T + (2 << 23), T + (2 << 23) + (1023 << 19), T - (1023 << 19), T - (1024 << 19)):
        for dlt in (-(1 << 19) - 1, -(1 << 13) - 1, -(1 << 13), -1, 0, 1, 1 << 13, (1 << 19) + 1):
            keys.add(base + dlt)
    keys |= set(_rng("probe", T).integers(0, 0x7F80_0001, 400).tolist())
    keys = np.array(sorted(k for k in keys if 0 <= k <= 0x7F80_0000), dtype=np.uint32)
    mag = _f(keys)
    return np.concatenate([mag, -mag])


@pytest.mark.parametrize("T", THRESHOLDS)
def test_rank_bin_is_monotone(kernel_bins, T):
    """v1 > v2 => bin(v1) <= bin(v2), and every bin inside the 8192-entry table (NaN included)."""
    v = _probe_values(T)
    b = kernel_bins(v, T).astype(np.int64)
    assert b.max() < 8192
    gt = v[:, None] > v[None, :]
    bad = np.argwhere(gt & (b[:, None] > b[None, :]))
    assert bad.size == 0, [(float(v[i]), float(v[j]), int(b[i]), int(b[j])) for i, j in bad[:5]]
    nan = kernel_bins(np.array([np.nan, -np.nan, _f(0x7FC0_0001), _f(0xFFFF_FFFF)], np.float32), T)
    assert nan.max() < 8192


@pytest.mark.parametrize("T", THRESHOLDS)
def test_rank_bin_equal_values_share_a_bin(kernel_bins, T):
    """v1 == v2 => bin(v1) == bin(v2).  The only equal pairs of distinct bits are +0.0 and -0.0: the stable descending
    sort treats them as equal and orders them by position, so the exact rank must see them in one bin."""
    v = _probe_values(T)
    b = kernel_bins(v, T).astype(np.int64)
    eq = v[:, None] == v[None, :]
    bad = np.argwhere(eq & (b[:, None] != b[None, :]))
    assert bad.size == 0, [(float(v[i]), float(v[j]), int(b[i]), int(b[j])) for i, j in bad[:5]]
