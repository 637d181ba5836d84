"""Piece-wise polynomial value codec (``'value': 'polyfit'`` / ``'polyfit_cpu'``).

Parity with reference pytorch/deepreduce.py:306-425 (``PolyFit``) and :558-688
(``PolyFitCPU``): sort values descending, split at the sign change and into the
``get_segments`` table (:362-377), least-squares fit a degree-``poly_degree``
polynomial per segment, ship coefficients + the permuted indices.

GPU-first changes (SURVEY §7.4 "Polyfit numerics"):

* the reference builds a monomial Vandermonde on x=1..n in fp64 and inverts the
  6×6 normal matrix **on the CPU** per segment (:326-338).  fp64 is the slow
  path on the GPU, so the fit uses the *Gram (discrete Chebyshev) polynomials*
  p_0..p_deg, which are **exactly orthogonal on the grid 0..n-1**::

      p_0 = 1,  p_1 = 1 - 2x/N,                       N = n-1
      (k+1)(N-k) p_{k+1} = (2k+1)(N-2x) p_k - k(N+k+1) p_{k-1}

  so the normal matrix is diagonal and ``c_k = Σ p_k y / Σ p_k²`` — one fused
  reduction pass, no solve, no host hop, |p_k| ≤ 1 so fp32 is enough.  The
  fitted *values* equal the monomial least-squares fit (same polynomial space).
* wire layout: ``float32[(deg+1)*seg_rows(N) + 1]`` where ``seg_rows(N)`` is the
  largest segment count ``get_segments`` can produce for N values (a function of N
  only: unused rows are zero, last word = num_pos bit-cast from int32), so every rank
  ships the same size and ``tensors_size_are_same`` is honestly True (the reference's
  size depends on num_pos — a latent bug, SURVEY §3.7) while a 368-value tensor
  carries 6 rows instead of the 22 of the largest table.
* zero-length / tiny segments are legal (degree clamps to n-1).
"""
from __future__ import annotations

import numpy as np
import torch

from .base import SparseCompressor, register, use_cuda

RATIOS = [1 / 5, 1 / 10, 1 / 30, 1 / 100, 1 / 300, 1 / 1000, 1 / 3000, 1 / 10000, 1 / 30000, 1 / 100000]
MAX_SEGMENTS = 2 * len(RATIOS) + 2
MAX_DEGREE = 7


def get_segments(N: int, num_pos: int = 0):
    """Segment lengths for a descending-sorted value vector with ``num_pos``
    positives — same table as reference :362-377."""
    pos, neg = [], []
    num_neg = N - num_pos
    for r in RATIOS:
        if int(num_pos * r) > 30:
            pos.append(int(num_pos * r))
        if int(num_neg * r) > 30:
            neg.append(int(num_neg * r))
    return pos[::-1] + [num_pos - sum(pos)] + [num_neg - sum(neg)] + neg


def seg_rows(N: int) -> int:
    """Upper bound of ``len(get_segments(N, p))`` over all p: both halves may use every ratio that passes for N."""
    return min(MAX_SEGMENTS, 2 * sum(1 for r in RATIOS if int(N * r) > 30) + 2)


def gram_basis(n: int, degree: int, device=None, dtype=torch.float64) -> torch.Tensor:
    """[n, degree+1] Gram polynomials on x = 0..n-1 (columns beyond n-1 are 0)."""
    P = torch.zeros(n, degree + 1, dtype=dtype, device=device)
    if n == 0:
        return P
    P[:, 0] = 1
    N = n - 1
    if degree >= 1 and N >= 1:
        x = torch.arange(n, dtype=dtype, device=device)
        P[:, 1] = (N - 2 * x) / N
        for k in range(1, min(degree, N)):
            P[:, k + 1] = ((2 * k + 1) * (N - 2 * x) * P[:, k] - k * (N + k + 1) * P[:, k - 1]) / ((k + 1) * (N - k))
    return P


def fit_segment_oracle(y: torch.Tensor, degree: int) -> torch.Tensor:
    n = y.numel()
    c = torch.zeros(degree + 1, dtype=torch.float64, device=y.device)
    if n == 0:
        return c
    P = gram_basis(n, degree, y.device)
    num = P.T @ y.double()
    den = (P * P).sum(dim=0)
    ok = den > 0
    c[ok] = num[ok] / den[ok]
    return c


def polyfit_fit_oracle(y_sorted: torch.Tensor, segments, degree: int) -> torch.Tensor:
    """-> float32[MAX_SEGMENTS*(degree+1)]"""
    out = torch.zeros(MAX_SEGMENTS, degree + 1, dtype=torch.float32, device=y_sorted.device)
    off = 0
    for s, n in enumerate(segments):
        out[s] = fit_segment_oracle(y_sorted[off:off + n], degree).float()
        off += n
    return out.flatten()


def polyfit_eval_oracle(coeffs: torch.Tensor, segments, degree: int) -> torch.Tensor:
    C = coeffs.view(MAX_SEGMENTS, degree + 1).double()
    ys = []
    for s, n in enumerate(segments):
        if n:
            ys.append(gram_basis(n, degree, coeffs.device) @ C[s])
    if not ys:
        return torch.empty(0, dtype=torch.float32, device=coeffs.device)
    return torch.cat(ys).float()


def _pack_num_pos(coeffs: torch.Tensor, num_pos: int) -> torch.Tensor:
    tail = torch.tensor([num_pos], dtype=torch.int32, device=coeffs.device).view(torch.float32)
    return torch.cat([coeffs, tail])


def _split_num_pos(wire: torch.Tensor):
    return wire[:-1], int(wire[-1:].view(torch.int32).item())


@register("polyfit")
class PolyFit(SparseCompressor):
    order_preserving = False
    kind = "value"

    @staticmethod
    def compress(sparse_tensor, params):
        degree = min(int(params.get('poly_degree', 5)), MAX_DEGREE)
        vals, idxs, shape = sparse_tensor
        N = idxs.numel()
        y_all = vals.float()
        if not params.get('sort', False):
            y_all, mapping = y_all.sort(descending=True)
            idxs = idxs[mapping]
        num_pos = int((y_all > 0).sum().item())
        segments = get_segments(N, num_pos)
        if use_cuda(y_all):
            from .. import ops
            coeffs = ops.polyfit_fit(y_all, segments, degree)
        else:
            coeffs = polyfit_fit_oracle(y_all, segments, degree)
        coeffs = coeffs[:seg_rows(N) * (degree + 1)]            # rows beyond seg_rows(N) can never be used
        return _pack_num_pos(coeffs, num_pos), idxs, shape

    @staticmethod
    def decompress(fitted_sparse_tensor, params):
        degree = min(int(params.get('poly_degree', 5)), MAX_DEGREE)
        wire, idxs, shape = fitted_sparse_tensor
        N = idxs.numel()
        coeffs, num_pos = _split_num_pos(wire)
        segments = get_segments(N, num_pos)
        full = MAX_SEGMENTS * (degree + 1)
        if coeffs.numel() < full:                                # kernels / oracle index a MAX_SEGMENTS table
            coeffs = torch.cat([coeffs, coeffs.new_zeros(full - coeffs.numel())])
        if use_cuda(coeffs):
            from .. import ops
            vals = ops.polyfit_eval(coeffs, segments, degree, N)
        else:
            vals = polyfit_eval_oracle(coeffs, segments, degree)
        return vals, idxs, shape


# ----------------------------------------------------------------------------
# CPU variant with data-driven knots (reference :558-688)
# ----------------------------------------------------------------------------
def find_breaks(curve: np.ndarray, num_of_breaks: int = 10):
    """Greedy knot search: repeatedly take the point farthest from the chord of
    the remaining suffix (reference :566-582; paper Lemma 1)."""
    y = curve
    breaks = []
    break_index = 0
    for _ in range(num_of_breaks):
        if len(y) < 20 * num_of_breaks:
            break
        line = np.linspace(y[0], y[-1], len(y))
        break_index += int(np.argmax(np.abs(line - y)))
        if (len(curve) - break_index) < 20 * num_of_breaks:
            break
        breaks.append(break_index)
        y = curve[break_index:]
    return breaks


def fit_curve(curve, breaks, poly_degree=5):
    breaks = [0] + list(breaks) + [len(curve)]
    coefficients = []
    for lo, hi in zip(breaks[:-1], breaks[1:]):
        n = hi - lo
        deg = max(0, min(poly_degree, n - 1))
        c = np.zeros(poly_degree + 1)
        if n > 0:
            # local, centred abscissa keeps the monomial fit well conditioned
            t = (np.arange(n) - (n - 1) / 2.0) / max(1.0, (n - 1) / 2.0)
            c[: deg + 1] = np.polynomial.polynomial.polyfit(t, curve[lo:hi], deg)
        coefficients.append(c)
    return coefficients, breaks


def restore_curve(coefficients, breaks):
    out = []
    for c, lo, hi in zip(coefficients, breaks[:-1], breaks[1:]):
        n = hi - lo
        if n > 0:
            t = (np.arange(n) - (n - 1) / 2.0) / max(1.0, (n - 1) / 2.0)
            out.append(np.polynomial.polynomial.polyval(t, c))
    return np.concatenate(out) if out else np.zeros(0)


@register("polyfit_cpu")
class PolyFitCPU(SparseCompressor):
    order_preserving = False
    kind = "value"

    @staticmethod
    def compress(sparse_tensor, params):
        vals, idxs, shape = sparse_tensor
        num_of_breaks = int(params.get('num_of_breaks', 5))
        poly_degree = int(params.get('poly_degree', 5))
        vals_sorted, mask = torch.sort(vals, descending=True)
        indices_sorted = idxs[mask]
        v = vals_sorted.detach().cpu().double().numpy()
        num_pos = int((v > 0).sum())
        if num_pos == 0:
            breaks = find_breaks(v, num_of_breaks)
        elif num_pos == len(v):
            b = find_breaks(v[::-1], num_of_breaks)
            breaks = [len(v) - x for x in b[::-1]]
        else:
            pos, neg = v[:num_pos], v[num_pos:]
            b = find_breaks(pos[::-1], num_of_breaks)
            breaks_pos = [len(pos) - x for x in b[::-1]]
            breaks_neg = [num_pos + x for x in find_breaks(neg, num_of_breaks)]
            breaks = breaks_pos + [num_pos] + breaks_neg
        breaks = sorted(set(x for x in breaks if 0 < x < len(v)))
        coefficients, breaks = fit_curve(v, breaks, poly_degree)
        # one flat float64 wire tensor [n_breaks, breaks..., coefficients...] — resolves the reference's
        # "todo: encode coeff_tensor and breaks_tensor into one tensor" (:672) so allgather can ship it
        flat = np.concatenate([[float(len(breaks))], np.asarray(breaks, dtype=np.float64),
                               np.asarray(coefficients, dtype=np.float64).reshape(-1)])
        return torch.tensor(flat, dtype=torch.float64, device=idxs.device), indices_sorted, shape

    @staticmethod
    def decompress(sparse_tensor, params):
        wire, idxs, shape = sparse_tensor
        if isinstance(wire, (tuple, list)):          # reference-style (coeff, breaks) tuple is still accepted
            coeff_tensor, breaks_tensor = wire
            breaks = breaks_tensor.cpu().numpy().astype(np.int64).tolist()
            coefficients = coeff_tensor.cpu().numpy().reshape(len(breaks) - 1, -1)
        else:
            w = wire.detach().cpu().numpy()
            nb = int(w[0])
            breaks = w[1:1 + nb].astype(np.int64).tolist()
            coefficients = w[1 + nb:].reshape(len(breaks) - 1, -1)
        vals = restore_curve(coefficients, breaks)
        return torch.tensor(vals, dtype=torch.float32, device=idxs.device), idxs, shape


# ----------------------------------------------------------------------------
# monomial-basis helpers with the reference's module-level names (:308-347).  The codec above does not use them
# (Gram basis, fp32, no explicit inverse); they exist so code written against the reference keeps working and so the
# tests can show that both bases span the same fit.
# ----------------------------------------------------------------------------
def GetInputMatrix_Polynomial(N: int, degree: int, device=None) -> torch.Tensor:
    """[N, degree+1] Vandermonde matrix on x = 1..N in float64 (reference :308-323)."""
    x = torch.arange(1, int(N) + 1, dtype=torch.float64, device=device)
    return torch.stack([x ** j for j in range(int(degree) + 1)], dim=1)


def LeastSquares(X: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """argmin ||X a - y||: the reference forms (X'X)^-1 X'y with the small inverse on the CPU (:326-338); here a
    rank-revealing solve on the input's own device (columns scaled first: x^5 reaches 1e25 for N = 1e5)."""
    X = X.double()
    scale = X.abs().amax(dim=0).clamp_min(1e-300)
    sol = torch.linalg.lstsq(X / scale, y.double().reshape(-1, 1)).solution[:, 0]
    return sol / scale


def RestoreValues(N: int, coefficients: torch.Tensor) -> torch.Tensor:
    """X(N) @ coefficients (reference :341-347)."""
    c = coefficients.double().flatten()
    return GetInputMatrix_Polynomial(N, c.numel() - 1, c.device) @ c
