// Double-exponential fit ("Fit-DExp"): y_k ~ a e^{p x_k} + b e^{q x_k} on x_k = (k+1)/K, shared by the per-tensor kernel
// (ops.cu::dexp_fit_kernel, one CTA of 1 024 threads) and the fused engine's fit phase (engine.cu::phase_fit, one CTA
// of kThreads per sign run of a 'dexp' tensor).
// Reference: tensorflow/deepreduce.py:66-144 (Jacquelin-style integral-equation regression: cumulative trapezoids
// S = int y, SS = int S; 4x4 normal system of  y ~ A SS + B S + C x + D;  p,q = (B +- sqrt(B^2 + 4A))/2;  then a
// 2x2 least squares for a, b) — a chain of TF GPU ops (cumsum, matmul, linalg.solve) upstream; here ONE CTA does the
// two scans, the 14 moment sums, both small solves and the second pass.  fp64 throughout like the reference (the sums
// span ~1e6 terms of very different magnitude); codecs/dexp.py::double_exponential_fit is the torch oracle.
#pragma once
#include "common.cuh"

namespace dr {

__device__ __forceinline__ double warp_incl_scan_f64(double v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double n = __shfl_up_sync(0xFFFFFFFFu, v, o);
    if (lane >= o) v += n;
  }
  return v;
}

// block-wide inclusive scan of one value per thread (blockDim = kBlock); `tot` gets the block total
template <int kBlock>
__device__ double block_incl_scan_f64(double v, double* warp_sums, double& tot) {
  constexpr int kW = kBlock / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_incl_scan_f64(v, lane);
  __syncthreads();
  if (lane == 31) warp_sums[warp] = v;
  __syncthreads();
  if (warp == 0) {
    double w = lane < kW ? warp_sums[lane] : 0.0;
    w = warp_incl_scan_f64(w, lane);
    warp_sums[lane] = w;
  }
  __syncthreads();
  const double base = warp ? warp_sums[warp - 1] : 0.0;
  tot = warp_sums[kW - 1];
  return v + base;
}

template <int kBlock>
__device__ double block_sum_f64(double v, double* scratch) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < kBlock / 32; ++w) t += scratch[w];
  return t;
}

// shared memory of one fit
struct DexpScratch {
  double ws[32];
  double sums[14];
  double pq[2];
};

// Fit of the K values y(0) .. y(K-1) (ascending; y(k) returns the k-th as a double).  Called by all kBlock threads of
// the CTA; thread 0 receives (a, b, p, q) in `out` (K <= 0: the zero curve).
template <int kBlock, typename LoadY>
__device__ __forceinline__ void dexp_fit_block(LoadY y, int64_t K, DexpScratch& sh, double out[4]) {
  const int tid = threadIdx.x;
  if (K <= 0) { out[0] = out[1] = out[2] = out[3] = 0.0; return; }
  double* ws = sh.ws;
  double* sums = sh.sums;
  const double dx = 1.0 / (double)K;
  double acc[14];
#pragma unroll
  for (int i = 0; i < 14; ++i) acc[i] = 0.0;
  double carry_S = 0.0, carry_SS = 0.0;     // S, SS at the last element of the previous chunk
  for (int64_t c0 = 0; c0 < K; c0 += kBlock) {
    const int64_t k = c0 + tid;
    const bool on = k < K;
    const double yk = on ? y(k) : 0.0;
    const double ym = (on && k > 0) ? y(k - 1) : 0.0;
    const double inc = (on && k > 0) ? 0.5 * (yk + ym) * dx : 0.0;
    double tot;
    const double S = carry_S + block_incl_scan_f64<kBlock>(inc, ws, tot);
    const double S_prev = S - inc;                                  // S_{k-1}
    const double inc2 = (on && k > 0) ? 0.5 * (S + S_prev) * dx : 0.0;
    double tot2;
    const double SS = carry_SS + block_incl_scan_f64<kBlock>(inc2, ws, tot2);
    carry_S += tot; carry_SS += tot2;
    if (on) {
      const double x = (double)(k + 1) * dx;
      const double col[4] = {SS, S, x, 1.0};
      int q = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = i; j < 4; ++j) acc[q++] += col[i] * col[j];     // 10 entries of the Gram matrix
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[10 + i] += col[i] * yk;         // right-hand side
    }
  }
  for (int i = 0; i < 14; ++i) {
    const double t = block_sum_f64<kBlock>(acc[i], ws);
    if (tid == 0) sums[i] = t;
  }
  __syncthreads();
  if (tid == 0) {
    double G[4][5];
    int q = 0;
    for (int i = 0; i < 4; ++i) for (int j = i; j < 4; ++j) { G[i][j] = sums[q]; G[j][i] = sums[q]; ++q; }
    for (int i = 0; i < 4; ++i) { G[i][i] += 1e-18; G[i][4] = sums[10 + i]; }
    for (int c = 0; c < 4; ++c) {                                     // Gaussian elimination, partial pivoting
      int piv = c;
      for (int r = c + 1; r < 4; ++r) if (fabs(G[r][c]) > fabs(G[piv][c])) piv = r;
      if (piv != c) for (int j = 0; j < 5; ++j) { const double t = G[c][j]; G[c][j] = G[piv][j]; G[piv][j] = t; }
      const double d = G[c][c];
      if (d != 0.0) for (int r = c + 1; r < 4; ++r) { const double f = G[r][c] / d; for (int j = c; j < 5; ++j) G[r][j] -= f * G[c][j]; }
    }
    double sol[4];
    for (int i = 3; i >= 0; --i) {
      double t = G[i][4];
      for (int j = i + 1; j < 4; ++j) t -= G[i][j] * sol[j];
      sol[i] = G[i][i] != 0.0 ? t / G[i][i] : 0.0;
    }
    const double A = sol[0], B = sol[1];
    const double disc = fmax(B * B + 4.0 * A, 0.0);
    sh.pq[0] = 0.5 * (B + sqrt(disc));
    sh.pq[1] = 0.5 * (B - sqrt(disc));
  }
  __syncthreads();
  const double p = sh.pq[0], qq = sh.pq[1];
  double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int64_t k = tid; k < K; k += kBlock) {
    const double x = (double)(k + 1) * dx, yk = y(k);
    const double bk = exp(p * x), ek = exp(qq * x);
    m[0] += bk * bk; m[1] += bk * ek; m[2] += ek * ek; m[3] += bk * yk; m[4] += ek * yk;
  }
  for (int i = 0; i < 5; ++i) {
    const double t = block_sum_f64<kBlock>(m[i], ws);
    if (tid == 0) sums[i] = t;
  }
  __syncthreads();
  if (tid == 0) {
    // p == q: the two basis functions are one and the 2x2 system is singular, but the contracted (FMA) determinant of
    // the equal sums is a rounding residue, not 0 — take the one-exponential fallback as the oracle's exact det does
    const double det = sums[0] * sums[2] - sums[1] * sums[1];
    double a, b;
    if (fabs(det) < 1e-300 || p == qq) { a = sums[0] != 0.0 ? sums[3] / sums[0] : 0.0; b = 0.0; }
    else { a = (sums[3] * sums[2] - sums[4] * sums[1]) / det; b = (sums[0] * sums[4] - sums[1] * sums[3]) / det; }
    out[0] = a; out[1] = b; out[2] = p; out[3] = qq;
  }
}

}  // namespace dr
