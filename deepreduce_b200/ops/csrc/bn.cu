// Training-mode BatchNorm for NHWC (channels_last) bf16 activations, fused with the ReLU and the residual add that
// follow it in ResNet-50.  The results are bitwise those of the unfused graph (native_batch_norm -> relu_ -> add ->
// relu_), because every expression and every bf16 rounding point is kept:
//   * per-channel mean / biased var come from torch's own channels-last Welford kernel (binding.cpp), so the
//     reduction order is torch's;
//   * running stats and invstd: the expressions of torch's batch_norm_update_stats_and_invert;
//   * apply: torch's channels-last transform w * (x - mean) * invstd + shift, which compiles to
//     fma(w * (x - mean), invstd, shift) (checked in the sm_90 SASS of batch_norm_transform_input_channels_last_kernel),
//     rounded to bf16;
//   * residual add: fp32 sum of the two bf16 values, rounded to bf16 once (torch's bf16 add);
//   * ReLU on the bf16 value (clamp_min(0): NaN passes through).
// What changes is the memory traffic: one read of each input and one 16-byte-vectorised write per output, where the
// unfused graph writes and re-reads the BN output, the sum and the ReLU output.
//
// The apply pass also writes the ReLU mask (one bit per element: !(out <= 0), threshold_backward's condition), and
// backward runs on it instead of threshold_backward + native_batch_norm_backward:
//   * reduce: per-channel sum(g) and sum(g * (x - mean)) with g = mask ? go : +0, in the reduction tree of torch's
//     batch_norm_backward_reduce_channels_last_kernel (see BwdTree), so the sums are bitwise torch's;
//   * elementwise: torch's dx expression, pinned to the FMA placement of its sm_90 SASS.
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "ops.h"

namespace dr {

namespace {

constexpr int kVec = 8;            // bf16 channels per thread: one 16-byte load / store
constexpr int kApplyThreads = 256;
constexpr int kReduceThreads = 128;   // at most; the reduce keeps 130-250 registers per thread

struct ChanParams {
  float m[kVec], inv[kVec], w[kVec], b[kVec];
};

__device__ __forceinline__ void load8(const float* __restrict__ p, float* d) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w;
  d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
}

__device__ __forceinline__ void load_params(const BnParams& p, int c, ChanParams& o) {
  load8(p.mean + c, o.m);
  load8(p.invstd + c, o.inv);
  load8(p.weight + c, o.w);
  load8(p.bias + c, o.b);
}

__device__ __forceinline__ float bn_elem(float x, float m, float inv, float w, float b) {
  return __fmaf_rn(__fmul_rn(w, __fsub_rn(x, m)), inv, b);
}

__device__ __forceinline__ __nv_bfloat16 relu_bf16(__nv_bfloat16 v) {
  return __bfloat162float(v) <= 0.f ? __float2bfloat16_rn(0.f) : v;
}

// kMode 0: relu(bn(x));  1: relu(bn(x) + z);  2: relu(bn(x) + bn_z(z)).
// Each thread owns one group of 8 channels for the whole launch (its parameters stay in registers) and walks rows.
// mask[row][C / 8]: bit i of a byte is channel 8 * group + i, set where !(out <= 0) (so a NaN output passes gradient).
template <int kMode>
__global__ void __launch_bounds__(kApplyThreads) bn_apply_kernel(const __nv_bfloat16* __restrict__ x, BnParams px,
                                                                 const __nv_bfloat16* __restrict__ z, BnParams pz,
                                                                 __nv_bfloat16* __restrict__ out,
                                                                 uint8_t* __restrict__ mask, int64_t rows, int C) {
  const int groups = C / kVec;
  const int rows_per_cta = blockDim.x / groups;
  const int rsub = threadIdx.x / groups;
  if (rsub >= rows_per_cta) return;
  const int c = (threadIdx.x % groups) * kVec;
  ChanParams a;
  load_params(px, c, a);
  ChanParams d;
  if (kMode == 2) load_params(pz, c, d);
  const int64_t step = (int64_t)gridDim.x * rows_per_cta;
#pragma unroll 2
  for (int64_t r = (int64_t)blockIdx.x * rows_per_cta + rsub; r < rows; r += step) {
    const int64_t off = r * C + c;
    const uint4 vx = *reinterpret_cast<const uint4*>(x + off);
    uint4 vz = make_uint4(0, 0, 0, 0);
    if (kMode != 0) vz = *reinterpret_cast<const uint4*>(z + off);
    const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&vx);
    const __nv_bfloat16* hz = reinterpret_cast<const __nv_bfloat16*>(&vz);
    uint4 vo;
    __nv_bfloat16* ho = reinterpret_cast<__nv_bfloat16*>(&vo);
    unsigned bits = 0;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      __nv_bfloat16 y = __float2bfloat16_rn(bn_elem(__bfloat162float(hx[i]), a.m[i], a.inv[i], a.w[i], a.b[i]));
      if (kMode != 0) {
        const __nv_bfloat16 s = kMode == 1 ? hz[i]
                                           : __float2bfloat16_rn(bn_elem(__bfloat162float(hz[i]), d.m[i], d.inv[i], d.w[i], d.b[i]));
        y = __float2bfloat16_rn(__fadd_rn(__bfloat162float(y), __bfloat162float(s)));
      }
      ho[i] = relu_bf16(y);
      bits |= (__bfloat162float(ho[i]) <= 0.f ? 0u : 1u) << i;
    }
    *reinterpret_cast<uint4*>(out + off) = vo;
    mask[r * groups + c / kVec] = (uint8_t)bits;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------------------------------
// The reduction tree of torch's batch_norm_backward_reduce_channels_last_kernel<4> for `rows` x C (launch config from
// flexible_launch_configs(rows, C, coop = true); block_x does not change a column's sums).  Virtual thread
// v = block * block_y + y (of S = block_y * grid_y) keeps kBwdLoads accumulators; accumulator j sums rows
// v + (i * kBwdLoads + j) * S for i = 0, 1, ... from 0.0f (rows past the end add g = 0, x = 0, as torch's loads do).  Then
// ((a0 + a1) + a2) + a3, a pairwise tree over y inside each block (offsets block_y / 2 ... 1), and for grid_y > 1 the
// same tree over y of 0.0f + s[y] + s[y + block_y] + ... of the block results s.  Nothing here is specific to the
// backward sums: a statistics kernel that mirrors torch's Welford tree indexes rows the same way.
struct BwdTree {
  int block_y, grid_y;
  __host__ __device__ int S() const { return block_y * grid_y; }
  __host__ __device__ int loops(int rows) const { return 1 + (rows - 1) / (S() * kBwdLoads); }
  static constexpr int kBwdLoads = 4;       // torch's ELEMENTS_PER_ITER
};

// Pairwise tree over y of kN columns per (y, column group) thread, as torch's merge_block_vertical_backward: the
// result is at y == 0.  sh holds n * width floats; every thread of the block calls this.
template <int kN>
__device__ __forceinline__ void tree_over_y(float* v, float* sh, int y, int n, int col, int width) {
  for (int off = n / 2; off > 0; off >>= 1) {
#pragma unroll
    for (int i = 0; i < kN; ++i) sh[y * width + col + i] = v[i];
    __syncthreads();
    if (y < off) {
#pragma unroll
      for (int i = 0; i < kN; ++i) v[i] = __fadd_rn(v[i], sh[(y + off) * width + col + i]);
    }
    __syncthreads();
  }
}

struct BwdOut {
  float* sums;          // [kSums][C]: sum_dy, sum_dy_xmu (, sum_dy_xmu_z)
  float* dw; float* db; float* dwz; float* dbz;
  float* staging;       // [kSums][grid_y][C] when grid_y > 1
};

// Writes the final per-channel results of sum k: the sums, and dw = sum_dy_xmu * invstd, db = sum_dy (fp32, torch's
// mixed-type branch: fp32 weight with bf16 input).
__device__ __forceinline__ void bwd_store(const BwdOut& o, int k, int c, int C, float v, const float* invstd,
                                         const float* invstd_z) {
  o.sums[k * C + c] = v;
  if (k == 0) {
    o.db[c] = v;
    if (o.dbz) o.dbz[c] = v;
  } else if (k == 1) {
    o.dw[c] = __fmul_rn(v, invstd[c]);
  } else {
    o.dwz[c] = __fmul_rn(v, invstd_z[c]);
  }
}

__device__ __forceinline__ float masked(__nv_bfloat16 go, unsigned bit) { return bit ? __bfloat162float(go) : 0.f; }

// One physical thread = 8 channels (16-byte loads, one mask byte) of one virtual thread.  Block = gpc channel groups x
// block_y virtual threads of one virtual block (blockIdx.y).  kMode 0: sums of g; 1: also writes g; 2: also the z sums.
template <int kMode>
__global__ void __launch_bounds__(kReduceThreads) bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ go,
                                                                       const uint8_t* __restrict__ mask,
                                                                       const __nv_bfloat16* __restrict__ x,
                                                                       const float* __restrict__ mean,
                                                                       const float* __restrict__ invstd,
                                                                       const __nv_bfloat16* __restrict__ z,
                                                                       const float* __restrict__ mean_z,
                                                                       const float* __restrict__ invstd_z,
                                                                       __nv_bfloat16* __restrict__ g_out, BwdOut o,
                                                                       BwdTree t, int rows, int C) {
  constexpr int kSums = kMode == 2 ? 3 : 2;
  constexpr int L = BwdTree::kBwdLoads;
  extern __shared__ float sh[];                    // block_y x (gpc * kVec)
  const int gpc = blockDim.x / t.block_y;
  const int tg = threadIdx.x % gpc, y = threadIdx.x / gpc;
  const int group = blockIdx.x * gpc + tg;
  const bool live = group * kVec < C;
  const int c = live ? group * kVec : 0;
  const int S = t.S();
  float m[kVec], mz[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    m[i] = mean[c + i];
    mz[i] = kMode == 2 ? mean_z[c + i] : 0.f;
  }
  float acc[kSums][L][kVec];
#pragma unroll
  for (int k = 0; k < kSums; ++k)
#pragma unroll
    for (int j = 0; j < L; ++j)
#pragma unroll
      for (int i = 0; i < kVec; ++i) acc[k][j][i] = 0.f;
  const int mgroups = C / kVec;
  int r = blockIdx.y * t.block_y + y;
  const int n_loops = t.loops(rows);
  // The tree fixes the thread count (S * C / kVec; 16 K threads for C = 64), so each thread keeps two iterations of loads
  // in flight: the next one is issued before the current one is summed.  Rows past the end load nothing and give 0.
  struct Batch {
    uint4 g[L], x[L], z[L];
    unsigned m[L];
  };
  auto load = [&](Batch& b, int r0) {
#pragma unroll
    for (int j = 0; j < L; ++j) {
      const int rr = r0 + j * S;
      if (live && rr < rows) {
        const int off = rr * C + c;
        b.g[j] = *reinterpret_cast<const uint4*>(go + off);
        b.x[j] = *reinterpret_cast<const uint4*>(x + off);
        if (kMode == 2) b.z[j] = *reinterpret_cast<const uint4*>(z + off);
        b.m[j] = mask[rr * mgroups + group];
      } else {
        b.g[j] = uint4{}; b.x[j] = uint4{}; b.z[j] = uint4{}; b.m[j] = 0;
      }
    }
  };
  Batch cur;
  load(cur, r);
  for (int it = 0; it < n_loops; ++it) {
    Batch nxt;
    load(nxt, r + L * S);
    const unsigned* mb = cur.m;
#pragma unroll
    for (int j = 0; j < L; ++j) {
      const __nv_bfloat16* hg = reinterpret_cast<const __nv_bfloat16*>(&cur.g[j]);
      const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&cur.x[j]);
      const __nv_bfloat16* hz = reinterpret_cast<const __nv_bfloat16*>(&cur.z[j]);
      uint4 vo;
      __nv_bfloat16* ho = reinterpret_cast<__nv_bfloat16*>(&vo);
#pragma unroll
      for (int i = 0; i < kVec; ++i) {
        const unsigned bit = (mb[j] >> i) & 1u;
        const float g = masked(hg[i], bit);
        if (kMode == 1) ho[i] = bit ? hg[i] : __float2bfloat16_rn(0.f);      // threshold_backward's bits, NaN too
        // torch's sm_90 SASS: FADD d = x - mean; FADD acc += g; FFMA acc_xmu = d * g + acc_xmu
        acc[0][j][i] = __fadd_rn(acc[0][j][i], g);
        acc[1][j][i] = __fmaf_rn(__fsub_rn(__bfloat162float(hx[i]), m[i]), g, acc[1][j][i]);
        if (kMode == 2) acc[2][j][i] = __fmaf_rn(__fsub_rn(__bfloat162float(hz[i]), mz[i]), g, acc[2][j][i]);
      }
      if (kMode == 1 && live && r + j * S < rows) *reinterpret_cast<uint4*>(g_out + (r + j * S) * C + c) = vo;
    }
    cur = nxt;
    r += L * S;
  }
#pragma unroll
  for (int k = 0; k < kSums; ++k) {
#pragma unroll
    for (int i = 0; i < kVec; ++i)
#pragma unroll
      for (int j = 1; j < L; ++j) acc[k][0][i] = __fadd_rn(acc[k][0][i], acc[k][j][i]);
    tree_over_y<kVec>(acc[k][0], sh, y, t.block_y, tg * kVec, gpc * kVec);
  }
  if (y != 0 || !live) return;
#pragma unroll
  for (int k = 0; k < kSums; ++k)
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      if (t.grid_y > 1) o.staging[((size_t)k * t.grid_y + blockIdx.y) * C + c + i] = acc[k][0][i];
      else bwd_store(o, k, c + i, C, acc[k][0][i], invstd, invstd_z);
    }
}

// grid_y > 1: the cross-block step of torch's tree.  Block = cols channels x block_y; thread (col, y) sums
// 0.0f + s[y] + s[y + block_y] + ... and the tree over y combines them.
__global__ void bn_bwd_finalize_kernel(BwdOut o, BwdTree t, int n_sums, int C, const float* __restrict__ invstd,
                                       const float* __restrict__ invstd_z) {
  extern __shared__ float sh[];
  const int cols = blockDim.x / t.block_y;
  const int col = threadIdx.x % cols, y = threadIdx.x / cols;
  const int c = blockIdx.x * cols + col;
  for (int k = 0; k < n_sums; ++k) {
    float v = 0.f;
    if (c < C)
      for (int b = y; b < t.grid_y; b += t.block_y) v = __fadd_rn(v, o.staging[((size_t)k * t.grid_y + b) * C + c]);
    tree_over_y<1>(&v, sh, y, t.block_y, col, cols);
    if (y == 0 && c < C) bwd_store(o, k, c, C, v, invstd, invstd_z);
  }
}

// Elementwise: torch's dx = (g - sum_dy * norm_fct - (x - mean) * f1) * f2 with f1 = ((invstd * invstd) * sum_dy_xmu)
// * norm_fct and f2 = weight * invstd.  Its sm_90 SASS contracts it to fma(-f1, x - mean, fma(-sum_dy, norm_fct, g))
// * f2, rounded to bf16 once.  kMode 1 reads the g the reduce wrote (gm = nullptr); 0 and 2 mask go; 2 also writes dz.
struct ElemtChan {
  float m[kVec], f1[kVec], f2[kVec], sdy[kVec];
};

__device__ __forceinline__ void elemt_params(const float* mean, const float* invstd, const float* w, const float* sdy,
                                             const float* sxmu, float norm, int c, ElemtChan& p) {
  float inv[kVec], ww[kVec], sx[kVec];
  load8(mean + c, p.m);
  load8(invstd + c, inv);
  load8(w + c, ww);
  load8(sdy + c, p.sdy);
  load8(sxmu + c, sx);
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    p.f1[i] = __fmul_rn(__fmul_rn(__fmul_rn(inv[i], inv[i]), sx[i]), norm);
    p.f2[i] = __fmul_rn(ww[i], inv[i]);
  }
}

__device__ __forceinline__ __nv_bfloat16 elemt(float g, float x, const ElemtChan& p, int i, float norm) {
  const float a = __fmaf_rn(-p.sdy[i], norm, g);
  return __float2bfloat16_rn(__fmul_rn(__fmaf_rn(-p.f1[i], __fsub_rn(x, p.m[i]), a), p.f2[i]));
}

struct ElemtArgs {
  const float *mean, *invstd, *weight, *sums;                // sums = [sum_dy, sum_dy_xmu(, sum_dy_xmu_z)] x C
  const float *mean_z, *invstd_z, *weight_z;
};

template <int kMode>
__global__ void __launch_bounds__(kApplyThreads) bn_bwd_elemt_kernel(const __nv_bfloat16* __restrict__ g_in,
                                                                     const uint8_t* __restrict__ mask,
                                                                     const __nv_bfloat16* __restrict__ x,
                                                                     const __nv_bfloat16* __restrict__ z, ElemtArgs a,
                                                                     __nv_bfloat16* __restrict__ dx,
                                                                     __nv_bfloat16* __restrict__ dz, float norm,
                                                                     int64_t rows, int C) {
  const int groups = C / kVec;
  const int rows_per_cta = blockDim.x / groups;
  const int rsub = threadIdx.x / groups;
  if (rsub >= rows_per_cta) return;
  const int c = (threadIdx.x % groups) * kVec;
  ElemtChan p;
  elemt_params(a.mean, a.invstd, a.weight, a.sums, a.sums + C, norm, c, p);
  ElemtChan q;
  if (kMode == 2) elemt_params(a.mean_z, a.invstd_z, a.weight_z, a.sums, a.sums + 2 * C, norm, c, q);
  const int64_t step = (int64_t)gridDim.x * rows_per_cta;
#pragma unroll 2
  for (int64_t r = (int64_t)blockIdx.x * rows_per_cta + rsub; r < rows; r += step) {
    const int64_t off = r * C + c;
    const uint4 vg = *reinterpret_cast<const uint4*>(g_in + off);
    const uint4 vx = *reinterpret_cast<const uint4*>(x + off);
    uint4 vz = make_uint4(0, 0, 0, 0);
    if (kMode == 2) vz = *reinterpret_cast<const uint4*>(z + off);
    const unsigned mb = kMode == 1 ? 0xffu : mask[r * groups + c / kVec];
    const __nv_bfloat16* hg = reinterpret_cast<const __nv_bfloat16*>(&vg);
    const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&vx);
    const __nv_bfloat16* hz = reinterpret_cast<const __nv_bfloat16*>(&vz);
    uint4 vo, vd;
    __nv_bfloat16* ho = reinterpret_cast<__nv_bfloat16*>(&vo);
    __nv_bfloat16* hd = reinterpret_cast<__nv_bfloat16*>(&vd);
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const float g = masked(hg[i], (mb >> i) & 1u);
      ho[i] = elemt(g, __bfloat162float(hx[i]), p, i, norm);
      if (kMode == 2) hd[i] = elemt(g, __bfloat162float(hz[i]), q, i, norm);
    }
    *reinterpret_cast<uint4*>(dx + off) = vo;
    if (kMode == 2) *reinterpret_cast<uint4*>(dz + off) = vd;
  }
}

// torch's batch_norm_update_stats_and_invert, per channel: running stats with the unbiased variance, and the biased
// variance turned into invstd in place.
__global__ void bn_update_stats_kernel(const float* __restrict__ mean, float* __restrict__ var_invstd,
                                       float* __restrict__ running_mean, float* __restrict__ running_var, int C,
                                       float momentum, float bessel, float eps) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float m = mean[c], v = var_invstd[c];
  const float unbiased_var = v * bessel;
  running_mean[c] = m * momentum + (1 - momentum) * running_mean[c];
  running_var[c] = unbiased_var * momentum + (1 - momentum) * running_var[c];
  var_invstd[c] = rsqrtf(v + eps);
}

// Grid of a row-walking pass (apply, backward elementwise): every row once, at most as many CTAs as fit on the device.
template <typename K>
cudaError_t rows_grid(K kernel, int64_t rows, int C, int& grid, int& threads) {
  const int groups = C / kVec;
  const int rows_per_cta = groups >= kApplyThreads ? 1 : kApplyThreads / groups;
  threads = groups * rows_per_cta;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0);
  if (e != cudaSuccess) return e;
  int64_t g = (rows + rows_per_cta - 1) / rows_per_cta;
  const int64_t cap = (int64_t)(per_sm > 0 ? per_sm : 1) * sm_count();
  grid = (int)(g > cap ? cap : g);
  return cudaSuccess;
}

template <int kMode>
cudaError_t launch_apply(const void* x, const BnParams& px, const void* z, const BnParams& pz, void* out, void* mask,
                         int64_t rows, int C, cudaStream_t st) {
  if (rows == 0) return cudaSuccess;
  int grid = 0, threads = 0;
  cudaError_t e = rows_grid(bn_apply_kernel<kMode>, rows, C, grid, threads);
  if (e != cudaSuccess) return e;
  count_launch();
  bn_apply_kernel<kMode><<<grid, threads, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), px,
                                                   reinterpret_cast<const __nv_bfloat16*>(z), pz,
                                                   reinterpret_cast<__nv_bfloat16*>(out),
                                                   reinterpret_cast<uint8_t*>(mask), rows, C);
  return cudaGetLastError();
}

int last_pow2(unsigned n) {       // torch's lastPow2 (ATen/native/cuda/LaunchUtils.h)
  n |= n >> 1; n |= n >> 2; n |= n >> 4; n |= n >> 8; n |= n >> 16;
  return std::max<int>(1, (int)(n - (n >> 1)));
}

// The vertical part of torch's flexible_launch_configs(rows, C, block, grid, coop = true): MAX_BLOCK_SIZE 512,
// OPTIMAL_TILE_W 32, ELEMENTS_PER_THREAD 16, MAX_H_BLOCK 128.
BwdTree bwd_tree(int rows, int C) {
  const int block_x = std::min(last_pow2((unsigned)C), 32);
  const int block_y = std::min(last_pow2((unsigned)((rows + 15) / 16)), 512 / block_x);
  int grid_y = std::min((rows + block_y * 16 - 1) / (block_y * 16), 128);
  if (grid_y < 8) grid_y = 1;
  return {block_y, grid_y};
}

template <int kMode>
cudaError_t launch_bwd_reduce(const BnBwd& b, const BwdTree& t, const BwdOut& o, int rows, int C, cudaStream_t st) {
  const int groups = C / kVec;
  const int gpc = std::min(groups, std::max(1, kReduceThreads / t.block_y));
  const dim3 grid((groups + gpc - 1) / gpc, t.grid_y);
  const int threads = gpc * t.block_y;
  count_launch();
  bn_bwd_reduce_kernel<kMode><<<grid, threads, threads * kVec * sizeof(float), st>>>(
      reinterpret_cast<const __nv_bfloat16*>(b.go), b.mask, reinterpret_cast<const __nv_bfloat16*>(b.x), b.px.mean,
      b.px.invstd, reinterpret_cast<const __nv_bfloat16*>(b.z), b.pz.mean, b.pz.invstd,
      reinterpret_cast<__nv_bfloat16*>(b.g), o, t, rows, C);
  return cudaGetLastError();
}

template <int kMode>
cudaError_t launch_bwd_elemt(const BnBwd& b, const ElemtArgs& a, int64_t rows, int C, cudaStream_t st) {
  int grid = 0, threads = 0;
  cudaError_t e = rows_grid(bn_bwd_elemt_kernel<kMode>, rows, C, grid, threads);
  if (e != cudaSuccess) return e;
  const float norm = (float)(1.0 / (double)rows);      // torch: static_cast<accscalar_t>(1.0 / reduction_size)
  count_launch();
  bn_bwd_elemt_kernel<kMode><<<grid, threads, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(kMode == 1 ? b.g : b.go), b.mask,
      reinterpret_cast<const __nv_bfloat16*>(b.x), reinterpret_cast<const __nv_bfloat16*>(b.z), a,
      reinterpret_cast<__nv_bfloat16*>(b.dx), reinterpret_cast<__nv_bfloat16*>(b.dz), norm, rows, C);
  return cudaGetLastError();
}

template <int kMode>
cudaError_t launch_backward(const BnBwd& b, int64_t rows64, int C, cudaStream_t st) {
  const int rows = (int)rows64;
  const BwdTree t = bwd_tree(rows, C);
  const BwdOut o{b.sums, b.dw, b.db, b.dwz, b.dbz, b.staging};
  cudaError_t e = launch_bwd_reduce<kMode>(b, t, o, rows, C, st);
  if (e != cudaSuccess) return e;
  if (t.grid_y > 1) {
    const int cols = std::max(1, 512 / t.block_y);
    const int threads = cols * t.block_y;
    count_launch();
    bn_bwd_finalize_kernel<<<(C + cols - 1) / cols, threads, threads * sizeof(float), st>>>(
        o, t, kMode == 2 ? 3 : 2, C, b.px.invstd, b.pz.invstd);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  const ElemtArgs a{b.px.mean, b.px.invstd, b.px.weight, b.sums, b.pz.mean, b.pz.invstd, b.pz.weight};
  return launch_bwd_elemt<kMode>(b, a, rows64, C, st);
}

}  // namespace

void bn_backward_tree(int64_t rows, int C, int* block_y, int* grid_y) {
  const BwdTree t = bwd_tree((int)rows, C);
  *block_y = t.block_y;
  *grid_y = t.grid_y;
}

cudaError_t launch_bn_backward(int mode, const BnBwd& b, int64_t rows, int C, cudaStream_t st) {
  if (rows == 0) return cudaSuccess;
  switch (mode) {
    case 0: return launch_backward<0>(b, rows, C, st);
    case 1: return launch_backward<1>(b, rows, C, st);
    case 2: return launch_backward<2>(b, rows, C, st);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_bn_update_stats(const float* mean, float* var_invstd, float* running_mean, float* running_var, int C,
                                   float momentum, float bessel, float eps, cudaStream_t st) {
  count_launch();
  bn_update_stats_kernel<<<(C + 255) / 256, 256, 0, st>>>(mean, var_invstd, running_mean, running_var, C, momentum,
                                                          bessel, eps);
  return cudaGetLastError();
}

cudaError_t launch_bn_apply(int mode, const void* x, const BnParams& px, const void* z, const BnParams& pz, void* out,
                            void* mask, int64_t rows, int C, cudaStream_t st) {
  switch (mode) {
    case 0: return launch_apply<0>(x, px, z, pz, out, mask, rows, C, st);
    case 1: return launch_apply<1>(x, px, z, pz, out, mask, rows, C, st);
    case 2: return launch_apply<2>(x, px, z, pz, out, mask, rows, C, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace dr
