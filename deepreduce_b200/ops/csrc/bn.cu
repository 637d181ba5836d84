// Training-mode BatchNorm for NHWC (channels_last) bf16 activations, fused with the ReLU and the residual add that
// follow it in ResNet-50.  The results are bitwise those of the unfused graph (native_batch_norm -> relu_ -> add ->
// relu_), because every expression and every bf16 rounding point is kept:
//   * per-channel mean / biased var: torch's channels-last Welford tree, operation for operation (bn_stats_kernel);
//   * running stats and invstd: the expressions of torch's batch_norm_update_stats_and_invert, in the same pass;
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
//     batch_norm_backward_reduce_channels_last_kernel (see RowTree), so the sums are bitwise torch's;
//   * elementwise: torch's dx expression, pinned to the FMA placement of its sm_90 SASS.
// The stem's relu(bn(x)) is pooled in the same pass (bn_apply_pool_kernel), which writes a winner code per pooled element
// instead of the ReLU output; backward mode 3 gathers the pooled gradient through the codes.
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

// The two gradients of a block input (conv1's and the skip path's), summed as autograd's bf16 add does: fp32 sum of the
// bf16 values, rounded once.  The operands commute, so the order autograd would have added them in does not matter.
__device__ __forceinline__ uint4 add_bf16x8(const uint4& a, const uint4& b) {
  uint4 s;
  const __nv_bfloat16* ha = reinterpret_cast<const __nv_bfloat16*>(&a);
  const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&b);
  __nv_bfloat16* hs = reinterpret_cast<__nv_bfloat16*>(&s);
#pragma unroll
  for (int i = 0; i < kVec; ++i) hs[i] = __float2bfloat16_rn(__fadd_rn(__bfloat162float(ha[i]), __bfloat162float(hb[i])));
  return s;
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
// stem: relu(bn(x)) -> max pool (kernel 3, stride 2, padding 1, dilation 1, floor mode)
// ---------------------------------------------------------------------------------------------------------------------
// Input x is N x H x W x C, the pooled output N x Ho x Wo x C with Ho = (H - 1) / 2 + 1 (PoolGeom).  Window (oh, ow)
// covers rows 2 oh - 1 .. 2 oh + 1 and columns 2 ow - 1 .. 2 ow + 1, clipped to the input.

// One thread = one output position x 8 channels; each thread keeps its channel group and walks output positions.  The
// window is scanned as torch's max_pool_forward_nhwc does (ih outer, iw inner, from -inf; the winner changes where
// v > best || isnan(v)), so the first of equal maxima and the last NaN win, on the bf16 value relu(bn(x)) of mode 0.
// codes[pos][c]: bits 0-6 the winner's slot (ih - (2 oh - 1)) * 3 + (iw - (2 ow - 1)) in the unclipped window, bit 7
// its ReLU mask !(y <= 0).  Backward needs nothing else: a position that wins a window has the same y in all of them.
__global__ void __launch_bounds__(kApplyThreads) bn_apply_pool_kernel(const __nv_bfloat16* __restrict__ x, BnParams px,
                                                                      __nv_bfloat16* __restrict__ out,
                                                                      uint8_t* __restrict__ codes, int64_t orows,
                                                                      PoolGeom pg, int C) {
  const int groups = C / kVec;
  const int rows_per_cta = blockDim.x / groups;
  const int rsub = threadIdx.x / groups;
  if (rsub >= rows_per_cta) return;
  const int c = (threadIdx.x % groups) * kVec;
  ChanParams a;
  load_params(px, c, a);
  const int64_t step = (int64_t)gridDim.x * rows_per_cta;
  for (int64_t r = (int64_t)blockIdx.x * rows_per_cta + rsub; r < orows; r += step) {
    const int ow = (int)(r % pg.Wo);
    const int64_t t = r / pg.Wo;
    const int oh = (int)(t % pg.Ho);
    const int64_t n = t / pg.Ho;
    const int h0 = 2 * oh - 1, w0 = 2 * ow - 1;
    uint4 v[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int ih = h0 + k / 3, iw = w0 + k % 3;
      v[k] = ih >= 0 && ih < pg.H && iw >= 0 && iw < pg.W
                 ? *reinterpret_cast<const uint4*>(x + ((n * pg.H + ih) * pg.W + iw) * C + c)
                 : uint4{};
    }
    __nv_bfloat16 best[kVec];
    unsigned slot[kVec];
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      best[i] = __float2bfloat16_rn(-INFINITY);
      slot[i] = 0;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int ih = h0 + k / 3, iw = w0 + k % 3;
      if (ih < 0 || ih >= pg.H || iw < 0 || iw >= pg.W) continue;
      const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&v[k]);
#pragma unroll
      for (int i = 0; i < kVec; ++i) {
        const __nv_bfloat16 y = relu_bf16(__float2bfloat16_rn(bn_elem(__bfloat162float(hx[i]), a.m[i], a.inv[i], a.w[i], a.b[i])));
        const float fy = __bfloat162float(y);
        if (fy > __bfloat162float(best[i]) || isnan(fy)) {
          best[i] = y;
          slot[i] = k;
        }
      }
    }
    uint4 vo;
    __nv_bfloat16* ho = reinterpret_cast<__nv_bfloat16*>(&vo);
    uint2 vc;
    uint8_t* hc = reinterpret_cast<uint8_t*>(&vc);
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      ho[i] = best[i];
      hc[i] = (uint8_t)(slot[i] | (__bfloat162float(best[i]) <= 0.f ? 0u : 0x80u));
    }
    *reinterpret_cast<uint4*>(out + r * C + c) = vo;
    *reinterpret_cast<uint2*>(codes + r * C + c) = vc;
  }
}

// The pooled gradient of input position (n, h, w), 8 channels, as torch's max_pool_backward_nhwc gives it, from the
// <= 2 x 2 windows that cover it (torch's p_start / p_end: windows h / 2 .. min((h + 1) / 2 + 1, Ho) - 1 along h):
//   * covered by one window: its gradient where the position won it, copied as bf16 (a -0.0 stays), else +0;
//   * covered by more: the fp32 sum from 0.0f, in (oh, ow) order, of the gradients of the windows it won, rounded to bf16.
struct PoolGather {
  uint4 g[4];
  uint2 code[4];     // window (h / 2 + a, w / 2 + b) in entry 2 a + b
  int off;           // element offset of window (h / 2, w / 2) in the pooled tensor, channel c
  int nh, nw;        // windows along h and w (0 for a row past the end)
  int sh, sw;        // h - (2 (h / 2) - 1), w - (2 (w / 2) - 1): the position's row / column in window (h / 2, w / 2)
};

__device__ __forceinline__ void pool_gather_codes(PoolGather& q, const uint8_t* __restrict__ codes, const PoolGeom& pg,
                                                  int row, int C, int c, bool valid) {
  const int w = row % pg.W, t = row / pg.W, h = t % pg.H, n = t / pg.H;
  const int ph = h >> 1, pw = w >> 1;
  q.nh = valid ? min((h + 1) / 2 + 1, pg.Ho) - ph : 0;
  q.nw = valid ? min((w + 1) / 2 + 1, pg.Wo) - pw : 0;
  q.sh = h - 2 * ph + 1;
  q.sw = w - 2 * pw + 1;
  q.off = ((n * pg.Ho + ph) * pg.Wo + pw) * C + c;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int a = k >> 1, b = k & 1;
    q.code[k] = a < q.nh && b < q.nw ? *reinterpret_cast<const uint2*>(codes + q.off + (a * pg.Wo + b) * C) : uint2{};
  }
}

// kTwo: the pooled output is a block input with two consumers; its gradient is the bf16 sum of gp and gp2, formed per
// pooled element before the gather.
template <bool kTwo>
__device__ __forceinline__ void pool_gather_grads(PoolGather& q, const __nv_bfloat16* __restrict__ gp,
                                                  const __nv_bfloat16* __restrict__ gp2, const PoolGeom& pg, int C) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int a = k >> 1, b = k & 1;
    const bool in = a < q.nh && b < q.nw;
    const int off = q.off + (a * pg.Wo + b) * C;
    q.g[k] = in ? *reinterpret_cast<const uint4*>(gp + off) : uint4{};
    if (kTwo && in) q.g[k] = add_bf16x8(q.g[k], *reinterpret_cast<const uint4*>(gp2 + off));
  }
}

// -> g (8 bf16: the pooled gradient of the position) and bits (bit i: the ReLU mask of channel i where the position won
// a window, else 0; g is +0 there anyway).
__device__ __forceinline__ void pool_gather_resolve(const PoolGather& q, uint4& g, unsigned& bits) {
  __nv_bfloat16* hg = reinterpret_cast<__nv_bfloat16*>(&g);
  const bool single = q.nh == 1 && q.nw == 1;
  bits = 0;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    float s = 0.f;
    __nv_bfloat16 one = __float2bfloat16_rn(0.f);
    unsigned bit = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int a = k >> 1, b = k & 1;
      const unsigned code = (reinterpret_cast<const uint8_t*>(&q.code[k]))[i];
      if (a < q.nh && b < q.nw && (int)(code & 0x7fu) == (q.sh - 2 * a) * 3 + (q.sw - 2 * b)) {
        const __nv_bfloat16 v = (reinterpret_cast<const __nv_bfloat16*>(&q.g[k]))[i];
        s = __fadd_rn(s, __bfloat162float(v));
        one = v;
        bit = code >> 7;
      }
    }
    hg[i] = single ? one : __float2bfloat16_rn(s);
    bits |= bit << i;
  }
}

// Backward of the stem, first pass: g = mask ? (pooled gradient gathered onto x's positions) : +0, bf16 in x's layout,
// which is threshold_backward(max_pool2d_with_indices_backward(...)) of the unfused graph.  Mode 3 of the reduce and the
// elementwise pass then read it as mode 1 reads the reduce's g.  Gathering inside the reduce instead left that
// latency-bound pass (16 K threads at C = 64) at a fraction of its bandwidth.  kTwo: the pooled gradient is gp + gp2.
template <bool kTwo>
__global__ void __launch_bounds__(kApplyThreads) bn_pool_grad_kernel(const __nv_bfloat16* __restrict__ gp,
                                                                     const __nv_bfloat16* __restrict__ gp2,
                                                                     const uint8_t* __restrict__ codes,
                                                                     __nv_bfloat16* __restrict__ g, PoolGeom pg,
                                                                     int64_t rows, int C) {
  const int groups = C / kVec;
  const int rows_per_cta = blockDim.x / groups;
  const int rsub = threadIdx.x / groups;
  if (rsub >= rows_per_cta) return;
  const int c = (threadIdx.x % groups) * kVec;
  const int64_t step = (int64_t)gridDim.x * rows_per_cta;
#pragma unroll 2
  for (int64_t r = (int64_t)blockIdx.x * rows_per_cta + rsub; r < rows; r += step) {
    PoolGather q;
    pool_gather_codes(q, codes, pg, (int)r, C, c, true);
    pool_gather_grads<kTwo>(q, gp, gp2, pg, C);
    uint4 v;
    unsigned bits;
    pool_gather_resolve(q, v, bits);
    __nv_bfloat16* hv = reinterpret_cast<__nv_bfloat16*>(&v);
#pragma unroll
    for (int i = 0; i < kVec; ++i)
      if (!((bits >> i) & 1u)) hv[i] = __float2bfloat16_rn(0.f);
    *reinterpret_cast<uint4*>(g + r * C + c) = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// reduction trees
// ---------------------------------------------------------------------------------------------------------------------
// The row indexing of torch's channels-last reductions (batch_norm_collect_statistics_channels_last_kernel<4> and
// batch_norm_backward_reduce_channels_last_kernel<4>) for `rows` x C, launch config from
// flexible_launch_configs(rows, C, coop = true); block_x does not change a column's result.  Virtual thread
// v = block * block_y + y (of S = block_y * grid_y) keeps kLoads accumulators; accumulator j takes rows
// v + (i * kLoads + j) * S for i < loops(rows).  Then ((a0 . a1) . a2) . a3, a pairwise tree over y inside each block
// (offsets block_y / 2 ... 1), and for grid_y > 1 the same tree over y of e . s[y] . s[y + block_y] . ... of the block
// results s, from the identity e.  For the backward sums "." is + and e = 0.0f; for the statistics it is Welford's merge
// and e = (count 0, mean 0, m2n 0).
struct RowTree {
  int block_y, grid_y;
  __host__ __device__ int S() const { return block_y * grid_y; }
  __host__ __device__ int loops(int rows) const { return 1 + (rows - 1) / (S() * kLoads); }
  static constexpr int kLoads = 4;       // torch's ELEMENTS_PER_ITER
};

// ---------------------------------------------------------------------------------------------------------------------
// forward statistics
// ---------------------------------------------------------------------------------------------------------------------
// Per-channel mean and biased variance, bitwise those of torch's batch_norm_collect_statistics_channels_last_kernel
// <Var, BFloat16, float, 4>: the same RowTree and the same fp32 operations, each pinned to the placement of that
// kernel's sm_90 SASS.  Only the thread layout differs: accumulator j of a virtual thread lives in a physical thread of
// its own (4 per virtual thread, 8 channels each, one 16-byte load per row), and the four are merged in torch's order
// through shared memory.
constexpr int kStatsThreads = 256;    // at most; 78 registers per thread, 3 blocks per SM

// Welford update of one element; inv = 1 / count (0 for a row past the end, with x = 0 and valid = 0: torch still runs
// this arithmetic there, and a non-finite mean makes it NaN).  SASS: FADD d0 = x - mean; FFMA mean = d0 * inv + mean;
// FADD d1 = x - mean; FMUL t = d0 * d1; FFMA m2n = t * valid + m2n.
__device__ __forceinline__ void welford_update(float x, float inv, float valid, float& mean, float& m2n) {
  const float d0 = __fsub_rn(x, mean);
  mean = __fmaf_rn(d0, inv, mean);
  const float d1 = __fsub_rn(x, mean);
  m2n = __fmaf_rn(__fmul_rn(d0, d1), valid, m2n);
}

// torch's welford_merge_element of (n_new, mean_new, m2n_new) into (n, mean, m2n), kN channels that share the counts.
// SASS: factor = 1.0f / max(1, n + n_new) (correctly rounded); FADD d = mean - mean_new;
// FMUL u = d * d; FMUL u *= n_new; FMUL u *= n; FFMA u = u * factor + m2n_new; FADD m2n += u;
// and mean = (mean_new * n_new + mean * n) * factor, whose contraction nvcc chose per inlined call site:
//   kFuseNew (the merge of the 4 accumulators): FMUL t = mean * n; FFMA mean = mean_new * n_new + t;
//   otherwise (the vertical tree, the cross-block merge): FMUL t = mean_new * n_new; FFMA mean = mean * n + t;
// then FMUL mean *= factor.
template <int kN, bool kFuseNew>
__device__ __forceinline__ void welford_merge(int& n, float* mean, float* m2n, int n_new, const float* mean_new,
                                              const float* m2n_new) {
  const float fn = (float)n, fn_new = (float)n_new;
  const float factor = __frcp_rn((float)max(1, n + n_new));
#pragma unroll
  for (int i = 0; i < kN; ++i) {
    const float d = __fsub_rn(mean[i], mean_new[i]);
    const float s = kFuseNew ? __fmaf_rn(mean_new[i], fn_new, __fmul_rn(mean[i], fn))
                             : __fmaf_rn(mean[i], fn, __fmul_rn(mean_new[i], fn_new));
    mean[i] = __fmul_rn(s, factor);
    const float u = __fmul_rn(__fmul_rn(__fmul_rn(d, d), fn_new), fn);
    m2n[i] = __fadd_rn(m2n[i], __fmaf_rn(u, factor, m2n_new[i]));
  }
  n += n_new;
}

// Shared-memory slots for a Welford merge across threads: mean[slots][kN], m2n[slots][kN], count[slots].
template <int kN>
struct WelfordSlots {
  float* mean; float* m2n; int* count;
  __device__ WelfordSlots(float* sh, int slots)
      : mean(sh), m2n(sh + slots * kN), count(reinterpret_cast<int*>(sh + 2 * slots * kN)) {}
  __device__ void put(int s, int n, const float* m, const float* q) const {
#pragma unroll
    for (int i = 0; i < kN; ++i) { mean[s * kN + i] = m[i]; m2n[s * kN + i] = q[i]; }
    count[s] = n;
  }
  template <bool kFuseNew>
  __device__ void merge_from(int s, int& n, float* m, float* q) const {
    float mn[kN], qn[kN];
#pragma unroll
    for (int i = 0; i < kN; ++i) { mn[i] = mean[s * kN + i]; qn[i] = m2n[s * kN + i]; }
    welford_merge<kN, kFuseNew>(n, m, q, count[s], mn, qn);
  }
  static size_t bytes(int slots) { return (size_t)slots * (2 * kN * sizeof(float) + sizeof(int)); }
};

// torch's welford_merge_block_vertical: pairwise tree over y (offsets block_y / 2 ... 1), result at y == 0.  Slot of y
// is base + y * stride; threads with !part take part in the barriers only.
template <int kN>
__device__ __forceinline__ void welford_tree_over_y(const WelfordSlots<kN>& sl, bool part, int y, int block_y, int base,
                                                    int stride, int& n, float* mean, float* m2n) {
  for (int off = block_y / 2; off > 0; off >>= 1) {
    if (part && y < 2 * off) sl.put(base + y * stride, n, mean, m2n);
    __syncthreads();
    if (part && y < off) sl.template merge_from<false>(base + (y + off) * stride, n, mean, m2n);
    __syncthreads();
  }
}

struct StatsOut {
  float* mean; float* invstd; float* running_mean; float* running_var;
  float* st_mean; float* st_m2n; int* st_count;     // [grid_y][C], [grid_y][C], [grid_y] when grid_y > 1
  float momentum, bessel, eps;
};

// The end of torch's statistics kernel (var = m2n / count, Var transform) followed by the expressions of
// batch_norm_update_stats_and_invert, as their SASS places them: FADD a = 1 - momentum; FMUL t = running * a;
// FFMA running = new * momentum + t; the unbiased variance is FMUL var * bessel; invstd = rsqrtf(var + eps).
__device__ __forceinline__ void stats_store(const StatsOut& o, int c, int n, float mean, float m2n) {
  const float var = __fdiv_rn(m2n, (float)n);
  const float keep = __fsub_rn(1.f, o.momentum);
  o.mean[c] = mean;
  o.invstd[c] = rsqrtf(__fadd_rn(var, o.eps));
  o.running_mean[c] = __fmaf_rn(mean, o.momentum, __fmul_rn(o.running_mean[c], keep));
  o.running_var[c] = __fmaf_rn(__fmul_rn(var, o.bessel), o.momentum, __fmul_rn(o.running_var[c], keep));
}

// Block = gpc channel groups x kLoads accumulators x block_y virtual threads of virtual block blockIdx.y; thread
// (g, j, y) walks rows v + (i * kLoads + j) * S with the loads of the next kAhead iterations issued before the current
// ones are used.  grid_y == 1: the block writes the final results; else its partial goes to staging.
__global__ void __launch_bounds__(kStatsThreads) bn_stats_kernel(const __nv_bfloat16* __restrict__ x, StatsOut o,
                                                                 RowTree t, int rows, int C) {
  constexpr int L = RowTree::kLoads;
  constexpr int kAhead = 4;
  extern __shared__ float sh[];
  const int gpc = blockDim.x / (L * t.block_y);
  const int g = threadIdx.x % gpc, j = (threadIdx.x / gpc) % L, y = threadIdx.x / (gpc * L);
  const int group = blockIdx.x * gpc + g;
  const bool live = group * kVec < C;
  const int c = live ? group * kVec : 0;
  const int S = t.S();
  const int n_loops = t.loops(rows);
  const int r0 = blockIdx.y * t.block_y + y + j * S;      // row of iteration i: r0 + i * L * S
  const int rstep = L * S;
  float mean[kVec], m2n[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) mean[i] = m2n[i] = 0.f;
  int n = 0;
  auto load = [&](uint4* b, int i0) {
#pragma unroll
    for (int u = 0; u < kAhead; ++u) {
      const int r = r0 + (i0 + u) * rstep;
      b[u] = live && i0 + u < n_loops && r < rows ? *reinterpret_cast<const uint4*>(x + (size_t)r * C + c) : uint4{};
    }
  };
  uint4 cur[kAhead];
  load(cur, 0);
  for (int i0 = 0; i0 < n_loops; i0 += kAhead) {
    uint4 nxt[kAhead];
    load(nxt, i0 + kAhead);
#pragma unroll
    for (int u = 0; u < kAhead; ++u) {
      const int i = i0 + u;
      if (i >= n_loops) break;
      // for a row in range, count = i + 1 in every accumulator, so 1 / count is one correctly rounded reciprocal
      const bool valid = r0 + i * rstep < rows;
      const float inv = valid ? __frcp_rn((float)(i + 1)) : 0.f;
      const float fv = valid ? 1.f : 0.f;
      n += valid;
      const __nv_bfloat16* hx = reinterpret_cast<const __nv_bfloat16*>(&cur[u]);
#pragma unroll
      for (int k = 0; k < kVec; ++k) welford_update(__bfloat162float(hx[k]), inv, fv, mean[k], m2n[k]);
    }
#pragma unroll
    for (int u = 0; u < kAhead; ++u) cur[u] = nxt[u];
  }
  // ((a0 . a1) . a2) . a3 in the thread of accumulator 0, then the tree over y
  const WelfordSlots<kVec> sl(sh, blockDim.x);
  sl.put(threadIdx.x, n, mean, m2n);
  __syncthreads();
  if (j == 0) {
#pragma unroll
    for (int a = 1; a < L; ++a) sl.merge_from<true>(threadIdx.x + a * gpc, n, mean, m2n);
  }
  __syncthreads();
  welford_tree_over_y<kVec>(sl, j == 0, y, t.block_y, g, gpc * L, n, mean, m2n);
  if (j != 0 || y != 0 || !live) return;
  if (t.grid_y == 1) {
#pragma unroll
    for (int i = 0; i < kVec; ++i) stats_store(o, c + i, n, mean[i], m2n[i]);
    return;
  }
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    o.st_mean[(size_t)blockIdx.y * C + c + i] = mean[i];
    o.st_m2n[(size_t)blockIdx.y * C + c + i] = m2n[i];
  }
  if (group == 0) o.st_count[blockIdx.y] = n;
}

// grid_y > 1: the cross-block step of torch's kernel (its last block's code).  Block = cols channels x block_y; thread
// (col, y) merges staging rows y, y + block_y, ... into (0, 0, 0), and the tree over y combines them.
__global__ void bn_stats_finalize_kernel(StatsOut o, RowTree t, int C) {
  extern __shared__ float sh[];
  const int cols = blockDim.x / t.block_y;
  const int col = threadIdx.x % cols, y = threadIdx.x / cols;
  const int c = blockIdx.x * cols + col;
  int n = 0;
  float mean = 0.f, m2n = 0.f;
  if (c < C)
    for (int b = y; b < t.grid_y; b += t.block_y) {
      const float mb = o.st_mean[(size_t)b * C + c], qb = o.st_m2n[(size_t)b * C + c];
      welford_merge<1, false>(n, &mean, &m2n, o.st_count[b], &mb, &qb);
    }
  const WelfordSlots<1> sl(sh, blockDim.x);
  welford_tree_over_y<1>(sl, true, y, t.block_y, col, cols, n, &mean, &m2n);
  if (y == 0 && c < C) stats_store(o, c, n, mean, m2n);
}

// ---------------------------------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------------------------------
// The backward sums run on the same RowTree as the statistics: accumulator j sums rows v + (i * kLoads + j) * S from
// 0.0f (rows past the end add g = 0, x = 0, as torch's loads do), then ((a0 + a1) + a2) + a3, the pairwise tree over y,
// and for grid_y > 1 the tree over y of 0.0f + s[y] + s[y + block_y] + ...

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
// block_y virtual threads of one virtual block (blockIdx.y).  kMode 0: sums of g; 1: also writes g; 2: also the z sums;
// 3: go is the masked gradient bn_pool_grad_kernel wrote (no mask).  kTwo (modes 1, 2): the output is a block input and
// its gradient is the bf16 sum of go and go2 (add_bf16x8), formed before the mask.
template <int kMode, bool kTwo>
__global__ void __launch_bounds__(kReduceThreads) bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ go,
                                                                       const __nv_bfloat16* __restrict__ go2,
                                                                       const uint8_t* __restrict__ mask,
                                                                       const __nv_bfloat16* __restrict__ x,
                                                                       const float* __restrict__ mean,
                                                                       const float* __restrict__ invstd,
                                                                       const __nv_bfloat16* __restrict__ z,
                                                                       const float* __restrict__ mean_z,
                                                                       const float* __restrict__ invstd_z,
                                                                       __nv_bfloat16* __restrict__ g_out, BwdOut o,
                                                                       RowTree t, int rows, int C) {
  constexpr int kSums = kMode == 2 ? 3 : 2;
  constexpr int L = RowTree::kLoads;
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
  // With two gradients the current batch's pair is summed before the next loads are issued, so only the next batch
  // holds a second gradient.  Mode 2 with two gradients has no room for a second batch (249 registers without it) and
  // runs at 64 K-262 K threads (C >= 256), so it loads at the top of each iteration instead.
  constexpr bool kAhead = !(kTwo && kMode == 2);
  struct Batch {
    uint4 g[L], g2[L], x[L], z[L];
    unsigned m[L];
  };
  auto load = [&](Batch& b, int r0) {
#pragma unroll
    for (int j = 0; j < L; ++j) {
      const int rr = r0 + j * S;
      if (live && rr < rows) {
        const int off = rr * C + c;
        b.g[j] = *reinterpret_cast<const uint4*>(go + off);
        if (kTwo) b.g2[j] = *reinterpret_cast<const uint4*>(go2 + off);
        b.x[j] = *reinterpret_cast<const uint4*>(x + off);
        if (kMode == 2) b.z[j] = *reinterpret_cast<const uint4*>(z + off);
        b.m[j] = kMode == 3 ? 0u : mask[rr * mgroups + group];      // mode 3's g is masked already
      } else {
        b.g[j] = uint4{}; b.g2[j] = uint4{}; b.x[j] = uint4{}; b.z[j] = uint4{}; b.m[j] = 0;
      }
    }
  };
  Batch cur;
  if (kAhead) load(cur, r);
  for (int it = 0; it < n_loops; ++it) {
    if (!kAhead) load(cur, r);
    if (kTwo) {
#pragma unroll
      for (int j = 0; j < L; ++j) cur.g[j] = add_bf16x8(cur.g[j], cur.g2[j]);
    }
    Batch nxt;
    if (kAhead) load(nxt, r + L * S);
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
        const float g = kMode == 3 ? __bfloat162float(hg[i]) : masked(hg[i], bit);
        if (kMode == 1) ho[i] = bit ? hg[i] : __float2bfloat16_rn(0.f);      // threshold_backward's bits, NaN too
        // torch's sm_90 SASS: FADD d = x - mean; FADD acc += g; FFMA acc_xmu = d * g + acc_xmu
        acc[0][j][i] = __fadd_rn(acc[0][j][i], g);
        acc[1][j][i] = __fmaf_rn(__fsub_rn(__bfloat162float(hx[i]), m[i]), g, acc[1][j][i]);
        if (kMode == 2) acc[2][j][i] = __fmaf_rn(__fsub_rn(__bfloat162float(hz[i]), mz[i]), g, acc[2][j][i]);
      }
      if (kMode == 1 && live && r + j * S < rows) *reinterpret_cast<uint4*>(g_out + (r + j * S) * C + c) = vo;
    }
    if (kAhead) cur = nxt;
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
__global__ void bn_bwd_finalize_kernel(BwdOut o, RowTree t, int n_sums, int C, const float* __restrict__ invstd,
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
// * f2, rounded to bf16 once.  kMode 1 reads the g the reduce wrote (gm = nullptr), 3 the g bn_pool_grad_kernel wrote;
// 0 and 2 mask go; 2 also writes dz.
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

// kTwo (mode 2): the gradient is the bf16 sum of g_in and g2_in, as in the reduce.
template <int kMode, bool kTwo>
__global__ void __launch_bounds__(kApplyThreads) bn_bwd_elemt_kernel(const __nv_bfloat16* __restrict__ g_in,
                                                                     const __nv_bfloat16* __restrict__ g2_in,
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
    uint4 vg = *reinterpret_cast<const uint4*>(g_in + off);
    if (kTwo) vg = add_bf16x8(vg, *reinterpret_cast<const uint4*>(g2_in + off));
    const unsigned mb = kMode == 1 || kMode == 3 ? 0xffu : mask[r * groups + c / kVec];
    const uint4 vx = *reinterpret_cast<const uint4*>(x + off);
    uint4 vz = make_uint4(0, 0, 0, 0);
    if (kMode == 2) vz = *reinterpret_cast<const uint4*>(z + off);
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
// A CTA holds one row's C / 8 threads at least, and the four row-walking kernels are __launch_bounds__(kApplyThreads),
// so C is capped at kBnMaxChannels (binding.cpp's check_bn_input, fused_bn._eligible_x).
static_assert(kBnMaxChannels / kVec <= kApplyThreads, "a row of kBnMaxChannels channels exceeds one apply CTA");
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
RowTree row_tree(int rows, int C) {
  const int block_x = std::min(last_pow2((unsigned)C), 32);
  const int block_y = std::min(last_pow2((unsigned)((rows + 15) / 16)), 512 / block_x);
  int grid_y = std::min((rows + block_y * 16 - 1) / (block_y * 16), 128);
  if (grid_y < 8) grid_y = 1;
  return {block_y, grid_y};
}

template <int kMode, bool kTwo>
cudaError_t launch_bwd_reduce(const BnBwd& b, const RowTree& t, const BwdOut& o, int rows, int C, cudaStream_t st) {
  const int groups = C / kVec;
  const int gpc = std::min(groups, std::max(1, kReduceThreads / t.block_y));
  const dim3 grid((groups + gpc - 1) / gpc, t.grid_y);
  const int threads = gpc * t.block_y;
  count_launch();
  bn_bwd_reduce_kernel<kMode, kTwo><<<grid, threads, threads * kVec * sizeof(float), st>>>(
      reinterpret_cast<const __nv_bfloat16*>(b.go), reinterpret_cast<const __nv_bfloat16*>(b.go2), b.mask,
      reinterpret_cast<const __nv_bfloat16*>(b.x), b.px.mean, b.px.invstd, reinterpret_cast<const __nv_bfloat16*>(b.z),
      b.pz.mean, b.pz.invstd, reinterpret_cast<__nv_bfloat16*>(b.g), o, t, rows, C);
  return cudaGetLastError();
}

template <int kMode, bool kTwo>
cudaError_t launch_bwd_elemt(const BnBwd& b, const ElemtArgs& a, int64_t rows, int C, cudaStream_t st) {
  int grid = 0, threads = 0;
  cudaError_t e = rows_grid(bn_bwd_elemt_kernel<kMode, kTwo>, rows, C, grid, threads);
  if (e != cudaSuccess) return e;
  const float norm = (float)(1.0 / (double)rows);      // torch: static_cast<accscalar_t>(1.0 / reduction_size)
  count_launch();
  bn_bwd_elemt_kernel<kMode, kTwo><<<grid, threads, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(kMode == 1 || kMode == 3 ? b.g : b.go),
      reinterpret_cast<const __nv_bfloat16*>(b.go2), b.mask, reinterpret_cast<const __nv_bfloat16*>(b.x),
      reinterpret_cast<const __nv_bfloat16*>(b.z), a, reinterpret_cast<__nv_bfloat16*>(b.dx),
      reinterpret_cast<__nv_bfloat16*>(b.dz), norm, rows, C);
  return cudaGetLastError();
}

// kTwo: b.go2 is set.  Mode 1 folds it in the reduce, which writes the summed, masked g for the elementwise pass; mode 2
// folds it in both passes; mode 3 in bn_pool_grad_kernel, whose g both passes read.
template <int kMode, bool kTwo>
cudaError_t launch_backward(const BnBwd& b, int64_t rows64, int C, cudaStream_t st) {
  const int rows = (int)rows64;
  const RowTree t = row_tree(rows, C);
  const BwdOut o{b.sums, b.dw, b.db, b.dwz, b.dbz, b.staging};
  cudaError_t e;
  if (kMode == 3) {
    int grid = 0, threads = 0;
    e = rows_grid(bn_pool_grad_kernel<kTwo>, rows64, C, grid, threads);
    if (e != cudaSuccess) return e;
    count_launch();
    bn_pool_grad_kernel<kTwo><<<grid, threads, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(b.go),
                                                        reinterpret_cast<const __nv_bfloat16*>(b.go2), b.mask,
                                                        reinterpret_cast<__nv_bfloat16*>(b.g), b.pool, rows64, C);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  BnBwd bb = b;
  if (kMode == 3) bb.go = b.g;           // the reduce reads the gathered, masked g
  e = launch_bwd_reduce<kMode, kTwo && kMode != 3>(bb, t, o, rows, C, st);
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
  return launch_bwd_elemt<kMode, kTwo && kMode == 2>(b, a, rows64, C, st);
}

cudaError_t launch_stats(const BnStats& s, int rows, int C, cudaStream_t st) {
  const RowTree t = row_tree(rows, C);
  const int grid_y = t.grid_y;
  const StatsOut o{s.mean, s.invstd, s.running_mean, s.running_var,
                   s.staging, s.staging + (size_t)grid_y * C, reinterpret_cast<int*>(s.staging + 2 * (size_t)grid_y * C),
                   s.momentum, s.bessel, s.eps};
  const int groups = C / kVec;
  const int gpc = std::min(groups, std::max(1, kStatsThreads / (RowTree::kLoads * t.block_y)));
  const int threads = gpc * RowTree::kLoads * t.block_y;
  count_launch();
  bn_stats_kernel<<<dim3((groups + gpc - 1) / gpc, grid_y), threads, WelfordSlots<kVec>::bytes(threads), st>>>(
      reinterpret_cast<const __nv_bfloat16*>(s.x), o, t, rows, C);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || grid_y == 1) return e;
  const int cols = std::max(1, 512 / t.block_y);
  const int fthreads = cols * t.block_y;
  count_launch();
  bn_stats_finalize_kernel<<<(C + cols - 1) / cols, fthreads, WelfordSlots<1>::bytes(fthreads), st>>>(o, t, C);
  return cudaGetLastError();
}

}  // namespace

void bn_row_tree(int64_t rows, int C, int* block_y, int* grid_y) {
  const RowTree t = row_tree((int)rows, C);
  *block_y = t.block_y;
  *grid_y = t.grid_y;
}

cudaError_t launch_bn_backward(int mode, const BnBwd& b, int64_t rows, int C, cudaStream_t st) {
  if (rows == 0) return cudaSuccess;
  const bool two = b.go2 != nullptr;
  switch (mode) {
    case 0: return two ? cudaErrorInvalidValue : launch_backward<0, false>(b, rows, C, st);
    case 1: return two ? launch_backward<1, true>(b, rows, C, st) : launch_backward<1, false>(b, rows, C, st);
    case 2: return two ? launch_backward<2, true>(b, rows, C, st) : launch_backward<2, false>(b, rows, C, st);
    case 3: return two ? launch_backward<3, true>(b, rows, C, st) : launch_backward<3, false>(b, rows, C, st);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_bn_stats(const BnStats& s, int64_t rows, int C, cudaStream_t st) {
  if (rows == 0) return cudaSuccess;
  return launch_stats(s, (int)rows, C, st);
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

cudaError_t launch_bn_apply_pool(const void* x, const BnParams& px, void* out, void* codes, int N, const PoolGeom& pg,
                                 int C, cudaStream_t st) {
  const int64_t orows = (int64_t)N * pg.Ho * pg.Wo;
  if (orows == 0) return cudaSuccess;
  int grid = 0, threads = 0;
  cudaError_t e = rows_grid(bn_apply_pool_kernel, orows, C, grid, threads);
  if (e != cudaSuccess) return e;
  count_launch();
  bn_apply_pool_kernel<<<grid, threads, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), px,
                                                 reinterpret_cast<__nv_bfloat16*>(out),
                                                 reinterpret_cast<uint8_t*>(codes), orows, pg, C);
  return cudaGetLastError();
}

}  // namespace dr
