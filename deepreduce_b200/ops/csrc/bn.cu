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
#include <cuda_bf16.h>

#include "common.cuh"
#include "ops.h"

namespace dr {

namespace {

constexpr int kVec = 8;            // bf16 channels per thread: one 16-byte load / store
constexpr int kApplyThreads = 256;

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
template <int kMode>
__global__ void __launch_bounds__(kApplyThreads) bn_apply_kernel(const __nv_bfloat16* __restrict__ x, BnParams px,
                                                                 const __nv_bfloat16* __restrict__ z, BnParams pz,
                                                                 __nv_bfloat16* __restrict__ out, int64_t rows, int C) {
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
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      __nv_bfloat16 y = __float2bfloat16_rn(bn_elem(__bfloat162float(hx[i]), a.m[i], a.inv[i], a.w[i], a.b[i]));
      if (kMode != 0) {
        const __nv_bfloat16 s = kMode == 1 ? hz[i]
                                           : __float2bfloat16_rn(bn_elem(__bfloat162float(hz[i]), d.m[i], d.inv[i], d.w[i], d.b[i]));
        y = __float2bfloat16_rn(__fadd_rn(__bfloat162float(y), __bfloat162float(s)));
      }
      ho[i] = relu_bf16(y);
    }
    *reinterpret_cast<uint4*>(out + off) = vo;
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

template <int kMode>
cudaError_t launch_apply(const void* x, const BnParams& px, const void* z, const BnParams& pz, void* out, int64_t rows,
                         int C, cudaStream_t st) {
  if (rows == 0) return cudaSuccess;
  const int groups = C / kVec;
  const int rows_per_cta = groups >= kApplyThreads ? 1 : kApplyThreads / groups;
  const int threads = groups * rows_per_cta;
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bn_apply_kernel<kMode>, threads, 0);
  if (e != cudaSuccess) return e;
  int64_t grid = (rows + rows_per_cta - 1) / rows_per_cta;
  const int64_t cap = (int64_t)(per_sm > 0 ? per_sm : 1) * sm_count();
  if (grid > cap) grid = cap;
  count_launch();
  bn_apply_kernel<kMode><<<(int)grid, threads, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), px,
                                                        reinterpret_cast<const __nv_bfloat16*>(z), pz,
                                                        reinterpret_cast<__nv_bfloat16*>(out), rows, C);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_bn_update_stats(const float* mean, float* var_invstd, float* running_mean, float* running_var, int C,
                                   float momentum, float bessel, float eps, cudaStream_t st) {
  count_launch();
  bn_update_stats_kernel<<<(C + 255) / 256, 256, 0, st>>>(mean, var_invstd, running_mean, running_var, C, momentum,
                                                          bessel, eps);
  return cudaGetLastError();
}

cudaError_t launch_bn_apply(int mode, const void* x, const BnParams& px, const void* z, const BnParams& pz, void* out,
                            int64_t rows, int C, cudaStream_t st) {
  switch (mode) {
    case 0: return launch_apply<0>(x, px, z, pz, out, rows, C, st);
    case 1: return launch_apply<1>(x, px, z, pz, out, rows, C, st);
    case 2: return launch_apply<2>(x, px, z, pz, out, rows, C, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace dr
