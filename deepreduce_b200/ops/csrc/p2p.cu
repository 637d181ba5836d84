// Symmetric arena over CUDA IPC: every rank cudaMalloc's one arena, exports its
// handle (exchanged once through torch.distributed), and maps every peer's arena.
// After that the engine kernel stores compressed slots straight into peers'
// memory over NVLink and signals with release/acquire flags — NCCL is only the
// bootstrap (SURVEY §5 "Distributed communication backend").
// Replaces the GRACE Allgather communicator's per-tensor, per-wire-component `dist.all_gather` calls (2-3 per tensor,
// +1 size gather when sizes differ; reference README.md:37, pytorch/deepreduce.py:59,108,267 — >= 322 NCCL calls
// per ResNet-50 step) and, on the TF side, Horovod's allgather of one blob per tensor
// (tensorflow/bloom_filter_compression.cc:112).
#include <cstdio>
#include <cstring>

#include <cuda_bf16.h>

#include "common.cuh"
#include "ops.h"

namespace dr {

void* arena_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
  cudaMemset(p, 0, bytes);
  cudaDeviceSynchronize();
  return p;
}

void arena_free(void* p) { if (p) cudaFree(p); }

ArenaHandle arena_export(void* p) {
  ArenaHandle h;
  static_assert(sizeof(cudaIpcMemHandle_t) <= sizeof(h.bytes), "handle size");
  cudaIpcMemHandle_t ih;
  memset(&h, 0, sizeof(h));
  if (cudaIpcGetMemHandle(&ih, p) == cudaSuccess) memcpy(h.bytes, &ih, sizeof(ih));
  return h;
}

void* arena_import(const ArenaHandle& h) {
  cudaIpcMemHandle_t ih;
  memcpy(&ih, h.bytes, sizeof(ih));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, ih, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    fprintf(stderr, "[deepreduce_b200] cudaIpcOpenMemHandle failed: %s\n", cudaGetErrorString(e));
    cudaGetLastError();
    return nullptr;
  }
  return p;
}

void arena_close(void* p) { if (p) cudaIpcCloseMemHandle(p); }

// Enable peer access from the current device to exactly the listed devices (the GPUs of the ranks of this
// communication group) — never to every GPU of the box: mapping devices outside the job showed up as activity on
// GPUs the job does not own (round-1 SCALE records).
int arena_enable_peer_access(const int* devices, int n) {
  int dev = 0, enabled = 0;
  cudaGetDevice(&dev);
  for (int i = 0; i < n; ++i) {
    const int p = devices[i];
    if (p == dev) continue;
    int can = 0;
    cudaDeviceCanAccessPeer(&can, dev, p);
    if (!can) continue;
    cudaError_t e = cudaDeviceEnablePeerAccess(p, 0);
    if (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled) ++enabled;
    cudaGetLastError();
  }
  return enabled;
}

namespace {
// uint8 NHWC image batch -> normalised bf16, same physical layout (channels_last).
__global__ void u8_to_nhwc_norm_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t n_pix,
                                       float m0, float m1, float m2, float s0, float s1, float s2) {
  // 4 pixels (12 bytes) per thread
  const int64_t n4 = n_pix / 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(in) + i * 3;
    const uint32_t w0 = p[0], w1 = p[1], w2 = p[2];
    const uint8_t b[12] = {(uint8_t)w0, (uint8_t)(w0 >> 8), (uint8_t)(w0 >> 16), (uint8_t)(w0 >> 24),
                           (uint8_t)w1, (uint8_t)(w1 >> 8), (uint8_t)(w1 >> 16), (uint8_t)(w1 >> 24),
                           (uint8_t)w2, (uint8_t)(w2 >> 8), (uint8_t)(w2 >> 16), (uint8_t)(w2 >> 24)};
    const float m[3] = {m0, m1, m2}, s[3] = {s0, s1, s2};
    __nv_bfloat16 o[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) o[j] = __float2bfloat16(((float)b[j] * (1.f / 255.f) - m[j % 3]) * s[j % 3]);
    const uint32_t* ow = reinterpret_cast<const uint32_t*>(o);
    // 24 bytes per thread: three 8-byte stores (24*i is only 8-byte aligned)
    uint2* q = reinterpret_cast<uint2*>(out + i * 12);
    q[0] = make_uint2(ow[0], ow[1]);
    q[1] = make_uint2(ow[2], ow[3]);
    q[2] = make_uint2(ow[4], ow[5]);
  }
  // tail pixels
  const int64_t start = n4 * 4;
  for (int64_t px = start + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; px < n_pix; px += (int64_t)gridDim.x * blockDim.x) {
    const float m[3] = {m0, m1, m2}, s[3] = {s0, s1, s2};
    for (int c = 0; c < 3; ++c) out[px * 3 + c] = __float2bfloat16(((float)in[px * 3 + c] * (1.f / 255.f) - m[c]) * s[c]);
  }
}
}  // namespace

void launch_u8_to_nhwc_norm(const uint8_t* in, void* out_bf16, int64_t n_pix, const float* mean, const float* inv_std,
                            cudaStream_t st) {
  if (n_pix == 0) return;
  count_launch();
  int64_t g = (n_pix / 4 + 255) / 256;
  if (g < 1) g = 1;
  const int64_t cap = 16LL * sm_count();           // grid-stride kernel: at most 16 CTAs per SM
  if (g > cap) g = cap;
  u8_to_nhwc_norm_kernel<<<(int)g, 256, 0, st>>>(in, reinterpret_cast<__nv_bfloat16*>(out_bf16), n_pix, mean[0], mean[1],
                                                  mean[2], inv_std[0], inv_std[1], inv_std[2]);
}

}  // namespace dr
