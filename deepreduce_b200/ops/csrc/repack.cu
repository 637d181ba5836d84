// Repack between a torch DDP gradient bucket and the fused engine's flat buffer (parallel/comm_hook.py).
//
// DDP lays a bucket's parameters back to back with no padding, at arbitrary element offsets.  The engine starts every
// tensor on a 32-element boundary (parallel/plan.py).  A per-layout segment table {ddp_off, eng_off, numel, vec_begin}
// maps one to the other; each segment is one parameter in its storage order.  One launch moves every segment:
//   * the work unit is one 16-byte vector of the ENGINE side (4 fp32 / 8 bf16 elements); segment s owns the vectors
//     [vec_begin[s], vec_begin[s + 1]), so a 1-element bias and a 2.4 M-element conv weight cost what their sizes say and
//     the grid is balanced over the total element count, not per segment;
//   * a block covers 256 * kItems consecutive vectors; two threads find the first and last segment of that range by
//     binary search and every item then searches only between them (almost always one segment: zero steps);
//   * the engine side is 16-byte aligned (eng_off % vector == 0, base checked by the binding): full vectors are one
//     16-byte load or store, the tail of a segment goes element by element so that the engine's padding is never
//     written;
//   * the DDP side is misaligned by arbitrary amounts.  A vector whose DDP address happens to be 16-byte aligned takes
//     one 16-byte access; any other reads or writes its elements one by one.  Consecutive threads touch consecutive
//     16-byte spans, so the scalar accesses of a warp still cover whole 128-byte lines (full sectors).  Measured on the
//     ResNet-50 layout with every DDP-side access scalar (profiles/README.md §12): 1-2 % slower for fp32, 5 % for bf16
//     pack, but half the speed for bf16 unpack (2-byte stores).  Only a bf16 bucket with segments off 16-byte
//     boundaries pays that; aligning the stores on the DDP side would be the fix there.
// The copy is bit for bit: the element type only sets the width (uint32 for fp32, uint16 for bf16).
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"
#include "ops.h"

namespace dr {

namespace {

constexpr int kRepackThreads = 256;
constexpr int kRepackItems = 4;

// largest s in [lo, hi] with vec_begin[s] <= v (row s of the table is {ddp_off, eng_off, numel, vec_begin})
__device__ __forceinline__ int repack_find(const int64_t* __restrict__ tab, int lo, int hi, int64_t v) {
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(tab + 4 * mid + 3) <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

template <typename T, bool kPack>
__global__ void __launch_bounds__(kRepackThreads) bucket_repack_kernel(const T* __restrict__ src, T* __restrict__ dst,
                                                                       const int64_t* __restrict__ tab, int n_seg,
                                                                       int64_t n_vec) {
  constexpr int V = 16 / sizeof(T);
  __shared__ int s_range[2];
  const int64_t base = (int64_t)blockIdx.x * (kRepackThreads * kRepackItems);
  if (threadIdx.x < 2) {
    const int64_t last = min(base + kRepackThreads * kRepackItems, n_vec) - 1;
    s_range[threadIdx.x] = repack_find(tab, 0, n_seg - 1, threadIdx.x == 0 ? base : last);
  }
  __syncthreads();
  const int lo = s_range[0], hi = s_range[1];
#pragma unroll
  for (int it = 0; it < kRepackItems; ++it) {
    const int64_t v = base + it * kRepackThreads + threadIdx.x;
    if (v >= n_vec) break;
    const int s = repack_find(tab, lo, hi, v);
    const int64_t ddp_off = __ldg(tab + 4 * s), eng_off = __ldg(tab + 4 * s + 1), numel = __ldg(tab + 4 * s + 2);
    const int64_t j = (v - __ldg(tab + 4 * s + 3)) * V;
    const int n = numel - j < V ? (int)(numel - j) : V;
    const T* in = src + (kPack ? ddp_off : eng_off) + j;
    T* out = dst + (kPack ? eng_off : ddp_off) + j;
    const T* ddp_ptr = kPack ? in : out;
    if (n == V && (reinterpret_cast<uintptr_t>(ddp_ptr) & 15) == 0) {
      *reinterpret_cast<uint4*>(out) = *reinterpret_cast<const uint4*>(in);
    } else if (n == V && !kPack) {
      // unpack: the engine side is aligned, one 16-byte load; the misaligned DDP side is stored element by element
      const uint4 w = *reinterpret_cast<const uint4*>(in);
      const T* e = reinterpret_cast<const T*>(&w);
#pragma unroll
      for (int i = 0; i < V; ++i) out[i] = e[i];
    } else if (n == V) {
      // pack: the misaligned DDP side is read element by element, the engine side gets one 16-byte store
      uint4 w;
      T* e = reinterpret_cast<T*>(&w);
#pragma unroll
      for (int i = 0; i < V; ++i) e[i] = in[i];
      *reinterpret_cast<uint4*>(out) = w;
    } else {
      for (int i = 0; i < n; ++i) out[i] = in[i];       // the segment's tail: the padding after it is not touched
    }
  }
}

template <typename T, bool kPack>
cudaError_t repack_launch(const void* src, void* dst, const int64_t* table, int n_seg, int64_t n_vec, cudaStream_t st) {
  if (n_seg == 0 || n_vec == 0) return cudaSuccess;
  const int64_t per_block = kRepackThreads * kRepackItems;
  const int64_t grid = (n_vec + per_block - 1) / per_block;
  bucket_repack_kernel<T, kPack><<<(unsigned)grid, kRepackThreads, 0, st>>>(
      static_cast<const T*>(src), static_cast<T*>(dst), table, n_seg, n_vec);
  count_launch();
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_bucket_repack(bool pack, int elem_bytes, const void* src, void* dst, const int64_t* table, int n_seg,
                                 int64_t n_vec, cudaStream_t st) {
  if (elem_bytes == 4)
    return pack ? repack_launch<uint32_t, true>(src, dst, table, n_seg, n_vec, st)
                : repack_launch<uint32_t, false>(src, dst, table, n_seg, n_vec, st);
  if (elem_bytes == 2)
    return pack ? repack_launch<uint16_t, true>(src, dst, table, n_seg, n_vec, st)
                : repack_launch<uint16_t, false>(src, dst, table, n_seg, n_vec, st);
  return cudaErrorInvalidValue;
}

}  // namespace dr
