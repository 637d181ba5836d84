// Microbenchmark: what costs HBM throughput in the engine's accumulate phase?
// Base traffic: read g, read r, write r' = r + g, write g = 0 (4 x 102 MB), persistent 264 x 512 threads, contiguous
// tile range per CTA.  Feature bits add the engine's extra work one by one:
//   1 = candidate compaction (|x| >= thr: ballot positions + 8-byte scattered stores into a (tile, warp) chunk)
//   2 = shared-memory histogram atomic per candidate (digit 1)
//   4 = second shared-memory histogram atomic (speculative digit 2)
//   8 = blocked-cyclic tile mapping (B = 4) instead of contiguous ranges
//  16 = loads staged through shared memory with cp.async (4 groups in flight per thread) instead of direct LDG
//  32 = second histogram only for keys whose digit 1 equals a guess (what the engine does)
//  (dyn_smem > 0: allocate that much dynamic shared memory, shrinking the L1)
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o stream_pattern_bench stream_pattern_bench.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

constexpr int kTile = 4096, kThreads = 512;

__global__ void __launch_bounds__(kThreads, 2) stream_kernel(float* __restrict__ g, float* __restrict__ r, uint2* __restrict__ cand,
                                                             unsigned* __restrict__ cand_cnt, int n_tiles, int feat, unsigned thr, unsigned guess) {
  __shared__ unsigned hist[4096];
  extern __shared__ __align__(16) unsigned char dyn[];
  for (int j = threadIdx.x; j < 4096; j += kThreads) hist[j] = 0;
  __syncthreads();
  const int G = gridDim.x, b = blockIdx.x;
  const int per = (n_tiles + G - 1) / G;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
  for (int i = 0; i < per; ++i) {
    int tile = (feat & 8) ? ((i / 4) * G + b) * 4 + (i % 4) : b * per + i;
    if (tile >= n_tiles) continue;
    float4* gp = reinterpret_cast<float4*>(g + (size_t)tile * kTile);
    float4* rp = reinterpret_cast<float4*>(r + (size_t)tile * kTile);
    uint2* chunk = cand + ((size_t)tile * 16 + warp) * 256;
    unsigned cnt = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = h * kThreads + threadIdx.x;
      float4 a, c;
      if (feat & 16) {
        // ring of 4 items (half-tiles) per thread: slot = item & 3; item sequence = (i, h)
        const int item = i * 2 + h;
        auto issue = [&](int it) {
          const int ti = it >> 1, hh = it & 1;
          int tl = (feat & 8) ? ((ti / 4) * G + b) * 4 + (ti % 4) : b * per + ti;
          if (ti < per && tl < n_tiles) {
            const float4* gs = reinterpret_cast<const float4*>(g + (size_t)tl * kTile) + hh * kThreads + threadIdx.x;
            const float4* rs = reinterpret_cast<const float4*>(r + (size_t)tl * kTile) + hh * kThreads + threadIdx.x;
            unsigned d = (unsigned)__cvta_generic_to_shared(dyn + ((it & 3) * 2 * kThreads + threadIdx.x) * 16);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(d), "l"(gs) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(d + kThreads * 16), "l"(rs) : "memory");
          }
          asm volatile("cp.async.commit_group;" ::: "memory");
        };
        if (item == 0) { issue(0); issue(1); issue(2); }
        issue(item + 3);
        asm volatile("cp.async.wait_group 3;" ::: "memory");
        const float4* sl = reinterpret_cast<const float4*>(dyn + ((item & 3) * 2 * kThreads + threadIdx.x) * 16);
        a = sl[0]; c = sl[kThreads];
      } else { a = gp[j]; c = rp[j]; }
      c.x += a.x; c.y += a.y; c.z += a.z; c.w += a.w;
      rp[j] = c;
      gp[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (feat & 1) {
        const unsigned key[4] = {__float_as_uint(c.x) & 0x7FFFFFFFu, __float_as_uint(c.y) & 0x7FFFFFFFu,
                                 __float_as_uint(c.z) & 0x7FFFFFFFu, __float_as_uint(c.w) & 0x7FFFFFFFu};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const bool f = key[q] >= thr;
          const unsigned bal = __ballot_sync(0xFFFFFFFFu, f);
          if (f) {
            chunk[cnt + __popc(bal & lt)] = make_uint2(key[q], (unsigned)(j * 4 + q));
            if (feat & 2) atomicAdd(&hist[key[q] >> 20], 1u);
            if ((feat & 4) && (!(feat & 32) || (key[q] >> 20) == guess)) atomicAdd(&hist[2048 + ((key[q] >> 9) & 0x7FFu)], 1u);
          }
          cnt += __popc(bal);
        }
      }
    }
    if ((feat & 1) && lane == 0) cand_cnt[tile * 16 + warp] = cnt;
  }
  if (feat & 6) {
    __syncthreads();
    for (int j = threadIdx.x; j < 4096; j += kThreads) if (hist[j]) atomicAdd(cand_cnt + (j & 15), hist[j]);
  }
}

int main(int argc, char** argv) {
  const int n_tiles = 6240;                         // ~25.56 M elements
  const size_t n = (size_t)n_tiles * kTile;
  float *g, *r, *flush, *src;
  uint2* cand; unsigned* cnt;
  cudaMalloc(&g, n * 4); cudaMalloc(&r, n * 4); cudaMalloc(&src, n * 4); cudaMalloc(&flush, 256u << 20);
  cudaMalloc(&cand, n * 8); cudaMalloc(&cnt, n_tiles * 16 * 4);
  float* h = (float*)malloc(n * 4);
  srand(1);
  for (size_t i = 0; i < n; ++i) h[i] = (float)rand() / RAND_MAX;      // uniform [0,1]: thr picks the candidate rate
  cudaMemcpy(src, h, n * 4, cudaMemcpyHostToDevice);
  cudaMemset(r, 0, n * 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int grid = 264;
  const float rates[3] = {0.07f, 0.16f, 1.0f};
  const int feats[] = {0, 16, 1, 3, 7, 39, 17, 19, 55, 0, 1, 17, 55};
  const int dyns[] =  {0, 65536, 0, 0, 0, 0, 65536, 65536, 65536, 81920, 81920, 81920, 81920};
  cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 90 * 1024);
  for (int fi = 0; fi < 13; ++fi) {
    for (int ri = 0; ri < 2; ++ri) {
      const int feat = feats[fi];
      const int dyn_smem = dyns[fi];
      if (!(feat & 1) && ri) continue;
      const float t = 1.0f - rates[ri];
      unsigned thr; memcpy(&thr, &t, 4);
      float best = 1e9f, sum = 0.f;
      for (int it = 0; it < 12; ++it) {
        cudaMemcpyAsync(g, src, n * 4, cudaMemcpyDeviceToDevice);
        cudaMemsetAsync(r, 0, n * 4);
        cudaMemsetAsync(flush, 1, 256u << 20);
        cudaEventRecord(e0);
        stream_kernel<<<grid, kThreads, dyn_smem>>>(g, r, cand, cnt, n_tiles, feat, thr, thr >> 20);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (it >= 2) { best = ms < best ? ms : best; sum += ms; }
      }
      printf("feat=%2d dyn=%5d cand_rate=%.2f  mean %.1f us  best %.1f us  -> %.0f GB/s of base traffic\n", feat, dyn_smem, (feat & 1) ? rates[ri] : 0.f,
             sum / 10 * 1e3, best * 1e3, 4.0 * n * 4 / (sum / 10 * 1e-3) / 1e9);
    }
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
