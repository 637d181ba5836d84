// Microbenchmark: do two co-resident 512-thread CTAs of an SM run an issue-bound streaming phase at the same speed?
// Work = the engine's accumulate phase in miniature (read g, read r, write r + g, write g = 0, candidate compaction by
// ballot, digit-1 SMEM histogram, conditional digit-2 histogram), one contiguous tile range per (virtual) CTA.
//   mode 0: 264 CTAs x 512 threads (2 per SM) — what the engine launches
//   mode 1: 132 CTAs x 1024 threads, virtual CTA = warps 0-15 / 16-31
//   mode 2: 132 CTAs x 1024 threads, virtual CTA = warps whose id has bit 2 clear / set (halves interleaved on every
//           scheduler: warp w runs on sub-partition w % 4)
// Prints the kernel time and the mean per-virtual-CTA duration of the first / second virtual CTA of every SM.
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o cta_age_bench cta_age_bench.cu
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cuda_runtime.h>

constexpr int kTile = 4096, kV = 512;

__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

template <int kThreads>
__global__ void __launch_bounds__(kThreads, 1024 / kThreads * 1) k(float* __restrict__ g, float* __restrict__ r, uint2* __restrict__ cand,
    unsigned* __restrict__ cand_cnt, int n_tiles, unsigned thr, unsigned guess, int mode, unsigned long long* times, unsigned* smids) {
  __shared__ unsigned hist2[2][4096];
  const unsigned W = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned half = 0, vwarp = W;
  if (kThreads == 1024) {
    if (mode == 1) { half = W >> 4; vwarp = W & 15; }
    else { half = (W >> 2) & 1; vwarp = (W & 3) | ((W >> 3) << 2); }
  }
  const unsigned vtid = vwarp * 32 + lane;
  const int halves = kThreads / kV;
  const int G = gridDim.x * halves, b = blockIdx.x * halves + half;
  unsigned* hist = hist2[half];
  for (int j = vtid; j < 4096; j += kV) hist[j] = 0;
  __syncthreads();
  unsigned long long t0 = 0;
  if (vtid == 0) t0 = gtime();
  const int per = (n_tiles + G - 1) / G;
  const unsigned lt = (1u << lane) - 1u;
  for (int i = 0; i < per; ++i) {
    const int tile = b * per + i;
    if (tile >= n_tiles) continue;
    float4* gp = reinterpret_cast<float4*>(g + (size_t)tile * kTile);
    float4* rp = reinterpret_cast<float4*>(r + (size_t)tile * kTile);
    uint2* chunk = cand + ((size_t)tile * 16 + vwarp) * 256;
    unsigned cnt = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = h * kV + vtid;
      float4 a = gp[j], c = rp[j];
      c.x += a.x; c.y += a.y; c.z += a.z; c.w += a.w;
      rp[j] = c;
      gp[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      const unsigned key[4] = {__float_as_uint(c.x) & 0x7FFFFFFFu, __float_as_uint(c.y) & 0x7FFFFFFFu,
                               __float_as_uint(c.z) & 0x7FFFFFFFu, __float_as_uint(c.w) & 0x7FFFFFFFu};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const bool f = key[q] >= thr;
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, f);
        if (f) {
          chunk[cnt + __popc(bal & lt)] = make_uint2(key[q], (unsigned)(j * 4 + q));
          atomicAdd(&hist[key[q] >> 20], 1u);
          if ((key[q] >> 20) == guess) atomicAdd(&hist[2048 + ((key[q] >> 9) & 0x7FFu)], 1u);
        }
        cnt += __popc(bal);
      }
    }
    if (lane == 0) cand_cnt[tile * 16 + vwarp] = cnt;
  }
  if (vtid == 0) {
    times[b] = gtime() - t0;
    unsigned s; asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
    smids[b] = s;
  }
  __syncthreads();
  for (int j = vtid; j < 4096; j += kV) if (hist[j]) atomicAdd(cand_cnt + (j & 15), hist[j]);
}

int main() {
  const int n_tiles = 6240;
  const size_t n = (size_t)n_tiles * kTile;
  float *g, *r, *flush, *src; uint2* cand; unsigned* cnt; unsigned long long* times; unsigned* smids;
  cudaMalloc(&g, n * 4); cudaMalloc(&r, n * 4); cudaMalloc(&src, n * 4); cudaMalloc(&flush, 256u << 20);
  cudaMalloc(&cand, n * 8); cudaMalloc(&cnt, n_tiles * 16 * 4); cudaMalloc(&times, 264 * 8); cudaMalloc(&smids, 264 * 4);
  float* h = (float*)malloc(n * 4);
  srand(1);
  for (size_t i = 0; i < n; ++i) h[i] = (float)rand() / RAND_MAX;
  cudaMemcpy(src, h, n * 4, cudaMemcpyHostToDevice);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const float t = 1.0f - 0.12f;                      // 12 % candidates
  unsigned thr; memcpy(&thr, &t, 4);
  for (int mode = 0; mode < 3; ++mode) {
    float best = 1e9f, sum = 0.f;
    double first = 0, second = 0, mx = 0;
    for (int it = 0; it < 12; ++it) {
      cudaMemcpyAsync(g, src, n * 4, cudaMemcpyDeviceToDevice);
      cudaMemsetAsync(r, 0, n * 4);
      cudaMemsetAsync(flush, 1, 256u << 20);
      cudaEventRecord(e0);
      if (mode == 0) k<512><<<264, 512>>>(g, r, cand, cnt, n_tiles, thr, thr >> 20, mode, times, smids);
      else k<1024><<<132, 1024>>>(g, r, cand, cnt, n_tiles, thr, thr >> 20, mode, times, smids);
      cudaEventRecord(e1); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      if (it >= 2) {
        best = ms < best ? ms : best; sum += ms;
        unsigned long long ht[264]; unsigned hs[264];
        cudaMemcpy(ht, times, 264 * 8, cudaMemcpyDeviceToHost); cudaMemcpy(hs, smids, 264 * 4, cudaMemcpyDeviceToHost);
        // first / second virtual CTA of an SM: by index order among the virtual CTAs that report the same smid
        int seen[512]; memset(seen, 0, sizeof(seen));
        double f = 0, s = 0; int nf = 0, ns = 0; double m = 0;
        for (int b = 0; b < 264; ++b) {
          const double us = ht[b] / 1e3;
          if (us > m) m = us;
          if (seen[hs[b] & 511]++ == 0) { f += us; ++nf; } else { s += us; ++ns; }
        }
        first += f / (nf ? nf : 1) / 10; second += s / (ns ? ns : 1) / 10; mx += m / 10;
      }
    }
    printf("mode %d: kernel mean %.1f us best %.1f us | per-virtual-CTA duration: first-of-SM %.1f us, second-of-SM %.1f us, max %.1f us\n",
           mode, sum / 10 * 1e3, best * 1e3, first, second, mx);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
