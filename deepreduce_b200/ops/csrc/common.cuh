// Shared device/host helpers for the DeepReduce-B200 kernels (sm_90a).
// Hash family and bit layout are normative: see deepreduce_b200/spec.py.
//
// Parity: the reference looks hashes up in a precomputed MurmurHash3 table `hash_table[d_max, k_max]`
// (pytorch/deepreduce.py:440,461-463,471; ~1.5 MB for ResNet-20, ~1 GB for NCF — paper p.29) and reduces them
// `% size`; here the k positions of an index are computed on the fly (two murmur3 finalisers, Kirsch-Mitzenmacher
// h_j = a + j*b, Lemire multiply-shift range reduction), so d is unbounded and no table is loaded.  The bit array is
// built bit-packed (uint32 words, LSB first) — the reference's bool array + cupy.packbits step (:446-455,529) is gone.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "plan.h"

#define DR_HD __host__ __device__ __forceinline__
#define DR_D __device__ __forceinline__

namespace dr {

constexpr uint32_t kGolden = 0x9E3779B1u;
constexpr uint32_t kBAdd = 0x7F4A7C15u;
constexpr int kThreads = 512;         // threads per CTA in the engine kernels
constexpr int kPerThread = kTile / kThreads;   // 8
constexpr int kWarps = kThreads / 32;          // 16

DR_HD uint32_t fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}

struct HashAB { uint32_t a, b; };

DR_HD HashAB hash_ab(uint32_t x, uint32_t seed) {
  uint32_t y = x ^ seed;
  HashAB r;
  r.a = fmix32(y);
  r.b = fmix32(y * kGolden + kBAdd) | 1u;
  return r;
}

DR_HD uint32_t mulhi32(uint32_t h, uint32_t m) {
#ifdef __CUDA_ARCH__
  return __umulhi(h, m);
#else
  return (uint32_t)(((uint64_t)h * (uint64_t)m) >> 32);
#endif
}

DR_HD uint32_t policy_hash(uint32_t x, uint32_t seed) {
  return fmix32((x * kGolden + seed) ^ 0x5BD1E995u);
}

// per-(step, tensor) seed of the 'random' policy (spec.py::policy_seed): sender, residual update and receivers agree
DR_HD uint32_t policy_seed(uint32_t step, uint32_t tensor_id) {
  return fmix32((step * 0x01000193u) ^ ((tensor_id + 1u) * kGolden));
}

// Membership test with early exit, two probes per iteration (both loads in flight).
// `filter` is a bit-packed uint32 array.
template <typename LoadFn>
DR_D bool bloom_test(uint32_t x, uint32_t seed, uint32_t n_hash, uint32_t m_bits, LoadFn ld) {
  HashAB h = hash_ab(x, seed);
  uint32_t v = h.a;
  uint32_t j = 0;
  for (; j + 1 < n_hash; j += 2) {
    const uint32_t p0 = mulhi32(v, m_bits), p1 = mulhi32(v + h.b, m_bits);
    const uint32_t w0 = ld(p0 >> 5), w1 = ld(p1 >> 5);
    if (!((w0 >> (p0 & 31u)) & (w1 >> (p1 & 31u)) & 1u)) return false;
    v += 2u * h.b;
  }
  if (j < n_hash) {
    const uint32_t p0 = mulhi32(v, m_bits);
    if (!((ld(p0 >> 5) >> (p0 & 31u)) & 1u)) return false;
  }
  return true;
}

DR_D void bloom_set(uint32_t* filter, uint32_t x, uint32_t seed, uint32_t n_hash, uint32_t m_bits) {
  HashAB h = hash_ab(x, seed);
  uint32_t v = h.a;
  for (uint32_t j = 0; j < n_hash; ++j) {
    uint32_t pos = mulhi32(v, m_bits);
    atomicOr(filter + (pos >> 5), 1u << (pos & 31u));
    v += h.b;
  }
}

// ---- memory-model helpers -------------------------------------------------
DR_D uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
DR_D uint64_t ld_acquire_gpu64(const uint64_t* p) {
  uint64_t v; asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
}
DR_D void st_release_gpu64(uint64_t* p, uint64_t v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
DR_D uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
DR_D void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
DR_D uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v; asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
// streaming 128-bit load that does not allocate in L1 (data touched once per pass)
DR_D float4 ld_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
DR_D uint4 ld_stream_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// ---- TMA bulk copy (cp.async.bulk, 1-D) + mbarrier helpers ------------------------------------
DR_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
DR_D void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
DR_D void mbar_inval(uint64_t* bar) {
  asm volatile("mbarrier.inval.shared::cta.b64 [%0];" :: "r"(smem_u32(bar)) : "memory");
}
DR_D void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
DR_D void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
// shared-memory-only variant: orders generic-proxy reads of an SMEM stage before the TMA (async-proxy) write that
// refills it.  The unqualified fence above lowers to MEMBAR.ALL.GPU + FENCE.VIEW.ASYNC and waits for every global
// store of the thread — it must stay out of the ring's refill path (profiles/: v11 accumulate phase).
DR_D void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
DR_D void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// global -> shared bulk copy executed by the TMA unit; completion is signalled on `bar` (complete_tx)
DR_D void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
DR_D void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
DR_D uint64_t globaltimer_ns() {
  uint64_t t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}
DR_D void mbar_wait(uint64_t* bar, uint32_t parity, uint32_t* status = nullptr) {
  uint32_t ok, spins = 0;
  do {
    if (++spins > (1u << 24)) { if (status) atomicExch(status, 5u); break; }   // watchdog: never hang the GPU
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}

// ---- cp.async (LDGSTS): global -> shared copies tracked by commit groups, not by the register scoreboard.  A
// software prefetch through registers dies at ~5 loads in flight per warp (6 scoreboard slots, counting semantics:
// waiting for the oldest load also waits for every newer one sharing its slot — v12 profile of the candidate walks)
DR_D void cp_async_8(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
DR_D void cp_async_4(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
DR_D void cp_async_16(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
DR_D void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
DR_D void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

// NVLS: a store to a multicast address is replicated by the NVSwitch into every bound GPU's memory
DR_D void multimem_st_v4(uint4* mc_addr, uint4 v) {
  asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc_addr), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
                  "f"(__uint_as_float(v.w)) : "memory");
}

DR_D void multimem_st_v2(uint2* mc_addr, uint2 v) {
  asm volatile("multimem.st.weak.global.v2.f32 [%0], {%1,%2};"
               :: "l"(mc_addr), "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)) : "memory");
}
DR_D void multimem_st_b32(uint32_t* mc_addr, uint32_t v) {
  asm volatile("multimem.st.weak.global.f32 [%0], %1;" :: "l"(mc_addr), "f"(__uint_as_float(v)) : "memory");
}

// Grid-wide barrier for a co-resident (cooperative-launch) grid.  `counter`
// is zeroed by the host before launch; `*epoch` is a per-thread-0 register
// copy counting barriers passed.
DR_D void grid_barrier(uint32_t* counter, uint32_t& epoch, uint32_t* status, uint32_t spin_limit) {
  fence_proxy_async();          // generic-proxy global writes of this phase vs. TMA (async-proxy) reads of the next
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += 1;
    const uint32_t target = epoch * gridDim.x;
    __threadfence();
    atomicAdd(counter, 1u);
    uint32_t spins = 0;
    while (ld_acquire_gpu(counter) < target) {
      __nanosleep(32);
      if (++spins > spin_limit) { atomicExch(status, 4u); break; }   // watchdog: never hang the GPU
    }
    __threadfence();
  }
  __syncthreads();
}

// Gram (discrete Chebyshev) polynomials on the grid x = 0..N (N = n-1), exactly orthogonal there:
// p_0=1, p_1=1-2x/N, (k+1)(N-k)p_{k+1} = (2k+1)(N-2x)p_k - k(N+k+1)p_{k-1}   (codecs/polyfit.py)
template <int kDegP1>
DR_D void gram_eval(float x, float N, int deg_eff, float (&p)[kDegP1]) {
  p[0] = 1.f;
#pragma unroll
  for (int k = 1; k < kDegP1; ++k) p[k] = 0.f;
  if (deg_eff >= 1) {
    const float u = N - 2.f * x;
    p[1] = u / N;
#pragma unroll
    for (int k = 1; k < kDegP1 - 1; ++k) {
      if (k < deg_eff)
        p[k + 1] = ((2.f * k + 1.f) * u * p[k] - (float)k * (N + k + 1.f) * p[k - 1]) / ((k + 1.f) * (N - k));
    }
  }
}

// launch accounting (bench.py's "gpu_launches")
void count_launch(int n = 1);
long long launch_count();

// SMs of the current device, read once per device: grid-stride kernels size their grids as a few CTAs per SM
int sm_count();

}  // namespace dr
