// DeepReduce-B200 fused bucket engine (sm_90a), v22.
//
// One persistent, cooperatively-launched kernel runs the whole per-bucket
// gradient exchange:
//
//   accumulate residual (TMA ring) + zero the dense output + candidate lists ->
//   per-tensor top-k threshold (2-digit radix select, digit 2 over the candidates
//   only) -> bloom insert + occupancy hint from the candidates -> membership test
//   of the hinted 32-element groups (two-level survivor queue) -> ordered
//   compaction from group bitmasks + FP-aware value gather + residual update ->
//   P2P store of the compressed slot into every peer's arena over NVLink ->
//   release / acquire flags -> decode of all W slots for this rank's slice ->
//   second in-kernel exchange of the exact slice lists.
//
// It replaces, per tensor, the reference's chain: GRACE residual add, torch.topk,
// Bloomfilter.add/query/policy (reference pytorch/deepreduce.py:457-492,506-533),
// cupy packbits, 2-3 NCCL all_gathers (SURVEY C1), W x Bloom.decompress (:536-555),
// W x zeros+scatter and the sum (SURVEY K1-K7, K13).  Phases can also be launched
// one at a time (phase_begin/phase_end) — the "unfused chain" debug mode.
//
// Work decomposition: the bucket is cut into 4096-element tiles that never cross a
// tensor; every streaming phase gives CTA b one contiguous tile range, cut on the host
// per phase class from per-tile costs and measured per-CTA speeds (tile_range, P.cuts).
// The universe is read exactly once (accumulate): everything after it works on
//   * the candidate list  — the (key, offset) pairs with |x| above a fraction of last
//     step's threshold, written per (tile, warp) at a fixed location (no allocation,
//     no overflow); digit 2 of the select and the bloom insert walk it instead of d;
//   * group bitmasks      — one 32-bit word per 32 consecutive elements: the query
//     leaves the positives there, emit / decode derive ordered ranks from popcounts.
// v10 -> v11 (profiles/): 4 passes over d -> 1, per-tile CTA barriers -> mbarrier
// full/empty ring + warp-private work, probe chains run on dense survivor batches.
#include "common.cuh"
#include "dexp_fit.cuh"
#include "fp8_values.cuh"
#include "plan.h"
#include "sign_values.cuh"
#include "tiles.cuh"

#include <cuda_bf16.h>

#include <atomic>
#include <cstdio>

namespace dr {

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n); }
long long launch_count() { return g_launches.load(); }

int sm_count() {
  constexpr int kMaxDevices = 64;
  static std::atomic<int> cached[kMaxDevices];
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < kMaxDevices) n = cached[dev].load(std::memory_order_relaxed);
  if (n > 0) return n;
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  if (n < 1) n = 1;
  if (dev >= 0 && dev < kMaxDevices) cached[dev].store(n, std::memory_order_relaxed);
  return n;
}

namespace {

constexpr uint32_t kErrPeerWait = 2u, kErrResolve = 3u, kErrS2Overflow = 6u, kErrDisagree = 7u;
constexpr uint32_t kNoTensor = 0xFFFFFFFFu;
constexpr uint32_t kChunk = 256;                      // candidate capacity per (tile, warp) = the elements a warp owns
constexpr uint32_t kHalf = kTile / 2;                 // elements per ring stage (g half-tile | r half-tile)
constexpr uint32_t kStageBytes = 2u * kHalf * 4u;     // 16 KB
constexpr uint32_t kMaxStages = 6;
constexpr uint32_t kCpStages = 4;                     // cp.async variant of the accumulate ring: fixed depth (wait_group needs a constant)
constexpr int kPF = 4;                                // candidate-list walks: chunk heads in flight per warp (cp.async ring)
constexpr uint32_t kHead = 64;                        // entries of a chunk head (512 B): with ~20 % of the elements above the history bound a
                                                      // chunk holds ~50, and entries past the head are fetched on demand (one exposed DRAM latency)
constexpr uint32_t kUnsafeWord = 8;                   // P.barrier[8]: tensors whose history bound hid the threshold
constexpr uint32_t kNeedHist2Word = 9;                // P.barrier[9]: tensors whose digit 2 could not be taken speculatively

struct ScanSmem {
  uint32_t warp_tot[kWarps];
  uint32_t res[4];                            // resolve results: bin, krem, bincount, spare
  uint32_t lb;                                // small CTA-wide scratch word / dynamic work counter
  uint32_t rle_pre[16];                       // kModeRle decode: running entry prefix per sender
};

struct Smem {
  union {
    uint32_t hist[2 * kHistBins];             // radix-select digit histogram | speculative digit-2 histogram (accumulate phase)
    float acc[kTile];                         // raw / rle decode accumulator
    uint32_t q[kWarps][64];                   // probe passes: per-warp survivor ring
    uint32_t excl[kTile];                     // emit: exclusive prefixes of a chunk of tiles
    uint32_t sel[kWarps][32];                 // insert: selected elements of one warp iteration
    DexpScratch dexp;                         // fit phase: one double-exponential fit
    double sign_ws[kWarps];                   // fix phase, kVmodeSign: the warp sums of one bucket's |v|
    uint32_t fp8_scales[kWarps / 4];          // fix phase, kVmodeFp8: the scale bytes of one task's 16 blocks
  } u;
  ScanSmem s;
  TensorDesc td;                              // current tensor
  uint64_t bar[16];                           // mbarriers of the TMA ring: full[0..8), empty[8..16)
  int seg_start[kMaxSeg + 2];                 // 'both': segment boundaries of the current (tensor, rank)
  int n_seg;
};

extern __shared__ __align__(16) uint32_t g_filter_smem[];   // dynamic: staged bloom filter / TMA ring / stage-2 staging

DR_D uint32_t* slot_ptr(uint32_t* arena, const EngineParams& P, uint32_t parity, int src) {
  return arena + slot_offset(P, parity, src);
}

DR_D uint32_t* s2_ptr(uint32_t* arena, const EngineParams& P, uint32_t parity, int src) {
  return arena + s2_offset(P, parity, src);
}

// this CTA's contiguous share of the decode span (decode and compact use the SAME split, so the CTA that decoded
// a tile is the one that compacts it — no grid barrier in between)
DR_D void decode_range(const EngineParams& P, uint32_t& tile, uint32_t& t_end) {
  uint32_t s_begin, s_end;
  decode_span(P, P.rank, s_begin, s_end);
  const uint32_t span = s_end - s_begin;
  tile = s_begin + (uint32_t)(((uint64_t)span * blockIdx.x) / gridDim.x);
  t_end = s_begin + (uint32_t)(((uint64_t)span * (blockIdx.x + 1)) / gridDim.x);
}

// final value of dense output element i: fp32 as is, bf16 rounded once to nearest-even
template <bool kB>
DR_D void put_out(const EngineParams& P, size_t i, float v) {
  if constexpr (kB) P.grad_bf16[i] = __bfloat16_as_ushort(__float2bfloat16_rn(v));
  else P.grad[i] = v;
}

// four consecutive bf16 (8 bytes, element 0 in the low half of x) widened to fp32 — exact
DR_D float4 widen_bf16x4(uint2 h) {
  return make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xFFFF0000u), __uint_as_float(h.y << 16),
                     __uint_as_float(h.y & 0xFFFF0000u));
}

// round to nearest even (a finite value past the largest bf16 becomes +-inf), every NaN to the quiet NaN 0x7FC0
DR_D uint32_t bf16_rne_bits(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x7FFFFFFFu) > 0x7F800000u ? 0x7FC0u : (u + 0x7FFFu + ((u >> 16) & 1u)) >> 16;
}

// at W == 1 emit has already scattered the tensor's decoded fp32 values into the output (bf16 values too: phase_accum).
// phase_compact writes it out in its two skip tests, where the vmode load stays behind the short-circuit.
DR_D bool emit_scatters(const EngineParams& P, uint32_t vmode) { return P.world == 1 && vmode == kVmodeFp32; }

// bf16 buckets' bloom tensors that phase_compact applies (every sender added into acc32, then rounded once)
DR_D bool bloom_applied(const EngineParams& P, uint32_t mode, uint32_t vmode) {
  return mode == (uint32_t)kModeBloom && !emit_scatters(P, vmode);
}

DR_D void load_tensor(const EngineParams& P, uint32_t t, Smem& sm) {
  __syncthreads();
  if (threadIdx.x < kDescWords) {
    reinterpret_cast<uint32_t*>(&sm.td)[threadIdx.x] =
        __ldg(reinterpret_cast<const uint32_t*>(P.tensors + t) + threadIdx.x);
  }
  __syncthreads();
}

DR_D size_t chunk_of(uint32_t tile, uint32_t warp) { return ((size_t)tile * kWarps + warp) * kChunk; }

// ---------------------------------------------------------------------------
// radix-select digit resolve: find the bin holding the k-th largest key.
// Result in s.res: [0] bin (0xFFFFFFFF if total < k), [1] k remaining inside
// the bin, [2] count in the bin.
// ---------------------------------------------------------------------------
DR_D uint32_t* hist_ptr(const EngineParams& P, int which, uint32_t t) {
  return P.hist + ((size_t)which * P.n_tensors + t) * kHistBins;
}

template <typename LoadFn>
DR_D void resolve_bins(LoadFn H, int nbins, uint32_t k, ScanSmem& s) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  __syncthreads();
  if (tid == 0) { s.res[0] = 0xFFFFFFFFu; s.res[1] = 0; s.res[2] = 0; }
  uint32_t c[4], sum = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int rb = (int)tid * 4 + i;            // reversed position: 0 = largest digit
    c[i] = (rb < nbins) ? H(nbins - 1 - rb) : 0u;
    sum += c[i];
  }
  const uint32_t incl = warp_incl_scan(sum, lane);
  if (lane == 31) s.warp_tot[warp] = incl;
  __syncthreads();
  uint32_t base = 0;
  for (uint32_t w = 0; w < warp; ++w) base += s.warp_tot[w];
  uint32_t cum = base + incl - sum;             // keys strictly above my first bin
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int rb = (int)tid * 4 + i;
    if (rb < nbins && cum < k && cum + c[i] >= k) {
      s.res[0] = (uint32_t)(nbins - 1 - rb);
      s.res[1] = k - cum;
      s.res[2] = c[i];
    }
    cum += c[i];
  }
  __syncthreads();
}

DR_D void clear_hist(Smem& sm) {
  __syncthreads();
  for (int j = threadIdx.x; j < kHistBins; j += kThreads) sm.u.hist[j] = 0;
  __syncthreads();
}

// Merge this CTA's SMEM histogram of tensor t into the global one `gh` (kBins == 2 * kHistBins: the speculative digit-2
// half that follows it in SMEM goes to `gh2`), zeroing the SMEM bins, and take the tensor's ticket of histogram
// `which`.  Returns true (CTA-uniform) in the CTA whose merge completes the tensor (ticket count == n_tiles).
template <int kBins>
DR_D bool merge_ticket(const EngineParams& P, Smem& sm, int which, uint32_t t, uint32_t* __restrict__ gh,
                       uint32_t* __restrict__ gh2, uint32_t n_mine, uint32_t n_tiles) {
  __syncthreads();
  for (int j = threadIdx.x; j < kBins; j += kThreads) {
    const uint32_t v = sm.u.hist[j];
    if (v) { atomicAdd((j < kHistBins ? gh : gh2 - kHistBins) + j, v); sm.u.hist[j] = 0; }
  }
  __threadfence();                              // merged counts are visible before the ticket is taken
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t before = atomicAdd(P.hist_total + (size_t)which * P.n_tensors + t, n_mine);
    sm.s.lb = (before + n_mine == n_tiles) ? 1u : 0u;
    __threadfence();
  }
  __syncthreads();
  const bool last = sm.s.lb != 0u;
  __syncthreads();
  return last;
}

// Finish one digit of one tensor for this CTA.  If the CTA owns every tile of the tensor the digit is
// resolved straight from the SMEM histogram; otherwise the histogram is merged into the global one and
// the CTA whose merge completes the tensor (ticket count == n_tiles) resolves it — once per tensor,
// inside the same phase, no extra grid barrier.  Returns true (CTA-uniform) if this CTA resolved; the
// result is then in sm.s.res.
DR_D bool finish_digit(const EngineParams& P, Smem& sm, int which, uint32_t t, uint32_t n_mine, uint32_t n_tiles,
                       uint32_t k) {
  if (n_mine == n_tiles) {
    resolve_bins([&](int b) { return sm.u.hist[b]; }, kHistBins, k, sm.s);
    clear_hist(sm);
    return true;
  }
  uint32_t* gh = hist_ptr(P, which, t);
  const bool last = merge_ticket<kHistBins>(P, sm, which, t, gh, nullptr, n_mine, n_tiles);
  if (last) resolve_bins([&](int b) { return __ldcg(gh + b); }, kHistBins, k, sm.s);
  return last;
}

// stage a bloom filter (global, 16-byte aligned) into the dynamic SMEM buffer; read through L2: the filter was just
// built by atomics (own) or by remote stores (peers)
DR_D void stage_filter(const uint32_t* __restrict__ filter, uint32_t n_words) {
  __syncthreads();                              // previous users of the buffer are done
  const uint4* src = reinterpret_cast<const uint4*>(filter);
  uint4* dst = reinterpret_cast<uint4*>(g_filter_smem);
  const uint32_t n4 = (n_words + 3u) >> 2;
  for (uint32_t i = threadIdx.x; i < n4; i += kThreads) dst[i] = __ldcg(src + i);
  __syncthreads();
}

// first tile index whose cumulative cost reaches `target` (cost_prefix is non-decreasing, [n_tiles + 1] entries)
DR_D uint32_t cost_lower_bound(const uint32_t* __restrict__ cp, uint32_t n, uint32_t target) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldg(cp + mid) < target) lo = mid + 1; else hi = mid; }
  return lo;
}

// This CTA's contiguous tile range.  Ranges have equal COST, not equal length: a tile of a tensor that ends inside the
// range costs a histogram merge + ticket + resolve on top of its elements, and with equal counts the ~20 CTAs that
// own the many small tensors of a model set the duration of every streaming phase (v15 timeline: accumulate median
// 79 us, max 124 us; query 42 / 68 us).
DR_D void tile_range(const EngineParams& P, int part, uint32_t& t_begin, uint32_t& t_end) {
  if (P.cuts && gridDim.x == P.cuts_grid) {      // host-computed partition of this phase class (calibrated per CTA)
    const uint32_t* c = P.cuts + (size_t)part * (P.cuts_grid + 1u) + blockIdx.x;
    t_begin = __ldg(c); t_end = __ldg(c + 1);
    return;
  }
  if (P.cost_prefix) {
    const uint32_t total = __ldg(P.cost_prefix + P.n_tiles);
    const uint32_t lo = (uint32_t)(((uint64_t)total * blockIdx.x) / gridDim.x);
    const uint32_t hi = (uint32_t)(((uint64_t)total * (blockIdx.x + 1)) / gridDim.x);
    t_begin = blockIdx.x == 0 ? 0u : cost_lower_bound(P.cost_prefix, P.n_tiles, lo);
    t_end = blockIdx.x + 1 == gridDim.x ? P.n_tiles : cost_lower_bound(P.cost_prefix, P.n_tiles, hi);
    return;
  }
  t_begin = (uint32_t)(((uint64_t)P.n_tiles * blockIdx.x) / gridDim.x);
  t_end = (uint32_t)(((uint64_t)P.n_tiles * (blockIdx.x + 1)) / gridDim.x);
}

// ===========================================================================
// phase 0: accumulate + dense-output zero fill + candidate lists + hist digit 1
// (+ the whole select for single-tile tensors)
//
// g and r tiles arrive through a TMA ring of half-tile stages (cp.async.bulk + full/empty mbarriers): the 16 warps
// of a CTA drift through the stages independently — a warp releases a stage with one mbarrier arrive, thread 0
// refills the stage released one item earlier — and meet only where a tensor ends (histogram merge).
// Thread `tid` owns elements h*2048 + tid*4 .. +3 of a tile (h = half), so warp w owns two runs of 128 consecutive
// elements and its candidates of a tile go to the fixed chunk (tile*16 + w) * 256.
// ===========================================================================
constexpr uint32_t kUnsafe = 0xFFFFFFFFu;   // sel.bin1 marker: history bound hid the threshold -> fallback phase

// kModeShared select key of the in-tensor index i (plan.h "Selection rule"): the smallest hash gets the largest key
DR_D uint32_t shared_key(uint32_t i, uint32_t seed) { return (0xFFFFFFFFu - policy_hash(i, seed)) >> 1; }

DR_D void write_digit1(const EngineParams& P, Smem& sm, uint32_t t) {
  if (threadIdx.x == 0) {
    P.sel[t].bin1 = sm.s.res[0]; P.sel[t].krem1 = sm.s.res[1]; P.sel[t].done_epoch = 0;
    if (sm.s.res[0] == kUnsafe) atomicAdd(P.barrier + kUnsafeWord, 1u);
  }
}

DR_D void write_final(const EngineParams& P, Smem& sm, uint32_t t, uint32_t bin1) {
  if (threadIdx.x == 0) {
    if (sm.s.res[0] == 0xFFFFFFFFu) atomicExch(P.status, kErrResolve);
    const uint32_t T22 = max((bin1 << 11) | sm.s.res[0], 1u);
    P.sel[t].bin2 = sm.s.res[0]; P.sel[t].krem2 = sm.s.res[1];
    P.sel[t].thr = T22 << 9; P.sel[t].n_ge = sm.s.res[2];
  }
}

// Digit 2 of a one-tile tensor, from this thread's 8 keys still in registers (0xFFFFFFFF: not an element), once digit 1
// resolved to (bin1, krem1) and the SMEM histogram is clear.  An unsafe bin1 is the caller's to handle.
DR_D void finish_single(const EngineParams& P, Smem& sm, uint32_t t, const uint32_t (&keys)[8], uint32_t bin1,
                        uint32_t krem1) {
  if (bin1 == kUnsafe) return;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (keys[i] != 0xFFFFFFFFu && (keys[i] >> 20) == bin1) atomicAdd(&sm.u.hist[(keys[i] >> 9) & 0x7FFu], 1u);
  resolve_bins([&](int b) { return sm.u.hist[b]; }, kHistBins, krem1, sm.s);
  write_final(P, sm, t, bin1);
  if (threadIdx.x == 0) P.sel[t].done_epoch = P.epoch;
  clear_hist(sm);
}

// Digit 1 AND (speculatively) digit 2 of a multi-tile tensor at the end of the accumulate phase.  Every CTA also
// binned digit 2 of its candidates under the guess that the threshold bin is last step's (`guess`).  The CTA that
// completes the tensor resolves digit 1; if the guess was right it resolves digit 2 on the spot and the tensor needs
// no digit-2 phase at all (no pass over the candidates, no grid barrier) — otherwise it discards the speculative
// counts and the tensor is counted in P.barrier[kNeedHist2Word], which switches the digit-2 phase on for this step.
DR_D void finish_spec(const EngineParams& P, Smem& sm, uint32_t t, uint32_t n_mine, uint32_t n_tiles, uint32_t k,
                      uint32_t guess) {
  const uint32_t tid = threadIdx.x;
  uint32_t* gh1 = hist_ptr(P, 0, t);
  uint32_t* gh2 = hist_ptr(P, 2, t);
  const bool whole = (n_mine == n_tiles);                 // this CTA saw every tile: resolve from shared memory
  if (!whole && !merge_ticket<2 * kHistBins>(P, sm, 0, t, gh1, gh2, n_mine, n_tiles)) return;
  if (whole) resolve_bins([&](int b) { return sm.u.hist[b]; }, kHistBins, k, sm.s);
  else resolve_bins([&](int b) { return __ldcg(gh1 + b); }, kHistBins, k, sm.s);
  const uint32_t bin1 = sm.s.res[0], krem1 = sm.s.res[1];
  write_digit1(P, sm, t);
  if (bin1 != kUnsafe && bin1 == guess) {
    if (whole) resolve_bins([&](int b) { return sm.u.hist[kHistBins + b]; }, kHistBins, krem1, sm.s);
    else resolve_bins([&](int b) { return __ldcg(gh2 + b); }, kHistBins, krem1, sm.s);
    write_final(P, sm, t, bin1);
    if (tid == 0) P.sel[t].done_epoch = P.epoch;
  } else {
    if (!whole) for (int j = tid; j < kHistBins; j += kThreads) gh2[j] = 0u;     // the digit-2 phase starts from zero
    if (tid == 0) atomicAdd(P.barrier + kNeedHist2Word, 1u);
  }
  if (whole) {
    __syncthreads();
    for (int j = tid; j < 2 * kHistBins; j += kThreads) sm.u.hist[j] = 0;
    __syncthreads();
  }
}

// Append this thread's flagged elements (bit j of m: element e0 + j, key key[j]) to the warp's candidate chunk.
// `cnt` (warp-uniform) is the number of entries already in the chunk.  One ballot per element slot gives every
// flagged lane its position (popcount of the lower lanes) — no shuffle scan, no per-element branches with their own
// reconvergence points (v11/v12: 155 of the ~260 instructions of a half-tile iteration).
DR_D void append_candidates(Smem& sm, uint32_t m, const uint32_t (&key)[4], uint32_t e0, uint2* chunk, uint32_t& cnt,
                            bool do_hist, uint32_t lane, uint32_t guess = 0xFFFFFFFFu) {
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const bool f = ((m >> j) & 1u) != 0u;
    const uint32_t b = __ballot_sync(kFullMask, f);
    if (f) {
      chunk[cnt + (uint32_t)__popc(b & lt)] = make_uint2(key[j], e0 + (uint32_t)j);
      if (do_hist) {
        atomicAdd(&sm.u.hist[key[j] >> 20], 1u);
        // speculative digit 2: last step's threshold bin is almost always this step's (see finish_spec)
        if ((key[j] >> 20) == guess) atomicAdd(&sm.u.hist[kHistBins + ((key[j] >> 9) & 0x7FFu)], 1u);
      }
    }
    cnt += (uint32_t)__popc(b);
  }
}

DR_D uint32_t round16(uint32_t bytes) { return (bytes + 15u) & ~15u; }

// 'dgc' weight decay: the four parameter values of plan tensor t at in-tensor elements e .. e + 3, of which the first n
// (>= 1) lie inside the tensor; the others are padding of the engine's buffers, which the parameter does not have, and
// read as 0.  One vector load when the address is aligned and all four are inside, else element by element.  A bf16
// bucket's parameters stay packed (low half first, as widen_bf16x4 takes them) until they are used: two registers
// instead of four across the ring wait.
DR_D float4 load_weights(const EngineParams& P, uint32_t t, uint32_t e, uint32_t n) {
  const float* w = reinterpret_cast<const float*>(__ldg(P.wparams + t)) + e;
  if (n >= 4u && (reinterpret_cast<uintptr_t>(w) & 15u) == 0u) return __ldg(reinterpret_cast<const float4*>(w));
  float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (uint32_t j = 0; j < 4u; ++j) if (j < n) v[j] = __ldg(w + j);
  return make_float4(v[0], v[1], v[2], v[3]);
}

DR_D uint2 load_weights_bf16(const EngineParams& P, uint32_t t, uint32_t e, uint32_t n) {
  const uint16_t* w = reinterpret_cast<const uint16_t*>(__ldg(P.wparams + t)) + e;
  if (n >= 4u && (reinterpret_cast<uintptr_t>(w) & 7u) == 0u) return __ldg(reinterpret_cast<const uint2*>(w));
  uint32_t h[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (uint32_t j = 0; j < 4u; ++j) if (j < n) h[j] = __ldg(w + j);
  return make_uint2(h[0] | (h[1] << 16), h[2] | (h[3] << 16));
}

// 'dgc' local gradient clipping.  A parameter's squared norm is the sum of fl64(g_i)^2 (each square exact) over its
// elements zero-padded to 4096 * 2^ceil(log2(tiles)), added by adjacent pairs level after level: a perfect binary tree,
// so a tile's pairwise sum is a subtree (clip_tile_sums) and the parameter's sum is the tree over its tiles' sums
// (clip_factors).  The fixed order is what engine_oracle and DgcMemory reproduce in torch.
constexpr uint32_t kClipLeaves = 2048;   // tile sums reduced per shared-memory tree (a larger tree runs in blocks)

DR_D double sumsq4(float4 g) {
  const double x = g.x, y = g.y, z = g.z, w = g.w;
  return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dadd_rn(__dmul_rn(z, z), __dmul_rn(w, w)));
}

// pairwise sum of buf[0 .. L) (L a power of two), each level written behind the previous one (buf holds 2L - 1
// doubles); every thread gets the result
DR_D double smem_pairwise(double* buf, uint32_t L) {
  uint32_t in = 0, out = L;
  for (uint32_t w = L >> 1; w != 0u; w >>= 1) {
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < w; i += kThreads) buf[out + i] = __dadd_rn(buf[in + 2u * i], buf[in + 2u * i + 1u]);
    in = out; out += w;
  }
  __syncthreads();
  const double s = buf[in];
  __syncthreads();
  return s;
}

// step 1: the pairwise sum of the squares of every tile of my accumulate range into clip_part.  Thread tid holds the
// aligned quads tid of both half-tiles; the shuffles add adjacent lanes, so every warp sum is a subtree of 128 elements,
// and thread 0 adds the 32 warp sums by pairs.  One more read of the gradient.
template <bool kB>
DR_D void clip_tile_sums(const EngineParams& P) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  double* red = reinterpret_cast<double*>(g_filter_smem);
  uint32_t t0, t_end;
  tile_range(P, kPartAccum, t0, t_end);
  for (uint32_t tile = t0; tile < t_end; ++tile) {
    const Tile ti = load_tile(P.tiles, tile);
#pragma unroll
    for (uint32_t h = 0; h < 2u; ++h) {
      const uint32_t e0 = h * kHalf + tid * 4u;
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
      if (e0 < ti.n) {
        if constexpr (kB) g = widen_bf16x4(__ldcs(reinterpret_cast<const uint2*>(P.grad_bf16 + ti.base + e0)));
        else g = __ldcs(reinterpret_cast<const float4*>(P.grad + ti.base + e0));
        if (e0 + 1u >= ti.n) g.y = 0.f;                                    // the buffers' padding is not the tensor's
        if (e0 + 2u >= ti.n) g.z = 0.f;
        if (e0 + 3u >= ti.n) g.w = 0.f;
      }
      double v = sumsq4(g);
#pragma unroll
      for (uint32_t o = 1; o < 32u; o <<= 1) {
        const double p = __shfl_down_sync(0xFFFFFFFFu, v, o);
        if ((lane & (2u * o - 1u)) == 0u) v = __dadd_rn(v, p);
      }
      if (lane == 0) red[h * kWarps + warp] = v;
    }
    __syncthreads();
    if (tid == 0) {
      for (uint32_t w = kWarps; w != 0u; w >>= 1)                          // in place: pair i reads 2i, 2i + 1 >= i
        for (uint32_t i = 0; i < w; ++i) red[i] = __dadd_rn(red[2u * i], red[2u * i + 1u]);
      __stcg(P.clip_part + tile, red[0]);
    }
    __syncthreads();
  }
}

// step 2 (after a grid barrier): the factor of every plan tensor from the tree over its parameter's tile sums.  The
// chunks of a split parameter each compute the same tree.  The factor is read by other CTAs after the next barrier.
DR_D void clip_factors(const EngineParams& P) {
  double* red = reinterpret_cast<double*>(g_filter_smem);                 // 2 * kClipLeaves - 1 doubles
  double* outer = red + 2u * kClipLeaves;                                  // block sums: <= 2^20 tiles / kClipLeaves
  for (uint32_t t = blockIdx.x; t < P.n_tensors; t += gridDim.x) {
    const uint2 ow = __ldg(reinterpret_cast<const uint2*>(P.clip_owner) + t);
    uint32_t L = 1;
    while (L < ow.y) L <<= 1;
    double s;
    if (L <= kClipLeaves) {
      for (uint32_t i = threadIdx.x; i < L; i += kThreads) red[i] = i < ow.y ? __ldcg(P.clip_part + ow.x + i) : 0.0;
      s = smem_pairwise(red, L);
    } else {
      for (uint32_t b = 0; b < L / kClipLeaves; ++b) {
        for (uint32_t i = threadIdx.x; i < kClipLeaves; i += kThreads) {
          const uint32_t j = b * kClipLeaves + i;
          red[i] = j < ow.y ? __ldcg(P.clip_part + ow.x + j) : 0.0;
        }
        const double sb = smem_pairwise(red, kClipLeaves);
        if (threadIdx.x == 0) outer[b] = sb;
      }
      s = smem_pairwise(outer, L / kClipLeaves);
    }
    if (threadIdx.x == 0) {
      // NaN is never > thr, and an infinite norm (an infinite element) leaves the gradient untouched too
      const double nrm = __dsqrt_rn(s);
      const float f = (nrm > P.clip_thr && isfinite(nrm)) ? __double2float_rn(__ddiv_rn(P.clip_thr, nrm)) : 1.0f;
      __stcg(P.clip_f + t, f);
    }
  }
}

// kTma = true : g / r half-tiles arrive through a CTA-wide TMA ring (cp.async.bulk + full/empty mbarriers, one producer
//               thread); kTma = false: every THREAD copies its own float4 of g and r with cp.async (LDGSTS) into a
//               private slot of the ring and reads it back itself — no mbarriers, no producer, warps never wait for
//               each other between tensor boundaries.  Selected by EngineParams::use_tma; both are kept because which
//               one feeds HBM better is measured, not derived (scripts/engine_microbench.py).
// kB = true    : bf16 bucket.  The g half of a stage holds the bf16 half-tile (4 KB, the rest of its 8 KB unused, so the
//               ring arithmetic is the same), each thread widens its 8 bytes in registers and zero-fills its 8 bytes of
//               the bf16 output; the rows of acc32 that the apply of this step adds into are zeroed here too.
// kDgc = true  : 'dgc' memory.  Each thread reads its float4 of the momentum u with a direct streaming load, issued
//               before it waits for the ring so that the load overlaps the wait, and writes u back the same way.  u
//               is not staged through the ring: the stage size, the ring depth and the shared-memory budget stay
//               the same as the existing variants', so u costs no ring space and no extra TMA bookkeeping, and each
//               element of u is read by exactly the thread that uses it.  With weight decay (P.weight_decay != 0 and
//               the tensor's P.decayed[t], read once per tensor run, CTA-uniform) the thread reads its four elements of
//               the parameter w the same way, next to u, and adds fl(weight_decay * w) to g before the momentum;
//               otherwise (no decay, or an excluded parameter) nothing is read or added.  With P.nesterov
//               (CTA-uniform) the residual adds fl(d + fl(momentum * u)) with the new u instead of u.
// kClip = true : 'dgc' local gradient clipping.  clip_tile_sums and clip_factors have run (two grid barriers ago), and
//               g = fl(g * f) with the tensor's factor f ahead of everything else, where f != 1.
template <bool kTma, bool kFull, bool kB, bool kDgc, bool kClip = false>
DR_D void phase_accum(const EngineParams& P, Smem& sm) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t parity_slot = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity_slot, P.rank);
  {  // zero the outgoing slot (filters, headers, prefix tables, hints)
    uint4* p = reinterpret_cast<uint4*>(my_slot);
    const uint32_t n4 = (P.payload_words + 3u) >> 2;
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (uint32_t i = blockIdx.x * kThreads + tid; i < n4; i += gridDim.x * kThreads) p[i] = z;
  }
  if (sharded(P) && blockIdx.x == 0 && tid == 0) *s2_ptr(P.arena[P.rank], P, parity_slot, P.rank) = 0u;
  // per-tile counts are accumulated by the insert (raw / rle) and query (bloom) phases of this step
  // (+ two per-tensor counters behind the tiles: filter positives and inserted elements — 'random' policy)
  for (uint32_t i = blockIdx.x * kThreads + tid; i < P.n_tiles + 2u * P.n_tensors; i += gridDim.x * kThreads) P.tile_count[i] = 0u;
  __syncthreads();
  for (int j = tid; j < 2 * kHistBins; j += kThreads) sm.u.hist[j] = 0;
  __syncthreads();
  const bool has_resid = (P.beta != 0.0f);
  uint32_t acc_begin = 0, acc_end = 0;         // bf16: the tiles this rank decodes own the rows of acc32
  if constexpr (kB) decode_span(P, P.rank, acc_begin, acc_end);
  uint32_t t0, t_end;
  tile_range(P, kPartAccum, t0, t_end);
  if (t0 >= t_end) return;
  uint8_t* ring = reinterpret_cast<uint8_t*>(g_filter_smem);
  const uint32_t n_stages = kTma ? min(kMaxStages, (P.filter_smem_words * 4u) / kStageBytes)   // host guarantees >= 2
                                 : kCpStages;                                               // ... and >= 64 KB when !use_tma
  uint64_t* full = sm.bar;
  uint64_t* empty = sm.bar + 8;
  // The producer is lane 0 of the LAST warp: the SMSP arbiter favours the highest warp id, so the refill is never
  // queued behind the consumers it feeds (thread 0 was starved: v11 profile, 41 % of the samples in the full-wait).
  constexpr uint32_t kProducer = kThreads - 32;
  if (kTma && tid == 0) {
    for (uint32_t i = 0; i < n_stages; ++i) {
      mbar_inval(&full[i]); mbar_init(&full[i], 1);
      mbar_inval(&empty[i]); mbar_init(&empty[i], kWarps);
    }
    mbar_fence_init();
    fence_proxy_async_smem();
  }
  __syncthreads();
  // ---- producer: the item sequence = every non-empty half-tile of my range, in order
  uint32_t p_tile = t0, p_half = 0, p_stage = 0;
  auto issue_next = [&]() -> bool {
    while (p_tile < t_end) {
      const Tile t = load_tile(P.tiles, p_tile);
      const uint32_t off = p_half * kHalf;
      if (p_half == 1u) { p_half = 0; ++p_tile; } else { p_half = 1u; }
      if (off < t.n) {
        uint8_t* dst = ring + (size_t)p_stage * kStageBytes;
        if (kTma) {
          const uint32_t bytes = round16(min(t.n - off, kHalf) * 4u);
          if constexpr (kB) {                           // tensors start at 32-element boundaries: 16-byte aligned source
            const uint32_t gbytes = round16(min(t.n - off, kHalf) * 2u);
            mbar_expect_tx(&full[p_stage], has_resid ? gbytes + bytes : gbytes);
            bulk_g2s(dst, P.grad_bf16 + t.base + off, gbytes, &full[p_stage]);
          } else {
            mbar_expect_tx(&full[p_stage], has_resid ? 2u * bytes : bytes);
            bulk_g2s(dst, P.grad + t.base + off, bytes, &full[p_stage]);
          }
          if (has_resid) bulk_g2s(dst + kHalf * 4u, P.resid + t.base + off, bytes, &full[p_stage]);
        } else {                                        // this thread's own 16 bytes of g and of r (bf16: 8 bytes of g)
          const uint32_t e0 = off + tid * 4u;
          if (e0 < t.n) {
            if constexpr (kB) cp_async_8(dst + tid * 8u, P.grad_bf16 + t.base + e0);
            else cp_async_16(dst + tid * 16u, P.grad + t.base + e0);
            if (has_resid) cp_async_16(dst + kHalf * 4u + tid * 16u, P.resid + t.base + e0);
          }
          cp_async_commit();
        }
        if (++p_stage == n_stages) p_stage = 0;
        return true;
      }
    }
    return false;
  };
  uint32_t n_issued = 0;                       // cp.async path: groups committed by this thread
  if (kTma) { if (tid == kProducer) for (uint32_t i = 0; i < n_stages; ++i) if (!issue_next()) break; }
  else { for (uint32_t i = 0; i + 1 < kCpStages; ++i) { if (issue_next()) ++n_issued; else cp_async_commit(); } }
  // ---- consumers
  uint32_t stage = 0, par = 0;                 // ring position of the next item to consume
  uint32_t prev_stage = 0, prev_par = 0;       // ... of the item consumed last (the stage the producer refills)
  bool first_item = true;
  uint32_t tile = t0;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const float beta = P.beta, gamma = P.gamma;
  while (tile < t_end) {
    Tile ti = load_tile(P.tiles, tile);
    const uint32_t cur = ti.tensor;
    const TensorDesc* tdp = P.tensors + cur;
    const uint32_t mode = __ldg(&tdp->mode), fixed = __ldg(&tdp->fixed_thr);
    bool zero_acc = false;                                                 // bf16: this tensor's rows of acc32 start from 0
    if constexpr (kB) zero_acc = bloom_applied(P, mode, __ldg(&tdp->vmode));
    // bf16 values at W == 1: emit scatters them, as it does fp32 values, and decode and compact do not run (they run at
    // W == 1 only for the fix phase's value codecs), so no acc32 row is applied
    if constexpr (kFull && kB) zero_acc = zero_acc && !(P.world == 1 && __ldg(&tdp->vmode) == kVmodeBf16);
    // 'randomk' (full kernel only): the keys are hashes of the element index (CTA-uniform per tensor), the candidate
    // bound is static
    const bool shared = kFull && (mode == (uint32_t)kModeShared);
    const uint32_t hseed = shared ? policy_seed(P.epoch, __ldg(&tdp->salt)) : 0u;
    uint32_t lower;
    if (fixed) lower = fixed;
    else if (shared) lower = __ldg(&tdp->shared_lb);
    else {
      const uint32_t prev = P.use_history ? __ldcg(&P.sel[cur].prev_thr) : 0u;
      lower = (prev > (1u << 23)) ? prev - (1u << P.hist_shift) : 0u;      // a fraction of last step's threshold
    }
    const bool do_hist = (fixed == 0u);
    const bool single = ti.single != 0u;
    // last step's threshold bin: the guess under which digit 2 is binned speculatively (one-tile tensors finish both
    // digits from registers below and need no guess)
    const uint32_t guess = (do_hist && !single) ? __ldcg(&P.sel[cur].bin1) : 0xFFFFFFFFu;
    float clip_f = 1.0f;
    if constexpr (kClip) clip_f = __ldcg(P.clip_f + cur);                 // written by another CTA in this launch
    bool dec = false;                                                      // CTA-uniform: this tensor takes the decay
    if constexpr (kDgc) dec = P.weight_decay != 0.0f && __ldg(P.decayed + cur) != 0;
    uint32_t n_mine = 0;
    uint32_t keys[8];
    while (true) {                                                         // tiles of this tensor inside my range
      uint32_t cnt = 0;
      uint2* chunk = P.cand + chunk_of(tile, warp);
      float* r_t = P.resid + ti.base + tid * 4u;                           // this thread's 4 elements of half 0
      float* g_t = P.grad + ti.base + tid * 4u;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t off = (uint32_t)h * kHalf;
        uint32_t key4[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};   // 0xFFFFFFFF = not an element
        if (off < ti.n) {                                                  // CTA-uniform
          float4 u_old = zero4, w = zero4;
          uint2 w_bf16 = make_uint2(0u, 0u);
          if constexpr (kDgc) {
            const uint32_t e0 = off + tid * 4u;
            if (e0 < ti.n) {
              u_old = __ldcs(reinterpret_cast<const float4*>(P.mom + ti.base + e0));
              if (dec) {
                if constexpr (kB) w_bf16 = load_weights_bf16(P, cur, ti.local0 + e0, ti.n - e0);
                else w = load_weights(P, cur, ti.local0 + e0, ti.n - e0);
              }
            }
          }
          if (kTma) {
            // refill first: the stage consumed one item ago is free as soon as every warp released it
            if (tid == kProducer && !first_item && p_tile < t_end) {
              mbar_wait(&empty[prev_stage], prev_par, P.status);
              fence_proxy_async_smem();
              issue_next();
            }
            mbar_wait(&full[stage], par, P.status);
          } else {
            // n_stages - 1 of my groups are in flight; issue the next one into the slot I read last time (only this
            // thread ever touches its 16-byte slots), then wait until the oldest group — this item — has landed
            if (issue_next()) ++n_issued;
            else cp_async_commit();                      // keep the group count uniform past the end of the range
            cp_async_wait<kCpStages - 1>();
            (void)n_issued;
          }
          const float4* sg = reinterpret_cast<const float4*>(ring + (size_t)stage * kStageBytes);
          const float4* sr = sg + kHalf / 4;
          const uint32_t e0 = off + tid * 4u;
          uint32_t m = 0;
          const bool whole = (ti.n - off) >= kHalf;                        // CTA-uniform fast path: no bounds checks
          if (whole || e0 < ti.n) {
            float4 g;
            if constexpr (kB) g = widen_bf16x4(reinterpret_cast<const uint2*>(sg)[tid]);
            else g = sg[tid];
            float4 a;
            if constexpr (kDgc) {                                          // two roundings each: no contracted FMA
              const float mu = P.momentum, wd = P.weight_decay;
              if constexpr (kClip) {
                if (clip_f != 1.0f) {                                      // CTA-uniform
                  g.x = __fmul_rn(g.x, clip_f); g.y = __fmul_rn(g.y, clip_f);
                  g.z = __fmul_rn(g.z, clip_f); g.w = __fmul_rn(g.w, clip_f);
                }
              }
              if (dec) {                                                   // d = fl(g + fl(wd * w)) replaces g
                if constexpr (kB) w = widen_bf16x4(w_bf16);
                g.x = __fadd_rn(g.x, __fmul_rn(wd, w.x)); g.y = __fadd_rn(g.y, __fmul_rn(wd, w.y));
                g.z = __fadd_rn(g.z, __fmul_rn(wd, w.z)); g.w = __fadd_rn(g.w, __fmul_rn(wd, w.w));
              }
              float4 u;
              u.x = __fadd_rn(__fmul_rn(mu, u_old.x), g.x); u.y = __fadd_rn(__fmul_rn(mu, u_old.y), g.y);
              u.z = __fadd_rn(__fmul_rn(mu, u_old.z), g.z); u.w = __fadd_rn(__fmul_rn(mu, u_old.w), g.w);
              __stcs(reinterpret_cast<float4*>(P.mom + ti.base + e0), u);
              if (P.nesterov) {                                            // v = fl(d + fl(mu * u)) replaces u
                u.x = __fadd_rn(g.x, __fmul_rn(mu, u.x)); u.y = __fadd_rn(g.y, __fmul_rn(mu, u.y));
                u.z = __fadd_rn(g.z, __fmul_rn(mu, u.z)); u.w = __fadd_rn(g.w, __fmul_rn(mu, u.w));
              }
              const float4 r = sr[tid];
              a.x = __fadd_rn(r.x, u.x); a.y = __fadd_rn(r.y, u.y); a.z = __fadd_rn(r.z, u.z); a.w = __fadd_rn(r.w, u.w);
            } else if (has_resid) {
              // fl(fl(beta * r) + fl(gamma * g)): three roundings, as ResidualMemory and engine_oracle make them in
              // torch.  Left to itself nvcc fuses one product into an FFMA (here gamma * g), which changes a and the
              // residual wherever that factor is not 0 or a power of two
              const float4 r = sr[tid];
              a.x = __fadd_rn(__fmul_rn(beta, r.x), __fmul_rn(gamma, g.x));
              a.y = __fadd_rn(__fmul_rn(beta, r.y), __fmul_rn(gamma, g.y));
              a.z = __fadd_rn(__fmul_rn(beta, r.z), __fmul_rn(gamma, g.z));
              a.w = __fadd_rn(__fmul_rn(beta, r.w), __fmul_rn(gamma, g.w));
            } else {
              a.x = gamma * g.x; a.y = gamma * g.y; a.z = gamma * g.z; a.w = gamma * g.w;
            }
            *reinterpret_cast<float4*>(r_t + off) = a;
            if constexpr (kB) {
              *reinterpret_cast<uint2*>(P.grad_bf16 + ti.base + e0) = make_uint2(0u, 0u);
              if (zero_acc && tile >= acc_begin && tile < acc_end)
                *reinterpret_cast<float4*>(P.acc32 + (size_t)(tile - acc_begin) * kTile + e0) = zero4;
            } else {
              *reinterpret_cast<float4*>(g_t + off) = zero4;              // the dense output starts from zero
            }
            uint32_t kv[4] = {__float_as_uint(a.x) & 0x7FFFFFFFu, __float_as_uint(a.y) & 0x7FFFFFFFu,
                              __float_as_uint(a.z) & 0x7FFFFFFFu, __float_as_uint(a.w) & 0x7FFFFFFFu};
            if (shared) {
#pragma unroll
              for (int j = 0; j < 4; ++j) kv[j] = shared_key(ti.local0 + e0 + (uint32_t)j, hseed);
            }
            if (whole) {
#pragma unroll
              for (int j = 0; j < 4; ++j) { key4[j] = kv[j]; if (kv[j] >= lower) m |= 1u << j; }
            } else {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                if (e0 + j < ti.n) { key4[j] = kv[j]; if (kv[j] >= lower) m |= 1u << j; }
              }
            }
          }
          if (kTma) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);                     // this warp is done with the stage
          }
          prev_stage = stage; prev_par = par; first_item = false;
          if (++stage == n_stages) { stage = 0; par ^= 1u; }
          append_candidates(sm, m, key4, e0, chunk, cnt, do_hist, lane, guess);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) keys[h * 4 + j] = key4[j];
      }
      if (lane == 0) P.cand_cnt[tile * kWarps + warp] = cnt;
      if (mode != (uint32_t)kModeBloom && lane < 8u) P.pos_mask[(size_t)tile * kGroupsPerTile + warp * 8u + lane] = 0u;
      n_mine += 1;
      ++tile;
      if (tile >= t_end) break;
      const Tile tn = load_tile(P.tiles, tile);
      if (tn.tensor != cur) break;
      ti = tn;
    }
    // ---- the tensor (or my part of it) is done
    if (fixed) {
      if (tid == 0) {
        SelState* st = P.sel + cur;
        st->thr = fixed; st->bin1 = 0; st->krem1 = 0; st->done_epoch = P.epoch;
      }
    } else if (single) {
      // one-tile tensor: finish the whole 2-digit select here, from the keys still in registers
      const uint32_t k = __ldg(&tdp->k);
      resolve_bins([&](int b) { return sm.u.hist[b]; }, kHistBins, k, sm.s);
      const uint32_t bin1 = sm.s.res[0], krem1 = sm.s.res[1];
      write_digit1(P, sm, cur);
      clear_hist(sm);
      finish_single(P, sm, cur, keys, bin1, krem1);
    } else {
      finish_spec(P, sm, cur, n_mine, __ldg(&tdp->n_tiles), __ldg(&tdp->k), guess);
    }
  }
}

// ===========================================================================
// phase 1 (rare): the history bound hid the threshold of some tensor (fewer than K candidates): redo digit 1 over
// all of its keys and rebuild its candidate lists in full, so the later phases stay candidate-only.
// ===========================================================================
template <bool kFull>
DR_D void phase_fallback(const EngineParams& P, Smem& sm) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  clear_hist(sm);
  uint32_t tile, t_end;
  tile_range(P, kPartAccum, tile, t_end);
  while (tile < t_end) {
    const Tile t0 = load_tile(P.tiles, tile);
    const uint32_t cur = t0.tensor;
    const TensorDesc* tdp = P.tensors + cur;
    const uint32_t seg_end = min(t_end, __ldg(&tdp->tile_begin) + __ldg(&tdp->n_tiles));
    const bool active = (__ldcg(&P.sel[cur].bin1) == kUnsafe) && (__ldcg(&P.sel[cur].done_epoch) != P.epoch) &&
                        (__ldg(&tdp->fixed_thr) == 0u);
    if (!active) { tile = seg_end; continue; }
    // 'randomk': the keys are the index hashes of phase 0, not the residual's bit patterns
    const bool shared = kFull && (__ldg(&tdp->mode) == (uint32_t)kModeShared);
    const uint32_t hseed = shared ? policy_seed(P.epoch, __ldg(&tdp->salt)) : 0u;
    uint32_t keys[8];
    for (uint32_t tl = tile; tl < seg_end; ++tl) {
      const Tile ti = load_tile(P.tiles, tl);
      uint32_t cnt = 0;
      uint2* chunk = P.cand + chunk_of(tl, warp);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t e0 = (uint32_t)h * kHalf + tid * 4u;
        uint32_t key4[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
        uint32_t m = 0;
        if (e0 < ti.n) {
          uint32_t kv[4];
          if (shared) {
#pragma unroll
            for (int j = 0; j < 4; ++j) kv[j] = shared_key(ti.local0 + e0 + (uint32_t)j, hseed);
          } else {
            const uint4 q = __ldcg(reinterpret_cast<const uint4*>(P.resid + ti.base + e0));
            kv[0] = q.x & 0x7FFFFFFFu; kv[1] = q.y & 0x7FFFFFFFu; kv[2] = q.z & 0x7FFFFFFFu; kv[3] = q.w & 0x7FFFFFFFu;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) if (e0 + j < ti.n) { key4[j] = kv[j]; m |= 1u << j; }
        }
        append_candidates(sm, m, key4, e0, chunk, cnt, true, lane);
#pragma unroll
        for (int j = 0; j < 4; ++j) keys[h * 4 + j] = key4[j];
      }
      if (lane == 0) P.cand_cnt[tl * kWarps + warp] = cnt;
    }
    const uint32_t k = __ldg(&tdp->k), nt = __ldg(&tdp->n_tiles);
    if (t0.single) {
      resolve_bins([&](int b) { return sm.u.hist[b]; }, kHistBins, k, sm.s);
      const uint32_t bin1 = sm.s.res[0], krem1 = sm.s.res[1];
      if (tid == 0) {
        if (bin1 == kUnsafe) atomicExch(P.status, kErrResolve);
        P.sel[cur].bin1 = bin1; P.sel[cur].krem1 = krem1;
      }
      clear_hist(sm);
      finish_single(P, sm, cur, keys, bin1, krem1);
    } else if (finish_digit(P, sm, 1, cur, seg_end - tile, nt, k)) {
      if (tid == 0) {
        if (sm.s.res[0] == kUnsafe) atomicExch(P.status, kErrResolve);
        P.sel[cur].bin1 = sm.s.res[0]; P.sel[cur].krem1 = sm.s.res[1]; P.sel[cur].done_epoch = 0;
      }
    }
    tile = seg_end;
  }
}

// ===========================================================================
// kModeRle helpers: 12-bit fields, LSB-first, entry j at bit 12*j of the stream
// ===========================================================================
DR_D void rle_put(uint32_t* stream, uint32_t j, uint32_t pos) {
  const uint32_t bit = 12u * j, w = bit >> 5, sh = bit & 31u;
  atomicOr(stream + w, pos << sh);
  if (sh > 20u) atomicOr(stream + w + 1, pos >> (32u - sh));
}

DR_D uint32_t rle_get(const uint32_t* stream, uint32_t j) {
  const uint32_t bit = 12u * j, w = bit >> 5, sh = bit & 31u;
  uint32_t v = __ldcg(stream + w) >> sh;
  if (sh > 20u) v |= __ldcg(stream + w + 1) << (32u - sh);
  return v & 0xFFFu;
}

// ===========================================================================
// kModeEf helpers (spec.py ef_layout): entry p with in-tile offset e in tile-local tile t puts e & (2^L - 1) at bit p*L
// of the low stream (off_idx) and sets bit p + t * (kTile >> L) + (e >> L) of the high stream (off_hi), LSB-first
// ===========================================================================
DR_D void ef_put(uint32_t* slot, const TensorDesc* td, uint32_t p, uint32_t t, uint32_t e) {
  const uint32_t L = __ldg(&td->ef_low_bits);
  if (L) {
    uint32_t* lo = slot + __ldg(&td->off_idx);
    const uint32_t f = e & ((1u << L) - 1u), bit = p * L, w = bit >> 5, sh = bit & 31u;
    atomicOr(lo + w, f << sh);
    if (sh + L > 32u) atomicOr(lo + w + 1, f >> (32u - sh));
  }
  const uint32_t hb = p + t * (kTile >> L) + (e >> L);
  atomicOr(slot + __ldg(&td->off_hi) + (hb >> 5), 1u << (hb & 31u));
}

DR_D uint32_t ef_low(const uint32_t* lo, uint32_t p, uint32_t L) {
  if (!L) return 0u;
  const uint32_t bit = p * L, w = bit >> 5, sh = bit & 31u;
  uint32_t v = __ldcg(lo + w) >> sh;
  if (sh + L > 32u) v |= __ldcg(lo + w + 1) << (32u - sh);
  return v & ((1u << L) - 1u);
}

// ===========================================================================
// Walk of a warp's candidate chunks (one per tile) with the heads of the next kPF chunks in flight: cp.async copies
// the first 32 entries (256 B) and the count of chunk tile+kPF into a warp-private SMEM ring while chunk `tile` is
// processed.  The lists were written a phase ago and sit in DRAM; every chunk head is a separate 256-byte request,
// so the walk lives on memory-level parallelism.
// ===========================================================================
struct CandWalk {
  uint2* ent;          // [kPF][kHead] this warp's ring
  uint32_t* cnt;       // [kPF]
  uint32_t lane, warp;
};

DR_D CandWalk cand_walk_init() {
  CandWalk w;
  w.lane = threadIdx.x & 31u; w.warp = threadIdx.x >> 5;
  uint8_t* base = reinterpret_cast<uint8_t*>(g_filter_smem);
  w.ent = reinterpret_cast<uint2*>(base) + (size_t)w.warp * kPF * kHead;
  w.cnt = reinterpret_cast<uint32_t*>(base + (size_t)kWarps * kPF * kHead * sizeof(uint2)) + w.warp * kPF;
  return w;
}

// issue the copy of chunk `tile`'s head into ring slot `slot` (or an empty group past the end: group counting stays uniform)
DR_D void cand_walk_issue(const EngineParams& P, const CandWalk& w, uint32_t tile, uint32_t t_end, uint32_t slot) {
  if (tile < t_end) {
    const uint2* src = P.cand + chunk_of(tile, w.warp);
    cp_async_16(w.ent + slot * kHead + 2u * w.lane, src + 2u * w.lane);       // 32 lanes x 16 B = the 64-entry head
    if (w.lane == 0) cp_async_4(w.cnt + slot, P.cand_cnt + tile * kWarps + w.warp);
  }
  cp_async_commit();
}

// ===========================================================================
// phase 2: digit 2 of the select over the candidate lists (keys whose digit 1 is the threshold bin)
// ===========================================================================
DR_D void phase_hist2(const EngineParams& P, Smem& sm) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  clear_hist(sm);
  const CandWalk cw = cand_walk_init();
  uint32_t tile, t_end;
  tile_range(P, kPartAccum, tile, t_end);
  while (tile < t_end) {
    const Tile t0 = load_tile(P.tiles, tile);
    const uint32_t cur = t0.tensor;
    const TensorDesc* tdp = P.tensors + cur;
    const uint32_t nt = __ldg(&tdp->n_tiles);
    const uint32_t seg_end = min(t_end, __ldg(&tdp->tile_begin) + nt);
    if (__ldcg(&P.sel[cur].done_epoch) == P.epoch) { tile = seg_end; continue; }     // one-tile / fixed-threshold tensors
    const uint32_t prefix = __ldcg(&P.sel[cur].bin1), k_cur = __ldcg(&P.sel[cur].krem1);
    if (prefix == kUnsafe && tid == 0) atomicExch(P.status, kErrResolve);
    __syncwarp();
#pragma unroll
    for (int p = 0; p < kPF; ++p) cand_walk_issue(P, cw, tile + (uint32_t)p, seg_end, (uint32_t)p);
    for (uint32_t tl = tile, i = 0; tl < seg_end; ++tl, ++i) {
      const uint32_t slot = i & (kPF - 1);
      cp_async_wait<kPF - 1>();                                            // the oldest group (chunk tl) has landed
      __syncwarp();
      const uint32_t c = cw.cnt[slot];
      const uint32_t ka = cw.ent[slot * kHead + lane].x, kb = cw.ent[slot * kHead + 32u + lane].x;
      __syncwarp();                                                        // everyone has read the slot: refill it
      cand_walk_issue(P, cw, tl + kPF, seg_end, slot);
      if (lane < c && (ka >> 20) == prefix) atomicAdd(&sm.u.hist[(ka >> 9) & 0x7FFu], 1u);
      if (lane + 32u < c && (kb >> 20) == prefix) atomicAdd(&sm.u.hist[(kb >> 9) & 0x7FFu], 1u);
      if (c > kHead) {
        const uint2* chunk = P.cand + chunk_of(tl, warp);
        for (uint32_t j = kHead + lane; j < c; j += 32u) {
          const uint32_t k = __ldcg(chunk + j).x;
          if ((k >> 20) == prefix) atomicAdd(&sm.u.hist[(k >> 9) & 0x7FFu], 1u);
        }
      }
    }
    cp_async_wait<0>();
    if (finish_digit(P, sm, 2, cur, seg_end - tile, nt, k_cur)) write_final(P, sm, cur, prefix);
    tile = seg_end;
  }
}

// ===========================================================================
// phase 3: the selected candidates (key >= threshold) build the index side of the slot.
//   bloom : occupancy-hint bit of the element's 32-group + n_hash filter bits (RED.OR into the outgoing slot)
//   raw / rle : the positive masks directly (there is no membership test to run) + per-tile counts
// Warp-private: a warp walks its own candidate chunks; the selected elements of one iteration are compacted into a
// 32-entry SMEM row so that every lane sets one (element, hash) bit — no divergent per-element hash loops.
// ===========================================================================
// 'random' policy: per-tensor counters behind the per-tile counts (zeroed with them in phase 0)
DR_D uint32_t* n_pos_of(const EngineParams& P, uint32_t t) { return P.tile_count + P.n_tiles + t; }
DR_D uint32_t* n_ins_of(const EngineParams& P, uint32_t t) { return P.tile_count + P.n_tiles + P.n_tensors + t; }

DR_D void phase_insert(const EngineParams& P, Smem& sm) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  uint32_t* row = sm.u.sel[warp];
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t tile, t_end;
  tile_range(P, kPartInsert, tile, t_end);
  if (tile >= t_end) return;
  uint32_t cur = kNoTensor, thr = 0xFFFFFFFFu, mode = 0, n_hash = 0, m_bits = 0, recip = 0, tile_begin = 0;
  uint32_t* filter = nullptr;
  uint32_t* hint = nullptr;
  auto process = [&](uint32_t tl, uint32_t local0, bool have, uint32_t k, uint32_t e, uint32_t& n_sel_tile) {
    const bool sel = have && k >= thr;
    const uint32_t b = __ballot_sync(kFullMask, sel);
    if (b == 0u) return;
    n_sel_tile += __popc(b);
    if (mode != (uint32_t)kModeBloom) {
      if (sel) atomicOr(P.pos_mask + (size_t)tl * kGroupsPerTile + (e >> 5), 1u << (e & 31u));
      return;
    }
    if (sel) {
      row[__popc(b & lt)] = local0 + e;
      if (hint) atomicOr(hint + 4u * (tl - tile_begin) + (e >> 10), 1u << ((e >> 5) & 31u));
    }
    __syncwarp();
    const uint32_t pairs = (uint32_t)__popc(b) * n_hash;
    for (uint32_t p = lane; p < pairs; p += 32u) {
      const uint32_t ent = (n_hash == 1u) ? p : __umulhi(p, recip);
      const uint32_t j = p - ent * n_hash;
      const HashAB h = hash_ab(row[ent], P.seed);
      const uint32_t pos = mulhi32(h.a + j * h.b, m_bits);
      atomicOr(filter + (pos >> 5), 1u << (pos & 31u));
    }
    __syncwarp();
  };
  auto tensor_params = [&](uint32_t t) {
    cur = t;
    const TensorDesc* tdp = P.tensors + cur;
    mode = __ldg(&tdp->mode); n_hash = __ldg(&tdp->n_hash); m_bits = __ldg(&tdp->m_bits);
    tile_begin = __ldg(&tdp->tile_begin);
    filter = my_slot + __ldg(&tdp->off_filter);
    const uint32_t oh = __ldg(&tdp->off_hint);
    hint = oh ? my_slot + oh : nullptr;
    recip = n_hash > 1u ? (0xFFFFFFFFu / n_hash) + 1u : 0u;
    thr = __ldcg(&P.sel[cur].thr);
  };
  const CandWalk cw = cand_walk_init();
#pragma unroll
  for (int p = 0; p < kPF; ++p) cand_walk_issue(P, cw, tile + (uint32_t)p, t_end, (uint32_t)p);
  for (uint32_t tl = tile, i = 0; tl < t_end; ++tl, ++i) {
    const uint32_t slot = i & (kPF - 1);
    const Tile ti = load_tile(P.tiles, tl);
    cp_async_wait<kPF - 1>();                                              // the oldest group (chunk tl) has landed
    __syncwarp();
    const uint32_t c = cw.cnt[slot];
    const uint2 ea = cw.ent[slot * kHead + lane], eb2 = cw.ent[slot * kHead + 32u + lane];
    __syncwarp();                                                          // everyone has read the slot: refill it
    cand_walk_issue(P, cw, tl + kPF, t_end, slot);
    if (ti.tensor != cur) tensor_params(ti.tensor);
    uint32_t n_sel_tile = 0;
    if (c) {                                                               // warp-uniform
      process(tl, ti.local0, lane < c, ea.x, ea.y, n_sel_tile);
      if (c > 32u) process(tl, ti.local0, lane + 32u < c, eb2.x, eb2.y, n_sel_tile);
      if (c > kHead) {
        const uint2* chunk = P.cand + chunk_of(tl, warp);
        for (uint32_t j0 = kHead; j0 < c; j0 += 32u) {
          const bool have = j0 + lane < c;
          const uint2 eb = have ? __ldcg(chunk + j0 + lane) : make_uint2(0, 0);
          process(tl, ti.local0, have, eb.x, eb.y, n_sel_tile);
        }
      }
    }
    if (lane == 0 && n_sel_tile) {
      if (mode != (uint32_t)kModeBloom) atomicAdd(P.tile_count + tl, n_sel_tile);
      else if (P.policy == kPolicyRandom) atomicAdd(n_ins_of(P, cur), n_sel_tile);   // the policy's target count
    }
  }
  cp_async_wait<0>();
}

// ===========================================================================
// Membership test of the hinted 32-element groups of a run of tiles against ONE filter -> group bitmasks.
//
// Work item = one hint word (32 groups = a quarter tile), handed out dynamically (SMEM counter) so the 16 warps
// stay balanced whatever the hint density.  A warp owns whole groups: lane l tests element 32*g + l.
// Two levels: level 1 runs the first two probes for every element of a hinted group (all lanes busy); the ~25 %
// survivors are appended to a per-warp ring in SMEM, and whenever 32 have gathered level 2 finishes their probe
// chains on a dense batch.  A hinted group always holds a true positive, which used to drag its whole warp through
// all n_hash probes at 1-2 active lanes (v10: 19/32 lane efficiency, ~230 warp-instructions per hinted group).
// Positives land in mask_out (word = group, bit = lane) by RED.OR; level 1 zeroes the word first.
// ===========================================================================
struct ProbeCtx {
  const uint32_t* hint;     // hint words of this tensor, 4 per tile (nullptr: every group is tested)
  const uint32_t* prefix;   // decode: the sender's per-tile prefix table (nullptr: query)
  uint32_t n_sel, cutoff;   // decode gating (query: 0xFFFFFFFF both)
  uint32_t* mask_out;       // [n_tiles * 128]
  uint32_t* tile_count;     // query: positives per tile (nullptr: not counted)
  uint32_t tile_begin;      // first global tile of the tensor
  uint32_t seg_a, seg_b;    // global tile range handled by this CTA
  uint32_t n_hash, m_bits, seed;
  uint32_t pol_T, pol_seed; // 'random' policy on the receiving side: a positive x survives iff policy_hash(x, pol_seed) <= pol_T
                            // (0xFFFFFFFF: no filter — the sender's own query, every other policy)
};

// caller: sm.s.lb = 0 and __syncthreads() before; __syncthreads() after
template <typename LoadFn>
DR_D void probe_segment(const EngineParams& P, Smem& sm, const ProbeCtx& c, LoadFn ld) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  uint32_t* q = sm.u.q[warp];
  uint32_t qh = 0, qn = 0;
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t n_items = (c.seg_b - c.seg_a) * 4u;
  const uint32_t m_bits = c.m_bits;
  auto level2 = [&](uint32_t n_take) {
    __syncwarp();
    if (lane < n_take) {
      const uint32_t gp = q[(qh + lane) & 63u];
      const uint32_t tile = gp >> 12, e = gp & 4095u;
      const uint32_t x = ((tile - c.tile_begin) << 12) + e;
      const HashAB h = hash_ab(x, c.seed);
      uint32_t v = h.a + 2u * h.b;
      bool pass = true;
      uint32_t j = 2;
      for (; j + 1 < c.n_hash; j += 2) {
        const uint32_t p0 = mulhi32(v, m_bits), p1 = mulhi32(v + h.b, m_bits);
        const uint32_t w0 = ld(p0 >> 5), w1 = ld(p1 >> 5);
        if (!((w0 >> (p0 & 31u)) & (w1 >> (p1 & 31u)) & 1u)) { pass = false; break; }
        v += 2u * h.b;
      }
      if (pass && j < c.n_hash) {
        const uint32_t p0 = mulhi32(v, m_bits);
        pass = ((ld(p0 >> 5) >> (p0 & 31u)) & 1u) != 0u;
      }
      if (pass && c.pol_T != 0xFFFFFFFFu) pass = policy_hash(x, c.pol_seed) <= c.pol_T;
      if (pass) {
        atomicOr(c.mask_out + (size_t)tile * kGroupsPerTile + (e >> 5), 1u << (e & 31u));
        if (c.tile_count) atomicAdd(c.tile_count + tile, 1u);
      }
    }
    qh = (qh + n_take) & 63u;
    qn -= n_take;
    __syncwarp();
  };
  while (true) {
    uint32_t it = 0;
    if (lane == 0) it = atomicAdd(&sm.s.lb, 1u);
    it = __shfl_sync(kFullMask, it, 0);
    if (it >= n_items) break;
    const uint32_t tile = c.seg_a + (it >> 2), qd = it & 3u;
    const Tile ti = load_tile(P.tiles, tile);
    const uint32_t tl = tile - c.tile_begin;
    if (c.prefix) {
      const uint32_t pre = __ldcg(c.prefix + tl);
      if (!ships_into(pre, c.n_sel, ti.local0, c.cutoff)) continue;        // tile-uniform: nothing of this sender lands here
    }
    uint32_t hw = c.hint ? __ldcg(c.hint + 4u * tl + qd) : 0xFFFFFFFFu;
    const uint32_t n_groups = (ti.n + 31u) >> 5, g0 = qd * 32u;
    if (g0 >= n_groups) continue;
    if (n_groups - g0 < 32u) hw &= (1u << (n_groups - g0)) - 1u;
    while (hw) {
      const uint32_t j = (uint32_t)__ffs((int)hw) - 1u;
      hw &= hw - 1u;
      const uint32_t g = g0 + j, e = g * 32u + lane, x = ti.local0 + e;
      const bool valid = e < ti.n && x <= c.cutoff;
      const HashAB h = hash_ab(x, c.seed);
      const uint32_t p0 = mulhi32(h.a, m_bits);
      uint32_t ok = ld(p0 >> 5) >> (p0 & 31u);
      if (c.n_hash >= 2u) {
        const uint32_t p1 = mulhi32(h.a + h.b, m_bits);
        ok &= ld(p1 >> 5) >> (p1 & 31u);
      }
      bool pass = valid && (ok & 1u);
      if (c.n_hash <= 2u && c.pol_T != 0xFFFFFFFFu) pass = pass && policy_hash(x, c.pol_seed) <= c.pol_T;
      const uint32_t b = __ballot_sync(kFullMask, pass);
      const size_t gi = (size_t)tile * kGroupsPerTile + g;
      if (c.n_hash <= 2u) {
        if (lane == 0) {
          c.mask_out[gi] = b;
          if (c.tile_count && b) atomicAdd(c.tile_count + tile, (uint32_t)__popc(b));
        }
      } else {
        if (lane == 0) c.mask_out[gi] = 0u;
        if (pass) q[(qh + qn + (uint32_t)__popc(b & lt)) & 63u] = (tile << 12) | e;
        qn += (uint32_t)__popc(b);
        if (qn >= 32u) level2(32u);
      }
    }
  }
  if (qn) level2(qn);
}

// ===========================================================================
// phase 4: universe query of my own filter (bloom tensors only) -> pos_mask + tile_count
// ===========================================================================
DR_D void phase_query(const EngineParams& P, Smem& sm) {
  const uint32_t tid = threadIdx.x;
  {  // the select histograms are free after the insert barrier: zero them for the next step
    uint4* h = reinterpret_cast<uint4*>(P.hist);
    const size_t n4 = (size_t)kNumHist * P.n_tensors * kHistBins / 4;
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (size_t i = (size_t)blockIdx.x * kThreads + tid; i < n4; i += (size_t)gridDim.x * kThreads) h[i] = z;
    for (uint32_t i = blockIdx.x * kThreads + tid; i < (uint32_t)kNumHist * P.n_tensors; i += gridDim.x * kThreads)
      P.hist_total[i] = 0u;
    if (blockIdx.x == 0 && tid == 0) { P.barrier[kUnsafeWord] = 0u; P.barrier[kNeedHist2Word] = 0u; }
  }
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  uint32_t tile, t_end;
  tile_range(P, kPartQuery, tile, t_end);
  while (tile < t_end) {
    const Tile t0 = load_tile(P.tiles, tile);
    load_tensor(P, t0.tensor, sm);
    const uint32_t seg_end = min(t_end, sm.td.tile_begin + sm.td.n_tiles);
    if (sm.td.mode == (uint32_t)kModeBloom) {
      const bool fits = sm.td.n_filter_words <= P.filter_smem_words;
      const uint32_t* filter = my_slot + sm.td.off_filter;
      if (fits) stage_filter(filter, sm.td.n_filter_words);
      if (tid == 0) sm.s.lb = 0;
      __syncthreads();
      ProbeCtx c;
      c.hint = sm.td.off_hint ? my_slot + sm.td.off_hint : nullptr;
      c.prefix = nullptr; c.n_sel = 0xFFFFFFFFu; c.cutoff = 0xFFFFFFFFu;
      c.mask_out = P.pos_mask; c.tile_count = P.tile_count;
      c.tile_begin = sm.td.tile_begin; c.seg_a = tile; c.seg_b = seg_end;
      c.n_hash = sm.td.n_hash; c.m_bits = sm.td.m_bits; c.seed = P.seed;
      c.pol_T = 0xFFFFFFFFu; c.pol_seed = 0u;
      if (fits) probe_segment(P, sm, c, [&](uint32_t w) { return g_filter_smem[w]; });
      else probe_segment(P, sm, c, [&](uint32_t w) { return __ldcg(filter + w); });
      __syncthreads();
      if (P.policy == kPolicyRandom) {                                     // raw positives of the tensor (emit derives the acceptance rate)
        uint32_t part = 0;
        for (uint32_t j = tile + tid; j < seg_end; j += kThreads) part += __ldcg(P.tile_count + j);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(kFullMask, part, o);
        if ((tid & 31u) == 0u && part) atomicAdd(n_pos_of(P, t0.tensor), part);
      }
    }
    tile = seg_end;
  }
}

// ===========================================================================
// phase 5: ordered compaction + value gather + residual update, one WARP per tile.
// The positives of a tile are 128 mask words; lane l owns groups 4l..4l+3, the in-tile rank of an element is a
// popcount prefix — no per-element flags, no CTA barrier in the tile loop.  The exclusive prefix of every tile of my
// range (count of positives in the tensor's earlier tiles) comes from one segmented warp scan over tile_count.
// W == 1 and plain fp32 values: the element is also written into the (zero-filled) dense output — the decode of a
// rank's own contribution costs nothing extra.
// ===========================================================================
// Expand this lane's 4 mask words into the warp's SMEM list: the element with local (in-tile) rank r goes to
// list[r - base] for r in [base, base + kListCap).  rank0 = local rank of this lane's first element.  Pure ALU + STS:
// the DRAM-latency work (value gathers) then runs over the list with all lanes busy and independent loads in flight
// (v11 walked the mask bits with one dependent gather per bit: emit 28 us, long-scoreboard bound).
constexpr uint32_t kListCap = 1024;            // u16 entries per warp: 2 KB x 16 warps of the dynamic SMEM buffer
DR_D void fill_list(uint16_t* list, const uint32_t (&mm)[4], uint32_t rank0, uint32_t base, uint32_t lane) {
  uint32_t lr = rank0 - base;                    // unsigned: entries before `base` wrap to huge values and are skipped
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t w = mm[j];
    while (w) {
      const uint32_t b = (uint32_t)__ffs((int)w) - 1u;
      w &= w - 1u;
      if (lr < kListCap) list[lr] = (uint16_t)((4u * lane + (uint32_t)j) * 32u + b);
      ++lr;
    }
  }
}

// 'random' policy (P1; reference pytorch/deepreduce.py:484-490 draws K of the positives with torch.randperm under a fixed
// global seed).  Here every positive x of a bloom tensor survives iff policy_hash(x, seed(step, tensor)) <= T with
// T = 2^32 * target / n_pos, target = the number of inserted elements (capped by the capacity): a seeded Bernoulli
// draw of rate target/n_pos — the expected count is the reference's K, false positives and true elements are
// dropped alike, and sender and receivers agree because T travels in the tensor's header word `thr_bits` (the
// receiver applies the same test inside its membership probe).  Runs at the head of the emit phase over this CTA's
// tiles: rewrites the positive masks and the per-tile counts in place; a grid barrier separates it from the
// compaction, which then is the leftmost policy on the surviving set.
DR_D void policy_filter(const EngineParams& P, Smem& sm) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, P.epoch & 1u, P.rank);
  uint32_t tile, t_end;
  tile_range(P, kPartEmit, tile, t_end);
  while (tile < t_end) {
    const Tile t0 = load_tile(P.tiles, tile);
    const TensorDesc* tdp = P.tensors + t0.tensor;
    const uint32_t tile_begin = __ldg(&tdp->tile_begin), n_tiles = __ldg(&tdp->n_tiles);
    const uint32_t seg_end = min(t_end, tile_begin + n_tiles);
    if (__ldg(&tdp->mode) == (uint32_t)kModeBloom) {
      const uint32_t n_pos = __ldcg(n_pos_of(P, t0.tensor)), n_ins = __ldcg(n_ins_of(P, t0.tensor));
      const uint32_t target = min(n_ins, min(__ldg(&tdp->k), __ldg(&tdp->val_cap)));
      const uint32_t T = (n_pos <= target) ? 0xFFFFFFFFu : (uint32_t)(((uint64_t)target << 32) / n_pos);
      const uint32_t pseed = policy_seed(P.epoch, __ldg(&tdp->salt));
      const uint32_t oh = __ldg(&tdp->off_hint);
      const uint32_t* hint = oh ? my_slot + oh : nullptr;
      if (tile == tile_begin && tid == 0) {                                // the CTA that owns the tensor's first tile
        DynHeader* dyn = reinterpret_cast<DynHeader*>(my_slot + kSlotHeaderWords) + t0.tensor;
        dyn->thr_bits = T;
        dyn->n_pos = n_pos;
      }
      if (T != 0xFFFFFFFFu) {
        for (uint32_t tl = tile + warp; tl < seg_end; tl += (uint32_t)kWarps) {
          const Tile ti = load_tile(P.tiles, tl);
          uint32_t mm[4];
          load_masks(P.pos_mask, tl, hint_nibble(hint, tl - tile_begin, lane), ti.n, lane, mm);
          uint32_t cnt = 0;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint32_t w = mm[j], keep = 0u;
            while (w) {
              const uint32_t b = (uint32_t)__ffs((int)w) - 1u;
              w &= w - 1u;
              const uint32_t x = ti.local0 + (4u * lane + (uint32_t)j) * 32u + b;
              if (policy_hash(x, pseed) <= T) keep |= 1u << b;
            }
            mm[j] = keep;
            cnt += (uint32_t)__popc(keep);
          }
          reinterpret_cast<uint4*>(P.pos_mask + (size_t)tl * kGroupsPerTile)[lane] = make_uint4(mm[0], mm[1], mm[2], mm[3]);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(kFullMask, cnt, o);
          if (lane == 0) P.tile_count[tl] = cnt;
        }
      }
    }
    tile = seg_end;
  }
}

template <bool kFull, bool kB, bool kDgc>
DR_D void phase_emit(const EngineParams& P, Smem& sm, uint32_t& bar_epoch) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  if (P.policy == kPolicyRandom) {                                         // grid-uniform
    policy_filter(P, sm);
    grid_barrier(P.barrier, bar_epoch, P.status, P.spin_limit);
  }
  if (blockIdx.x == 0 && tid == 0) {
    my_slot[0] = kMagic; my_slot[1] = P.epoch; my_slot[2] = P.n_tensors; my_slot[3] = P.payload_words;
    my_slot[4] = (uint32_t)P.rank;
  }
  uint32_t t0, t_end;
  tile_range(P, kPartEmit, t0, t_end);
  for (uint32_t c0 = t0; c0 < t_end; c0 += (uint32_t)kTile) {
    const uint32_t n_chunk = min((uint32_t)kTile, t_end - c0);
    // ---- exclusive prefix of every tile of the chunk inside its tensor
    const Tile first = load_tile(P.tiles, c0);
    {
      const uint32_t tb = __ldg(&P.tensors[first.tensor].tile_begin);
      uint32_t part = 0;
      for (uint32_t j = tb + tid; j < c0; j += kThreads) part += __ldcg(P.tile_count + j);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(kFullMask, part, o);
      __syncthreads();
      if (tid == 0) sm.s.lb = 0;
      __syncthreads();
      if (lane == 0 && part) atomicAdd(&sm.s.lb, part);
      __syncthreads();
    }
    if (warp == 0) {
      uint32_t carry = sm.s.lb, carry_tensor = first.tensor;
      for (uint32_t i0 = 0; i0 < n_chunk; i0 += 32u) {
        const uint32_t i = i0 + lane;
        const bool valid = i < n_chunk;
        const uint32_t v = valid ? __ldcg(P.tile_count + c0 + i) : 0u;
        const uint32_t tens = valid ? load_tile(P.tiles, c0 + i).tensor : 0xFFFFFFFEu;
        uint32_t prev_t = __shfl_up_sync(kFullMask, tens, 1);
        if (lane == 0) prev_t = carry_tensor;
        uint32_t fl = (tens != prev_t) ? 1u : 0u;                          // a new tensor starts at this tile
        uint32_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t y = __shfl_up_sync(kFullMask, x, o);
          const uint32_t g = __shfl_up_sync(kFullMask, fl, o);
          if (lane >= (uint32_t)o) { if (!fl) x += y; fl |= g; }
        }
        if (!fl) x += carry;                                               // still inside the tensor the previous 32 ended in
        if (valid) sm.u.excl[i] = x - v;
        carry = __shfl_sync(kFullMask, x, 31);
        carry_tensor = __shfl_sync(kFullMask, tens, 31);
      }
    }
    if (tid == kThreads - 1) sm.s.res[3] = 0u;                             // dynamic tile counter of this chunk
    __syncthreads();
    // ---- one warp per tile, tiles handed out dynamically (a tile's cost follows its number of positives)
    uint32_t cur = kNoTensor;
    uint32_t mode = 0, k = 0, val_cap = 0, off_vals = 0, off_idx = 0, off_prefix = 0, tile_begin = 0, n_tiles = 0,
             vmode = kVmodeFp32, off_selidx = 0, thr = 0;
    const uint32_t* hint = nullptr;
    uint16_t* list = reinterpret_cast<uint16_t*>(g_filter_smem) + warp * kListCap;
    while (true) {
      uint32_t i = 0;
      if (lane == 0) i = atomicAdd(&sm.s.res[3], 1u);
      i = __shfl_sync(kFullMask, i, 0);
      if (i >= n_chunk) break;
      const uint32_t tile = c0 + i;
      const Tile ti = load_tile(P.tiles, tile);
      if (ti.tensor != cur) {
        cur = ti.tensor;
        const TensorDesc* tdp = P.tensors + cur;
        mode = __ldg(&tdp->mode); k = __ldg(&tdp->k); val_cap = __ldg(&tdp->val_cap);
        off_vals = __ldg(&tdp->off_vals); off_idx = __ldg(&tdp->off_idx); off_prefix = __ldg(&tdp->off_prefix);
        tile_begin = __ldg(&tdp->tile_begin); n_tiles = __ldg(&tdp->n_tiles);
        vmode = __ldg(&tdp->vmode); off_selidx = __ldg(&tdp->off_selidx);
        const uint32_t oh = __ldg(&tdp->off_hint);
        hint = (mode == (uint32_t)kModeBloom && oh) ? my_slot + oh : nullptr;
        thr = __ldcg(&P.sel[cur].thr);
      }
      const uint32_t excl = sm.u.excl[i];
      const uint32_t tile_local = tile - tile_begin;
      uint32_t mm[4];
      load_masks(P.pos_mask, tile, hint_nibble(hint, tile_local, lane), ti.n, lane, mm);
      const uint32_t c = (uint32_t)(__popc(mm[0]) + __popc(mm[1]) + __popc(mm[2]) + __popc(mm[3]));
      const uint32_t incl = warp_incl_scan(c, lane);
      const uint32_t total = __shfl_sync(kFullMask, incl, 31);
      const uint32_t limit = (mode == (uint32_t)kModeBloom && P.policy != kPolicyP0) ? min(k, val_cap) : val_cap;
      DynHeader* dyn = reinterpret_cast<DynHeader*>(my_slot + kSlotHeaderWords) + cur;
      float* vals = reinterpret_cast<float*>(my_slot + off_vals);
      uint32_t* idxs = my_slot + off_idx;
      const bool scatter = emit_scatters(P, vmode);
      const uint32_t n_emit = excl < limit ? min(total, limit - excl) : 0u;      // elements of this tile that are shipped
      for (uint32_t base = 0; base < n_emit; base += kListCap) {
        fill_list(list, mm, incl - c, base, lane);
        __syncwarp();
        const uint32_t n_here = min(kListCap, n_emit - base);
        for (uint32_t q0 = 0; q0 < n_here; q0 += 64u) {                    // two independent gathers per lane in flight
          const uint32_t qa = q0 + lane, qb = q0 + 32u + lane;
          const bool ha = qa < n_here, hb = qb < n_here;
          const uint32_t ea = ha ? list[qa] : 0u, eb = hb ? list[qb] : 0u;
          const size_t ga = (size_t)ti.base + ea, gb = (size_t)ti.base + eb;
          float va = 0.f, vb = 0.f;
          if (ha) va = __ldcg(P.resid + ga);
          if (hb) vb = __ldcg(P.resid + gb);
          auto put = [&](bool have, uint32_t q, uint32_t e, size_t gi, float v) {
            if (!have) return;
            const uint32_t rp = excl + base + q;
            if constexpr (kFull) {
              if (vmode == kVmodeBf16) {
                // bf16 values: v rounded goes on the wire and its rounding error, exact, stays in the residual (0
                // where the rounded value is not finite, as for fp32 values).  dec is what every receiver adds into
                // its zero-filled output, so a value that rounds to -0.0 lands as +0.0 here too.
                const uint32_t h = bf16_rne_bits(v);
                reinterpret_cast<uint16_t*>(vals)[rp] = (uint16_t)h;
                const float w = __uint_as_float(h << 16), dec = __fadd_rn(w, 0.0f);
                P.resid[gi] = isfinite(w) ? __fsub_rn(v, w) : 0.0f;
                if constexpr (kDgc) { if (dec != 0.0f) P.mom[gi] = 0.0f; }
                if (P.world == 1) put_out<kB>(P, gi, dec * P.scale);
                if (mode == (uint32_t)kModeRaw) idxs[rp] = ti.local0 + e;
                else if (mode == (uint32_t)kModeRle) rle_put(idxs, rp, e);
                else if (mode == (uint32_t)kModeEf) ef_put(my_slot, P.tensors + cur, rp, tile_local, e);
                if (rp == limit - 1u) dyn->cutoff = ti.local0 + e;
                return;
              }
            }
            vals[rp] = v;
            P.resid[gi] = 0.0f;                                            // residual is exactly 0 on the shipped set
            // momentum factor masking where the own decoded value is this fp32 value (coded values: phase_fix)
            if constexpr (kDgc) { if (vmode == kVmodeFp32 && v != 0.0f) P.mom[gi] = 0.0f; }
            if (scatter) put_out<kB>(P, gi, v * P.scale);
            if (mode == (uint32_t)kModeRaw) idxs[rp] = ti.local0 + e;
            else if (kFull && mode == (uint32_t)kModeRle) rle_put(idxs, rp, e);
            else if (kFull && mode == (uint32_t)kModeEf) ef_put(my_slot, P.tensors + cur, rp, tile_local, e);
            if (kFull && vmode != kVmodeFp32) my_slot[off_selidx + rp] = (uint32_t)gi;
            if (rp == limit - 1u) dyn->cutoff = ti.local0 + e;
          };
          put(ha, qa, ea, ga, va);
          put(hb, qb, eb, gb, vb);
        }
        __syncwarp();
      }
      if (lane == 0) {
        // bloom: shipped prefix table; shared: sender-local scratch that the decode reads back from the own slot
        if (mode == (uint32_t)kModeBloom || (kFull && mode == (uint32_t)kModeShared)) my_slot[off_prefix + tile_local] = min(excl, limit);
        else if (kFull && (mode == (uint32_t)kModeRle || mode == (uint32_t)kModeEf))
          reinterpret_cast<uint16_t*>(my_slot + off_prefix)[tile_local] =
              (uint16_t)(excl >= limit ? 0u : min(total, limit - excl));
        if (tile_local + 1u == n_tiles) {
          const uint32_t all = excl + total;
          dyn->n_sel = min(all, limit);
          if (!(P.policy == kPolicyRandom && mode == (uint32_t)kModeBloom)) {   // else: written by policy_filter
            dyn->n_pos = all;
            dyn->thr_bits = thr;
          }
          if (all < limit) dyn->cutoff = 0xFFFFFFFFu;
          P.sel[cur].prev_thr = thr;
        }
      }
    }
    __syncthreads();                                                       // sm.u.excl is rewritten by the next chunk
  }
}

// ===========================================================================
// 'both' (bloom index + polynomial value fit): phases rank / fit / fix and the decode-side evaluation.
// Replaces the reference's PolyFit (sort + per-segment Vandermonde normal equations with a CPU 6x6
// inverse per segment, reference pytorch/deepreduce.py:306-425) and the int64 `mapping` (:263-267).
// ===========================================================================
// segment table of reference get_segments (:362-377): fine segments at both steep ends of the descending curve
DR_D void build_segments(int n, int num_pos, int* start, int& n_seg) {
  const double ratios[10] = {1.0 / 5, 1.0 / 10, 1.0 / 30, 1.0 / 100, 1.0 / 300, 1.0 / 1000, 1.0 / 3000, 1.0 / 10000, 1.0 / 30000, 1.0 / 100000};
  int pos[10], neg[10], np = 0, nn = 0, sp = 0, sn = 0;
  const int num_neg = n - num_pos;
  for (int i = 0; i < 10; ++i) {
    const int a = (int)((double)num_pos * ratios[i]);
    if (a > 30) { pos[np++] = a; sp += a; }
    const int b = (int)((double)num_neg * ratios[i]);
    if (b > 30) { neg[nn++] = b; sn += b; }
  }
  int s = 0, acc = 0;
  for (int i = np - 1; i >= 0; --i) { start[s++] = acc; acc += pos[i]; }
  start[s++] = acc; acc += num_pos - sp;
  start[s++] = acc; acc += num_neg - sn;
  for (int i = 0; i < nn; ++i) { start[s++] = acc; acc += neg[i]; }
  start[s] = acc;                               // == n
  n_seg = s;
}

DR_D float poly_value(const float* __restrict__ coef, const int* start, int n_seg, int deg, uint32_t j) {
  int s = 0;
  for (int i = 0; i < n_seg; ++i) if (start[i + 1] > start[i] && (int)j >= start[i]) s = i;
  const int len = start[s + 1] - start[s];
  float p[kMaxDeg + 1];
  gram_eval<kMaxDeg + 1>((float)((int)j - start[s]), (float)(len - 1), min(deg, len - 1), p);
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k <= kMaxDeg; ++k) if (k <= deg) acc += __ldcg(coef + s * (deg + 1) + k) * p[k];
  return acc;
}

// 'dexp' (kVmodeDexp): two double-exponential curves per tensor, over the rank map's two sign runs.  Coefficient words
// (fp32): {a, b, p, q} of the positive run by ascending value, then {a, b, p, q} of the magnitudes of the rest (the
// values <= 0) by ascending |v|; each on its own abscissa x_i = (i + 1) / run length.
DR_D bool ranked(uint32_t vmode) { return vmode == kVmodePolyfit || vmode == kVmodeDexp; }

// words before the {num_pos, n} tail of a ranked tensor's header
DR_D uint32_t coef_words(uint32_t vmode, uint32_t deg) { return vmode == kVmodeDexp ? kDexpCoefWords : kMaxSeg * (deg + 1u); }

// fitted value of rank j (descending order) from the shipped fp32 words: the sender's residual and every receiver's
// decode go through this one evaluation, in fp64 without contraction (the oracle's torch order), rounded once
DR_D float dexp_value(const float* __restrict__ coef, uint32_t num_pos, uint32_t n, uint32_t j) {
  const bool pos = j < num_pos;
  const uint32_t len = pos ? num_pos : n - num_pos, i = pos ? num_pos - 1u - j : j - num_pos;
  const float* c = coef + (pos ? 0 : 4);
  const double x = (double)(i + 1u) / (double)len;
  const double v = __dadd_rn(__dmul_rn((double)__ldcg(c), exp(__dmul_rn((double)__ldcg(c + 2), x))),
                             __dmul_rn((double)__ldcg(c + 1), exp(__dmul_rn((double)__ldcg(c + 3), x))));
  return pos ? (float)v : -(float)v;
}

DR_D uint32_t load_rank(const uint32_t* slot, const TensorDesc& td, uint32_t p) {
  return td.rank_u32 ? __ldcg(slot + td.off_rankmap + p)
                     : (uint32_t)__ldcg(reinterpret_cast<const uint16_t*>(slot + td.off_rankmap) + p);
}

// ---- exact descending rank: counting sort on 13 bits of the order-preserving key + all-pairs inside a bin ----
// order_key: the float's bits made monotone as an unsigned integer (sign-magnitude flipped), with -0.0 folded onto
// +0.0.  Equal values get equal keys, so ties (the two zeros included) are broken by position alone, as the stable
// descending sort of the specification does; and a NaN still gets a key, so the ranks are a permutation whatever
// the values are (a NaN's place among them is unspecified).
DR_D uint32_t order_key(float v) {
  const uint32_t b = __float_as_uint(v) == 0x80000000u ? 0u : __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Bins are monotone non-increasing in the order key and centred on the tensor's selection threshold T (31-bit
// magnitude key): per sign 1024 coarse bins above 4T (16 per octave), 2048 fine bins on [T, 4T) (relative width
// 2^-10) and 1024 coarse bins below T (false positives carry arbitrary small values).  Exactness never depends on
// the binning — phase 9 counts inside the bin — only the amount of in-bin work does.
DR_D uint32_t rank_bin(uint32_t ok, uint32_t T) {
  const bool neg = !(ok & 0x80000000u);
  const uint32_t key = (neg ? ~ok : ok) & 0x7FFFFFFFu;
  uint32_t pb;                                   // 0 = largest magnitude ... 4095 = smallest
  if (key >= T) {
    const uint32_t d = key - T;
    if (d < (2u << 23)) pb = 1024u + (2047u - (d >> 13));
    else pb = 1023u - min(1023u, (key >> 19) - ((T + (2u << 23)) >> 19));
  } else {
    pb = 3072u + min(1023u, (T >> 19) - (key >> 19));
  }
  return neg ? (4096u + (4095u - pb)) : pb;
}

// phase 6: bin populations
DR_D void phase_rank_hist(const EngineParams& P, Smem& sm) {
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  for (uint32_t task = blockIdx.x; task < P.n_poly_tasks; task += gridDim.x) {
    const uint32_t t = __ldg(P.poly_tasks + 2 * task), p0 = __ldg(P.poly_tasks + 2 * task + 1);
    load_tensor(P, t, sm);
    if (!ranked(sm.td.vmode)) continue;
    const DynHeader* dyn = reinterpret_cast<const DynHeader*>(my_slot + kSlotHeaderWords) + t;
    const uint32_t n = __ldcg(&dyn->n_sel), p = p0 + threadIdx.x;
    if (p < n) {
      const float v = __ldcg(reinterpret_cast<const float*>(my_slot + sm.td.off_vals) + p);
      atomicAdd(P.poly_bins + (size_t)sm.td.poly_ord * 2 * kRankBins + rank_bin(order_key(v), __ldcg(&P.sel[t].thr)), 1u);
    }
  }
}

// phase 7: per tensor, exclusive prefix of the bin counts -> bin starts (second half of the bin table)
DR_D void phase_rank_scan(const EngineParams& P, Smem& sm) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (uint32_t o = blockIdx.x; o < P.n_poly; o += gridDim.x) {
    uint32_t* cnt = P.poly_bins + (size_t)o * 2 * kRankBins;
    uint32_t* start = cnt + kRankBins;
    constexpr int kPer = kRankBins / kThreads;                    // 16 consecutive bins per thread
    uint32_t c[kPer], sum = 0;
#pragma unroll
    for (int i = 0; i < kPer; ++i) { c[i] = __ldcg(cnt + threadIdx.x * kPer + i); sum += c[i]; }
    uint32_t incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t nb = __shfl_up_sync(kFullMask, incl, d); if (lane >= (uint32_t)d) incl += nb; }
    __syncthreads();
    if (lane == 31) sm.s.warp_tot[warp] = incl;
    __syncthreads();
    uint32_t base = 0;
    for (uint32_t w = 0; w < warp; ++w) base += sm.s.warp_tot[w];
    uint32_t run = base + incl - sum;
#pragma unroll
    for (int i = 0; i < kPer; ++i) { start[threadIdx.x * kPer + i] = run; run += c[i]; }
  }
}

// phase 8: group values by bin (order inside a bin is arbitrary here; phase 9 makes the rank exact)
DR_D void phase_rank_scatter(const EngineParams& P, Smem& sm) {
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  for (uint32_t task = blockIdx.x; task < P.n_poly_tasks; task += gridDim.x) {
    const uint32_t t = __ldg(P.poly_tasks + 2 * task), p0 = __ldg(P.poly_tasks + 2 * task + 1);
    load_tensor(P, t, sm);
    if (!ranked(sm.td.vmode)) continue;
    const DynHeader* dyn = reinterpret_cast<const DynHeader*>(my_slot + kSlotHeaderWords) + t;
    const uint32_t n = __ldcg(&dyn->n_sel), p = p0 + threadIdx.x;
    if (p < n) {
      const float v = __ldcg(reinterpret_cast<const float*>(my_slot + sm.td.off_vals) + p);
      uint32_t* tab = P.poly_bins + (size_t)sm.td.poly_ord * 2 * kRankBins;
      const uint32_t b = rank_bin(order_key(v), __ldcg(&P.sel[t].thr));
      // the count array is re-used as the running cursor: it is decremented down to 0 while filling the bin
      const uint32_t within = atomicSub(tab + b, 1u) - 1u;
      const uint32_t pos = __ldcg(tab + kRankBins + b) + within;
      P.bucket_val[sm.td.poly_off + pos] = v;
      P.bucket_pos[sm.td.poly_off + pos] = p;
    }
  }
}

// phase 9: exact rank = bin start + #(bin mates that sort before me); writes rank map, sorted values, num_pos
DR_D void phase_rank_exact(const EngineParams& P, Smem& sm) {
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  for (uint32_t task = blockIdx.x; task < P.n_poly_tasks; task += gridDim.x) {
    const uint32_t t = __ldg(P.poly_tasks + 2 * task), p0 = __ldg(P.poly_tasks + 2 * task + 1);
    load_tensor(P, t, sm);
    if (!ranked(sm.td.vmode)) continue;
    const DynHeader* dyn = reinterpret_cast<const DynHeader*>(my_slot + kSlotHeaderWords) + t;
    const uint32_t n = __ldcg(&dyn->n_sel), i = p0 + threadIdx.x;   // i = position in the grouped arrays
    float v = 0.f;
    if (i < n) {
      const float* bv = P.bucket_val + sm.td.poly_off;
      const uint32_t* bp = P.bucket_pos + sm.td.poly_off;
      v = __ldcg(bv + i);
      const uint32_t p = __ldcg(bp + i), k = order_key(v), b = rank_bin(k, __ldcg(&P.sel[t].thr));
      const uint32_t* start = P.poly_bins + (size_t)sm.td.poly_ord * 2 * kRankBins + kRankBins;
      const uint32_t lo = __ldcg(start + b), hi = (b + 1 < (uint32_t)kRankBins) ? __ldcg(start + b + 1) : n;
      uint32_t rank = lo;
      for (uint32_t q = lo; q < hi; ++q) {               // (key, position) is a strict total order: a permutation
        const uint32_t kw = order_key(__ldcg(bv + q));
        rank += (kw > k || (kw == k && __ldcg(bp + q) < p)) ? 1u : 0u;
      }
      if (sm.td.rank_u32) my_slot[sm.td.off_rankmap + p] = rank;
      else reinterpret_cast<uint16_t*>(my_slot + sm.td.off_rankmap)[p] = (uint16_t)rank;
      reinterpret_cast<float*>(my_slot + sm.td.off_sorted)[rank] = v;
    }
    const uint32_t pc = __syncthreads_count(i < n && v > 0.f);
    if (threadIdx.x == 0) {
      uint32_t* tail = my_slot + sm.td.off_coef + coef_words(sm.td.vmode, sm.td.poly_degree);
      if (pc) atomicAdd(tail, pc);
      if (p0 == 0) tail[1] = n;
    }
  }
}

// phase 10: one warp per (tensor, segment): Gram least squares  c_k = sum p_k y / sum p_k^2;
// 'dexp' tensors: one CTA per (tensor, sign run), the double-exponential regression of dexp_fit.cuh
DR_D void phase_fit(const EngineParams& P, Smem& sm) {
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t gw = blockIdx.x * kWarps + (threadIdx.x >> 5), nw = gridDim.x * kWarps;
  for (uint32_t task = gw; task < P.n_poly * kMaxSeg; task += nw) {
    const uint32_t t = __ldg(P.poly_tensors + task / kMaxSeg), s = task % kMaxSeg;
    const TensorDesc* td = P.tensors + t;
    if (__ldg(&td->vmode) != kVmodePolyfit) continue;
    const uint32_t off_coef = __ldg(&td->off_coef), off_sorted = __ldg(&td->off_sorted);
    const int deg = (int)__ldg(&td->poly_degree);
    const uint32_t* tail = my_slot + off_coef + kMaxSeg * (deg + 1);
    const int num_pos = (int)__ldcg(tail), n = (int)__ldcg(tail + 1);
    int start[kMaxSeg + 2], n_seg;
    build_segments(n, num_pos, start, n_seg);
    if ((int)s >= n_seg) continue;
    const int len = start[s + 1] - start[s];
    if (len <= 0) continue;
    const float* y = reinterpret_cast<const float*>(my_slot + off_sorted) + start[s];
    const int deg_eff = min(deg, len - 1);
    // recurrence constants of this segment (no divisions in the inner loop):
    //   p_{k+1} = ra[k] * (N - 2x) * p_k - rb[k] * p_{k-1}
    const float N = (float)(len - 1), invN = len > 1 ? 1.f / N : 0.f;
    float ra[kMaxDeg], rb[kMaxDeg];
#pragma unroll
    for (int k = 1; k < kMaxDeg; ++k) {
      const float dnm = (k + 1.f) * (N - k);
      ra[k] = (k < deg_eff) ? (2.f * k + 1.f) / dnm : 0.f;
      rb[k] = (k < deg_eff) ? (float)k * (N + k + 1.f) / dnm : 0.f;
    }
    float num[kMaxDeg + 1], den[kMaxDeg + 1];
#pragma unroll
    for (int k = 0; k <= kMaxDeg; ++k) { num[k] = 0.f; den[k] = 0.f; }
    for (int x0 = lane; x0 < len; x0 += 32 * 8) {                  // 8 independent loads in flight per lane
      float yv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) yv[u] = (x0 + 32 * u < len) ? __ldcg(y + x0 + 32 * u) : 0.f;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int x = x0 + 32 * u;
        if (x < len) {
          float p[kMaxDeg + 1];
          const float uu = N - 2.f * (float)x;
          p[0] = 1.f;
          p[1] = deg_eff >= 1 ? uu * invN : 0.f;
#pragma unroll
          for (int k = 1; k < kMaxDeg; ++k) p[k + 1] = ra[k] * uu * p[k] - rb[k] * p[k - 1];
#pragma unroll
          for (int k = 0; k <= kMaxDeg; ++k) { num[k] += p[k] * yv[u]; den[k] += p[k] * p[k]; }
        }
      }
    }
#pragma unroll
    for (int k = 0; k <= kMaxDeg; ++k) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        num[k] += __shfl_xor_sync(kFullMask, num[k], o);
        den[k] += __shfl_xor_sync(kFullMask, den[k], o);
      }
    }
    float* coef = reinterpret_cast<float*>(my_slot + off_coef) + s * (deg + 1);
#pragma unroll
    for (int k = 0; k <= kMaxDeg; ++k)
      if ((int)lane == k && k <= deg) coef[k] = (k <= deg_eff && den[k] > 0.f) ? num[k] / den[k] : 0.f;
  }
  // 'dexp': one CTA per (tensor, sign run) runs the fp64 regression over the sorted values of that run
  for (uint32_t task = blockIdx.x; task < 2u * P.n_poly; task += gridDim.x) {
    const uint32_t t = __ldg(P.poly_tensors + task / 2u), neg = task & 1u;
    const TensorDesc* td = P.tensors + t;
    if (__ldg(&td->vmode) != kVmodeDexp) continue;
    float* coef = reinterpret_cast<float*>(my_slot + __ldg(&td->off_coef));
    const uint32_t* tail = my_slot + __ldg(&td->off_coef) + kDexpCoefWords;
    const uint32_t num_pos = __ldcg(tail), n = __ldcg(tail + 1);
    const float* ys = reinterpret_cast<const float*>(my_slot + __ldg(&td->off_sorted)) + num_pos;   // the split
    double c[4];
    // positive run: descending ranks num_pos-1 .. 0; the rest: |v| = -v in rank order
    dexp_fit_block<kThreads>([&](int64_t k) { return neg ? -(double)__ldcg(ys + k) : (double)__ldcg(ys - 1 - k); },
                             (int64_t)(neg ? n - num_pos : num_pos), sm.u.dexp, c);
    if (threadIdx.x == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) coef[4 * neg + i] = (float)c[i];
    }
  }
}

// kVmodeSign fix task: this CTA owns one 512-value bucket and its 16 bit words (lane 0 of each warp writes its ballot).
// Not inlined, so that its fp64 sums do not take registers from the rest of the kernel.
template <bool kDgc>
__device__ __noinline__ void fix_sign(const EngineParams& P, Smem& sm, uint32_t* my_slot, uint32_t t, uint32_t p0) {
  const DynHeader* dyn = reinterpret_cast<const DynHeader*>(my_slot + kSlotHeaderWords) + t;
  const uint32_t nq = __ldcg(&dyn->n_sel);
  if (p0 >= nq) return;
  const uint32_t p = p0 + threadIdx.x;
  const float v = p < nq ? __ldcg(reinterpret_cast<const float*>(my_slot + sm.td.off_vals) + p) : 0.f;
  const float mu = sign_scale(v, min(nq - p0, kSignBucket), sm.u.sign_ws);
  const uint32_t word = sign_word(v);
  if (threadIdx.x == 0) reinterpret_cast<float*>(my_slot + sm.td.off_coef)[p0 >> 9] = mu;
  if (p < nq) {
    if ((threadIdx.x & 31u) == 0) my_slot[sm.td.off_rankmap + (p >> 5)] = word;
    // the residual keeps v - d, 0 where d is not finite (a NaN or inf in the bucket); the sign bit follows v, so
    // v - d cannot overflow
    const float d = sign_decoded(v < 0.f, mu);
    const uint32_t gi = __ldcg(my_slot + sm.td.off_selidx + p);
    P.resid[gi] = isfinite(d) ? __fsub_rn(v, d) : 0.0f;
    if constexpr (kDgc) { if (d != 0.0f) P.mom[gi] = 0.0f; }
  }
}

// kVmodeFp8 fix task: this CTA owns 512 values, 16 blocks of 32 (one per warp).  The 16 scale bytes are collected in
// shared memory and written as 4 whole words; lanes 0, 4, .., 28 of each warp write the element words.  A task starts
// at a multiple of 512 values, so no word is shared between tasks.  Not inlined, as fix_sign.
template <bool kDgc>
__device__ __noinline__ void fix_fp8(const EngineParams& P, Smem& sm, uint32_t* my_slot, uint32_t t, uint32_t p0) {
  const DynHeader* dyn = reinterpret_cast<const DynHeader*>(my_slot + kSlotHeaderWords) + t;
  const uint32_t nq = __ldcg(&dyn->n_sel);
  if (p0 >= nq) return;
  const uint32_t p = p0 + threadIdx.x, lane = threadIdx.x & 31u;
  const float v = p < nq ? __ldcg(reinterpret_cast<const float*>(my_slot + sm.td.off_vals) + p) : 0.f;
  const uint32_t s = fp8_block_scale(v);              // blocks past the end: A = 0, scale byte 0
  const uint32_t word = fp8_elem_word(v, s);
  if (lane == 0) reinterpret_cast<uint8_t*>(sm.u.fp8_scales)[threadIdx.x >> 5] = (uint8_t)s;
  __syncthreads();
  if (threadIdx.x < kWarps / 4 && p0 + 128u * threadIdx.x < nq)
    my_slot[sm.td.off_coef + (p0 >> 7) + threadIdx.x] = sm.u.fp8_scales[threadIdx.x];
  if (p < nq) {
    if ((lane & 3u) == 0) my_slot[sm.td.off_rankmap + (p >> 2)] = word;
    // the residual keeps v - d, 0 where d is not finite (an inf or a NaN in the block)
    const float d = fp8_decoded(s, word & 0xFFu);     // every lane's own byte is the low byte of its word
    const uint32_t gi = __ldcg(my_slot + sm.td.off_selidx + p);
    P.resid[gi] = isfinite(d) ? __fsub_rn(v, d) : 0.0f;
    if constexpr (kDgc) { if (d != 0.0f) P.mom[gi] = 0.0f; }
  }
}

// phase 11: error feedback sees the fit error: resid[idx_p] = value_p - fitted_p
// (kDgc: and the momentum of idx_p is cleared when the decoded value, the one every receiver rebuilds, is non-zero)
template <bool kDgc>
DR_D void phase_fix(const EngineParams& P, Smem& sm) {
  const uint32_t parity = P.epoch & 1u;
  uint32_t* my_slot = slot_ptr(P.arena[P.rank], P, parity, P.rank);
  for (uint32_t task = blockIdx.x; task < P.n_poly_tasks; task += gridDim.x) {
    const uint32_t t = __ldg(P.poly_tasks + 2 * task), p0 = __ldg(P.poly_tasks + 2 * task + 1);
    load_tensor(P, t, sm);
    if (sm.td.vmode == kVmodeQsgd) {
      // bucketed QSGD (reference QSGD, pytorch/deepreduce.py:849-907, which syncs the host once per bucket):
      // this CTA owns one 512-value bucket: L2 norm, stochastic rounding with a counter-based RNG, int8 level
      const DynHeader* dyn = reinterpret_cast<const DynHeader*>(my_slot + kSlotHeaderWords) + t;
      const uint32_t nq = __ldcg(&dyn->n_sel);
      if (p0 >= nq) continue;
      const uint32_t p = p0 + threadIdx.x;
      const float v = p < nq ? __ldcg(reinterpret_cast<const float*>(my_slot + sm.td.off_vals) + p) : 0.f;
      float ss = v * v;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(kFullMask, ss, o);
      __syncthreads();
      if ((threadIdx.x & 31u) == 0) sm.s.warp_tot[threadIdx.x >> 5] = __float_as_uint(ss);
      __syncthreads();
      float tot = 0.f;
      for (int w = 0; w < kWarps; ++w) tot += __uint_as_float(sm.s.warp_tot[w]);
      const float norm = sqrtf(tot), q = (float)sm.td.poly_degree;
      if (threadIdx.x == 0) reinterpret_cast<float*>(my_slot + sm.td.off_coef)[p0 >> 9] = norm;
      if (p < nq) {
        const float lf = (norm > 0.f ? q / norm : 0.f) * fabsf(v);
        const float prev = floorf(lf);
        const float u = (float)((double)policy_hash(p, 0x51EDu + P.epoch) / 4294967296.0);
        float l = prev + ((u < (lf - prev)) ? 1.f : 0.f);
        l = fminf(l, q);     // lf can round above q when norm == |v|; the residual below follows the clamped level
        l = v > 0.f ? l : (v < 0.f ? -l : 0.f);
        if (sm.td.rank_u32) reinterpret_cast<int16_t*>(my_slot + sm.td.off_rankmap)[p] = (int16_t)l;   // quantum_num >= 128
        else reinterpret_cast<int8_t*>(my_slot + sm.td.off_rankmap)[p] = (int8_t)l;
        P.resid[__ldcg(my_slot + sm.td.off_selidx + p)] = v - norm / q * l;
        if constexpr (kDgc) { if (__fmul_rn(norm / q, l) != 0.0f) P.mom[__ldcg(my_slot + sm.td.off_selidx + p)] = 0.0f; }
      }
      continue;
    }
    if (sm.td.vmode == kVmodeSign) { fix_sign<kDgc>(P, sm, my_slot, t, p0); continue; }
    if (sm.td.vmode == kVmodeFp8) { fix_fp8<kDgc>(P, sm, my_slot, t, p0); continue; }
    const int deg = (int)sm.td.poly_degree;
    const uint32_t* tail = my_slot + sm.td.off_coef + coef_words(sm.td.vmode, deg);
    const int num_pos = (int)__ldcg(tail), n = (int)__ldcg(tail + 1);
    if ((int)p0 >= n) continue;
    const bool dexp = sm.td.vmode == kVmodeDexp;
    if (threadIdx.x == 0 && !dexp) build_segments(n, num_pos, sm.seg_start, sm.n_seg);
    __syncthreads();
    const uint32_t p = p0 + threadIdx.x;
    if ((int)p < n) {
      const float* coef = reinterpret_cast<const float*>(my_slot + sm.td.off_coef);
      const uint32_t rank = load_rank(my_slot, sm.td, p);
      const float fitted = dexp ? dexp_value(coef, num_pos, n, rank) : poly_value(coef, sm.seg_start, sm.n_seg, deg, rank);
      const float v = __ldcg(reinterpret_cast<const float*>(my_slot + sm.td.off_vals) + p);
      P.resid[__ldcg(my_slot + sm.td.off_selidx + p)] = v - fitted;
      if constexpr (kDgc) { if (fitted != 0.0f) P.mom[__ldcg(my_slot + sm.td.off_selidx + p)] = 0.0f; }
    }
  }
}

// phase 14: evaluate every rank's fitted curve once (dense, all lanes busy); decode then gathers fitted[rank]
DR_D void phase_expand(const EngineParams& P, Smem& sm) {
  const uint32_t parity = P.epoch & 1u;
  uint32_t* arena = P.arena[P.rank];
  for (uint32_t wt = blockIdx.x; wt < P.n_poly_tasks * (uint32_t)P.world; wt += gridDim.x) {
    const uint32_t r = wt / P.n_poly_tasks, task = wt - r * P.n_poly_tasks;
    const uint32_t t = __ldg(P.poly_tasks + 2 * task), j0 = __ldg(P.poly_tasks + 2 * task + 1);
    load_tensor(P, t, sm);
    if (!ranked(sm.td.vmode)) continue;
    const uint32_t* slot = slot_ptr(arena, P, parity, (int)r);
    const int deg = (int)sm.td.poly_degree;
    const uint32_t* tail = slot + sm.td.off_coef + coef_words(sm.td.vmode, deg);
    const int num_pos = (int)__ldcg(tail), n = (int)__ldcg(tail + 1);
    if ((int)j0 >= n) continue;
    const bool dexp = sm.td.vmode == kVmodeDexp;
    if (threadIdx.x == 0 && !dexp) build_segments(n, num_pos, sm.seg_start, sm.n_seg);
    __syncthreads();
    const uint32_t j = j0 + threadIdx.x;
    const float* coef = reinterpret_cast<const float*>(slot + sm.td.off_coef);
    if ((int)j < n)
      P.expand_buf[(size_t)r * P.poly_total + sm.td.poly_off + j] =
          dexp ? dexp_value(coef, num_pos, n, j) : poly_value(coef, sm.seg_start, sm.n_seg, deg, j);
  }
}


// ===========================================================================
// push + flags.  Every CTA copies its share of the finished slot into each peer's arena (16-byte P2P stores over
// NVLink, or ONE multimem store that the NVSwitch replicates), fences at system scope and takes a ticket; the CTA
// that takes the last ticket releases the epoch flags — the copy needs no grid barrier before the signal.
// ===========================================================================
DR_D void phase_push(const EngineParams& P, Smem& sm) {
  const uint32_t parity = P.epoch & 1u;
  const uint4* src = reinterpret_cast<const uint4*>(slot_ptr(P.arena[P.rank], P, parity, P.rank));
  const uint32_t n4 = (P.payload_words + 3u) >> 2;
  if (P.mc_arena) {                                      // NVLS: one multimem store lands in every GPU's arena (the switch replicates)
    uint4* dst = reinterpret_cast<uint4*>(slot_ptr(P.mc_arena, P, parity, P.rank));
    for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n4; i += gridDim.x * kThreads) multimem_st_v4(dst + i, __ldcg(src + i));
  } else {
    for (int h = 1; h < P.world; ++h) {
      const int peer = (P.rank + h) % P.world;             // stagger so peers are not hit in lock-step
      uint4* dst = reinterpret_cast<uint4*>(slot_ptr(P.arena[peer], P, parity, P.rank));
      for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n4; i += gridDim.x * kThreads) {
        const uint4 v = __ldcg(src + i);
        asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                     :: "l"(dst + i), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
      }
    }
  }
  __syncthreads();                                       // every thread's peer stores are issued ...
  if (threadIdx.x == 0) {
    __threadfence_system();                              // ... and ordered (cumulatively) before the ticket
    const uint32_t t = atomicAdd(P.barrier + 1, 1u);
    sm.s.lb = (t == gridDim.x - 1u) ? 1u : 0u;
  }
  __syncthreads();
  if (sm.s.lb && P.fault != 1) {                         // last CTA: every share of the slot is in the peers' memory
    __threadfence_system();
    const int p = threadIdx.x;
    if (p < P.world && p != P.rank) st_release_sys(P.arena[p] + P.rank, P.epoch);
  }
  __syncthreads();
}

// Wait for every peer's epoch flag (flag word `base + peer` of my arena).  A peer that never shows up is fatal: the
// wait is bounded by WALL TIME (peer_timeout_ms — a rank can legitimately be seconds late: checkpoint, dataloader
// stall, first-step autotune), and on expiry the status word is set, the output is poisoned with NaN and the CTA
// leaves the kernel without decoding slots the peer may still be writing.  Returns false (CTA-uniform) on timeout.
template <bool kB>
DR_D bool wait_flags(const EngineParams& P, uint32_t base, uint32_t aux_base) {
  const int p = threadIdx.x;
  int bad = 0;
  if (p < P.world && p != P.rank) {
    const uint32_t* flag = P.arena[P.rank] + base + p;
    uint32_t spins = 0;
    uint64_t t_start = 0;
    while ((int32_t)(ld_acquire_sys(flag) - P.epoch) < 0) {
      if ((++spins & 1023u) == 0u) {
        const uint64_t now = globaltimer_ns();
        if (t_start == 0) t_start = now;
        else if (now - t_start > (uint64_t)P.peer_timeout_ms * 1000000ull) { bad = 1; break; }
      }
      __nanosleep(64);
    }
    if (bad) { atomicExch(P.status, kErrPeerWait); atomicExch(P.status + 1, aux_base + (uint32_t)p); }
  }
  const int any_bad = __syncthreads_or(bad);
  if (any_bad && threadIdx.x == 0) {                     // poison: the aggregate of this step does not exist
    uint32_t tile, t_end;
    decode_range(P, tile, t_end);
    if (tile < t_end) {
      if constexpr (kB) P.grad_bf16[load_tile(P.tiles, tile).base] = 0x7FC0u;
      else P.grad[load_tile(P.tiles, tile).base] = __uint_as_float(0x7FC00000u);
    }
  }
  return !any_bad;
}


// value of the p-th shipped coordinate of a sender's tensor under its value codec
template <bool kFull>
DR_D float coded_value(const uint32_t* slot, const TensorDesc& td, const float* vals, const float* fitted, uint32_t rp) {
  if (kFull && ranked(td.vmode)) return __ldcg(fitted + load_rank(slot, td, rp));
  if constexpr (kFull) {
    if (td.vmode == kVmodeBf16) return __uint_as_float((uint32_t)__ldcg(reinterpret_cast<const uint16_t*>(vals) + rp) << 16);
    if (td.vmode == kVmodeSign)
      return sign_decoded((__ldcg(slot + td.off_rankmap + (rp >> 5)) >> (rp & 31u)) & 1u,
                          __ldcg(reinterpret_cast<const float*>(slot + td.off_coef) + (rp >> 9)));
    if (td.vmode == kVmodeFp8)        // block rp / 32's scale byte, then the element byte; byte j in bits 8j
      return fp8_decoded((__ldcg(slot + td.off_coef + (rp >> 7)) >> ((rp >> 2) & 24u)) & 0xFFu,
                         (__ldcg(slot + td.off_rankmap + (rp >> 2)) >> ((rp & 3u) << 3)) & 0xFFu);
  }
  if (kFull && td.vmode == kVmodeQsgd) {
    const float norm = __ldcg(reinterpret_cast<const float*>(slot + td.off_coef) + (rp >> 9));
    const float lvl = td.rank_u32 ? (float)__ldcg(reinterpret_cast<const int16_t*>(slot + td.off_rankmap) + rp)
                                  : (float)__ldcg(reinterpret_cast<const int8_t*>(slot + td.off_rankmap) + rp);
    return norm / (float)td.poly_degree * lvl;
  }
  return __ldcg(vals + rp);
}

// ===========================================================================
// phases 15 + 16: decode of this rank's slice (all tiles when unsharded) for all W senders.
//
// phase 15 (probe pass).  The work is the concatenation, over the senders r != me, of my slice's tiles; every CTA
// takes one contiguous piece of that sequence.  A CTA therefore stages ONE sender's filter per tensor and probes a
// long run of tiles with it (v11-v15 walked sender-major inside every small per-CTA tile range and staged W filters
// per tensor for a handful of tiles: decode 35 us median / 67 us max at W = 2 — and it grows with W).  Positives go
// to dec_mask, one slot per (sender, tile of my slice).  My own positives are already in pos_mask (query phase).
//
// phase 16 (apply + compact + push).  After a grid barrier, one WARP per tile of my slice: for the senders in rank
// order, masks -> in-tile ranks (prefix table + popcounts) -> value gather -> accumulate into the zero-filled dense
// output (same warp and lane own an element for every sender: the sum order is rank-major and deterministic).  When
// sharded, the same warp then re-reads the finished tile (L2-hot), compacts its non-zeros into a small SMEM stage
// and stores them straight into every peer's stage-2 slot (P2P or one multimem store); the last CTA (ticket) writes
// the entry count and releases the second flag set.  No separate compaction pass over the slice, no second barrier.
// ===========================================================================
DR_D uint32_t lower_bound_u32(const uint32_t* a, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (__ldcg(a + mid) < x) lo = mid + 1; else hi = mid; }
  return lo;
}

template <bool kFull>
DR_D void phase_decode(const EngineParams& P, Smem& sm) {
  const uint32_t tid = threadIdx.x;
  const uint32_t parity = P.epoch & 1u;
  uint32_t* arena = P.arena[P.rank];
  if (kFull) {
    for (uint32_t i = blockIdx.x * kThreads + tid; i < P.n_poly * 2u * kRankBins; i += gridDim.x * kThreads)
      P.poly_bins[i] = 0u;
  }
  if (P.world == 1) return;
  uint32_t s_begin, s_end;
  decode_span(P, P.rank, s_begin, s_end);
  const uint32_t span = s_end - s_begin;
  const uint64_t total = (uint64_t)(P.world - 1) * span;                   // (sender != me, tile of my slice) pairs
  uint64_t w0 = total * blockIdx.x / gridDim.x, w1 = total * (blockIdx.x + 1) / gridDim.x;
  while (w0 < w1) {
    const uint32_t k = (uint32_t)(w0 / span);
    const int r = other_sender(k, P.rank);
    const uint32_t tile = s_begin + (uint32_t)(w0 - (uint64_t)k * span);
    const uint32_t piece_end = s_begin + (uint32_t)min((uint64_t)span, w1 - (uint64_t)k * span);
    const Tile t0 = load_tile(P.tiles, tile);
    load_tensor(P, t0.tensor, sm);
    const uint32_t seg_end = min(piece_end, sm.td.tile_begin + sm.td.n_tiles);
    if (sm.td.mode == (uint32_t)kModeBloom) {
      const uint32_t* slot = slot_ptr(arena, P, parity, r);
      const DynHeader* dyn = reinterpret_cast<const DynHeader*>(slot + kSlotHeaderWords) + t0.tensor;
      const uint32_t n_sel = __ldcg(&dyn->n_sel), cutoff = __ldcg(&dyn->cutoff);
      if (n_sel != 0u) {                                                   // CTA-uniform
        const uint32_t* filter = slot + sm.td.off_filter;
        const bool fits = sm.td.n_filter_words <= P.filter_smem_words;
        if (fits) stage_filter(filter, sm.td.n_filter_words);
        __syncthreads();
        if (tid == 0) sm.s.lb = 0;
        __syncthreads();
        ProbeCtx c;
        c.hint = sm.td.off_hint ? slot + sm.td.off_hint : nullptr;
        c.prefix = slot + sm.td.off_prefix; c.n_sel = n_sel; c.cutoff = cutoff;
        c.mask_out = dec_mask_base(P.dec_mask, r, s_begin, span); c.tile_count = nullptr;
        c.tile_begin = sm.td.tile_begin; c.seg_a = tile; c.seg_b = seg_end;
        c.n_hash = sm.td.n_hash; c.m_bits = sm.td.m_bits; c.seed = P.seed;
        c.pol_T = 0xFFFFFFFFu; c.pol_seed = 0u;
        if (P.policy == kPolicyRandom) {                                   // the sender's acceptance threshold rides in its header
          c.pol_T = __ldcg(&dyn->thr_bits);
          c.pol_seed = policy_seed(P.epoch, sm.td.salt);
        }
        if (fits) probe_segment(P, sm, c, [&](uint32_t w) { return g_filter_smem[w]; });
        else probe_segment(P, sm, c, [&](uint32_t w) { return __ldcg(filter + w); });
        __syncthreads();
      }
    }
    w0 += seg_end - tile;
  }
}

constexpr uint32_t kS2Stage = 256;             // per-warp stage of the slice list: entries (index | value), flushed at > 128

// debug timeline: sub-step stamps of the apply/compact phase go to the (otherwise unused at kVmodeFp32) slots 6..9
DR_D void dbg_stamp(const EngineParams& P, int slot, int which) {
  if (P.debug_times && threadIdx.x == 0) P.debug_times[((size_t)slot * gridDim.x + blockIdx.x) * 2 + which] = globaltimer_ns();
}

// Bloom apply of sender r to tile tl (tile_local inside tensor t) of my decode span, one warp: the sender's positives of
// the tile (my own query's, or the probe pass's in dec_mask) -> in-tile ranks (prefix table + popcounts) -> values.
// add(e, coded) runs for every shipped positive, e = in-tile element offset (distinct per sender), coded() = its value
// before scaling: the caller writes the whole add expression, whose FMA contraction decides the bits.
// kGateFirst: the header words and the prefix decide whether the tile is skipped before the hint and the masks are
// loaded (rank-ordered loop); otherwise all of them are issued first, one round trip (item loop).
template <bool kFull, bool kGateFirst, typename AddFn>
DR_D void apply_bloom(const EngineParams& P, uint32_t* arena, uint32_t parity, const TensorDesc& td, uint32_t t, int r,
                      uint32_t tl, uint32_t tile_local, const Tile& ti, uint32_t s_begin, uint32_t span, uint16_t* list,
                      uint32_t lane, AddFn add) {
  const uint32_t* slot = slot_ptr(arena, P, parity, r);
  const DynHeader* dyn = reinterpret_cast<const DynHeader*>(slot + kSlotHeaderWords) + t;
  const uint32_t n_sel = __ldcg(&dyn->n_sel), cutoff = __ldcg(&dyn->cutoff);
  if (kGateFirst && n_sel == 0u) return;
  const uint32_t pre = __ldcg(slot + td.off_prefix + tile_local);
  if (kGateFirst && !ships_into(pre, n_sel, ti.local0, cutoff)) return;     // warp-uniform: nothing of rank r lands here
  const uint32_t* hint = td.off_hint ? slot + td.off_hint : nullptr;
  const float* vals = reinterpret_cast<const float*>(slot + td.off_vals);
  const float* fitted = P.expand_buf + (size_t)r * P.poly_total + td.poly_off;   // 'both': rank r's curve
  const uint32_t* masks = (r == P.rank) ? P.pos_mask : dec_mask_base(P.dec_mask, r, s_begin, span);
  uint32_t mm[4];
  load_masks(masks, tl, hint_nibble(hint, tile_local, lane), ti.n, lane, mm);
  if (!kGateFirst && !ships_into(pre, n_sel, ti.local0, cutoff)) return;
  const uint32_t c = (uint32_t)(__popc(mm[0]) + __popc(mm[1]) + __popc(mm[2]) + __popc(mm[3]));
  const uint32_t incl = warp_incl_scan(c, lane);
  const uint32_t total = __shfl_sync(kFullMask, incl, 31);
  const uint32_t n_take = min(total, n_sel - pre);                         // positives beyond the sender's n_sel were not shipped
  for (uint32_t base = 0; base < n_take; base += kListCap) {
    fill_list(list, mm, incl - c, base, lane);
    __syncwarp();
    const uint32_t n_here = min(kListCap, n_take - base);
    for (uint32_t q = lane; q < n_here; q += 32u)
      add(list[q], [&]() { return coded_value<kFull>(slot, td, vals, fitted, pre + base + q); });
    __syncwarp();
  }
}

// Reserve n entries of my stage-2 slice list at its cursor s2 and store the entries (idx[j], val[j]) there in every
// peer's arena as interleaved (index, value) pairs: one 8-byte store per entry and peer, or one multicast store.  Run by
// a group of kN threads (a warp or the CTA), of which this thread is number i; `bcast` hands every thread of the group
// thread 0's reservation and orders the group's writes of idx / val before the stores.  Entries past s2_cap are
// dropped: status 6.
template <uint32_t kN, typename BcastFn>
DR_D void s2_store(const EngineParams& P, uint32_t parity, uint32_t* s2, uint32_t i, uint32_t n, const uint32_t* idx,
                   const float* val, BcastFn bcast) {
  uint32_t gbase = 0;
  if (i == 0 && n) gbase = atomicAdd(s2, n);
  gbase = bcast(gbase);
  uint32_t n_ok = n;
  if (gbase + n > P.s2_cap) {
    if (i == 0) atomicExch(P.status, kErrS2Overflow);                      // stage-2 capacity exceeded
    n_ok = gbase < P.s2_cap ? P.s2_cap - gbase : 0u;
  }
  if (P.mc_arena) {
    uint2* dst = reinterpret_cast<uint2*>(s2_ptr(P.mc_arena, P, parity, P.rank) + 4) + gbase;
    for (uint32_t j = i; j < n_ok; j += kN) multimem_st_v2(dst + j, make_uint2(idx[j], __float_as_uint(val[j])));
  } else {
    for (int h = 1; h < P.world; ++h) {
      const int peer = (P.rank + h) % P.world;
      uint2* dst = reinterpret_cast<uint2*>(s2_ptr(P.arena[peer], P, parity, P.rank) + 4) + gbase;
      for (uint32_t j = i; j < n_ok; j += kN) dst[j] = make_uint2(idx[j], __float_as_uint(val[j]));
    }
  }
}

template <bool kFull, bool kB>
DR_D void phase_compact(const EngineParams& P, Smem& sm, uint32_t& bar_epoch) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t parity = P.epoch & 1u;
  uint32_t* arena = P.arena[P.rank];
  const bool stage2 = sharded(P);
  uint32_t s_begin, s_end;
  decode_span(P, P.rank, s_begin, s_end);
  const uint32_t span = s_end - s_begin;
  uint32_t t_first, t_last;
  decode_range(P, t_first, t_last);
  // ---- (1) CTA-level: tensors without a filter (plain pairs, run-length) accumulate a tile in SMEM, rank-major
  for (uint32_t tile = t_first; tile < t_last;) {
    const Tile t0 = load_tile(P.tiles, tile);
    const uint32_t t = t0.tensor;
    {  // filter-coded tensors (and everything emit already scattered at W == 1) are skipped without a CTA barrier
      const TensorDesc* tdp = P.tensors + t;
      const uint32_t seg_end0 = min(t_last, __ldg(&tdp->tile_begin) + __ldg(&tdp->n_tiles));
      if (__ldg(&tdp->mode) == (uint32_t)kModeBloom || (P.world == 1 && __ldg(&tdp->vmode) == kVmodeFp32)) { tile = seg_end0; continue; }
    }
    load_tensor(P, t, sm);
    const uint32_t seg_end = min(t_last, sm.td.tile_begin + sm.td.n_tiles);
    if (kFull && sm.td.mode == (uint32_t)kModeShared) {
      // 'randomk': every rank holds the same selection, so my own positive mask and my own per-tile prefix place every
      // sender's p-th value.  A sender whose header words differ from mine drew a different set: status 7, not added.
      const uint32_t* own = slot_ptr(arena, P, parity, P.rank);
      const DynHeader* od = reinterpret_cast<const DynHeader*>(own + kSlotHeaderWords) + t;
      const uint32_t o_sel = __ldcg(&od->n_sel), o_cut = __ldcg(&od->cutoff), o_thr = __ldcg(&od->thr_bits);
      uint16_t* list = reinterpret_cast<uint16_t*>(g_filter_smem);          // in-tile offset of the rank-th positive
      for (; tile < seg_end; ++tile) {
        const Tile ti = load_tile(P.tiles, tile);
        const uint32_t pre = __ldcg(own + sm.td.off_prefix + (tile - sm.td.tile_begin));
        __syncthreads();
        for (int j = tid; j < kTile; j += kThreads) sm.u.acc[j] = 0.0f;
        if (warp == 0) {
          uint32_t mm[4];
          load_masks(P.pos_mask, tile, 0xFu, ti.n, lane, mm);
          const uint32_t c = (uint32_t)(__popc(mm[0]) + __popc(mm[1]) + __popc(mm[2]) + __popc(mm[3]));
          const uint32_t incl = warp_incl_scan(c, lane);
          uint32_t lr = incl - c;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            for (uint32_t w = mm[j]; w; w &= w - 1u)
              list[lr++] = (uint16_t)((4u * lane + (uint32_t)j) * 32u + (uint32_t)(__ffs((int)w) - 1));
          }
          if (lane == 31u) sm.s.lb = incl;
        }
        __syncthreads();
        const uint32_t n_take = pre < o_sel ? min(sm.s.lb, o_sel - pre) : 0u;
        for (int r = 0; r < P.world; ++r) {
          const uint32_t* slot = slot_ptr(arena, P, parity, r);
          const DynHeader* dyn = reinterpret_cast<const DynHeader*>(slot + kSlotHeaderWords) + t;
          if (__ldcg(&dyn->n_sel) != o_sel || __ldcg(&dyn->cutoff) != o_cut || __ldcg(&dyn->thr_bits) != o_thr) {
            if (tid == 0) { atomicExch(P.status, kErrDisagree); atomicExch(P.status + 1, (uint32_t)r); }
            continue;                                                      // CTA-uniform
          }
          const float* vals = reinterpret_cast<const float*>(slot + sm.td.off_vals);
          const float* fitted = P.expand_buf + (size_t)r * P.poly_total + sm.td.poly_off;
          for (uint32_t j = tid; j < n_take; j += kThreads) {
            const uint32_t e = list[j];                                    // distinct per sender: no atomics
            sm.u.acc[e] = sm.u.acc[e] + __fmul_rn(coded_value<kFull>(slot, sm.td, vals, fitted, pre + j), P.scale);
          }
          __syncthreads();                                                 // senders are added in rank order
        }
        for (uint32_t e = tid; e < ti.n; e += kThreads) put_out<kB>(P, ti.base + e, sm.u.acc[e]);
      }
    } else if (kFull && (sm.td.mode == (uint32_t)kModeRle || sm.td.mode == (uint32_t)kModeEf)) {
      // running entry prefix of every sender at my first tile of this tensor = sum of the earlier tiles' counts
      __syncthreads();
      if (tid < 16) sm.s.rle_pre[tid] = 0u;
      __syncthreads();
      const uint32_t first_local = tile - sm.td.tile_begin;
      for (int r = 0; r < P.world; ++r) {
        const uint16_t* cnt = reinterpret_cast<const uint16_t*>(slot_ptr(arena, P, parity, r) + sm.td.off_prefix);
        uint32_t part = 0;
        for (uint32_t j = tid; j < first_local; j += kThreads) part += __ldcg(cnt + j);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(kFullMask, part, o);
        if (lane == 0 && part) atomicAdd(&sm.s.rle_pre[r], part);
      }
      for (; tile < seg_end; ++tile) {
        const Tile ti = load_tile(P.tiles, tile);
        __syncthreads();
        for (int j = tid; j < kTile; j += kThreads) sm.u.acc[j] = 0.0f;
        __syncthreads();
        for (int r = 0; r < P.world; ++r) {
          const uint32_t* slot = slot_ptr(arena, P, parity, r);
          const uint32_t c = __ldcg(reinterpret_cast<const uint16_t*>(slot + sm.td.off_prefix) + (tile - sm.td.tile_begin));
          const uint32_t pre = sm.s.rle_pre[r];
          const float* vals = reinterpret_cast<const float*>(slot + sm.td.off_vals);
          const float* fitted = P.expand_buf + (size_t)r * P.poly_total + sm.td.poly_off;   // 'both': rank r's curve
          if (sm.td.mode == (uint32_t)kModeRle) {
            for (uint32_t j = tid; j < c; j += kThreads) {
              const uint32_t rp = pre + j;
              if (rp < sm.td.val_cap)                       // distinct positions per sender
                sm.u.acc[rle_get(slot + sm.td.off_idx, rp)] += coded_value<kFull>(slot, sm.td, vals, fitted, rp) * P.scale;
            }
          } else if (c) {
            // Elias-Fano: the tile's high-stream range [pre + t*B, pre + t*B + c + B) (at most 256 words), funnel-shifted
            // to its start, one word per thread; the popcount scan gives every set bit its rank j and the thread lists
            // its high part q - j at j (SMEM), then every thread takes one entry, as the run-length loop does: offset
            // (q - j) << L | its low field.  Bits past the range (the next tile's) are masked off.
            const uint32_t L = sm.td.ef_low_bits, B = kTile >> L;
            const uint32_t s = pre + (tile - sm.td.tile_begin) * B, len = c + B, nw = (len + 31u) >> 5;
            const uint32_t* hi = slot + sm.td.off_hi;
            const uint32_t hi_words = (sm.td.val_cap + sm.td.n_tiles * B + 31u) >> 5;
            uint32_t x = 0u;
            if (tid < nw) {
              const uint32_t w = (s >> 5) + tid;
              const uint32_t a = w < hi_words ? __ldcg(hi + w) : 0u, b = w + 1u < hi_words ? __ldcg(hi + w + 1u) : 0u;
              x = __funnelshift_r(a, b, s & 31u);
              if (len - 32u * tid < 32u) x &= (1u << (len - 32u * tid)) - 1u;
            }
            const uint32_t n = (uint32_t)__popc(x), incl = warp_incl_scan(n, lane);
            if (lane == 31u) sm.s.warp_tot[warp] = incl;
            __syncthreads();
            uint16_t* list = reinterpret_cast<uint16_t*>(g_filter_smem);   // high part of the j-th entry
            uint32_t j = incl - n;
            for (uint32_t w = 0; w < warp; ++w) j += sm.s.warp_tot[w];
            for (; x; x &= x - 1u, ++j) {
              const uint32_t h = 32u * tid + (uint32_t)(__ffs((int)x) - 1) - j;
              if (j < c) list[j] = (uint16_t)min(h, B);     // B: not in this tile's range (a malformed stream)
            }
            __syncthreads();
            for (uint32_t q = tid; q < c; q += kThreads) {
              const uint32_t h = list[q], rp = pre + q;
              if (h < B && rp < sm.td.val_cap)              // distinct positions per sender
                sm.u.acc[(h << L) | ef_low(slot + sm.td.off_idx, rp, L)] += coded_value<kFull>(slot, sm.td, vals, fitted, rp) * P.scale;
            }
          }
          __syncthreads();                                  // senders are added in rank order: deterministic sums
          if (tid == 0) sm.s.rle_pre[r] = pre + c;
        }
        for (uint32_t e = tid; e < ti.n; e += kThreads) put_out<kB>(P, ti.base + e, sm.u.acc[e]);
      }
    } else {
      for (; tile < seg_end; ++tile) {
        const Tile ti = load_tile(P.tiles, tile);
        __syncthreads();
        for (int j = tid; j < kTile; j += kThreads) sm.u.acc[j] = 0.0f;
        __syncthreads();
        for (int r = 0; r < P.world; ++r) {
          const uint32_t* slot = slot_ptr(arena, P, parity, r);
          const DynHeader* dyn = reinterpret_cast<const DynHeader*>(slot + kSlotHeaderWords) + t;
          const uint32_t n_sel = min(__ldcg(&dyn->n_sel), sm.td.val_cap);
          const uint32_t* idxs = slot + sm.td.off_idx;
          const float* vals = reinterpret_cast<const float*>(slot + sm.td.off_vals);
          const float* fitted = P.expand_buf + (size_t)r * P.poly_total + sm.td.poly_off;
          if (n_sel <= 2048u) {
            // short lists (the <= 1000-element bypass tensors ship <= 10 pairs): one pass over the list — two binary
            // searches are ~20 dependent L2 round trips per sender and tile (W = 2 timeline: 3-12 us of this phase)
            for (uint32_t j = tid; j < n_sel; j += kThreads) {
              const uint32_t off = __ldcg(idxs + j) - ti.local0;
              if (off < ti.n) atomicAdd(&sm.u.acc[off], coded_value<kFull>(slot, sm.td, vals, fitted, j) * P.scale);
            }
          } else {
            const uint32_t lo = lower_bound_u32(idxs, n_sel, ti.local0);
            const uint32_t hi = lower_bound_u32(idxs, n_sel, ti.local0 + ti.n);
            for (uint32_t j = lo + tid; j < hi; j += kThreads)
              atomicAdd(&sm.u.acc[__ldcg(idxs + j) - ti.local0], coded_value<kFull>(slot, sm.td, vals, fitted, j) * P.scale);
          }
          __syncthreads();                                  // rank-major: one sender at a time
        }
        for (uint32_t e = tid; e < ti.n; e += kThreads) put_out<kB>(P, ti.base + e, sm.u.acc[e]);
      }
    }
  }
  __syncthreads();
  dbg_stamp(P, 6, 0);
  // ---- (2) one warp per tile: bloom apply (all senders, rank order), then the slice list of the finished tile
  uint8_t* dyn_base = reinterpret_cast<uint8_t*>(g_filter_smem);
  uint16_t* list = reinterpret_cast<uint16_t*>(dyn_base) + warp * kListCap;                         // 2 KB per warp
  uint32_t* st_idx = reinterpret_cast<uint32_t*>(dyn_base + (size_t)kWarps * kListCap * 2u) + warp * 2u * kS2Stage;
  float* st_val = reinterpret_cast<float*>(st_idx + kS2Stage);
  uint32_t* s2 = s2_ptr(arena, P, parity, P.rank);                          // s2[0]: list cursor (zeroed in the accumulate phase)
  uint32_t n_st = 0;                                                         // entries in my warp's stage (warp-uniform)
  const uint32_t lt = (1u << lane) - 1u;
  // fast mode: the warps' stages are gathered in a CTA-wide stage (the list region, free once the apply items are
  // done) and the CTA reserves its part of the slice list with ONE global atomic — per-warp reservations were ~5 000
  // same-address atomics in a few microseconds and cost more than the compaction itself (timeline: 17 us)
  uint32_t* cta_idx = reinterpret_cast<uint32_t*>(dyn_base);
  float* cta_val = reinterpret_cast<float*>(dyn_base + (size_t)kWarps * kListCap);
  constexpr uint32_t kCtaCap = kWarps * kListCap / 4u;                       // 4096 entries (idx | val halves of the 32 KB list region)
  const bool cta_stage = (!P.deterministic && P.world > 1);
  auto flush = [&]() {                                                       // warp-uniform
    if (n_st == 0u) return;
    if (cta_stage) {
      uint32_t pos = 0;
      if (lane == 0) pos = atomicAdd(&sm.s.res[2], n_st);
      pos = __shfl_sync(kFullMask, pos, 0);
      if (pos + n_st <= kCtaCap) {
        for (uint32_t j = lane; j < n_st; j += 32u) { cta_idx[pos + j] = st_idx[j]; cta_val[pos + j] = st_val[j]; }
        __syncwarp();
        n_st = 0;
        return;
      }
      // does not fit (dense tiles): this and every later reservation go straight to the peers; the CTA stage ends
      // at the first failed position (reservations are monotonic, so everything below it was written)
      if (lane == 0) atomicMin(&sm.s.warp_tot[0], pos);
    }
    s2_store<32u>(P, parity, s2, lane, n_st, st_idx, st_val,
                  [&](uint32_t g) { g = __shfl_sync(kFullMask, g, 0); __syncwarp(); return g; });
    __syncwarp();
    n_st = 0;
  };
  uint32_t cur = kNoTensor;
  TensorDesc td;                                                             // this warp's current tensor (registers / local)
  auto warp_tensor = [&](uint32_t t) {
    cur = t;
    const TensorDesc& src = P.tensors[cur];
    td.mode = __ldg(&src.mode); td.n_hash = 0; td.tile_begin = __ldg(&src.tile_begin);
    td.off_vals = __ldg(&src.off_vals); td.off_prefix = __ldg(&src.off_prefix); td.off_hint = __ldg(&src.off_hint);
    td.vmode = __ldg(&src.vmode); td.off_coef = __ldg(&src.off_coef); td.off_rankmap = __ldg(&src.off_rankmap);
    td.poly_degree = __ldg(&src.poly_degree); td.rank_u32 = __ldg(&src.rank_u32); td.poly_off = __ldg(&src.poly_off);
  };
  const bool fast = !P.deterministic && P.world > 1;
  if (fast) {
    // ---- (2a) every (sender, tile of my slice) pair is an independent work item of one warp: masks -> ranks -> value
    // gather -> RED.ADD into the zero-filled dense output.  No read-modify-write latency, W x more parallelism than
    // walking the senders of a tile in turn (one tile per warp at W = 8 left 13 of 16 warps idle).
    const uint64_t n_items = (uint64_t)P.world * span;
    const uint64_t n_warps = (uint64_t)gridDim.x * kWarps;
    for (uint64_t it = (uint64_t)blockIdx.x * kWarps + warp; it < n_items; it += n_warps) {
      const int r = (int)(it / span);
      const uint32_t tl = s_begin + (uint32_t)(it - (uint64_t)r * span);
      const Tile ti = load_tile(P.tiles, tl);
      if (ti.tensor != cur) warp_tensor(ti.tensor);
      if (td.mode != (uint32_t)kModeBloom) continue;
      apply_bloom<kFull, false>(P, arena, parity, td, cur, r, tl, tl - td.tile_begin, ti, s_begin, span, list, lane,
                                [&](uint32_t e, auto coded) {
        const float v = coded() * P.scale;
        if constexpr (kB) atomicAdd(P.acc32 + (size_t)(tl - s_begin) * kTile + e, v);   // the tile's acc32 row
        else atomicAdd(P.grad + ti.base + e, v);
      });
    }
    __syncthreads();
    dbg_stamp(P, 6, 1);
    dbg_stamp(P, 7, 0);
    grid_barrier(P.barrier, bar_epoch, P.status, P.spin_limit);            // every tile of my slice is final
    dbg_stamp(P, 7, 1);
    cur = kNoTensor;
  }
  if (tid == 0) { sm.s.res[2] = 0u; sm.s.warp_tot[0] = 0xFFFFFFFFu; }       // CTA stage cursor / first failed reservation
  __syncthreads();
  dbg_stamp(P, 8, 0);
  for (uint32_t tl = t_first + warp; tl < t_last; tl += kWarps) {
    const Tile ti = load_tile(P.tiles, tl);
    if (ti.tensor != cur) warp_tensor(ti.tensor);
    const bool apply = !fast && td.mode == (uint32_t)kModeBloom && !(P.world == 1 && td.vmode == kVmodeFp32);
    if (apply) {
      const uint32_t tile_local = tl - td.tile_begin;
      for (int r = 0; r < P.world; ++r) {
        apply_bloom<kFull, true>(P, arena, parity, td, cur, r, tl, tile_local, ti, s_begin, span, list, lane,
                                 [&](uint32_t e, auto coded) {
          float* o;                                                        // bf16: the tile's acc32 row
          if constexpr (kB) o = P.acc32 + (size_t)(tl - s_begin) * kTile + e;
          else o = P.grad + ti.base + e;
          *o = *o + coded() * P.scale;
        });
      }
    }
    if constexpr (kB) {
      // every sender of the tile is in its acc32 row: round once into the bf16 output (the row was zeroed in phase 0 up
      // to the tile's element count rounded up to 4, so the 4-wide pass below reads only zeroed words)
      if (bloom_applied(P, td.mode, td.vmode)) {
        __syncwarp();
        const float4* row = reinterpret_cast<const float4*>(P.acc32 + (size_t)(tl - s_begin) * kTile);
        const uint32_t n4 = (ti.n + 3u) >> 2;
        for (uint32_t i = lane; i < n4; i += 32u) {
          const float4 a = __ldcg(row + i);
          const uint32_t lo = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(a.x)) |
                              ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(a.y)) << 16);
          const uint32_t hi = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(a.z)) |
                              ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(a.w)) << 16);
          reinterpret_cast<uint2*>(P.grad_bf16 + ti.base)[i] = make_uint2(lo, hi);
        }
      }
    }
    if (stage2) {
      // the tile is final (every sender added, or written by part (1)): its non-zeros go to the peers (bf16: the rounded
      // values, shipped as their exact fp32 widening)
      __syncwarp();
      const float4* src4 = reinterpret_cast<const float4*>(P.grad + ti.base);
      const uint32_t n4 = (ti.n + 3u) >> 2;                                  // tensors are padded to 32 floats
      for (uint32_t i0 = 0; i0 < n4; i0 += 128u) {                           // four independent 512-byte loads in flight
        float4 v4[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const uint32_t i = i0 + (uint32_t)u * 32u + lane;
          if constexpr (kB) v4[u] = i < n4 ? widen_bf16x4(__ldcg(reinterpret_cast<const uint2*>(P.grad_bf16 + ti.base) + i))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
          else v4[u] = i < n4 ? __ldcg(src4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const uint32_t i = i0 + (uint32_t)u * 32u + lane;
          const float vv[4] = {v4[u].x, v4[u].y, v4[u].z, v4[u].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            // bf16: a rounded -0 (an fp32 aggregate never is -0: every sum starts from +0) travels like any value, so
            // the receivers' bits stay the owner's; only +0 is the zero fill every rank already holds
            bool nz;
            if constexpr (kB) nz = __float_as_uint(vv[j]) != 0u && (i * 4u + (uint32_t)j) < ti.n;
            else nz = vv[j] != 0.f && (i * 4u + (uint32_t)j) < ti.n;
            const uint32_t bal = __ballot_sync(kFullMask, nz);
            if (nz) {
              const uint32_t pos = n_st + (uint32_t)__popc(bal & lt);
              st_idx[pos] = ti.base + i * 4u + (uint32_t)j;
              st_val[pos] = vv[j];
            }
            n_st += (uint32_t)__popc(bal);
          }
          if (n_st > kS2Stage - 128u) flush();
        }
      }
    }
  }
  if (stage2) {
    flush();
    __syncthreads();                                                         // every warp's entries are staged / stored
    if (cta_stage) {
      const uint32_t n = min(min(sm.s.res[2], kCtaCap), sm.s.warp_tot[0]);
      s2_store<(uint32_t)kThreads>(P, parity, s2, tid, n, cta_idx, cta_val, [&](uint32_t g) {
        if (tid == 0) sm.s.res[3] = g;
        __syncthreads();
        return sm.s.res[3];
      });
      __syncthreads();
    }
    dbg_stamp(P, 8, 1);
    if (tid == 0) {
      __threadfence_system();                                                // ... and ordered before the ticket (cumulative)
      const uint32_t t = atomicAdd(P.barrier + 2, 1u);
      sm.s.res[1] = (t == gridDim.x - 1u) ? 1u : 0u;
    }
    __syncthreads();
    if (sm.s.res[1]) {                                                       // last CTA: every chunk is in the peers' memory
      const int p = tid;
      if (p < P.world && p != P.rank) {
        __threadfence_system();
        const uint32_t n = min(__ldcg(s2), P.s2_cap);
        uint32_t* dst = s2_ptr(P.arena[p], P, parity, P.rank);
        dst[0] = n; dst[1] = P.epoch;
        __threadfence_system();
        st_release_sys(P.arena[p] + kArenaFlagWords + P.rank, P.epoch);
      }
    }
    __syncthreads();
  }
}

template <bool kB>
DR_D void phase_scatter(const EngineParams& P) {
  const uint32_t parity = P.epoch & 1u;
  const uint32_t gtid = blockIdx.x * kThreads + threadIdx.x, gsz = gridDim.x * kThreads;
  for (int h = 1; h < P.world; ++h) {
    const int r = (P.rank + h) % P.world;
    const uint32_t* s2 = s2_ptr(P.arena[P.rank], P, parity, r);
    const uint32_t n = min(__ldcg(s2), P.s2_cap);
    const uint2* pairs = reinterpret_cast<const uint2*>(s2 + 4);             // interleaved (index, value)
    for (uint32_t i = gtid; i < n; i += gsz) { const uint2 e = __ldcg(pairs + i); put_out<kB>(P, e.x, __uint_as_float(e.y)); }
  }
}

// Which phases do anything for this configuration (CTA-uniform, decided before the phase runs so that the grid
// barrier in front of a phase is only paid when it does).
template <bool kFull>
DR_D bool phase_active(const EngineParams& P, int ph) {
  switch (ph) {
    case kPhAccum: case kPhInsert: case kPhQuery: case kPhEmit: return true;
    case kPhFallback: return __ldcg(P.barrier + kUnsafeWord) != 0u;
    case kPhHist2: return __ldcg(P.barrier + kNeedHist2Word) != 0u;
    case kPhRankHist: case kPhRankScan: case kPhRankScatter: case kPhRankExact: case kPhFit: case kPhExpand:
      return kFull && P.n_poly != 0u;
    case kPhFix: return kFull && P.n_poly_tasks != 0u;
    case kPhPush: case kPhSignal: return P.world > 1;
    case kPhDecode: case kPhCompact: return P.world > 1 || (kFull && P.n_poly_tasks != 0u);
    case kPhSignal2: case kPhScatter: return sharded(P);
    default: return false;
  }
}

template <int kMinBlocks, bool kFull, bool kB, bool kDgc = false, bool kClip = false>
__global__ void __launch_bounds__(kThreads, kMinBlocks) dr_engine_kernel(const __grid_constant__ EngineParams P) {
  __shared__ Smem sm;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 16; ++i) mbar_init(&sm.bar[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  uint32_t bar_epoch = 0;
  bool pending = false;        // a phase ran since the last grid barrier of this launch
  bool prev_wait = false;      // the previous active phase was a peer-flag wait
  for (int ph = P.phase_begin; ph < P.phase_end; ++ph) {
    // the fallback decision reads a word written in the accumulate phase: it is taken after the barrier that the
    // digit-2 phase needs anyway
    if (ph == kPhFallback && pending) { grid_barrier(P.barrier, bar_epoch, P.status, P.spin_limit); pending = false; }
    if (!phase_active<kFull>(P, ph)) continue;
    const bool is_wait = (ph == kPhSignal || ph == kPhSignal2);
    // no barrier: in front of a flag wait; after one (every CTA waited itself)
    if (pending && !is_wait && !prev_wait) {
      grid_barrier(P.barrier, bar_epoch, P.status, P.spin_limit);
      pending = false;
    }
    if (P.debug_times && threadIdx.x == 0) {
      P.debug_times[((size_t)ph * gridDim.x + blockIdx.x) * 2] = globaltimer_ns();
      if (ph == P.phase_begin) {
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        P.debug_times[((size_t)kPhEnd * gridDim.x + blockIdx.x) * 2] = smid;
      }
    }
    switch (ph) {
      case kPhAccum:
        if constexpr (kClip) {                 // every CTA passes both barriers, also one without tiles or tensors
          clip_tile_sums<kB>(P);
          grid_barrier(P.barrier, bar_epoch, P.status, P.spin_limit);
          clip_factors(P);
          grid_barrier(P.barrier, bar_epoch, P.status, P.spin_limit);
        }
        if (P.use_tma) phase_accum<true, kFull, kB, kDgc, kClip>(P, sm); else phase_accum<false, kFull, kB, kDgc, kClip>(P, sm);
        break;
      case kPhFallback: phase_fallback<kFull>(P, sm); break;
      case kPhHist2: phase_hist2(P, sm); break;
      case kPhInsert: phase_insert(P, sm); break;
      case kPhQuery: phase_query(P, sm); break;
      case kPhEmit: phase_emit<kFull, kB, kDgc>(P, sm, bar_epoch); break;
      case kPhRankHist: if constexpr (kFull) phase_rank_hist(P, sm); break;
      case kPhRankScan: if constexpr (kFull) phase_rank_scan(P, sm); break;
      case kPhRankScatter: if constexpr (kFull) phase_rank_scatter(P, sm); break;
      case kPhRankExact: if constexpr (kFull) phase_rank_exact(P, sm); break;
      case kPhFit: if constexpr (kFull) phase_fit(P, sm); break;
      case kPhFix: if constexpr (kFull) phase_fix<kDgc>(P, sm); break;
      case kPhExpand: if constexpr (kFull) phase_expand(P, sm); break;
      case kPhPush: phase_push(P, sm); break;
      case kPhSignal: if (!wait_flags<kB>(P, 0u, 0u)) return; break;
      case kPhDecode: phase_decode<kFull>(P, sm); break;
      case kPhCompact: phase_compact<kFull, kB>(P, sm, bar_epoch); break;
      case kPhSignal2: if (!wait_flags<kB>(P, kArenaFlagWords, 100u)) return; break;
      case kPhScatter: phase_scatter<kB>(P); break;
      default: break;
    }
    if (P.debug_times) {
      __syncthreads();
      if (threadIdx.x == 0) P.debug_times[((size_t)ph * gridDim.x + blockIdx.x) * 2 + 1] = globaltimer_ns();
    }
    prev_wait = is_wait;
    pending = true;
  }
}

}  // namespace

// ---------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------
// Two register budgets of the same kernel: <1> = 128 regs, one CTA per SM, up to 200 KB of
// filter staging; <2> = 64 regs, two CTAs per SM, up to 88 KB each.
static bool g_attr_set = false;

// ... x two feature sets: <.., false, ..> index-only (plain pairs / bloom), <.., true, ..> + value codecs (bf16 values
// included), run-length and Elias-Fano indices (has_rle) and the shared 'randomk' index; ... x the gradient type: <.., .., false> fp32 buckets,
// <.., .., true> bf16 buckets (a separate instantiation, so the fp32 kernels are compiled from exactly the code they had
// before bf16 existed)
static const void* kernel_for(int blocks_per_sm, bool full, bool bf16) {
  if (bf16) {
    if (blocks_per_sm >= 2) return full ? (const void*)dr_engine_kernel<2, true, true> : (const void*)dr_engine_kernel<2, false, true>;
    return full ? (const void*)dr_engine_kernel<1, true, true> : (const void*)dr_engine_kernel<1, false, true>;
  }
  if (blocks_per_sm >= 2) return full ? (const void*)dr_engine_kernel<2, true, false> : (const void*)dr_engine_kernel<2, false, false>;
  return full ? (const void*)dr_engine_kernel<1, true, false> : (const void*)dr_engine_kernel<1, false, false>;
}

// ... and the 'dgc' memory (momentum correction + factor masking): the full feature set only, fp32 or bf16 buckets, a
// separate instantiation again, so that the eight kernels above are compiled from unchanged code; with local gradient
// clipping one more (<.., true, .., true, true>), so that the 'dgc' kernels without it are unchanged too
static const void* dgc_kernel_for(int blocks_per_sm, bool bf16, bool clip) {
  if (clip) {
    if (blocks_per_sm >= 2) return bf16 ? (const void*)dr_engine_kernel<2, true, true, true, true> : (const void*)dr_engine_kernel<2, true, false, true, true>;
    return bf16 ? (const void*)dr_engine_kernel<1, true, true, true, true> : (const void*)dr_engine_kernel<1, true, false, true, true>;
  }
  if (blocks_per_sm >= 2) return bf16 ? (const void*)dr_engine_kernel<2, true, true, true> : (const void*)dr_engine_kernel<2, true, false, true>;
  return bf16 ? (const void*)dr_engine_kernel<1, true, true, true> : (const void*)dr_engine_kernel<1, true, false, true>;
}

static void ensure_attr() {
  if (!g_attr_set) {
    for (int bf16 = 0; bf16 < 2; ++bf16) {
      for (int full = 0; full < 2; ++full) {
        cudaFuncSetAttribute(kernel_for(1, full, bf16), cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(kernel_for(2, full, bf16), cudaFuncAttributeMaxDynamicSharedMemorySize, 88 * 1024);
      }
      for (int clip = 0; clip < 2; ++clip) {
        cudaFuncSetAttribute(dgc_kernel_for(1, bf16, clip), cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        cudaFuncSetAttribute(dgc_kernel_for(2, bf16, clip), cudaFuncAttributeMaxDynamicSharedMemorySize, 88 * 1024);
      }
    }
    g_attr_set = true;
  }
}

int engine_max_grid(int blocks_per_sm, int dyn_smem_bytes) {
  int dev = 0, sms = 0, occ = 0;
  ensure_attr();
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel_for(blocks_per_sm, true, false), kThreads, (size_t)dyn_smem_bytes);
  for (int v = 1; v < 4; ++v) {                  // the grid must be co-resident whichever variant a bucket launches
    int o = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kernel_for(blocks_per_sm, v & 1, v >> 1), kThreads, (size_t)dyn_smem_bytes);
    if (o < occ) occ = o;
  }
  for (int v = 0; v < 4; ++v) {
    int o = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, dgc_kernel_for(blocks_per_sm, v & 1, v >> 1), kThreads, (size_t)dyn_smem_bytes);
    if (o < occ) occ = o;
  }
  if (occ < 1) occ = 1;
  if (blocks_per_sm > 0 && blocks_per_sm < occ) occ = blocks_per_sm;
  return occ * sms;
}

cudaError_t engine_launch(const EngineParams& P, int grid, int blocks_per_sm, int dyn_smem_bytes, cudaStream_t stream) {
  ensure_attr();
  if (dyn_smem_bytes < 64 * 1024) return cudaErrorInvalidValue;     // TMA ring, candidate rings, emit / decode lists + slice stage
  if (!P.use_tma && dyn_smem_bytes < (int)(kCpStages * kStageBytes)) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(P.barrier, 0, 4 * sizeof(uint32_t), stream);  // grid barrier + the two tickets
  if (e != cudaSuccess) return e;
  void* args[] = {const_cast<EngineParams*>(&P)};
  count_launch(1);
  const bool full = P.n_poly != 0 || P.n_poly_tasks != 0 || P.has_rle != 0 || P.has_shared != 0 || P.has_bf16_values != 0;
  const void* kernel = P.mom != nullptr ? dgc_kernel_for(blocks_per_sm, P.bf16 != 0, P.clip_part != nullptr)
                                        : kernel_for(blocks_per_sm, full, P.bf16 != 0);
  return cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(kThreads), args, (size_t)dyn_smem_bytes, stream);
}

}  // namespace dr
