// P2 ('conflict_sets', paper Alg. 1) bloom policy of the fused engine (sm_90a): kernels launched between phase-range
// launches of dr_engine_kernel, so the engine kernels themselves are compiled from exactly the code they have without P2.
//
// Whether a positive is picked depends on every other positive of its tensor that shares a filter bit, so a receiver
// that decodes one slice of the tiles cannot redraw the pick.  The sender draws it once per tensor and ships it:
//   pos_prefix[n_tiles]      positives before each tile (capped at pos_cap)
//   pick[ceil(pos_cap / 32)] bit q set <=> the q-th positive (ascending) carries a value
// A receiver keeps the positive of in-tile positive rank j of tile t iff q = pos_prefix[t] + j < pos_cap and bit q of
// the pick is set; its value index is the tile prefix plus the kept positives before it in the tile, which is what
// the engine's leftmost decode computes on the thinned masks.
//
// Sender (p2_pick_kernel, between the query and emit phases; one CTA per P2 tensor, all tensors in flight at once):
//   positive ranks (tile counts -> prefix, masks -> element of every positive q < pos_cap) -> counting sort of the
//   (filter bit, positive) pairs over m_bits, a positive once per bit, members ascending -> sets ordered by
//   (size, bit) -> one warp draws (sequential by definition) -> pick into the slot, positive masks and tile counts
//   thinned to the pick.  Emit then runs unchanged: leftmost on the surviving set.
// p2_header_kernel (after emit): header words cutoff = 0xFFFFFFFF and n_pos = the positives (emit wrote the picks).
// Receiver (p2_thin_kernel, between the probe pass and the apply pass): every (sender, tile) of the probed masks is
// thinned with that sender's pick.
// The draw is bit-exact with codecs/bloom.py::conflict_sets_oracle on pos[:pos_cap] (tests/test_gpu_p2_fused.py).
#include "common.cuh"
#include "conflict_sets.cuh"
#include "ops.h"
#include "plan.h"
#include "tiles.cuh"

namespace dr {
namespace {

constexpr int kPickThreads = 1024;
constexpr int kPickWarps = kPickThreads / 32;
constexpr uint32_t kSizeCap = 32;                 // sets of >= kSizeCap members are ordered by an all-pairs rank pass
constexpr uint32_t kMaxHash = 16;

// Keep the positives of a tile whose rank q = q0 + (in-tile rank) is below pos_cap and set in `pick`; returns the
// kept count of the warp's tile (warp-uniform) and leaves the kept masks in mm.
template <typename PickFn>
DR_D uint32_t thin_tile(uint32_t (&mm)[4], uint32_t q0, uint32_t pos_cap, uint32_t lane, PickFn picked) {
  const uint32_t c = (uint32_t)(__popc(mm[0]) + __popc(mm[1]) + __popc(mm[2]) + __popc(mm[3]));
  uint32_t q = q0 + warp_incl_scan(c, lane) - c, kept = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t w = mm[j], keep = 0u;
    while (w) {
      const uint32_t b = (uint32_t)__ffs((int)w) - 1u;
      w &= w - 1u;
      if (q < pos_cap && picked(q)) keep |= 1u << b;
      ++q;
    }
    mm[j] = keep;
    kept += (uint32_t)__popc(keep);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(kFullMask, kept, o);
  return kept;
}

// filter bits of element x, each once (a positive enters a conflict set once); returns their number
DR_D uint32_t distinct_bits(uint32_t x, uint32_t seed, uint32_t n_hash, uint32_t m_bits, uint32_t (&bits)[kMaxHash]) {
  const HashAB h = hash_ab(x, seed);
  uint32_t n = 0, v = h.a;
  for (uint32_t j = 0; j < n_hash; ++j, v += h.b) {
    const uint32_t b = mulhi32(v, m_bits);
    bool dup = false;
    for (uint32_t i = 0; i < n; ++i) dup |= bits[i] == b;
    if (!dup) bits[n++] = b;
  }
  return n;
}

// inclusive block scan of one value per thread (1024 threads); returns the inclusive prefix, total = block sum.
// s_warp: kPickWarps + 1 words of shared memory
DR_D uint32_t block_scan_incl(uint32_t v, uint32_t* s_warp, uint32_t& total) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t incl = warp_incl_scan(v, lane);
  __syncthreads();
  if (lane == 31u) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const uint32_t w = s_warp[lane];
    const uint32_t wi = warp_incl_scan(w, lane);
    s_warp[lane] = wi - w;
    if (lane == 31u) s_warp[kPickWarps] = wi;
  }
  __syncthreads();
  total = s_warp[kPickWarps];
  const uint32_t r = s_warp[warp] + incl;
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kPickThreads) p2_pick_kernel(const P2Args A) {
  extern __shared__ uint32_t chosen[];                       // one bit per positive rank, ceil(pos_cap / 32) words
  __shared__ uint32_t s_warp[kPickWarps + 1];
  __shared__ uint32_t s_cls[kPickWarps][kSizeCap + 1];       // per (warp range, size class): count, then placement cursor
  __shared__ uint32_t s_misc[4];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const P2Entry E = A.entries[blockIdx.x];
  const TensorDesc* td = A.tensors + E.tensor;
  const uint32_t tile_begin = __ldg(&td->tile_begin), n_tiles = __ldg(&td->n_tiles);
  const uint32_t m_bits = __ldg(&td->m_bits), n_hash = __ldg(&td->n_hash), pos_cap = __ldg(&td->pos_cap);
  const uint32_t oh = __ldg(&td->off_hint);
  const uint32_t* hint = oh ? A.slot + oh : nullptr;
  uint32_t* pos_prefix = A.slot + __ldg(&td->off_pos_prefix);
  uint32_t* pick = A.slot + __ldg(&td->off_pick);
  uint32_t* pos_idx = A.scratch + E.pos_idx;
  uint32_t* set_off = A.scratch + E.set_off;
  uint32_t* cursor = A.scratch + E.cursor;
  uint32_t* members = A.scratch + E.members;
  uint32_t* ord = A.scratch + E.ord;
  uint32_t* last = A.scratch + E.last;
  uint32_t* tmp = A.scratch + E.tmp;
  const uint32_t n_words = (pos_cap + 31u) >> 5;
  for (uint32_t i = tid; i < m_bits; i += kPickThreads) cursor[i] = 0u;
  for (uint32_t i = tid; i < n_words; i += kPickThreads) chosen[i] = 0u;

  // ---- (1) positives before every tile (capped) and in the tensor
  uint32_t carry = 0;
  for (uint32_t c0 = 0; c0 < n_tiles; c0 += kPickThreads) {
    const uint32_t i = c0 + tid;
    const uint32_t v = i < n_tiles ? __ldcg(A.tile_count + tile_begin + i) : 0u;
    uint32_t tot;
    const uint32_t incl = block_scan_incl(v, s_warp, tot);
    if (i < n_tiles) pos_prefix[i] = min(carry + incl - v, pos_cap);
    carry += tot;
  }
  const uint32_t n_pos = carry, np = min(n_pos, pos_cap);
  __syncthreads();
  // ---- (2) element of every positive rank q < pos_cap: one warp per tile
  for (uint32_t t = warp; t < n_tiles; t += kPickWarps) {
    const uint32_t pre = pos_prefix[t];
    if (pre >= pos_cap) continue;                                            // warp-uniform
    const Tile ti = load_tile(A.tiles, tile_begin + t);
    uint32_t mm[4];
    load_masks(A.pos_mask, tile_begin + t, hint_nibble(hint, t, lane), ti.n, lane, mm);
    const uint32_t c = (uint32_t)(__popc(mm[0]) + __popc(mm[1]) + __popc(mm[2]) + __popc(mm[3]));
    uint32_t q = pre + warp_incl_scan(c, lane) - c;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      for (uint32_t w = mm[j]; w; w &= w - 1u, ++q)
        if (q < pos_cap) pos_idx[q] = ti.local0 + (4u * lane + (uint32_t)j) * 32u + (uint32_t)(__ffs((int)w) - 1);
    }
  }
  __syncthreads();
  // ---- (3) members per filter bit, (4) their offsets in bit order, (5) the members, (6) ascending inside a set
  for (uint32_t q = tid; q < np; q += kPickThreads) {
    uint32_t bits[kMaxHash];
    const uint32_t n = distinct_bits(__ldcg(pos_idx + q), A.seed, n_hash, m_bits, bits);
    for (uint32_t i = 0; i < n; ++i) atomicAdd(cursor + bits[i], 1u);
  }
  __syncthreads();
  carry = 0;
  const uint32_t R = ((m_bits + 32u * kPickWarps - 1u) / (32u * kPickWarps)) * 32u;   // bits per warp range (step 7)
  for (uint32_t i = tid; i < (uint32_t)kPickWarps * (kSizeCap + 1u); i += kPickThreads) (&s_cls[0][0])[i] = 0u;
  for (uint32_t c0 = 0; c0 < m_bits; c0 += kPickThreads) {
    const uint32_t i = c0 + tid;
    const uint32_t v = i < m_bits ? __ldcg(cursor + i) : 0u;
    uint32_t tot;
    const uint32_t incl = block_scan_incl(v, s_warp, tot);
    if (i < m_bits) {
      set_off[i] = carry + incl - v;
      cursor[i] = carry + incl - v;
      if (v) atomicAdd(&s_cls[i / R][min(v, kSizeCap)], 1u);
    }
    carry += tot;
  }
  if (tid == 0) set_off[m_bits] = carry;
  __syncthreads();
  for (uint32_t q = tid; q < np; q += kPickThreads) {
    uint32_t bits[kMaxHash];
    const uint32_t n = distinct_bits(__ldcg(pos_idx + q), A.seed, n_hash, m_bits, bits);
    for (uint32_t i = 0; i < n; ++i) members[atomicAdd(cursor + bits[i], 1u)] = q;
  }
  __syncthreads();
  for (uint32_t b = tid; b < m_bits; b += kPickThreads) {
    const uint32_t o = __ldcg(set_off + b), e = __ldcg(set_off + b + 1);
    for (uint32_t i = o + 1; i < e; ++i) {                                   // sets are short: insertion sort
      const uint32_t x = members[i];
      uint32_t j = i;
      for (; j > o && members[j - 1] > x; --j) members[j] = members[j - 1];
      members[j] = x;
    }
  }
  // ---- (7) visit order (size, bit): a stable counting sort by size class over the warps' bit ranges, in bit order
  __syncthreads();
  if (warp == 0) {
    uint32_t base = 0;
    for (uint32_t cls = 1; cls <= kSizeCap; ++cls) {
      const uint32_t v = s_cls[lane][cls];
      const uint32_t incl = warp_incl_scan(v, lane);
      s_cls[lane][cls] = base + incl - v;
      if (cls == kSizeCap && lane == 0) s_misc[1] = base;                  // first large set
      base += __shfl_sync(kFullMask, incl, 31);
    }
    if (lane == 0) s_misc[0] = base;                                        // number of sets
  }
  __syncthreads();
  const uint32_t n_sets = s_misc[0], ov_begin = s_misc[1];
  {
    const uint32_t lo = warp * R, hi = min(lo + R, m_bits);
    const uint32_t lt = (1u << lane) - 1u;
    for (uint32_t b0 = lo; b0 < hi; b0 += 32u) {
      const uint32_t b = b0 + lane;
      const uint32_t s = b < hi ? __ldcg(set_off + b + 1) - __ldcg(set_off + b) : 0u;
      const uint32_t cls = s ? min(s, kSizeCap) : 0xFFFFFFFFu;
      const uint32_t peers = __match_any_sync(kFullMask, cls);
      if (s) ord[s_cls[warp][cls] + (uint32_t)__popc(peers & lt)] = b;
      __syncwarp();
      if (s && (peers & lt) == 0u) s_cls[warp][cls] += (uint32_t)__popc(peers);
      __syncwarp();
    }
  }
  __syncthreads();
  const uint32_t n_ov = n_sets - ov_begin;                                  // large sets, in bit order so far
  if (n_ov > 1u) {
    for (uint32_t i = tid; i < n_ov; i += kPickThreads) {
      const uint32_t b = __ldcg(ord + ov_begin + i);
      const uint64_t key = ((uint64_t)(__ldcg(set_off + b + 1) - __ldcg(set_off + b)) << 32) | b;
      uint32_t r = 0;
      for (uint32_t j = 0; j < n_ov; ++j) {
        const uint32_t bj = __ldcg(ord + ov_begin + j);
        r += (((uint64_t)(__ldcg(set_off + bj + 1) - __ldcg(set_off + bj)) << 32) | bj) < key ? 1u : 0u;
      }
      tmp[r] = b;
    }
    __syncthreads();
    for (uint32_t i = tid; i < n_ov; i += kPickThreads) ord[ov_begin + i] = __ldcg(tmp + i);
  }
  __syncthreads();
  for (uint32_t i = tid; i < n_sets; i += kPickThreads) {
    const uint32_t b = __ldcg(ord + i);
    last[i] = __ldcg(set_off + b + 1) - __ldcg(set_off + b);                 // untouched: the alive count is the size
  }
  __syncthreads();
  // ---- (8) the draw (conflict_sets.cuh), one warp, sets in visit order through `ord`
  if (warp == 0) {
    conflict_sets_draw(
        [&](uint32_t i) { const uint32_t b = __ldcg(ord + i), off = __ldcg(set_off + b); return make_uint2(off, __ldcg(set_off + b + 1) - off); },
        [&](uint32_t j) { return __ldcg(members + j); }, last, n_sets, np, __ldg(&td->k),
        policy_seed(A.epoch, __ldg(&td->salt)), chosen);
  }
  __syncthreads();
  // ---- (9) ship the pick; thin my positive masks and tile counts to it (emit then is leftmost on the picked set)
  for (uint32_t i = tid; i < n_words; i += kPickThreads) pick[i] = chosen[i];
  for (uint32_t t = warp; t < n_tiles; t += kPickWarps) {
    const uint32_t tile = tile_begin + t;
    const Tile ti = load_tile(A.tiles, tile);
    uint32_t mm[4];
    load_masks(A.pos_mask, tile, hint_nibble(hint, t, lane), ti.n, lane, mm);
    const uint32_t kept = thin_tile(mm, pos_prefix[t], pos_cap, lane,
                                    [&](uint32_t q) { return ((chosen[q >> 5] >> (q & 31u)) & 1u) != 0u; });
    reinterpret_cast<uint4*>(A.pos_mask + (size_t)tile * kGroupsPerTile)[lane] = make_uint4(mm[0], mm[1], mm[2], mm[3]);
    if (lane == 0) A.tile_count[tile] = kept;
  }
  if (tid == 0) A.scratch[E.misc] = n_pos;
}

// after emit: the header of a P2 tensor carries no cutoff (the pick says which positives are shipped) and the number of
// positives (emit wrote the number of picks there)
__global__ void p2_header_kernel(const P2Args A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n_entries) return;
  const P2Entry E = A.entries[i];
  DynHeader* dyn = reinterpret_cast<DynHeader*>(A.slot + kSlotHeaderWords) + E.tensor;
  dyn->cutoff = 0xFFFFFFFFu;
  dyn->n_pos = __ldcg(A.scratch + E.misc);
}

// receiver: one warp per (sender other than me, tile of my decode span); P2 tensors' probed masks are thinned with the
// sender's pick — tiles the sender ships nothing into were not probed and are skipped, as the apply pass skips them
__global__ void __launch_bounds__(256) p2_thin_kernel(const P2Thin T) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t n_items = (uint64_t)(T.world - 1) * T.span;
  const uint64_t n_warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t it = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); it < n_items; it += n_warps) {
    const uint32_t k = (uint32_t)(it / T.span);
    const int r = other_sender(k, T.rank);
    const uint32_t tl = T.s_begin + (uint32_t)(it - (uint64_t)k * T.span);
    const Tile ti = load_tile(T.tiles, tl);
    const TensorDesc* td = T.tensors + ti.tensor;
    const uint32_t pos_cap = __ldg(&td->pos_cap);
    if (pos_cap == 0u || __ldg(&td->mode) != (uint32_t)kModeBloom) continue;
    const uint32_t* slot = T.slots + (size_t)r * T.slot_words;
    const DynHeader* dyn = reinterpret_cast<const DynHeader*>(slot + kSlotHeaderWords) + ti.tensor;
    const uint32_t n_sel = __ldcg(&dyn->n_sel), cutoff = __ldcg(&dyn->cutoff);
    const uint32_t tile_local = tl - __ldg(&td->tile_begin);
    const uint32_t pre = __ldcg(slot + __ldg(&td->off_prefix) + tile_local);
    if (!ships_into(pre, n_sel, ti.local0, cutoff)) continue;
    const uint32_t oh = __ldg(&td->off_hint);
    uint32_t* masks = dec_mask_base(T.dec_mask, r, T.s_begin, T.span);
    uint32_t mm[4];
    load_masks(masks, tl, hint_nibble(oh ? slot + oh : nullptr, tile_local, lane), ti.n, lane, mm);
    const uint32_t* pick = slot + __ldg(&td->off_pick);
    thin_tile(mm, __ldcg(slot + __ldg(&td->off_pos_prefix) + tile_local), pos_cap, lane,
              [&](uint32_t q) { return ((__ldcg(pick + (q >> 5)) >> (q & 31u)) & 1u) != 0u; });
    reinterpret_cast<uint4*>(masks + (size_t)tl * kGroupsPerTile)[lane] = make_uint4(mm[0], mm[1], mm[2], mm[3]);
  }
}

}  // namespace

cudaError_t p2_prepare() {
  return cudaFuncSetAttribute(p2_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kP2MaxSmemBytes);
}

cudaError_t p2_pick_launch(const P2Args& A, uint32_t max_pos_cap, cudaStream_t st) {
  if (A.n_entries == 0) return cudaSuccess;
  const size_t smem = (size_t)((max_pos_cap + 31u) >> 5) * 4u;
  if (smem > kP2MaxSmemBytes) return cudaErrorInvalidValue;
  count_launch(1);
  p2_pick_kernel<<<A.n_entries, kPickThreads, smem, st>>>(A);
  return cudaGetLastError();
}

cudaError_t p2_header_launch(const P2Args& A, cudaStream_t st) {
  if (A.n_entries == 0) return cudaSuccess;
  count_launch(1);
  p2_header_kernel<<<(A.n_entries + 127u) / 128u, 128, 0, st>>>(A);
  return cudaGetLastError();
}

cudaError_t p2_thin_launch(const P2Thin& T, cudaStream_t st) {
  if (T.world < 2 || T.span == 0) return cudaSuccess;
  const uint64_t warps = (uint64_t)(T.world - 1) * T.span;
  const uint64_t want = (warps + 7u) / 8u, cap = (uint64_t)sm_count() * 8u;
  const int grid = (int)(want < cap ? want : cap);
  count_launch(1);
  p2_thin_kernel<<<grid, 256, 0, st>>>(T);
  return cudaGetLastError();
}

}  // namespace dr
