// P2 / conflict sets (paper Alg. 1; reference tensorflow/policies.hpp:43-146): the draw, shared by the per-tensor kernel
// (ops.cu::conflict_sets_pick_kernel, sets in visit order) and the fused engine's sender stage
// (p2.cu::p2_pick_kernel, sets reached through a visit-order table).  Normative: codecs/bloom.py::conflict_sets_oracle.
#pragma once
#include "common.cuh"

namespace dr {

// The draw is sequential BY DEFINITION (the r-th pick's random number and every set's "untouched since my last visit"
// test depend on all earlier picks), so ONE warp walks the conflict sets in (size, bit position) order:
//   * the chosen flags of the positives are a bitmap indexed by positive rank (`chosen`, zeroed by the caller; shared
//     memory in both callers);
//   * 32 sets are fetched at a time (offset, size, last-visit count, first 4 member ranks per lane) and then visited one
//     by one with warp shuffles — no memory latency on the sequential path for sets of <= 4 members (the vast majority:
//     a set is the list of positives hashing to one filter bit);
//   * a set erases its chosen members implicitly (alive = not chosen); `last[i]` holds the alive count of set i at its
//     previous visit (the set's size before the first), exactly the `cs.size() == before` test of the reference;
//   * a pass without a pick falls back to the leftmost unchosen positives (the reference would spin forever).
// set_of(i) -> {first member, size} of the i-th set in visit order; member(j) -> rank of the j-th member entry.
// Picks min(K, n_pos) positives.  Called by all 32 lanes of one warp.
template <typename SetFn, typename MemberFn>
DR_D void conflict_sets_draw(SetFn set_of, MemberFn member, uint32_t* last, uint32_t n_sets, uint32_t n_pos, uint32_t K,
                             uint32_t pseed, uint32_t* chosen) {
  const uint32_t lane = threadIdx.x & 31u;
  auto is_chosen = [&](uint32_t r) { return (chosen[r >> 5] >> (r & 31u)) & 1u; };
  uint32_t left = min(K, n_pos), draw = 0;
  while (left > 0) {
    bool picked = false;
    for (uint32_t base = 0; base < n_sets && left > 0; base += 32u) {
      const uint32_t i = base + lane;
      const bool valid = i < n_sets;
      const uint2 s = valid ? set_of(i) : make_uint2(0u, 0u);
      const uint32_t off = s.x, sz = s.y;
      uint32_t lc = valid ? last[i] : 0u;
      uint32_t m[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) m[j] = ((uint32_t)j < sz) ? member(off + j) : 0u;
      const uint32_t n_here = min(32u, n_sets - base);
      for (uint32_t sidx = 0; sidx < n_here && left > 0; ++sidx) {        // warp-uniform, sequential by definition
        const uint32_t ssz = __shfl_sync(0xFFFFFFFFu, sz, sidx), soff = __shfl_sync(0xFFFFFFFFu, off, sidx);
        const uint32_t slc = __shfl_sync(0xFFFFFFFFu, lc, sidx);
        uint32_t a[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) a[j] = __shfl_sync(0xFFFFFFFFu, m[j], sidx);
        uint32_t cnt = 0;
        if (ssz <= 4u) {
#pragma unroll
          for (int j = 0; j < 4; ++j) cnt += ((uint32_t)j < ssz && !is_chosen(a[j])) ? 1u : 0u;
        } else {
          for (uint32_t t = lane; t < ssz; t += 32u) cnt += is_chosen(member(soff + t)) ? 0u : 1u;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, o);
        }
        uint32_t nl = cnt;
        if (cnt == slc && cnt > 0u) {                                       // untouched since my last visit: draw one member
          uint32_t r = policy_hash(draw, pseed) % cnt;
          ++draw;
          uint32_t pick = 0;
          if (ssz <= 4u) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if ((uint32_t)j < ssz && !is_chosen(a[j])) { if (r == 0u) pick = a[j]; --r; }
            }
          } else {
            for (uint32_t t = 0; t < ssz; ++t) {                            // every lane walks the (rare) long set identically
              const uint32_t x = member(soff + t);
              if (!is_chosen(x)) { if (r == 0u) { pick = x; break; } --r; }
            }
          }
          __syncwarp();
          if (lane == 0) chosen[pick >> 5] |= 1u << (pick & 31u);
          __syncwarp();
          --left;
          picked = true;
          nl = cnt - 1u;
        }
        if (lane == sidx) lc = nl;
      }
      if (valid) last[i] = lc;
    }
    if (!picked && left > 0) {                                               // termination fallback: leftmost unchosen positives
      for (uint32_t r = 0; r < n_pos && left > 0; ++r) {
        if (!is_chosen(r)) {
          __syncwarp();
          if (lane == 0) chosen[r >> 5] |= 1u << (r & 31u);
          __syncwarp();
          --left;
        }
      }
    }
  }
  __syncwarp();
}

}  // namespace dr
