// Tile table, positive masks and the decode's (sender, tile) layout, shared by the engine kernel (engine.cu) and the
// P2 kernels launched between its phases (p2.cu): both must read the same tile, the same mask bits and the same
// dec_mask slot for a (sender, tile) pair.
#pragma once
#include "common.cuh"

namespace dr {

constexpr uint32_t kFullMask = 0xFFFFFFFFu;
constexpr uint32_t kGroupsPerTile = kTile / 32;       // 128 mask words per tile

struct Tile { uint32_t tensor, base, n, local0, single; };   // `single`: the tensor has exactly one tile

DR_D Tile load_tile(const TileInfo* tiles, uint32_t tile) {
  const uint4 q = __ldg(reinterpret_cast<const uint4*>(tiles) + tile);
  Tile t; t.tensor = q.x; t.base = q.y; t.n = q.z & 0xFFFFu; t.local0 = q.w; t.single = q.z >> 31;
  return t;
}

DR_D uint32_t warp_incl_scan(uint32_t v, uint32_t lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(kFullMask, v, o);
    if (lane >= (uint32_t)o) v += n;
  }
  return v;
}

// this lane's 4 bits of a tile's occupancy hint (4 hint words per tile, bit g <=> group g holds a selected element)
DR_D uint32_t hint_nibble(const uint32_t* hint, uint32_t tile_local, uint32_t lane) {
  if (!hint) return 0xFu;
  const uint32_t hw = __ldcg(hint + 4u * tile_local + (lane >> 3));
  return (hw >> ((lane & 7u) * 4u)) & 0xFu;
}

// this lane's 4 mask words of a tile, restricted to hinted groups that hold real elements
DR_D void load_masks(const uint32_t* masks, uint32_t tile, uint32_t nib, uint32_t n, uint32_t lane, uint32_t (&mm)[4]) {
  const uint4 m4 = __ldcg(reinterpret_cast<const uint4*>(masks + (size_t)tile * kGroupsPerTile) + lane);
  const uint32_t raw[4] = {m4.x, m4.y, m4.z, m4.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t g = 4u * lane + (uint32_t)j;
    mm[j] = (((nib >> j) & 1u) && g * 32u < n) ? raw[j] : 0u;
  }
}

// The decode's work items are the (sender other than me, tile of my decode span) pairs, sender-major: item i is tile
// i % span of the k-th sender other than me, k = i / span.
DR_D int other_sender(uint32_t k, int rank) { return (int)k + ((int)k >= rank ? 1 : 0); }

// dec_mask slot of (sender r, tile): senders are laid out back to back, each with `span` tiles of my slice
DR_D uint32_t* dec_mask_base(uint32_t* dec_mask, int r, uint32_t s_begin, uint32_t span) {
  // probe_segment / load_masks index with the GLOBAL tile id: shift the base so that base + tile*128 is the slot
  return dec_mask + ((size_t)r * span) * kGroupsPerTile - (size_t)s_begin * kGroupsPerTile;
}

// a sender ships values into a tile iff its prefix at the tile is below its n_sel and the tile starts at or before its
// cutoff (the largest shipped index); nothing else of the sender lands there
DR_D bool ships_into(uint32_t pre, uint32_t n_sel, uint32_t local0, uint32_t cutoff) {
  return pre < n_sel && local0 <= cutoff;
}

}  // namespace dr
