// Bucket plan + engine parameter block shared by host (binding.cpp) and device
// (engine.cu).  The plan is built in Python (parallel/plan.py) and uploaded as
// int32 tensors; field order here is normative for that builder.
//
// Parity notes (reference = hangxu0304/DeepReduce):
//  * a TensorDesc carries what the reference recomputes per call from `params`: K = max(1, int(d * ratio))
//    (GRACE top-k), bloom m / hash count (pytorch/deepreduce.py:495-500,511-512), the 1000-element bypass
//    (:68,84,114), polyfit degree (:385), QSGD quantum_num / bucket 512 (:857-858);
//  * a slot replaces the per-tensor wire tuples `(vals, packed bit array)` (:529), `(coefficients, idxs)` (:413-414)
//    and `(vals', idxs', mapping)` (:267) — all tensors of a bucket in one buffer with static offsets, so the
//    size all_gather + pad-to-max of the GRACE communicator (tensors_size_are_same=False, :59,108) disappears;
//  * DynHeader.n_sel/cutoff is policy `leftmost` / `p0` (:479-492) expressed so the receiver needs no sort.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace dr {

constexpr int kMaxWorld = 16;
constexpr int kTile = 4096;           // elements per tile (wire-visible: per-tile prefix table)
constexpr uint32_t kDefaultSeed = 0x9747B28Cu;

enum TensorMode : uint32_t {
  kModeRaw = 0,     // plain (value, index) pairs — small-tensor bypass / plain top-k
  kModeBloom = 1,   // bloom-filter index codec, fp32 values
  kModeRle = 2,     // lossless tile-local run coding: u16 count per 4096-element tile (off_prefix) + the cumulative
                    // zero-run offset of every selected element inside its tile, 12 bits each, LSB-first (off_idx)
  kModeShared = 3,  // 'randomk': the index set is a seeded draw every rank computes itself (selection rule below), so
                    // only the values travel; off_prefix is sender-local scratch (per-tile exclusive prefix)
  kModeEf = 4,      // lossless tile-local Elias-Fano (spec.py ef_layout): kModeRle's u16 count per tile (off_prefix), the
                    // L low bits of every entry's in-tile offset (off_idx) and its unary high part (off_hi), L = ef_low_bits
};

enum ValueMode : uint32_t {  // TensorDesc::vmode: how a tensor's values travel in the slot (parallel/plan.py VMODE_*)
  kVmodeFp32 = 0,     // fp32 values
  kVmodePolyfit = 1,  // piece-wise Gram-polynomial fit + rank map
  kVmodeQsgd = 2,     // bucketed QSGD (int8 levels, or int16 when rank_u32 is set: quantum_num >= 128)
  kVmodeDexp = 3,     // double-exponential fit of each sign run + rank map
  kVmodeBf16 = 4,     // bf16 values: the p-th value's bits in half p % 2 (low half first) of word off_vals + p / 2,
                      // rounded by emit, which also writes the residual (no scratch, no rank / fit / fix phase)
  kVmodeSign = 5,     // scaled sign (sign_values.cuh): per 512-value bucket b one fp32 scale mu_b at off_coef + b, then
                      // one bit per value at off_rankmap, LSB first (value p is bit p % 32 of word p / 32, 1 <=> v < 0);
                      // decodes to bit ? -mu_b : +mu_b.  off_vals / off_selidx are sender-local scratch (fix phase)
  kVmodeFp8 = 6,      // E4M3 values (fp8_values.cuh), a scale byte per 32-value block: the scale bytes at off_coef, then
                      // the element bytes at off_rankmap, each packed four per word (byte p in bits 8 (p % 4) of word
                      // p / 4).  off_vals / off_selidx are sender-local scratch (fix phase)
};

// kPolicyP2 ('conflict_sets', opt-in): the sender draws the pick over its positives and ships it as a bitmask (p2.cu);
// the engine kernel itself treats it as leftmost on the thinned positives
enum Policy : int { kPolicyLeftmost = 0, kPolicyRandom = 1, kPolicyP0 = 2, kPolicyP2 = 3 };

// 32 x uint32 per tensor (kDescWords)
struct TensorDesc {
  uint32_t elem_off;     // offset into the flat grad/residual buffers (elements, multiple of 4)
  uint32_t numel;        // d_i
  uint32_t k;            // K_i = max(1, int(d_i * ratio)), <= numel
  uint32_t tile_begin;   // first global tile id
  uint32_t n_tiles;      // ceil(numel / kTile)
  uint32_t mode;         // TensorMode
  uint32_t m_bits;       // bloom bits (multiple of 32)
  uint32_t n_hash;       // bloom hash count
  uint32_t off_vals;     // payload word offsets (within a slot)
  uint32_t off_filter;
  uint32_t off_prefix;   // per-tile exclusive prefix of selected counts (n_tiles words)
  uint32_t off_idx;      // raw mode: indices
  uint32_t val_cap;      // capacity of the value region (K, or K+slack for p0)
  uint32_t salt;         // tensor id (policy seeds)
  uint32_t n_filter_words;
  uint32_t off_hint;     // 0 = none; else 4 words per tile: bit g set <=> 32-element group g holds a selected element
  // ---- value codec ('both': bloom index + polynomial fit of the values) ----
  uint32_t vmode;        // ValueMode
  uint32_t off_coef;     // [kMaxSeg * (deg+1)] (kVmodeDexp: [kDexpCoefWords]) float coefficients, then {num_pos, n}
  uint32_t off_rankmap;  // rank of the p-th shipped value in the descending sort (u16 if val_cap <= 65536 else u32)
  uint32_t off_selidx;   // scratch (not shipped): element index of the p-th shipped value
  uint32_t off_sorted;   // scratch (not shipped): values in descending order
  uint32_t poly_degree;
  uint32_t rank_u32;     // 1: rank map entries are 32-bit
  uint32_t poly_off;     // offset of this tensor's values in the engine's per-value scratch arrays
  uint32_t poly_ord;     // ordinal among the ranked (kVmodePolyfit, kVmodeDexp) tensors (selects its bin table)
  uint32_t fixed_thr;    // != 0: 'threshold' sparsifier — select key >= fixed_thr (31-bit |x| pattern), no radix select, variable K
  uint32_t shared_lb;    // kModeShared: static candidate bound on the hash key (multiple of 512; replaces the history bound)
  // ---- P2 ('conflict_sets') bloom tensors; 0 otherwise ----
  uint32_t pos_cap;        // the pick runs over the first min(n_pos, pos_cap) positives
  uint32_t off_pos_prefix; // [n_tiles] positives before each tile, capped at pos_cap
  uint32_t off_pick;       // [ceil(pos_cap / 32)] pick bitmask: bit q <=> the q-th positive carries a value
  // ---- kModeEf tensors; 0 otherwise ----
  uint32_t ef_low_bits;    // L: low bits per entry (0..12); the high stream gives each tile kTile >> L bits + its count
  uint32_t off_hi;         // [ceil((val_cap + n_tiles * (kTile >> L)) / 32)] high stream
};
static_assert(sizeof(TensorDesc) == 128, "TensorDesc must be 32 words");
constexpr int kDescWords = 32;
constexpr int kRankBins = 8192;        // 'both': counting-sort bins = sign + 8 exponent + 4 mantissa bits
constexpr int kMaxSeg = 22;            // codecs/polyfit.py MAX_SEGMENTS
constexpr int kMaxDeg = 7;
constexpr uint32_t kDexpCoefWords = 8;  // kVmodeDexp: {a, b, p, q} of the positive run, then of the non-positive run

// payload slot layout (uint32 words):
//   [0..8)                      : magic, epoch, n_tensors, payload_words, rank, 0,0,0
//   [8 .. 8+4*n_tensors)        : DynHeader per tensor
//   then per-tensor regions at the TensorDesc offsets
constexpr uint32_t kSlotHeaderWords = 8;
constexpr uint32_t kDynWords = 4;
constexpr uint32_t kMagic = 0xD33B2000u;
struct DynHeader {
  uint32_t n_sel;      // number of values actually shipped
  uint32_t cutoff;     // largest selected index (leftmost); 0xFFFFFFFF = no cut
  uint32_t thr_bits;   // |g| threshold bits chosen by the select
  uint32_t n_pos;      // filter positives in the universe (diagnostics / FP count)
};

// per-tensor select state (persists across steps; thr history drives the
// pass-1 lower bound): 8 words
struct SelState {
  uint32_t bin1, krem1, bin2, krem2;
  uint32_t thr;         // selection threshold as a key lower bound: (T22 << 9), T22 = 22-bit prefix
  uint32_t n_ge;        // diagnostics: keys in the threshold bin
  uint32_t done_epoch;  // == epoch when the accumulate phase already finished the select (one-tile tensors)
  uint32_t prev_thr;    // thr of the previous step (0 = none)
};

constexpr int kHistBins = 2048;
constexpr int kNumHist = 3;
// hist arrays: [3][n_tensors][kHistBins]  (pass1, pass1-fallback, pass2);  hist_total: [3][n_tensors] merge tickets

// arena layout per rank (uint32 words): [flags: 64][stage-2 flags: 64][slots: 2 * world * slot_words]
//                                       [stage-2 slots: 2 * world * s2_words]
constexpr uint32_t kArenaFlagWords = 64;
constexpr uint32_t kArenaHdrWords = 128;

// Selection rule (normative, mirrored by parallel/engine.py::select_topk_oracle):
//   key  = |x| bit pattern (31 bits);  T22 = (key of the K-th largest |x|) >> 9
//   selected  <=>  (key >> 9) >= max(T22, 1)
// i.e. the threshold is resolved to 22 bits (8 exponent + 14 mantissa): at least K elements are
// selected, plus the few that share the threshold's 22-bit prefix; exact zeros are never selected.
//
// kModeShared ('randomk', mirrored by parallel/engine.py::select_randomk_oracle): the key of the in-tensor index i is
//   key(i) = (0xFFFFFFFF - policy_hash(i, policy_seed(epoch, salt))) >> 1      (smallest hash -> largest key)
// and the same 22-bit rule applies to it: a superset of the K smallest hashes, plus ~numel / 2^22 elements sharing the
// threshold's prefix.  The set depends on (numel, K, epoch, salt) only, so every rank computes the same one.
enum Phase : int {
  kPhAccum = 0,      // r = beta*r + gamma*g (dgc: [g = f*g,] d = g [+ wd*w], u = m*u + d, r = r + (nesterov ? d + m*u : u)) ; dense grad <- 0 ; zero slot ; candidate lists (keys >= history bound) ; hist digit 1
  kPhFallback = 1,   // (only if some bound was unsafe) digit 1 redone without the bound, candidate lists rebuilt in full
  kPhHist2 = 2,      // digit 2 of the candidate keys in the threshold bin
  kPhInsert = 3,     // selected candidates -> bloom filter + occupancy hint (bloom) / positive masks (raw, rle)
  kPhQuery = 4,      // hinted 32-element groups of the universe vs my filter -> positive masks + per-tile counts
  kPhEmit = 5,       // ordered compaction from the masks + value gather + residual zeroing (+ dense scatter when W == 1)
  // 'both' (bloom index + polynomial value fit): exact descending rank of every shipped value by a
  // counting sort on 13 key bits + an all-pairs count inside each bin, then the fit
  kPhRankHist = 6,   // bin populations
  kPhRankScan = 7,   // per-tensor exclusive prefix over the bins
  kPhRankScatter = 8,// group the values by bin
  kPhRankExact = 9,  // exact rank inside the bin -> rank map + sorted values + num_pos
  kPhFit = 10,       // per-segment Gram-polynomial least squares on the sorted values ('dexp': per sign run, fp64)
  kPhFix = 11,       // residual <- value - fitted value (error feedback sees the fit error)
  kPhPush = 12,      // copy the finished slot into every peer's arena (P2P stores over NVLink); the CTA that finishes last
                     // (ticket) releases the flags — no grid barrier between the copy and the signal
  kPhSignal = 13,    // acquire peers' flags
  kPhExpand = 14,    // 'both': evaluate every rank's fitted curve once (dense), decode then only gathers
  kPhDecode = 15,    // membership test on every rank's filter, rank->value, sum, scale, dense write
                     // (sharded mode, W>1: only this rank's 1/W slice of the tiles, for all W senders)
  // sharded decode (W > 1): the decoded slice is exchanged as an exact (index, value) list — decode work per rank
  // no longer grows with W; NVLink carries the extra ~2 MB/rank
  kPhCompact = 16,   // compact the non-zeros of my decoded slice (same CTA that decoded the tile) and store them straight
                     // into every peer's stage-2 slot; last CTA (ticket) writes the count and releases the second flag set
  kPhPush2 = 17,     // (folded into kPhCompact; kept so phase numbers stay stable)
  kPhSignal2 = 18,   // acquire peers' second flags
  kPhScatter = 19,   // write every peer's slice list into the dense gradient
  kPhEnd = 20
};

// phase classes with their own tile -> CTA partition (the phases have different cost profiles, and the SMs of the two dies
// run the memory-heavy phases at different speeds): accumulate / fallback / hist2, insert, query, emit
enum Part : int { kPartAccum = 0, kPartInsert = 1, kPartQuery = 2, kPartEmit = 3, kNumParts = 4 };

// per-tile table (uint4): {tensor id, element offset of the tile in the flat buffers, valid count, offset inside tensor}
struct TileInfo { uint32_t tensor, base, n, local0; };

struct EngineParams {
  const TensorDesc* tensors;
  const TileInfo* tiles;         // [n_tiles]
  const uint32_t* cost_prefix;   // [n_tiles + 1] cumulative cost of the tiles (host plan: elements + per-tensor overheads); the
                                 // streaming phases cut the tile sequence into equal-COST ranges (nullptr: equal counts)
  uint32_t n_tensors;
  uint32_t n_tiles;
  uint32_t slot_words;           // words reserved per slot
  uint32_t payload_words;        // words actually used (pushed)
  float* grad;                   // in: local dense grad; out: aggregated dense grad
  float* resid;                  // residual accumulator (persists across steps)
  uint32_t* hist;                // [3][n_tensors][kHistBins]
  uint32_t* hist_total;          // [3][n_tensors] merge tickets (#tiles whose histogram was merged)
  SelState* sel;                 // [n_tensors]
  uint32_t* tile_count;          // [n_tiles] selected/positive count of every tile (insert / query phase)
  uint32_t* pos_mask;            // [n_tiles * 128] positives of this rank, one bit per element, one word per 32-element group
  uint32_t* dec_mask;            // [n_tiles * 128] decode scratch: positives of the sender being decoded
  uint2* cand;                   // [n_tiles * 4096] candidates {key = |x| pattern >= the history bound, in-tile element offset},
                                 // 256 slots per (tile, warp) at a fixed place
  uint32_t* cand_cnt;            // [n_tiles * 16] candidates per (tile, warp)
  uint32_t* barrier;             // [0] grid barrier counter, [1] push ticket, [2] stage-2 ticket (zeroed by the host per
                                 // launch); [8] number of tensors whose history bound hid the threshold (device-managed)
  uint32_t* status;              // [8] error / watchdog words (device-local)
  uint32_t* arena[kMaxWorld];    // peer-mapped arena base of every rank (arena[rank] is local)
  int rank;
  int world;
  uint32_t epoch;                // 1-based step counter; slot parity = epoch & 1
  float beta, gamma, scale;
  uint32_t seed;
  int policy;
  int use_history;               // pass-1 lower bound from prev_thr
  int phase_begin, phase_end;
  uint32_t spin_limit;           // watchdog for flag / look-back / barrier spins
  uint32_t filter_smem_words;    // capacity of the dynamic-SMEM buffer (filter staging / TMA tile ring)
  int use_tma;                   // streaming phases fetch tiles with cp.async.bulk into an SMEM ring
  uint32_t hist_shift;           // history bound = prev_thr - (1 << hist_shift): 23 -> x0.5, 22 -> ~x0.7
  const uint32_t* poly_tensors;  // ids of the ranked (kVmodePolyfit, kVmodeDexp) tensors (largest K first)
  uint32_t n_poly;
  const uint32_t* poly_tasks;    // per-value tasks: {tensor id, first value of a 512-value chunk}
  uint32_t n_poly_tasks;
  uint32_t* poly_bins;           // [n_poly][2][kRankBins]: bin counts | bin starts/cursors (zeroed in decode)
  float* bucket_val;             // [sum K] values grouped by bin
  uint32_t* bucket_pos;          // [sum K] original position p of the grouped values
  float* expand_buf;             // [world][sum K] fitted curves of every rank
  uint32_t poly_total;           // sum K over the ranked tensors
  unsigned long long* debug_times;  // optional [kPhEnd + 1][grid][2] globaltimer ns at phase entry / exit of every CTA (nullptr: off);
                                    // row kPhEnd: {%smid of the CTA, 0}
  const uint32_t* cuts;          // optional per-phase-class tile partitions [kNumParts][cuts_grid + 1] (first tile of every CTA,
  uint32_t cuts_grid;            // host-computed: per-phase cost weights x per-CTA speeds); used when gridDim.x == cuts_grid
  int deterministic;             // 1: decode adds the senders of a tile in rank order by one warp (bit-reproducible sums);
                                 // 0 (default): every (sender, tile) pair is an independent work item that adds with RED.ADD.F32 —
                                 // identical on all ranks (owner computes), order-dependent in the last ulp only where >= 3
                                 // senders hit the same element
  uint32_t peer_timeout_ms;      // peer-flag waits give up after this long (status 2, output poisoned with NaN, CTA exits)
  int fault;                     // fault injection (tests): 1 = this rank never releases its stage-1 flags
  uint32_t* mc_arena;            // NVLS multicast mapping of the symmetric arena (nullptr: per-peer P2P stores)
  int has_rle;                   // some tensor uses kModeRle or kModeEf (their bit streams are OR-ed into the slot, which is
                                 // zeroed every step; only the <.., true> kernels carry those paths)
  int has_shared;                // some tensor uses kModeShared ('randomk': only the <.., true> kernel carries that path)
  int shard;                     // 1: sharded decode + stage-2 exchange (when world > 1)
  uint32_t s2_words;             // words per stage-2 slot: [count, epoch, 0, 0][idx x cap][val x cap]
  uint32_t s2_cap;               // entries per stage-2 slot
  // bf16 buckets (bf16 != 0, the <.., .., true> kernels; grad is unused): the dense gradient is bf16 in and out, the
  // residual, the select, the codecs and the wire stay fp32 (widening is exact), and the aggregate is rounded once
  // (round-to-nearest-even) where it is final.  The bloom apply adds in fp32 into acc32 first; the warp that finishes a
  // tile rounds it into grad_bf16.
  uint16_t* grad_bf16;           // [total elements] bf16 bit patterns
  float* acc32;                  // [acc_tiles * kTile] apply accumulator, row = tile - first tile this rank decodes; zeroed
                                 // in the accumulate phase for the bloom tiles that are applied
  uint32_t acc_tiles;            // rows of acc32 (0: no tensor needs the apply)
  int bf16;
  // 'dgc' memory (mom != nullptr, the <.., true, .., true> kernels; beta = gamma = 1): momentum correction before the
  // select, u = fl(fl(momentum * u) + g) and r = fl(r + u), and momentum factor masking, u = 0 wherever this rank's
  // own decoded contribution is non-zero (emit for fp32 values, fix for coded values)
  float* mom;                    // [total elements] fp32 momentum u (persists across steps)
  float momentum;
  int has_bf16_values;           // some tensor ships bf16 values (kVmodeBf16: only the <.., true> kernels carry that path)
  // 'dgc' weight decay (weight_decay != 0, the dgc kernels only): the accumulate phase adds weight_decay * w to the
  // gradient of every plan tensor t with decayed[t] != 0 ahead of the momentum, d = fl(g + fl(weight_decay * w)), with w
  // read from the parameter itself.  A tensor with decayed[t] == 0 (a parameter excluded from the decay) reads no w and
  // adds nothing.  The factor stays one scalar (the constant bank, no register across the tile loop); per tensor only
  // the on/off flag is read, once per tensor run.
  // wparams[t]: address of plan tensor t's first element in its parameter's storage (the bucket's dtype; a chunk of a
  // split parameter points at its offset).  Only the tensor's numel elements are read: the padding takes w = 0.
  // These fields and the ones below are read by the dgc kernels only.
  const unsigned long long* wparams;  // [n_tensors]
  float weight_decay;
  const uint8_t* decayed;             // [n_tensors] 1: the tensor takes the decay, 0: excluded (a chunk: its parameter's)
  // 'dgc' Nesterov momentum (nesterov != 0): the residual adds v = fl(d + fl(momentum * u)) with the new u, not u
  int nesterov;
  // 'dgc' local gradient clipping (clip_part != nullptr, the <.., true, .., true, true> kernels): the accumulate phase
  // first sums the squares of every parameter's gradient in fp64 by adjacent pairs (per tile into clip_part, then over
  // the parameter's tiles), and where nrm = sqrt(sum) is finite and > clip_thr it multiplies the gradient by
  // f = fl32(clip_thr / nrm) ahead of the weight decay and the momentum.  A split parameter's chunks share one norm.
  double* clip_part;             // [n_tiles] scratch: pairwise sum of the squares of each tile's gradient
  float* clip_f;                 // [n_tensors] scratch: factor of each plan tensor (1: not clipped)
  const uint32_t* clip_owner;    // [2 * n_tensors] {first tile, tile count} of the parameter the plan tensor belongs to
  double clip_thr;               // c / sqrt(W)
};

// Slot and slice layout, shared by the kernel and the host that launches it (binding.cpp)
#ifdef __CUDACC__
#define DR_PLAN_HD __host__ __device__ __forceinline__
#else
#define DR_PLAN_HD inline
#endif

DR_PLAN_HD bool sharded(const EngineParams& P) { return P.shard && P.world > 1; }

// tiles rank `owner` decodes: everything (W == 1 / unsharded) or its 1/W slice
DR_PLAN_HD void decode_span(const EngineParams& P, int owner, uint32_t& s_begin, uint32_t& s_end) {
  if (sharded(P)) {
    s_begin = (uint32_t)(((uint64_t)P.n_tiles * (uint32_t)owner) / (uint32_t)P.world);
    s_end = (uint32_t)(((uint64_t)P.n_tiles * ((uint32_t)owner + 1u)) / (uint32_t)P.world);
  } else { s_begin = 0; s_end = P.n_tiles; }
}

// word offset in an arena of sender `src`'s slot of the given parity (parallel/plan.py BucketPlan.slot_offset)
DR_PLAN_HD size_t slot_offset(const EngineParams& P, uint32_t parity, int src) {
  return kArenaHdrWords + (size_t)(parity * (uint32_t)P.world + (uint32_t)src) * P.slot_words;
}

// word offset in an arena of sender `src`'s stage-2 slot of the given parity (BucketPlan.stage2_offset)
DR_PLAN_HD size_t s2_offset(const EngineParams& P, uint32_t parity, int src) {
  return kArenaHdrWords + (size_t)2 * (uint32_t)P.world * P.slot_words +
         (size_t)(parity * (uint32_t)P.world + (uint32_t)src) * P.s2_words;
}

}  // namespace dr
