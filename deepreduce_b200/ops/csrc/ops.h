// Launcher declarations (implemented in ops.cu / engine.cu / p2p.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "plan.h"

namespace dr {

// engine.cu
int engine_max_grid(int blocks_per_sm, int dyn_smem_bytes);
cudaError_t engine_launch(const EngineParams& P, int grid, int blocks_per_sm, int dyn_smem_bytes, cudaStream_t stream);
void count_launch(int n);
long long launch_count();

// p2.cu — the P2 ('conflict_sets') bloom policy of the fused engine, launched between phase ranges of the engine
struct P2Entry {               // one P2 tensor: its id and word offsets into the scratch buffer (parallel/plan.py p2_tables)
  uint32_t tensor, pos_idx, set_off, cursor, members, ord, last, tmp, misc, pair_cap;
};
struct P2Args {                // sender stage
  const TensorDesc* tensors;
  const TileInfo* tiles;
  const P2Entry* entries;
  uint32_t n_entries;
  uint32_t* scratch;
  uint32_t* pos_mask;          // [n_tiles * 128] my positives (thinned to the pick)
  uint32_t* tile_count;        // [n_tiles] my positives per tile (thinned to the pick)
  uint32_t* slot;              // my slot of this step
  uint32_t epoch, seed;
};
struct P2Thin {                // receiver: thin the probed masks of every sender but me
  const TensorDesc* tensors;
  const TileInfo* tiles;
  const uint32_t* slots;       // slot of sender 0 of this step's parity in my arena (senders slot_words apart)
  uint32_t slot_words;
  uint32_t* dec_mask;          // [world * span * 128], as the engine's decode lays it out
  int rank, world;
  uint32_t s_begin, span;      // the tiles I decode
};
constexpr size_t kP2MaxSmemBytes = 128 * 1024;   // the pick's chosen bitmap: up to 2^20 positives (plan.py P2_MAX_POS_CAP)
// the pick kernel's shared-memory limit, set for the CURRENT device (a function attribute is per device): call it on
// every device that launches p2_pick_launch, before the first launch
cudaError_t p2_prepare();
cudaError_t p2_pick_launch(const P2Args& A, uint32_t max_pos_cap, cudaStream_t st);
cudaError_t p2_header_launch(const P2Args& A, cudaStream_t st);
cudaError_t p2_thin_launch(const P2Thin& T, cudaStream_t st);

// ops.cu
void launch_bloom_insert(const int64_t* idx, int64_t n, uint32_t* filter, uint32_t n_hash, uint32_t m_bits,
                         uint32_t seed, cudaStream_t st);
void launch_bloom_count(const uint32_t* filter, uint32_t d, uint32_t n_hash, uint32_t m_bits, uint32_t seed,
                        uint32_t* tile_counts, uint32_t* tile_excl, cudaStream_t st);
void launch_bloom_emit(const uint32_t* filter, uint32_t d, uint32_t n_hash, uint32_t m_bits, uint32_t seed,
                       const uint32_t* tile_excl, int64_t* out, uint32_t limit, cudaStream_t st);
void launch_qsgd_encode(const float* v, int64_t K, int bucket, int q, uint32_t seed, void* lvl, bool i16, float* norms,
                        cudaStream_t st);
void launch_qsgd_decode(const void* lvl, bool i16, const float* norms, int64_t K, int bucket, int q, float* out,
                        cudaStream_t st);
void launch_sign_encode(const float* v, int64_t K, uint32_t* bits, float* scales, cudaStream_t st);
void launch_sign_decode(const uint32_t* bits, const float* scales, int64_t K, float* out, cudaStream_t st);
void launch_fp8_encode(const float* v, int64_t K, uint32_t* scales, uint32_t* elems, cudaStream_t st);
void launch_fp8_decode(const uint32_t* scales, const uint32_t* elems, int64_t K, float* out, cudaStream_t st);
void launch_pack_bits(const int64_t* vals, int64_t n, int bits, uint32_t* out, int64_t n_words, cudaStream_t st);
void launch_unpack_bits(const uint32_t* in, int64_t n_words, int64_t n, int bits, int64_t* out, cudaStream_t st);
void launch_polyfit_fit(const float* y, const int* seg_off, const int* seg_len, int n_seg, int degree, float* coeffs,
                        cudaStream_t st);
void launch_polyfit_eval(const float* coeffs, const int* seg_off, const int* seg_len, int n_seg, int degree,
                         int64_t total, float* out, cudaStream_t st);
cudaError_t launch_conflict_sets_pick(const uint32_t* set_off, const uint32_t* members, uint32_t* last, uint32_t n_sets, uint32_t n_pos,
                                      uint32_t K, uint32_t pseed, uint32_t* chosen_out, cudaStream_t st);
void launch_dexp_fit(const float* y, int64_t K, double* out_abpq, cudaStream_t st);
void launch_bp128_widths(const int64_t* idx, int64_t n, uint32_t* widths, cudaStream_t st);
void launch_bp128_pack(const int64_t* idx, int64_t n, const uint32_t* widths, const int64_t* word_off, uint32_t* out,
                       cudaStream_t st);
void launch_bp128_unpack(const uint32_t* in, int64_t n, int64_t* word_off, int64_t* deltas, cudaStream_t st);
void launch_rle_count(const int64_t* idx, int64_t n, uint32_t* counts, uint32_t* excl, cudaStream_t st);
void launch_rle_runs(const int64_t* idx, int64_t n, const uint32_t* excl, int64_t* start_pos, int64_t* end_pos,
                     int64_t n_runs, int64_t d, int64_t* runs, cudaStream_t st);
void launch_rle_expand(const int64_t* ones_excl, const int64_t* run_start, int64_t n_runs, int64_t total, int64_t* out,
                       cudaStream_t st);

// repack.cu — DDP gradient bucket <-> engine flat buffer.  table: int64 [n_seg + 1][4] on the device, row s =
// {ddp_off, eng_off, numel, vec_begin} (elements; vec_begin counts 16-byte engine-side vectors), row n_seg =
// {0, 0, 0, n_vec}.  pack: src = DDP buffer, dst = engine buffer; unpack: the other way.  elem_bytes: 4 or 2.
cudaError_t launch_bucket_repack(bool pack, int elem_bytes, const void* src, void* dst, const int64_t* table, int n_seg,
                                 int64_t n_vec, cudaStream_t st);

// p2p.cu — symmetric arena over CUDA IPC
struct ArenaHandle { unsigned char bytes[64]; };
void* arena_alloc(size_t bytes);                       // cudaMalloc + zero
void arena_free(void* p);
ArenaHandle arena_export(void* p);
void* arena_import(const ArenaHandle& h);              // cudaIpcOpenMemHandle
void arena_close(void* p);
int arena_enable_peer_access(const int* devices, int n);   // peers = the listed devices only; returns #enabled
void launch_u8_to_nhwc_norm(const uint8_t* in, void* out_bf16, int64_t n_pix, const float* mean, const float* inv_std,
                            cudaStream_t st);

// bn.cu — training BatchNorm (+ ReLU, + residual add) on NHWC bf16, C % 8 == 0, C <= kBnMaxChannels; per-channel fp32
// parameters.  The row-walking passes (apply, pool, pool gradient, backward elementwise) run one thread per 8 channels
// of a row in a CTA of at most 256 threads, so 2048 channels is the most they cover.
constexpr int kBnMaxChannels = 2048;
struct BnParams { const float* mean; const float* invstd; const float* weight; const float* bias; };
// The (block_y, grid_y) of torch's channels-last reduction tree for rows x C (flexible_launch_configs, coop = true);
// bn_stats and bn_backward reproduce it, and need block_y * grid_y <= rows.
void bn_row_tree(int64_t rows, int C, int* block_y, int* grid_y);
// Training statistics, bitwise torch's channels-last Welford kernel + batch_norm_update_stats_and_invert: writes mean
// and invstd, updates running_mean / running_var.  staging: 2 * grid_y * C + grid_y floats when grid_y > 1.
struct BnStats {
  const void* x;
  float* mean; float* invstd; float* running_mean; float* running_var;
  float* staging;
  float momentum, bessel, eps;
};
cudaError_t launch_bn_stats(const BnStats& s, int64_t rows, int C, cudaStream_t st);
// torch's batch_norm_update_stats_and_invert on the (mean, var) of torch's statistics kernel; var becomes invstd.
cudaError_t launch_bn_update_stats(const float* mean, float* var_invstd, float* running_mean, float* running_var, int C,
                                   float momentum, float bessel, float eps, cudaStream_t st);
// mode 0: relu(bn(x)); 1: relu(bn(x) + z); 2: relu(bn(x) + bn_z(z)).  Also writes the ReLU mask, uint8 [rows][C / 8].
cudaError_t launch_bn_apply(int mode, const void* x, const BnParams& px, const void* z, const BnParams& pz, void* out,
                            void* mask, int64_t rows, int C, cudaStream_t st);
// The stem's max pool (kernel 3, stride 2, padding 1, dilation 1, floor mode) on x of N x H x W x C: Ho = (H - 1) / 2 + 1,
// Wo = (W - 1) / 2 + 1.
struct PoolGeom { int H, W, Ho, Wo; };
// maxpool(relu(bn(x))) (mode 0's relu(bn(x)), then torch's NHWC max pool): writes the pooled output, N x Ho x Wo x C,
// and a code byte per pooled element, uint8 [N * Ho * Wo][C]: bits 0-6 the winner's slot (3 * row + column) in the
// unclipped window, bit 7 the winner's ReLU mask.
cudaError_t launch_bn_apply_pool(const void* x, const BnParams& px, void* out, void* codes, int N, const PoolGeom& pg,
                                 int C, cudaStream_t st);
// Backward of bn_apply's mode from the output gradient go and the mask.  bf16 tensors have x's shape; per-channel fp32
// outputs have C elements; sums = [sum_dy, sum_dy_xmu(, sum_dy_xmu_z)] x C; staging = same x grid_y (bn_row_tree)
// when grid_y > 1.  Mode 1 also writes the masked gradient g; mode 2 reads z and writes dz, dwz, dbz.  Mode 3 is the
// backward of bn_apply_pool: go is the pooled gradient (N x Ho x Wo x C), mask its codes, pool the geometry, and g
// (x's shape) receives the masked gradient of the ReLU output, which both passes then read.  go2 (modes 1-3, may be
// null): a second gradient of go's shape; the output gradient is then the bf16 sum go + go2, autograd's sum at a block
// input with two consumers, formed as the kernels load it.
struct BnBwd {
  const void* go; const void* go2; const uint8_t* mask; const void* x; const void* z;
  BnParams px, pz;      // bias unused
  void* dx; void* dz; void* g;
  float* sums; float* staging; float* dw; float* db; float* dwz; float* dbz;
  PoolGeom pool;        // mode 3
};
cudaError_t launch_bn_backward(int mode, const BnBwd& b, int64_t rows, int C, cudaStream_t st);

}  // namespace dr
