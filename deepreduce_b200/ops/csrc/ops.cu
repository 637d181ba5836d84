// Stand-alone sm_90a kernels behind the GRACE-compatible per-tensor codec API
// (deepreduce_b200/codecs/*): bloom insert / universe query+select, QSGD, scaled sign,
// fp8 values, bit packing, Gram-polynomial fit/eval, delta+bp128 integer coding.
// Each has a plain-torch oracle in the codec module; tests compare them.
#include "common.cuh"
#include "conflict_sets.cuh"
#include "dexp_fit.cuh"
#include "fp8_values.cuh"
#include "ops.h"
#include "sign_values.cuh"

namespace dr {
namespace {

// ---------------------------------------------------------------------------
// bloom
// ---------------------------------------------------------------------------
__global__ void bloom_insert_kernel(const int64_t* __restrict__ idx, int64_t n, uint32_t* filter,
                                    uint32_t n_hash, uint32_t m_bits, uint32_t seed) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    bloom_set(filter, (uint32_t)idx[i], seed, n_hash, m_bits);
}

// pass A: positives per tile;  pass C: emit ascending indices with rank < limit
template <bool kEmit>
__global__ void __launch_bounds__(kThreads) bloom_query_kernel(const uint32_t* __restrict__ filter, uint32_t d,
                                                               uint32_t n_hash, uint32_t m_bits, uint32_t seed,
                                                               uint32_t* __restrict__ tile_counts,
                                                               const uint32_t* __restrict__ tile_excl,
                                                               int64_t* __restrict__ out, uint32_t limit) {
  __shared__ uint32_t cnt[kPerThread * kWarps + 1];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (uint32_t tile = blockIdx.x; tile * (uint32_t)kTile < d; tile += gridDim.x) {
    const uint32_t local0 = tile * kTile;
    uint32_t ball[kPerThread];
#pragma unroll
    for (int c = 0; c < kPerThread; ++c) {
      const uint32_t gi = local0 + c * kThreads + threadIdx.x;
      const bool hit = gi < d && bloom_test(gi, seed, n_hash, m_bits, [&](uint32_t w) { return __ldg(filter + w); });
      ball[c] = __ballot_sync(0xFFFFFFFFu, hit);
    }
    __syncthreads();
    if (lane == 0) {
#pragma unroll
      for (int c = 0; c < kPerThread; ++c) cnt[c * kWarps + warp] = __popc(ball[c]);
    }
    __syncthreads();
    if (warp == 0) {
      uint32_t v[4], sum = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) { v[i] = cnt[lane * 4 + i]; sum += v[i]; }
      uint32_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { uint32_t nb = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (uint32_t)o) incl += nb; }
      uint32_t run = incl - sum;
#pragma unroll
      for (int i = 0; i < 4; ++i) { cnt[lane * 4 + i] = run; run += v[i]; }
      if (lane == 31) cnt[kPerThread * kWarps] = incl;
    }
    __syncthreads();
    if (!kEmit) {
      if (threadIdx.x == 0) tile_counts[tile] = cnt[kPerThread * kWarps];
    } else {
      const uint32_t excl = tile_excl[tile];
      const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
      for (int c = 0; c < kPerThread; ++c) {
        if ((ball[c] >> lane) & 1u) {
          const uint32_t rp = excl + cnt[c * kWarps + warp] + __popc(ball[c] & lt);
          if (rp < limit) out[rp] = (int64_t)(local0 + c * kThreads + threadIdx.x);
        }
      }
    }
  }
}

// single-CTA exclusive scan of tile counts (n up to a few 10k); total -> excl[n]
__global__ void __launch_bounds__(1024) scan_counts_kernel(const uint32_t* __restrict__ counts, uint32_t* __restrict__ excl, uint32_t n) {
  __shared__ uint32_t wsum[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (uint32_t base = 0; base < n; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < n ? counts[i] : 0u;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t nb = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (uint32_t)o) incl += nb; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = wsum[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { uint32_t nb = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= (uint32_t)o) wi += nb; }
      wsum[lane] = wi - w;
    }
    __syncthreads();
    const uint32_t c = carry;
    if (i < n) excl[i] = c + wsum[warp] + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry = c + wsum[warp] + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) excl[n] = carry;
}

// ---------------------------------------------------------------------------
// QSGD: one CTA per bucket
// ---------------------------------------------------------------------------
template <typename OutT>
__global__ void __launch_bounds__(256) qsgd_encode_kernel(const float* __restrict__ v, int64_t K, int bucket, int q,
                                                          uint32_t seed, OutT* __restrict__ lvl, float* __restrict__ norms) {
  __shared__ float red[8];
  const int64_t b0 = (int64_t)blockIdx.x * bucket;
  const int n = (int)min((int64_t)bucket, K - b0);
  float ss = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { const float x = v[b0 + i]; ss += x * x; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xFFFFFFFFu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
  const float norm = sqrtf(tot);
  if (threadIdx.x == 0) norms[blockIdx.x] = norm;
  const float scale = norm > 0.f ? (float)q / norm : 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float x = v[b0 + i];
    const float lf = scale * fabsf(x);
    const float prev = floorf(lf);
    const float u = (float)((double)policy_hash((uint32_t)(b0 + i), seed) / 4294967296.0);
    float l = prev + ((u < (lf - prev)) ? 1.f : 0.f);
    // lf rounds to q(1 + 2^-23) when norm == |x| (a bucket dominated by one value): level q + 1 would wrap the
    // integer type and flip the sign on the wire
    l = fminf(l, (float)q);
    l = x > 0.f ? l : (x < 0.f ? -l : 0.f);
    lvl[b0 + i] = (OutT)l;
  }
}

template <typename InT>
__global__ void qsgd_decode_kernel(const InT* __restrict__ lvl, const float* __restrict__ norms, int64_t K, int bucket,
                                   int q, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < K; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = norms[i / bucket] / (float)q * (float)lvl[i];
}

// ---------------------------------------------------------------------------
// scaled sign: one 512-thread CTA per 512-value bucket (the fused engine's fix phase runs the same rule per task)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) sign_encode_kernel(const float* __restrict__ v, int64_t K,
                                                               uint32_t* __restrict__ bits, float* __restrict__ scales) {
  __shared__ double ws[kWarps];
  const int64_t p = (int64_t)blockIdx.x * kSignBucket + threadIdx.x;
  const float x = p < K ? v[p] : 0.f;
  const float mu = sign_scale(x, (uint32_t)min((int64_t)kSignBucket, K - (int64_t)blockIdx.x * kSignBucket), ws);
  const uint32_t word = sign_word(x);
  if (threadIdx.x == 0) scales[blockIdx.x] = mu;
  if ((threadIdx.x & 31u) == 0 && p < K) bits[p >> 5] = word;
}

__global__ void sign_decode_kernel(const uint32_t* __restrict__ bits, const float* __restrict__ scales, int64_t K,
                                   float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < K; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = sign_decoded((bits[i >> 5] >> (i & 31)) & 1u, scales[i / kSignBucket]);
}

// ---------------------------------------------------------------------------
// fp8 values: one warp per 32-value block, four blocks (one scale word) per 128-thread CTA (the fused engine's fix
// phase runs the same rule per task)
// ---------------------------------------------------------------------------
constexpr int kFp8Threads = 4 * kFp8Block;

__global__ void __launch_bounds__(kFp8Threads) fp8_encode_kernel(const float* __restrict__ v, int64_t K,
                                                                 uint32_t* __restrict__ scales,
                                                                 uint32_t* __restrict__ elems) {
  __shared__ uint32_t sw;
  const int64_t p = (int64_t)blockIdx.x * kFp8Threads + threadIdx.x;
  const float x = p < K ? v[p] : 0.f;
  const uint32_t s = fp8_block_scale(x);                // blocks past the end: scale byte 0
  const uint32_t word = fp8_elem_word(x, s);
  if ((threadIdx.x & 31u) == 0) reinterpret_cast<uint8_t*>(&sw)[threadIdx.x >> 5] = (uint8_t)s;
  __syncthreads();
  if (threadIdx.x == 0) scales[blockIdx.x] = sw;
  if ((threadIdx.x & 3u) == 0 && p < K) elems[p >> 2] = word;
}

__global__ void fp8_decode_kernel(const uint32_t* __restrict__ scales, const uint32_t* __restrict__ elems, int64_t K,
                                  float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < K; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = fp8_decoded((scales[i >> 7] >> ((i >> 2) & 24)) & 0xFFu, (elems[i >> 2] >> ((i & 3) << 3)) & 0xFFu);
}

// ---------------------------------------------------------------------------
// bit packing: thread per output word / per value
// ---------------------------------------------------------------------------
__global__ void pack_bits_kernel(const int64_t* __restrict__ vals, int64_t n, int bits, uint32_t* __restrict__ out, int64_t n_words) {
  for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bit0 = w * 32;
    int64_t i = bit0 / bits;
    uint32_t word = 0;
    for (; i < n && i * bits < bit0 + 32; ++i) {
      const uint64_t v = (uint64_t)vals[i] & ((bits >= 64) ? ~0ull : ((1ull << bits) - 1ull));
      const int64_t s = i * bits - bit0;               // position of value bit 0 relative to the word
      if (s >= 0) word |= (uint32_t)(v << s);
      else word |= (uint32_t)(v >> (-s));
    }
    out[w] = word;
  }
}

__global__ void unpack_bits_kernel(const uint32_t* __restrict__ in, int64_t n_words, int64_t n, int bits, int64_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bit0 = i * bits;
    const int64_t w = bit0 >> 5;
    const int s = (int)(bit0 & 31);
    uint64_t lo = in[w];
    uint64_t hi = (w + 1 < n_words) ? in[w + 1] : 0u;
    uint64_t v = (lo | (hi << 32)) >> s;
    if (s + bits > 64) {                              // the value spans three words: its top bits are in in[w + 2]
      const uint64_t top = (w + 2 < n_words) ? in[w + 2] : 0u;
      v |= top << (64 - s);
    }
    out[i] = (int64_t)(v & ((1ull << bits) - 1ull));
  }
}

// ---------------------------------------------------------------------------
// Gram-polynomial least squares: one CTA per segment.
// p_0=1, p_1=1-2x/N, (k+1)(N-k)p_{k+1} = (2k+1)(N-2x)p_k - k(N+k+1)p_{k-1}
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) polyfit_fit_kernel(const float* __restrict__ y, const int* __restrict__ seg_off,
                                                          const int* __restrict__ seg_len, int degree,
                                                          float* __restrict__ coeffs) {
  __shared__ float red[2][kMaxDeg + 1][8];
  const int s = blockIdx.x;
  const int n = seg_len[s], off = seg_off[s];
  const int deg_eff = min(degree, n - 1);
  float num[kMaxDeg + 1], den[kMaxDeg + 1];
#pragma unroll
  for (int k = 0; k <= kMaxDeg; ++k) { num[k] = 0.f; den[k] = 0.f; }
  const float N = (float)(n - 1);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float p[kMaxDeg + 1];
    gram_eval<kMaxDeg + 1>((float)i, N, deg_eff, p);
    const float yi = y[off + i];
#pragma unroll
    for (int k = 0; k <= kMaxDeg; ++k) { num[k] += p[k] * yi; den[k] += p[k] * p[k]; }
  }
#pragma unroll
  for (int k = 0; k <= kMaxDeg; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      num[k] += __shfl_xor_sync(0xFFFFFFFFu, num[k], o);
      den[k] += __shfl_xor_sync(0xFFFFFFFFu, den[k], o);
    }
    if ((threadIdx.x & 31) == 0) { red[0][k][threadIdx.x >> 5] = num[k]; red[1][k][threadIdx.x >> 5] = den[k]; }
  }
  __syncthreads();
  if ((int)threadIdx.x <= degree) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < 8; ++w) { a += red[0][threadIdx.x][w]; b += red[1][threadIdx.x][w]; }
    coeffs[s * (degree + 1) + threadIdx.x] = (n > 0 && (int)threadIdx.x <= max(deg_eff, 0) && b > 0.f) ? a / b : 0.f;
  }
}

__global__ void polyfit_eval_kernel(const float* __restrict__ coeffs, const int* __restrict__ seg_off,
                                    const int* __restrict__ seg_len, int n_seg, int degree, int64_t total,
                                    float* __restrict__ out) {
  __shared__ int s_off[32], s_len[32];
  if ((int)threadIdx.x < n_seg) { s_off[threadIdx.x] = seg_off[threadIdx.x]; s_len[threadIdx.x] = seg_len[threadIdx.x]; }
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int s = 0;
    for (int j = 0; j < n_seg; ++j) if (s_len[j] > 0 && i >= s_off[j]) s = j;
    const int n = s_len[s];
    const int deg_eff = min(degree, n - 1);
    float p[kMaxDeg + 1];
    gram_eval<kMaxDeg + 1>((float)(i - s_off[s]), (float)(n - 1), deg_eff, p);
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k <= kMaxDeg; ++k) if (k <= degree) acc += coeffs[s * (degree + 1) + k] * p[k];
    out[i] = acc;
  }
}

// ---------------------------------------------------------------------------
// delta + bp128: one warp per block of 128 sorted indices (4 per lane).
// block wire: [width][4*width words]; value j of the block occupies bits
// [j*width, (j+1)*width) of the block's little-endian bit stream.
// ---------------------------------------------------------------------------
__global__ void bp128_width_kernel(const int64_t* __restrict__ idx, int64_t n, uint32_t* __restrict__ widths) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t n_blocks = (n + 127) / 128;
  if (warp >= n_blocks) return;
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int64_t i = warp * 128 + j * 32 + lane;
    if (i < n) {
      const uint32_t d = (uint32_t)(idx[i] - (i > 0 ? idx[i - 1] : 0));
      m |= d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m |= __shfl_xor_sync(0xFFFFFFFFu, m, o);
  if (lane == 0) widths[warp] = 32 - __clz(m);
}

__global__ void bp128_pack_kernel(const int64_t* __restrict__ idx, int64_t n, const uint32_t* __restrict__ widths,
                                  const int64_t* __restrict__ word_off, uint32_t* __restrict__ out) {
  __shared__ uint32_t sv[8][128];
  const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t n_blocks = (n + 127) / 128;
  if (warp >= n_blocks) return;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int64_t i = warp * 128 + j * 32 + lane;
    sv[wl][j * 32 + lane] = i < n ? (uint32_t)(idx[i] - (i > 0 ? idx[i - 1] : 0)) : 0u;
  }
  __syncwarp();
  const uint32_t width = widths[warp];
  uint32_t* dst = out + word_off[warp];
  if (lane == 0) dst[0] = width;
  for (uint32_t w = lane; w < 4 * width; w += 32) {
    const uint32_t bit0 = w * 32;
    uint32_t j = bit0 / width, word = 0;
    for (; j < 128 && j * width < bit0 + 32; ++j) {
      const uint64_t v = sv[wl][j];
      const int s = (int)(j * width) - (int)bit0;
      word |= s >= 0 ? (uint32_t)(v << s) : (uint32_t)(v >> (-s));
    }
    dst[1 + w] = word;
  }
}

// decode: one warp per block; deltas -> inclusive scan inside the block + block base (second kernel adds bases)
__global__ void bp128_unpack_kernel(const uint32_t* __restrict__ in, const int64_t* __restrict__ word_off, int64_t n,
                                    int64_t* __restrict__ deltas) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int64_t n_blocks = (n + 127) / 128;
  if (warp >= n_blocks) return;
  const uint32_t* src = in + word_off[warp];
  const uint32_t width = src[0];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int v = j * 32 + lane;
    const int64_t i = warp * 128 + v;
    if (i < n) {
      uint64_t val = 0;
      if (width) {
        const uint32_t bit0 = v * width;
        const uint32_t w = bit0 >> 5, s = bit0 & 31u;
        const uint64_t lo = src[1 + w];
        const uint64_t hi = (w + 1 < 4 * width) ? src[2 + w] : 0u;
        val = ((lo | (hi << 32)) >> s) & ((1ull << width) - 1ull);
      }
      deltas[i] = (int64_t)val;
    }
  }
}

__global__ void bp128_header_scan_kernel(const uint32_t* __restrict__ in, int64_t n_blocks, int64_t* __restrict__ word_off) {
  // sequential walk over block headers (n_blocks is K/128: small); single thread.
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    int64_t off = 0;
    for (int64_t b = 0; b < n_blocks; ++b) { word_off[b] = off; off += 1 + 4 * (int64_t)in[off]; }
    word_off[n_blocks] = off;
  }
}

// ---------------------------------------------------------------------------
// bit-level run-length index coding (reference RunLength, pytorch/deepreduce.py:805-846, which loops over all d
// bits in Python).  Runs are derived from the sorted indices: a run of ones starts where idx[i] != idx[i-1]+1.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) rle_count_kernel(const int64_t* __restrict__ idx, int64_t n, uint32_t* __restrict__ counts) {
  const int64_t i = blockIdx.x * 1024ll + threadIdx.x;
  const bool start = i < n && (i == 0 || idx[i] != idx[i - 1] + 1);
  const int c = __syncthreads_count(start);
  if (threadIdx.x == 0) counts[blockIdx.x] = c;
}

__global__ void __launch_bounds__(1024) rle_mark_kernel(const int64_t* __restrict__ idx, int64_t n, const uint32_t* __restrict__ excl,
                                                        int64_t* __restrict__ start_pos, int64_t* __restrict__ end_pos) {
  __shared__ uint32_t wsum[32];
  const int64_t i = blockIdx.x * 1024ll + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const bool start = i < n && (i == 0 || idx[i] != idx[i - 1] + 1);
  const bool end = i < n && (i == n - 1 || idx[i + 1] != idx[i] + 1);
  const uint32_t ball = __ballot_sync(0xFFFFFFFFu, start);
  if (lane == 0) wsum[warp] = __popc(ball);
  __syncthreads();
  if (warp == 0) {
    uint32_t w = wsum[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t nb = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= (uint32_t)o) wi += nb; }
    wsum[lane] = wi - w;
  }
  __syncthreads();
  // inclusive count of starts up to and including element i
  const uint32_t incl = excl[blockIdx.x] + wsum[warp] + __popc(ball & ((2u << lane) - 1u));
  if (start) start_pos[incl - 1] = i;
  if (end) end_pos[incl - 1] = i;               // an end closes the run opened by the latest start
}

__global__ void rle_runs_kernel(const int64_t* __restrict__ idx, const int64_t* __restrict__ start_pos,
                                const int64_t* __restrict__ end_pos, int64_t n_runs, int64_t d, int64_t* __restrict__ runs) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_runs; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = start_pos[r], e = end_pos[r];
    const int64_t prev_end = r ? idx[end_pos[r - 1]] : -1;
    runs[2 * r] = idx[s] - prev_end - 1;
    runs[2 * r + 1] = e - s + 1;
    if (r == n_runs - 1) { const int64_t tail = d - 1 - idx[e]; if (tail > 0) runs[2 * n_runs] = tail; }
  }
}

// decode: thread j finds the run holding the j-th index (binary search over the cumulative ones counts)
__global__ void rle_expand_kernel(const int64_t* __restrict__ ones_excl, const int64_t* __restrict__ run_start, int64_t n_runs,
                                  int64_t total, int64_t* __restrict__ out) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < total; j += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n_runs;                 // largest r with ones_excl[r] <= j
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (ones_excl[mid] <= j) lo = mid; else hi = mid; }
    out[j] = run_start[lo] + (j - ones_excl[lo]);
  }
}

inline int grid_for(int64_t n, int threads, int ctas_per_sm = 8) {   // grid-stride kernels: at most 8 CTAs per SM
  const int64_t cap = (int64_t)ctas_per_sm * sm_count();
  int64_t g = (n + threads - 1) / threads;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

}  // namespace

// ---------------------------------------------------------------------------
// launchers (C ABI used by binding.cpp)
// ---------------------------------------------------------------------------
void launch_bloom_insert(const int64_t* idx, int64_t n, uint32_t* filter, uint32_t n_hash, uint32_t m_bits,
                         uint32_t seed, cudaStream_t st) {
  if (n == 0) return;
  count_launch();
  bloom_insert_kernel<<<grid_for(n, 256), 256, 0, st>>>(idx, n, filter, n_hash, m_bits, seed);
}

void launch_bloom_count(const uint32_t* filter, uint32_t d, uint32_t n_hash, uint32_t m_bits, uint32_t seed,
                        uint32_t* tile_counts, uint32_t* tile_excl, cudaStream_t st) {
  const uint32_t n_tiles = (d + kTile - 1) / kTile;
  count_launch(2);
  bloom_query_kernel<false><<<min(n_tiles, 148u * 4u), kThreads, 0, st>>>(filter, d, n_hash, m_bits, seed, tile_counts,
                                                                         nullptr, nullptr, 0);
  scan_counts_kernel<<<1, 1024, 0, st>>>(tile_counts, tile_excl, n_tiles);
}

void launch_bloom_emit(const uint32_t* filter, uint32_t d, uint32_t n_hash, uint32_t m_bits, uint32_t seed,
                       const uint32_t* tile_excl, int64_t* out, uint32_t limit, cudaStream_t st) {
  const uint32_t n_tiles = (d + kTile - 1) / kTile;
  count_launch();
  bloom_query_kernel<true><<<min(n_tiles, 148u * 4u), kThreads, 0, st>>>(filter, d, n_hash, m_bits, seed, nullptr,
                                                                        tile_excl, out, limit);
}

void launch_qsgd_encode(const float* v, int64_t K, int bucket, int q, uint32_t seed, void* lvl, bool i16, float* norms,
                        cudaStream_t st) {
  if (K == 0) return;
  const int nb = (int)((K + bucket - 1) / bucket);
  count_launch();
  if (i16) qsgd_encode_kernel<int16_t><<<nb, 256, 0, st>>>(v, K, bucket, q, seed, (int16_t*)lvl, norms);
  else qsgd_encode_kernel<int8_t><<<nb, 256, 0, st>>>(v, K, bucket, q, seed, (int8_t*)lvl, norms);
}

void launch_qsgd_decode(const void* lvl, bool i16, const float* norms, int64_t K, int bucket, int q, float* out,
                        cudaStream_t st) {
  if (K == 0) return;
  count_launch();
  if (i16) qsgd_decode_kernel<int16_t><<<grid_for(K, 256), 256, 0, st>>>((const int16_t*)lvl, norms, K, bucket, q, out);
  else qsgd_decode_kernel<int8_t><<<grid_for(K, 256), 256, 0, st>>>((const int8_t*)lvl, norms, K, bucket, q, out);
}

void launch_sign_encode(const float* v, int64_t K, uint32_t* bits, float* scales, cudaStream_t st) {
  if (K == 0) return;
  count_launch();
  sign_encode_kernel<<<(unsigned)((K + kSignBucket - 1) / kSignBucket), kThreads, 0, st>>>(v, K, bits, scales);
}

void launch_sign_decode(const uint32_t* bits, const float* scales, int64_t K, float* out, cudaStream_t st) {
  if (K == 0) return;
  count_launch();
  sign_decode_kernel<<<grid_for(K, 256), 256, 0, st>>>(bits, scales, K, out);
}

void launch_fp8_encode(const float* v, int64_t K, uint32_t* scales, uint32_t* elems, cudaStream_t st) {
  if (K == 0) return;
  count_launch();
  fp8_encode_kernel<<<(unsigned)((K + kFp8Threads - 1) / kFp8Threads), kFp8Threads, 0, st>>>(v, K, scales, elems);
}

void launch_fp8_decode(const uint32_t* scales, const uint32_t* elems, int64_t K, float* out, cudaStream_t st) {
  if (K == 0) return;
  count_launch();
  fp8_decode_kernel<<<grid_for(K, 256), 256, 0, st>>>(scales, elems, K, out);
}

void launch_pack_bits(const int64_t* vals, int64_t n, int bits, uint32_t* out, int64_t n_words, cudaStream_t st) {
  if (n_words == 0) return;
  count_launch();
  pack_bits_kernel<<<grid_for(n_words, 256), 256, 0, st>>>(vals, n, bits, out, n_words);
}

void launch_unpack_bits(const uint32_t* in, int64_t n_words, int64_t n, int bits, int64_t* out, cudaStream_t st) {
  if (n == 0) return;
  count_launch();
  unpack_bits_kernel<<<grid_for(n, 256), 256, 0, st>>>(in, n_words, n, bits, out);
}

// ---------------------------------------------------------------------------
// Double-exponential fit ("Fit-DExp"): one CTA runs the regression of dexp_fit.cuh over y = |values| ascending.
// ---------------------------------------------------------------------------
constexpr int kDexpThreads = 1024;

__global__ void __launch_bounds__(kDexpThreads) dexp_fit_kernel(const float* __restrict__ y, int64_t K, double* __restrict__ out) {
  __shared__ DexpScratch sh;
  double c[4];
  dexp_fit_block<kDexpThreads>([&](int64_t k) { return (double)y[k]; }, K, sh, c);
  if (threadIdx.x == 0) { out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3]; }
}

void launch_dexp_fit(const float* y, int64_t K, double* out, cudaStream_t st) {
  count_launch();
  dexp_fit_kernel<<<1, kDexpThreads, 0, st>>>(y, K, out);
}

// ---------------------------------------------------------------------------
// P2 / conflict sets (paper Alg. 1; reference tensorflow/policies.hpp:43-146 — a host C++ routine upstream, and up to
// round 1 a device -> host -> device bounce here): one warp runs the draw of conflict_sets.cuh over the sets in visit
// order, with the chosen flags of the positives in shared memory.
// Bit-exact with ops/csrc/cpu/native_cpu.cpp::conflict_sets_impl (tests/test_gpu_engine.py).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(32) conflict_sets_pick_kernel(const uint32_t* __restrict__ set_off, const uint32_t* __restrict__ members,
                                                                 uint32_t* __restrict__ last, uint32_t n_sets, uint32_t n_pos, uint32_t K,
                                                                 uint32_t pseed, uint32_t* __restrict__ chosen_out) {
  extern __shared__ uint32_t chosen[];                     // ceil(n_pos / 32) words
  const uint32_t lane = threadIdx.x;
  const uint32_t n_words = (n_pos + 31u) >> 5;
  for (uint32_t i = lane; i < n_words; i += 32u) chosen[i] = 0u;
  __syncwarp();
  conflict_sets_draw([&](uint32_t i) { const uint32_t off = set_off[i]; return make_uint2(off, set_off[i + 1] - off); },
                     [&](uint32_t j) { return members[j]; }, last, n_sets, n_pos, K, pseed, chosen);
  for (uint32_t i = lane; i < n_words; i += 32u) chosen_out[i] = chosen[i];
}

cudaError_t launch_conflict_sets_pick(const uint32_t* set_off, const uint32_t* members, uint32_t* last, uint32_t n_sets, uint32_t n_pos,
                                      uint32_t K, uint32_t pseed, uint32_t* chosen_out, cudaStream_t st) {
  const size_t smem = (size_t)((n_pos + 31u) >> 5) * 4u;
  if (smem > 200 * 1024) return cudaErrorInvalidValue;                       // > 1.6 M positives: the caller falls back to the host routine
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(conflict_sets_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); attr = true; }
  count_launch();
  conflict_sets_pick_kernel<<<1, 32, smem, st>>>(set_off, members, last, n_sets, n_pos, K, pseed, chosen_out);
  return cudaGetLastError();
}

void launch_polyfit_fit(const float* y, const int* seg_off, const int* seg_len, int n_seg, int degree, float* coeffs,
                        cudaStream_t st) {
  count_launch();
  polyfit_fit_kernel<<<n_seg, 256, 0, st>>>(y, seg_off, seg_len, degree, coeffs);
}

void launch_polyfit_eval(const float* coeffs, const int* seg_off, const int* seg_len, int n_seg, int degree,
                         int64_t total, float* out, cudaStream_t st) {
  if (total == 0) return;
  count_launch();
  polyfit_eval_kernel<<<grid_for(total, 256), 256, 0, st>>>(coeffs, seg_off, seg_len, n_seg, degree, total, out);
}

void launch_bp128_widths(const int64_t* idx, int64_t n, uint32_t* widths, cudaStream_t st) {
  if (n == 0) return;
  const int64_t n_blocks = (n + 127) / 128;
  count_launch();
  bp128_width_kernel<<<(int)((n_blocks * 32 + 255) / 256), 256, 0, st>>>(idx, n, widths);
}

void launch_bp128_pack(const int64_t* idx, int64_t n, const uint32_t* widths, const int64_t* word_off, uint32_t* out,
                       cudaStream_t st) {
  if (n == 0) return;
  const int64_t n_blocks = (n + 127) / 128;
  count_launch();
  bp128_pack_kernel<<<(int)((n_blocks * 32 + 255) / 256), 256, 0, st>>>(idx, n, widths, word_off, out);
}

void launch_rle_count(const int64_t* idx, int64_t n, uint32_t* counts, uint32_t* excl, cudaStream_t st) {
  const uint32_t nb = (uint32_t)((n + 1023) / 1024);
  count_launch(2);
  rle_count_kernel<<<nb, 1024, 0, st>>>(idx, n, counts);
  scan_counts_kernel<<<1, 1024, 0, st>>>(counts, excl, nb);
}

void launch_rle_runs(const int64_t* idx, int64_t n, const uint32_t* excl, int64_t* start_pos, int64_t* end_pos,
                     int64_t n_runs, int64_t d, int64_t* runs, cudaStream_t st) {
  const uint32_t nb = (uint32_t)((n + 1023) / 1024);
  count_launch(2);
  rle_mark_kernel<<<nb, 1024, 0, st>>>(idx, n, excl, start_pos, end_pos);
  rle_runs_kernel<<<grid_for(n_runs, 256), 256, 0, st>>>(idx, start_pos, end_pos, n_runs, d, runs);
}

void launch_rle_expand(const int64_t* ones_excl, const int64_t* run_start, int64_t n_runs, int64_t total, int64_t* out,
                       cudaStream_t st) {
  if (total == 0) return;
  count_launch();
  rle_expand_kernel<<<grid_for(total, 256), 256, 0, st>>>(ones_excl, run_start, n_runs, total, out);
}

void launch_bp128_unpack(const uint32_t* in, int64_t n, int64_t* word_off, int64_t* deltas, cudaStream_t st) {
  if (n == 0) return;
  const int64_t n_blocks = (n + 127) / 128;
  count_launch(2);
  bp128_header_scan_kernel<<<1, 32, 0, st>>>(in, n_blocks, word_off);
  bp128_unpack_kernel<<<(int)((n_blocks * 32 + 255) / 256), 256, 0, st>>>(in, word_off, n, deltas);
}

}  // namespace dr
