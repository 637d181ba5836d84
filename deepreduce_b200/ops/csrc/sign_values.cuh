// Scaled-sign values ('value': 'sign'): the bucket rule, shared by the per-tensor kernels (ops.cu sign_encode_kernel)
// and the fused engine's fix phase (engine.cu phase_fix).  Normative: codecs/sign.py::sign_encode_oracle.
//
// A bucket is 512 consecutive shipped values, one per thread of a 512-thread CTA (thread t holds position t of the
// bucket, 0.0 past its end).  Its scale is mu = fl32(S / n), S the fp64 sum of |v| over the bucket zero-padded to 512
// in a fixed adjacent-pair tree: the warp butterfly xor 1, 2, 4, 8, 16 (IEEE addition commutes, so both lanes of a
// pair hold the same bits), then the 16 warp sums in adjacent pairs.  A value ships as its sign bit (v < 0, so -0.0,
// +0.0 and NaN give 0) and decodes to bit ? -mu : +mu.
#pragma once
#include "common.cuh"
#include "tiles.cuh"   // kFullMask

namespace dr {

constexpr uint32_t kSignBucket = 512;
static_assert(kThreads == (int)kSignBucket && kWarps == 16, "one 512-value bucket per 512-thread CTA");

// mu of the CTA's bucket of n values (1 <= n <= 512); every thread returns the same bits.  ws: kWarps doubles of
// shared memory, which the caller must not reuse before a barrier.
DR_D float sign_scale(float v, uint32_t n, double* ws) {
  double s = (double)fabsf(v);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) s += __shfl_xor_sync(kFullMask, s, o);
  if ((threadIdx.x & 31u) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  // the 16 warp sums in adjacent pairs: the same butterfly over lanes 0..15 (and again over 16..31)
  s = ws[threadIdx.x & 15u];
#pragma unroll
  for (int o = 1; o < kWarps; o <<= 1) s += __shfl_xor_sync(kFullMask, s, o);
  return __double2float_rn(s / (double)n);
}

// the warp's 32 sign bits, LSB first: bit l <=> lane l's value is < 0
DR_D uint32_t sign_word(float v) { return __ballot_sync(kFullMask, v < 0.0f); }

DR_D float sign_decoded(bool neg, float mu) { return neg ? -mu : mu; }

}  // namespace dr
