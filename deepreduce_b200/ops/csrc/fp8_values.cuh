// FP8 values ('value': 'fp8'): the block rule, shared by the per-tensor kernels (ops.cu fp8_encode_kernel /
// fp8_decode_kernel) and the fused engine (engine.cu fix_fp8 and coded_value).  Normative: codecs/fp8.py.
//
// A block is 32 consecutive shipped values, one per lane of a warp (0.0 past the end of the values).  Its scale byte s
// comes from A, the largest |v| bit pattern of the block (one integer max):
//   * A >= 0x7F800000 (an inf or a NaN in the block): s = 0xFF, every element byte 0x00, every value decodes to NaN;
//   * otherwise s = e + 127, e the smallest integer with float(A) * 2^-e <= 448 (E4M3's largest finite value), clamped
//     below at -127: for a = m * 2^E with m in [1, 2), e = E - 8 if m <= 1.75, else E - 7; e = -127 for 0 and fp32
//     subnormals.  The scale rounds UP, so no element saturates (OCP MXFP8's floor(log2 a) - 8 can clip the block
//     maximum by up to 12.5 %; the bytes differ from OCP's on blocks whose maximum has m > 1.75).
// Element byte: q = RNE_E4M3(v * 2^-e), the E4M3 "fn" code (no inf, largest 448); v * 2^-e is exact wherever it can
// round to a non-zero code, and |v * 2^-e| <= 448, so cvt.rn.satfinite never saturates.  Decode: widen(q) * 2^e, exact
// in fp32 (at most 4 significant bits, the lowest at 2^-136 or above) unless it exceeds FLT_MAX, which only a block
// maximum of at least 1.9375 * 2^127 can reach (it then decodes to inf).
#pragma once
#include "common.cuh"
#include "tiles.cuh"   // kFullMask

#include <cuda_fp16.h>
#include <cuda_fp8.h>

namespace dr {

constexpr uint32_t kFp8Block = 32;
constexpr uint32_t kFp8NonFinite = 0xFFu;   // scale byte of a block holding an inf or a NaN

// the scale byte of a block from A, its largest |v| bit pattern
DR_D uint32_t fp8_scale_byte(uint32_t A) {
  if (A >= 0x7F800000u) return kFp8NonFinite;
  const uint32_t E8 = A >> 23;                           // biased exponent; 0 for 0 and the subnormals
  if (E8 == 0u) return 0u;
  const int s = (int)E8 - ((A & 0x7FFFFFu) <= 0x600000u ? 8 : 7);   // e + 127, m <= 1.75 <=> mantissa <= 0x600000
  return (uint32_t)max(s, 0);
}

// the scale byte of the warp's block: every lane holds one value (0.0 past the end) and gets the same byte
DR_D uint32_t fp8_block_scale(float v) {
  return fp8_scale_byte(__reduce_max_sync(kFullMask, __float_as_uint(v) & 0x7FFFFFFFu));
}

// the warp's 32 element bytes, four per word: lane l with l % 4 == 0 returns the word of values l .. l + 3 (value l + j
// in bits 8j); every lane's own byte is the low byte of what it returns.  The lanes pair up for one fp32x2 -> e4m3x2
// conversion (cvt.rn.satfinite.e4m3x2.f32).
DR_D uint32_t fp8_elem_word(float v, uint32_t s) {
  // 2^-e = 2^(127 - s), biased exponent 254 - s in [7, 254]: a normal number, so the product is exact (see above)
  const float x = s == kFp8NonFinite ? 0.0f : __fmul_rn(v, __uint_as_float((254u - s) << 23));
  const float x1 = __shfl_down_sync(kFullMask, x, 1);
  const uint32_t pair = __nv_cvt_float2_to_fp8x2(make_float2(x, x1), __NV_SATFINITE, __NV_E4M3);   // x in the low byte
  const uint32_t hi = __shfl_down_sync(kFullMask, pair, 2);
  return (pair & 0xFFFFu) | (hi << 16);
}

// the value of element byte q in a block of scale byte s
DR_D float fp8_decoded(uint32_t s, uint32_t q) {
  if (s == kFp8NonFinite) return __uint_as_float(0x7FC00000u);
  const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)q, __NV_E4M3);
  const float w = __half2float(__half(h));                                      // exact
  const float p2 = s ? __uint_as_float(s << 23) : __uint_as_float(0x00400000u);  // 2^(s - 127); s = 0: 2^-127
  return __fmul_rn(w, p2);
}

}  // namespace dr
