// gptq_unpack.cuh -- unit decoders of the packed 2 / 3-bit GPTQ layouts, shared by the dequant-matmul
// (gptq_lowbit.cu) and its input gradient (gptq_dgrad.cu).
//
// Packed layouts (QuantLinear.pack, utils/quant.py:210-258), LSB first, rows along K:
//   2-bit: 16 values per int32 word.
//   3-bit: 32 values per 3 words; value 10 straddles words 0/1 (2 + 1 bits), value 21 straddles
//          words 1/2 (1 + 2 bits); the other 30 sit at 3 j (+1, +2 in words 1, 2).
// A "unit" is 32 consecutive k (2 words for 2-bit, 3 words for 3-bit).
#pragma once
#include <cstdint>

namespace sb200 {

// integer 0..7 -> float without I2F: OR the bits into the mantissa of 2^23 and subtract 2^23
__device__ __forceinline__ float small_to_float(uint32_t v) { return __uint_as_float(0x4B000000u | v) - 8388608.0f; }

template <int BITS>
__device__ __forceinline__ void decode_unit(const uint32_t* w, float (&q)[32]);

template <>
__device__ __forceinline__ void decode_unit<2>(const uint32_t* w, float (&q)[32]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    q[j] = small_to_float((w[0] >> (2 * j)) & 3u);
    q[16 + j] = small_to_float((w[1] >> (2 * j)) & 3u);
  }
}

template <>
__device__ __forceinline__ void decode_unit<3>(const uint32_t* w, float (&q)[32]) {
#pragma unroll
  for (int j = 0; j < 10; ++j) {
    q[j] = small_to_float((w[0] >> (3 * j)) & 7u);
    q[11 + j] = small_to_float((w[1] >> (3 * j + 1)) & 7u);
    q[22 + j] = small_to_float((w[2] >> (3 * j + 2)) & 7u);
  }
  q[10] = small_to_float((w[0] >> 30) | ((w[1] & 1u) << 2));
  q[21] = small_to_float((w[1] >> 31) | ((w[2] & 3u) << 1));
}

}  // namespace sb200
