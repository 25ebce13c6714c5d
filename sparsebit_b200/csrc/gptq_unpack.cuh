// gptq_unpack.cuh -- the packed 2 / 3 / 4-bit GPTQ layouts, shared by the dequant-matmul (gptq_simt.cu), its input
// gradient (gptq_dgrad.cu) and the argument checks of the entry points (gptq.cu).
//
// Packed layouts (QuantLinear.pack, utils/quant.py:210-258), LSB first, rows along K:
//   4-bit: 8 values per int32 word.
//   2-bit: 16 values per int32 word.
//   3-bit: 32 values per 3 words; value 10 straddles words 0/1 (2 + 1 bits), value 21 straddles
//          words 1/2 (1 + 2 bits); the other 30 sit at 3 j (+1, +2 in words 1, 2).
// A "unit" is 32 consecutive k: BITS packed words.  A K block of the SIMT dequant-matmul is 64 k (2-bit) or 128 k
// (3 / 4-bit); it never straddles a group because group_size % 64 (2-bit) or % 128 == 0
// (cuda_kernel_2bit.cu:58, cuda_kernel_3bit.cu:60, cuda_kernel_4bit.cu:60).
#pragma once
#include <cstdint>

namespace sb200 {

template <int BITS>
struct GptqFmt {
  static_assert(BITS == 2 || BITS == 3 || BITS == 4, "GPTQ packs 2, 3 or 4 bits");
  static constexpr int kUnitWords = BITS;               // packed words of one 32-k unit
  static constexpr int kUnits = BITS == 2 ? 2 : 4;      // units per K block
  static constexpr int kBlockK = 32 * kUnits;
  static constexpr int kBlockWords = kUnitWords * kUnits;
};

// Rows of the packed matrix QuantLinear allocates for K (utils/quant.py:172-184): ceil(K * bits / (32 p)) * p, p = 3
// for 3-bit, else 1.
inline long long gptq_packed_rows(int bits, long long k) {
  return bits == 4 ? (k + 7) / 8 : (bits == 2 ? (k + 15) / 16 : ((k * 3 + 95) / 96) * 3);
}

// integer 0..15 -> float without I2F: OR the bits into the mantissa of 2^23 and subtract 2^23
__device__ __forceinline__ float small_to_float(uint32_t v) { return __uint_as_float(0x4B000000u | v) - 8388608.0f; }

template <int BITS>
__device__ __forceinline__ void decode_unit(const uint32_t* w, float (&q)[32]);

template <>
__device__ __forceinline__ void decode_unit<4>(const uint32_t* w, float (&q)[32]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int j = 0; j < 8; ++j) q[8 * r + j] = small_to_float((w[r] >> (4 * j)) & 15u);
}

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
