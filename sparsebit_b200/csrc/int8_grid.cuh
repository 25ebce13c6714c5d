// int8_grid.cuh -- the stored int8 grid of the integer-grid kernels (int8_linear.cu, int8_group_conv.cu,
// int8_attention.cu): the one quantizer they all store an element through, the storage rules of that grid and the host
// checks their entry points share.
#pragma once

#include "common.cuh"

namespace sb200 {

// The stored grid value g - off of v (QP / quant_round<0>, as the QDQ kernels); NaN sets `nan` and stores 0.
__device__ __forceinline__ int stored_grid(float v, const QP& p, int off, bool& nan) {
  float g = __fadd_rn(quant_round<0>(v, p, 0), p.zp);
  g = fmax_nan(fmin_nan(g, p.qmax), p.qmin);
  if (g != g) {
    nan = true;
    return 0;
  }
  return (int)g - off;
}

// The s8 storage offset: a grid value g is stored as g - off, off = 128 for unsigned ranges and 0 otherwise.
static inline int grid_offset(int qmin) { return qmin >= 0 ? 128 : 0; }

// A stored row of K elements is padded with zeros to Kp = round_up(K, 16) bytes.
static inline long long padded_k(long long k) { return (k + 15) / 16 * 16; }

// The integer range [qmin, qmax] must fit s8 after the offset.
static inline int check_range(const char* fn, int qmin, int qmax) {
  SB_REQUIRE(qmin <= qmax, "%s: qmin %d > qmax %d", fn, qmin, qmax);
  SB_REQUIRE((long long)qmax - qmin <= 255, "%s: integer range [%d, %d] is wider than 8 bits", fn, qmin, qmax);
  const int off = grid_offset(qmin);
  SB_REQUIRE(qmin - off >= -128 && qmax - off <= 127,
             "%s: integer range [%d, %d] is neither signed 8-bit [-128, 127] nor unsigned 8-bit [0, 255]", fn, qmin, qmax);
  return SB200_OK;
}

// The caller's workspace must hold `need` bytes (the workspace queries include the alignment of its base).
static inline int check_workspace(const char* fn, size_t have, size_t need) {
  if (have >= need) return SB200_OK;
  set_error("%s: workspace too small (%zu bytes, need %zu)", fn, have, need);
  return SB200_E_WORKSPACE;
}

// int8_linear.cu: the conv geometry checks of sb200_int8_conv2d that come before the range check (a non-positive
// geometry, an empty output, M = n OH OW >= 2^31: SB200_E_INVALID); on success sets the output size.
int int8_check_conv(const char* fn, const sb200_conv2d_geom* g, long long* oh, long long* ow);

}  // namespace sb200
