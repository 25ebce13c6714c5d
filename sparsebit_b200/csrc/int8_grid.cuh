// int8_grid.cuh -- the stored int8 grid of the integer-grid kernels (int8_linear.cu, int8_group_conv.cu): the one
// quantizer they all store an element through, and the host checks int8_linear.cu shares with the grouped conv.
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

// int8_linear.cu: the conv geometry checks of sb200_int8_conv2d that come before the range check (a non-positive
// geometry, an empty output, M = n OH OW >= 2^31: SB200_E_INVALID), the integer range rule, and the s8 storage offset
// (128 for unsigned ranges, 0 otherwise).
int int8_check_conv(const char* fn, const sb200_conv2d_geom* g);
int int8_check_range(const char* fn, int qmin, int qmax);
int int8_grid_offset(int qmin);

}  // namespace sb200
