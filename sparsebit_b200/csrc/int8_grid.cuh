// int8_grid.cuh -- the stored int8 grid of the integer-grid kernels (int8_linear.cu, int8_group_conv.cu,
// int8_attention.cu, int8_sparse24.cu): the one quantizer they all store an element through, the storage rules of that
// grid, the host checks their entry points share, and the lowering of an activation onto the grid (int8_linear.cu).
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

// The stored grid value of an activation element v: stored_grid(v), or, kDoReFa, stored_grid of DoReFa's normalised
// tanh(v) / m (dorefa_norm of common.cuh, the op sequence of sb200_dorefa_fwd), m = max |tanh| over the whole input,
// rm = dorefa_rcp(m).
// A NaN m, or m = 0 (an all-zero input: 0 / 0), makes every element NaN, as in the fake-quant op.  Padding taps are
// not elements: they stay at the grid point of a real 0.
template <bool kDoReFa>
__device__ __forceinline__ int input_grid(float v, double rm, const QP& p, int off, bool& nan) {
  if constexpr (kDoReFa) {
    float t;
    v = dorefa_norm(v, rm, t);
  }
  return stored_grid(v, p, off, nan);
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

// The _dorefa entry points make every check of their plain counterpart, then this one: a null x_absmax is
// SB200_E_INVALID (dorefa = false: the plain entry point, nothing to check).
static inline int check_absmax(const char* fn, bool dorefa, const float* x_absmax) {
  SB_REQUIRE(!dorefa || x_absmax, "%s: null x_absmax", fn);
  return SB200_OK;
}

// |a|, |b| <= 128 on the stored grid: the s32 accumulator holds |sum a b| <= K * 2^14 for K < 2^17
constexpr long long kI8MaxK = 1LL << 17;

// Conv geometry on the device; every product is 64-bit (M Kp passes 2^31 at ResNet-50 stem sizes from batch ~1024).
struct ConvDims {
  long long H, W, HW, CHW;     // input plane, image
  long long sh, sw, dh, dw;    // stride, dilation
  long long pt, pl;            // top / left padding
  long long OW, P, M;          // output width, pixels per image, output pixels
  int KH, KW, K, Kp;           // taps, taps padded to 16
};

// The lowered activations of M rows of K elements in a workspace whose base is aligned up to 1024 bytes: the stored
// grid q [M, Kp] at the base, the int32 row sums 1024-aligned behind it, the NaN flags 256-aligned behind those.
struct I8Lowered {
  int8_t* q;
  int* sum;
  uint8_t* nan;
};

// ---- int8_linear.cu
I8Lowered i8_lowered(void* workspace, long long m, long long k);
// K < kI8MaxK, else SB200_E_UNSUPPORTED
int check_k(const char* fn, long long k);
// The conv geometry checks that come before the range check (a non-positive geometry, an empty output,
// M = n OH OW >= 2^31: SB200_E_INVALID); on success fills `d` (K saturated at kI8MaxK).
int check_conv(const char* fn, const sb200_conv2d_geom* g, ConvDims* d);
// The lowering launches: the row quantizer (x [rows, K], per-tensor or per-row qparams) and the conv2d lowering
// (one row per output pixel).  Unchecked: the caller has made every check of sb200_int8_quantize_rows /
// sb200_int8_im2col_quantize, q included (16-byte aligned).  x_absmax: NULL, or the device m of a DoReFa input
// (input_grid<true>).
int launch_rows(const float* x, const float* scale, const float* zero_point, int per_row, int qmin, int qmax, int8_t* q,
                int* row_sum, uint8_t* nan_flag, long long rows, long long k, cudaStream_t st,
                const float* x_absmax = nullptr);
int launch_im2col(const float* x, const ConvDims& d, const float* scale, const float* zero_point, int qmin, int qmax,
                  int8_t* q, int* row_sum, uint8_t* nan_flag, cudaStream_t st, const float* x_absmax = nullptr);
// The same lowering of an x stored NHWC with c channels; a stride-1, unpadded 1 x 1 conv runs the row quantizer.
int launch_im2col_nhwc(const float* x, const ConvDims& d, int c, const float* scale, const float* zero_point, int qmin,
                       int qmax, int8_t* q, int* row_sum, uint8_t* nan_flag, cudaStream_t st,
                       const float* x_absmax = nullptr);

}  // namespace sb200
