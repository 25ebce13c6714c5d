// int8_attention.cuh -- what the fused integer-grid attention (int8_attention.cu) and the attention over an int8
// key/value cache (int8_attention_cache.cu) share: the kernel parameters, the per-element steps of the softmax on the
// grid (the score epilogue, exp_diff, p's grid, the p @ v epilogue, the NaN rules) and the host checks and launches.
// Both files compute every score, p and output through these functions, so the two paths agree operation for
// operation wherever they see the same operands.
#pragma once

#include "int8_grid.cuh"
#include "tc_common.cuh"

namespace sb200 {

constexpr int kAtRows = 128;                    // query rows per CTA (two consumer warpgroups x 64)
constexpr int kAtKeys = 128;                    // keys per block: wgmma N of q k^T, K of p v
constexpr int kAtMaxDim = 128;                  // d, dv
constexpr long long kAtMaxTk = 1LL << 17;       // exact s32 sums of p v

struct AtParams {
  const int* q_sum;
  const uint8_t* q_nan;
  const int* k_sum;
  const uint8_t* k_nan;
  const int* v_sum;
  const uint8_t* v_nan;
  const float *q_scale, *q_zero, *k_scale, *k_zero, *p_scale, *p_zero, *v_scale, *v_zero;
  int q_off, k_off, p_off, v_off;
  float p_qmin, p_qmax;
  int has_scale;
  float scale;
  float* out;
  int8_t* p_q;  // [B, Tq, Tkp] or null
  int Tq, Tk, Tkp, d, dp, dv, vec2;
  int ks;  // entry stride of k_sum / k_nan: Tk, or the capacity of a key/value cache
};

// The mask of the masked instantiation, a separate kernel argument so that AtParams keeps its layout.  Entry b of the
// batch reads mask + (b / inner) stride_outer + (b % inner) stride_inner + i stride_row + j (all 64-bit).
struct AtMask {
  const float* mask;  // or null
  long long stride_outer, stride_inner, stride_row;
  const int* v_pre;  // causal: [B, dv, nkb] running column sums of v^T over the key blocks
  int inner, causal, batch;
};

// The fp32 score of an exact integer dot product I (zero points removed): s = RN32(fp64(I) (fp64(s_q) fp64(s_k))),
// the epilogue of int8_matmul_gemm_kernel, then RN32(s * scale) with a scale.
__device__ __forceinline__ float at_score(long long I, double sqk, int has_scale, float scale) {
  float sc = __double2float_rn((double)I * sqk);
  if (has_scale) sc = __fmul_rn(sc, scale);
  return sc;
}

// The masked score: -inf where the causal band hides the key, then one fp32 add of the mask value (mrow: the row of
// the mask, or null).
__device__ __forceinline__ float at_masked(float sc, bool seen, const float* mrow, int key) {
  if (!seen) sc = -INFINITY;
  if (mrow != nullptr) sc = __fadd_rn(sc, __ldg(mrow + key));
  return sc;
}

// The entry's offset into the mask (batch entry b).
__device__ __forceinline__ long long at_mask_base(const AtMask& mk, int b) {
  return (long long)(b / mk.inner) * mk.stride_outer + (long long)(b % mk.inner) * mk.stride_inner;
}

// exp(s - m) for fp32 s <= m: the difference is split exactly into hi + lo (TwoSum), expf(hi) is corrected by lo.
// Differences below -104 underflow to 0 in fp32 anyway and return 0 (also for a masked s = -inf); NaN propagates.
__device__ __forceinline__ float exp_diff(float s, float m) {
  const float hi = __fsub_rn(s, m);
  if (s == -INFINITY || hi < -104.f) return 0.f;
  const float bb = __fsub_rn(hi, s);
  const float lo = __fadd_rn(__fsub_rn(s, __fsub_rn(hi, bb)), __fsub_rn(-m, bb));
  const float e = expf(hi);
  return __fmaf_rn(e, lo, e);
}

// A partial sum l of exp(s - m_part) in fp64 moved to the row max m >= m_part (an empty part stays 0).
__device__ __forceinline__ double at_rescale(double l, float m_part, float m) {
  return l == 0.0 ? 0.0 : l * exp((double)m_part - (double)m);
}

// The stored grid of p = exp(s - m) * RN32(1 / l) (inv), with p's qparams; a NaN p sets `nan`.
__device__ __forceinline__ int at_p_grid(float s, float m, float inv, const QP& pp, int off, bool& nan) {
  return stored_grid(__fmul_rn(exp_diff(s, m), inv), pp, off, nan);
}

// The NaN rule of an output row: a NaN in its q row, a NaN key it sees, a NaN p, or no visible key at all.
__device__ __forceinline__ bool at_row_nan(bool q_nan, bool k_nan, bool p_nan, bool no_key) {
  return q_nan || k_nan || p_nan || no_key;
}

// out = RN32(fp64(I_pv) (fp64(s_p) fp64(s_v))), or NaN for a NaN row or a NaN column of v.
__device__ __forceinline__ float at_out(long long I, double spv, bool nan) {
  const float y = __double2float_rn((double)I * spv);
  return nan ? __int_as_float(0x7fc00000) : y;
}

// ---- int8_attention.cu
// 0 when the dimensions are acceptable (d, dv <= 128, tk < 2^17, batch tq and batch tk < 2^31), else the SB200 code.
int at_check_dims(const char* fn, int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv);
// The checks of the remaining arguments of sb200_int8_attention_masked (ranges, scale, p_q, causal, the mask over
// [batch, tq, tk]); mask == null skips the mask's.
int at_check_args(const char* fn, const int (&ranges)[4][2], int has_scale, float scale, const int8_t* p_q, int causal,
                  const float* mask, int64_t mask_stride_outer, int64_t mask_stride_inner, int64_t mask_inner,
                  int64_t mask_stride_row, int64_t batch, int64_t tq, int64_t tk);
// The q, k, p and v parts of AtParams from the qparams (device pointers) and ranges; the caller fills the rest.
void at_set_qparams(AtParams& a, const float* const (&qparams)[8], const int (&ranges)[4][2], int has_scale, float scale);
// Causal: bytes of the running column sums of v^T, [batch dv, ceil(tk / 128)] int32.
size_t at_vpre_bytes(long long batch, long long tk, long long dv);
// Launch int8_attention_kernel (masked when mk.mask or mk.causal) over ctas = batch ceil(Tq / 128) CTAs, preceded
// under causal by int8_attention_vprefix_kernel over the v^T rows (row stride vt_stride bytes) into mk.v_pre.
int at_launch(const CUtensorMap& map_q, const CUtensorMap& map_k, const CUtensorMap& map_v, const AtParams& a, AtMask mk,
              const int8_t* vt, long long vt_stride, int* v_pre, long long batch, cudaStream_t st);

}  // namespace sb200
