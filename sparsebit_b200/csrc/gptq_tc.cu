// gptq_tc.cu -- GPTQ int4 group-wise dequant-matmul on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces the M-serial SIMT loop of VecQuant4MatMulKernel
// (large_language_models/llama/quantization/cuda/cuda_kernel_4bit.cu:88-180) for prefill-sized M:
//   out[m, n] += sum_k (scales[n, k/gs] * q[k, n] - zeros[n, k/gs]) * x[m, k]
//
// Numerics.  The reference pins fp32 results at rtol = atol = 1e-5 (test_cuda_kernel.py:47), which a
// single fp16/bf16 tensor-core pass cannot meet.  Here the 4-bit integers q in [0, 15] enter the MMA
// EXACTLY (they are fp16 integers), the fp32 activations are split x * 2^-e = hi + lo into two fp16
// operands (e = per-row power of two so that hi never overflows; 22 significant bits survive), both
// products accumulate in fp32 registers, and the affine part is applied per 128-wide K group on the
// integer dot product:   sum_k (s q - z) x  =  s * (sum_k q x) - z * (sum_k x).
// The reference's group_size is a multiple of 128 (cuda_kernel_4bit.cu:60), so one (s, z) pair per
// 128-K block -- the same blocking the reference uses (BLOCKLEN = 128).
//
// Pipeline (tc_common.cuh): one CTA = 128 features x 128 tokens, a 5-stage TMA ring of 64-K stages.  Each consumer
// thread unpacks its own A fragments (q - zero for two feature rows) from the packed words of the stage, issues
// 4 (+4 lo) wgmma.m64n128k16 into a per-group partial accumulator, and after every 128 K folds
// acc += scale * partial (- zero * xsum) in fp32 registers -- the per-group rescale costs one FMA per accumulator,
// since the accumulator never leaves the registers.
// A prologue kernel splits x into (hi, lo), computes the per-(row, 128-K) sums and the row scales.
//
// fp16 activations (sb200_gptq4_linear_f16): the activations are the hi plane as they are, the lo pass never runs, and
// the epilogue writes out_h = fp16(bias + x @ W) instead of accumulating into the fp32 `out`.
#include "gptq_launch.cuh"
#include "tc_common.cuh"

namespace sb200 {

constexpr int kTcStages = 5;
constexpr int kGroupK = 128;  // fold granularity (= the reference's BLOCKLEN)

// ---------------------------------------------------------------------------------- prologue kernel
// Row m of x -> A_hi[m, :], A_lo[m, :] (fp16, K order permuted inside every 8 as 0,4,1,5,2,6,3,7 to
// match the nibble pairs the unpacker extracts with one AND per pair), xsum[m, g] = sum of the scaled
// row over K group g, rowscale[m] = 2^e.
__global__ void __launch_bounds__(256) gptq_split_kernel(const float* __restrict__ x, __half* __restrict__ a_hi,
                                                         __half* __restrict__ a_lo, float* __restrict__ xsum,
                                                         float* __restrict__ rowscale, int* __restrict__ need_lo,
                                                         int K, int G) {
  __shared__ float red[8];
  const int m = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const float* xr = x + (size_t)m * K;
  float amax = 0.f;
  for (int k = tid * 4; k < K; k += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (lane == 0) red[wid] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) amax = fmaxf(amax, red[i]);
  // scaled row max in [2^14, 2^15): fp16 never overflows, the low part keeps as many bits as possible.  e >= -126 (as
  // the decode kernel clamps its exponent) keeps 2^-e and 2^e finite normal numbers for rows with max |x| < 2^-112:
  // below 2^-113, 2^-e would overflow to +inf and turn the whole output row into NaN (0 * inf, inf - inf)
  int e = 0;
  if (amax > 0.f && amax < __int_as_float(0x7f800000)) e = max(ilogbf(amax) - 14, -126);
  const float down = ldexpf(1.f, -e);
  if (tid == 0) rowscale[m] = ldexpf(1.f, e);
  const int nchunk = K >> 3;
  bool any_lo = false;
  for (int c0 = 0; c0 < nchunk; c0 += 256) {
    const int c = c0 + tid;
    float s = 0.f;
    if (c < nchunk) {
      const float4 u = *reinterpret_cast<const float4*>(xr + c * 8);
      const float4 w = *reinterpret_cast<const float4*>(xr + c * 8 + 4);
      const float v[8] = {u.x * down, w.x * down, u.y * down, w.y * down, u.z * down, w.z * down, u.w * down, w.w * down};
      __half hi[8], lo[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        hi[j] = __float2half_rn(v[j]);
        lo[j] = __float2half_rn(v[j] - __half2float(hi[j]));
        any_lo |= (__half_as_ushort(lo[j]) & 0x7FFFu) != 0;
        s += v[j];
      }
      *reinterpret_cast<uint4*>(a_hi + (size_t)m * K + c * 8) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(a_lo + (size_t)m * K + c * 8) = *reinterpret_cast<const uint4*>(lo);
    }
    // a 128-K group = 16 consecutive chunks = 16 consecutive lanes
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((lane & 15) == 0 && (c >> 4) < G) xsum[(size_t)m * G + (c >> 4)] = s;
  }
  // activations that are exactly fp16-representable after the row scaling (the reference's model path
  // feeds fp16 activations cast to fp32, utils/quant.py:262-277) leave lo == 0 everywhere: the GEMM then
  // skips the second MMA pass and its TMA traffic, with bit-identical results.
  if (__any_sync(0xffffffffu, any_lo) && lane == 0) atomicOr(need_lo, 1);
}

// fp16 activations: the hi plane IS the input (no row scaling needed: |x| <= 65504 and |q - zero| <= 1039 keep every
// product inside fp32), copied with every 8 K permuted to (0, 4, 1, 5, 2, 6, 3, 7) to match the nibble pairs one LOP3
// extracts; xsum[m, g] = sum over the 128-K block (only read when some zero point has a fractional part).
__global__ void __launch_bounds__(256) gptq_permute_f16_kernel(const __half* __restrict__ x, __half* __restrict__ a_hi,
                                                               float* __restrict__ xsum, float* __restrict__ rowscale, int K,
                                                               int G) {
  const int m = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const __half* xr = x + (size_t)m * K;
  if (tid == 0) rowscale[m] = 1.f;
  const int nchunk = K >> 3;
  for (int c0 = 0; c0 < nchunk; c0 += 256) {
    const int c = c0 + tid;
    float s = 0.f;
    if (c < nchunk) {
      const uint4 raw = *reinterpret_cast<const uint4*>(xr + c * 8);
      const __half* h = reinterpret_cast<const __half*>(&raw);
      const __half p[8] = {h[0], h[4], h[1], h[5], h[2], h[6], h[3], h[7]};
#pragma unroll
      for (int j = 0; j < 8; ++j) s += __half2float(h[j]);
      *reinterpret_cast<uint4*>(a_hi + (size_t)m * K + c * 8) = *reinterpret_cast<const uint4*>(p);
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((lane & 15) == 0 && (c >> 4) < G) xsum[(size_t)m * G + (c >> 4)] = s;
  }
}

// ---------------------------------------------------------------------------------- zero-point probe
// GPTQ checkpoints store zeros = zero * scale with an INTEGER zero (utils/quant.py:188, find_params
// :83-89).  When that holds for every (n, g), (q - zero) is an exact fp16 integer that can go into the
// MMA directly and the epilogue needs a single FMA per element.  The probe recovers zero = rint(z/s),
// verifies |z - zero*s| <= 2^-20 |z| (fp32 rounding of the product is 2^-24) and |zero| <= 1024, and
// clears *flag otherwise -- then the kernel uses the general (scale, zeros) epilogue.
__global__ void gptq_zero_probe_kernel(const float* __restrict__ scales, const float* __restrict__ zeros, long long n,
                                       __half* __restrict__ zint, int* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = scales[i], z = zeros[i];
  const float zi = rintf(z / s);
  const bool ok = (fabsf(zi) <= 1024.f) && (fabsf(fmaf(-zi, s, z)) <= fabsf(z) * 0x1p-20f + 1e-30f);
  zint[i] = __float2half_rn(ok ? zi : 0.f);
  if (!ok) atomicAnd(flag, 0);
}

// ---------------------------------------------------------------------------------- main kernel
// F16_OUT: out_h[m, n] = fp16(bias[n] + rowscale[m] * acc), overwritten and never read, bias may be NULL; otherwise
// out[m, n] += rowscale[m] * acc (the reference's accumulate-in-place contract) and out_h / bias are unused.
template <bool F16_OUT>
__global__ void __launch_bounds__(kWgThreads, 1)
gptq4_tc_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                const __grid_constant__ CUtensorMap map_q, float* __restrict__ out, const float* __restrict__ scales,
                const float* __restrict__ zeros, const float* __restrict__ xsum, const float* __restrict__ rowscale,
                const __half* __restrict__ zint, const int* __restrict__ int_zero_flag, int M, int K, int N, int Gq,
                int G128, int group_size, int backoff_ns, __half* __restrict__ out_h, const float* __restrict__ bias) {
  extern __shared__ unsigned char smem_raw[];
  // stage buffers first (1024-byte aligned for SWIZZLE_128B), bookkeeping after them
  unsigned char* stage_base = smem_align1024(smem_raw);
  auto& ring = *reinterpret_cast<StageRing<kTcStages>*>(stage_base + (size_t)kTcStages * kWgStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + kWgTok - 1) / kWgTok;
  const int m0 = (int)(blockIdx.x % (unsigned)tiles_m) * kWgTok, n0 = (int)(blockIdx.x / (unsigned)tiles_m) * kWgFeat;
  const int num_kb = (K + kWgBK - 1) / kWgBK;
  const bool int_zero = int_zero_flag[0] != 0;  // uniform: every zeros[n,g] is an integer multiple of scales[n,g]
  const bool need_lo = int_zero_flag[1] != 0;   // uniform: some activation has a non-zero fp16 low part

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_hi);
    prefetch_tensormap(&map_lo);
    prefetch_tensormap(&map_q);
    ring.init();
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================================================== TMA producer
    reg_dec<40>();
    if (threadIdx.x == 0)
      wg_produce(stage_base, ring, &map_hi, &map_lo, &map_q, m0, n0, num_kb, need_lo, backoff_ns);
    return;
  }
  // ==================================================================== consumers: 64 features x 128 tokens each
  reg_inc<232>();
  const int q = lane & 3;
  const int f0 = ((warp - 4) >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);  // feature rows f0, f0 + 8 of the tile
  const int na = n0 + f0, nb = na + 8;
  const bool live_a = na < N, live_b = nb < N;
  const NibblePair unpack(q);
  const uint32_t stage0 = smem_u32(stage_base);
  float acc[64], part[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int g = kb >> 1;                                            // 128-K group
    const int gq = (int)((long long)g * kGroupK / group_size);        // quantisation group
    // this group's parameters, requested before the wait for the stage
    const float sa = live_a ? __ldg(scales + (size_t)na * Gq + gq) : 0.f;
    const float sb = live_b ? __ldg(scales + (size_t)nb * Gq + gq) : 0.f;
    const float zfa = (!int_zero && live_a) ? __ldg(zeros + (size_t)na * Gq + gq) : 0.f;
    const float zfb = (!int_zero && live_b) ? __ldg(zeros + (size_t)nb * Gq + gq) : 0.f;
    // integer-zero mode: (q - zero) enters the MMA and the fold is one FMA; otherwise q alone and zeros * xsum
    const float za = (int_zero && live_a) ? __half2float(zint[(size_t)na * Gq + gq]) : 0.f;
    const float zb = (int_zero && live_b) ? __half2float(zint[(size_t)nb * Gq + gq]) : 0.f;
    const __half2 offa = unpack.offset(za), offb = unpack.offset(zb);
    const int s = ring.wait(kb);
    const uint32_t* bq = reinterpret_cast<const uint32_t*>(stage_base + (size_t)s * kWgStageBytes + 2 * kWgXBytes);
    uint32_t a[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {  // 16 K = packed rows 2j (K 0..7) and 2j + 1 (K 8..15)
      a[j][0] = h2u(unpack(bq[(2 * j) * kWgFeat + f0], offa));
      a[j][1] = h2u(unpack(bq[(2 * j) * kWgFeat + f0 + 8], offb));
      a[j][2] = h2u(unpack(bq[(2 * j + 1) * kWgFeat + f0], offa));
      a[j][3] = h2u(unpack(bq[(2 * j + 1) * kWgFeat + f0 + 8], offb));
    }
    const uint32_t xh = stage0 + (uint32_t)s * kWgStageBytes;
    const uint64_t dh = gmma_desc_sw128(xh), dl = gmma_desc_sw128(xh + kWgXBytes);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      wgmma_m64n128k16_rs(part, a[j], dh + 2 * j, !((kb & 1) == 0 && j == 0));
      if (need_lo) wgmma_m64n128k16_rs(part, a[j], dl + 2 * j, 1);
    }
    wgmma_commit();
    wgmma_wait_all(part);
    ring.release(kb, lane);
    if ((kb & 1) == 1 || kb == num_kb - 1) {
      // acc[n, m] += s[n] * part (- z[n] * xsum[m, g]);  d[j]: feature f0 + 8 * ((j >> 1) & 1), token 8 (j >> 2) + 2q + (j & 1)
      if (int_zero) {
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] = fmaf((j & 2) ? sb : sa, part[j], acc[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 64; ++j) {
          const int m = m0 + 8 * (j >> 2) + 2 * q + (j & 1);
          const float nxs = (m < M) ? -__ldg(xsum + (size_t)m * G128 + g) : 0.f;
          acc[j] = fmaf((j & 2) ? sb : sa, part[j], fmaf((j & 2) ? zfb : zfa, nxs, acc[j]));
        }
      }
    }
  }
  if constexpr (F16_OUT) {
    const float bna = (bias && live_a) ? __ldg(bias + na) : 0.f;
    const float bnb = (bias && live_b) ? __ldg(bias + nb) : 0.f;
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      const int m = m0 + 8 * (j >> 2) + 2 * q + (j & 1);
      const int n = (j & 2) ? nb : na;
      if (m < M && n < N) out_h[(size_t)m * N + n] = __float2half_rn(fmaf(__ldg(rowscale + m), acc[j], (j & 2) ? bnb : bna));
    }
  } else {
    // out[m, n] += rowscale[m] * acc   (out is pre-initialised with the bias by the caller)
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      const int m = m0 + 8 * (j >> 2) + 2 * q + (j & 1);
      const int n = (j & 2) ? nb : na;
      if (m < M && n < N) {
        float* o = out + (size_t)m * N + n;
        *o = fmaf(__ldg(rowscale + m), acc[j], *o);
      }
    }
  }
}

// ---------------------------------------------------------------------------------- host side
struct TcWorkspace {
  size_t off_hi, off_lo, off_xsum, off_rs, off_zint, off_flag, total;
};
static TcWorkspace tc_layout(long long M, long long K, long long N = 0, long long Gq = 0) {
  TcWorkspace w;
  const long long G128 = (K + kGroupK - 1) / kGroupK;
  w.off_hi = 0;
  w.off_lo = align_up((size_t)M * K * 2, 1024);
  w.off_xsum = w.off_lo + align_up((size_t)M * K * 2, 1024);
  w.off_rs = w.off_xsum + align_up((size_t)M * G128 * 4, 1024);
  w.off_zint = w.off_rs + align_up((size_t)M * 4, 1024);
  w.off_flag = w.off_zint + align_up((size_t)N * Gq * 2, 1024);
  w.total = w.off_flag + 1024;
  return w;
}

int gptq_launch_split(const float* x, __half* a_hi, __half* a_lo, float* xsum, float* rowscale, int* need_lo, long long M,
                      int K, int G, cudaStream_t st) {
  gptq_split_kernel<<<(unsigned)M, 256, 0, st>>>(x, a_hi, a_lo, xsum, rowscale, need_lo, K, G);
  SB_LAUNCHED();
  return SB200_OK;
}

static int g_tc_backoff_ns = 0;
void gptq4_tc_set_backoff(int ns) { g_tc_backoff_ns = ns; }
int gptq4_tc_backoff() { return g_tc_backoff_ns; }

bool gptq4_tc_supported(const void* x, const int32_t* qweight, const float* out, long long M, long long K, long long N,
                        long long KW, int group_size) {
  (void)out;
  (void)KW;
  if (!get_encode()) return false;
  if (K % 8 != 0 || N % 4 != 0) return false;               // TMA global strides must be multiples of 16 B
  if (group_size % kGroupK != 0) return false;              // one (scale, zero) per 128-K block
  if (!aligned16(x) || !aligned16(qweight)) return false;
  if (M < 1 || K < 8 || N < 4) return false;
  return true;
}

size_t gptq4_tc_workspace(long long M, long long K, long long N, int group_size) {
  if (K % 8 != 0 || N % 4 != 0 || group_size % kGroupK != 0) return 0;
  return tc_layout(M, K, N, (K + group_size - 1) / group_size).total + 1024;
}

// x_h != nullptr: fp16 activations in, fp16 `out_h = bias + x @ W` out (sb200_gptq4_linear_f16); else the fp32 contract.
int gptq4_tc(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
             long long K, long long N, long long KW, int group_size, void* workspace, size_t workspace_bytes,
             cudaStream_t st, const __half* x_h, __half* out_h, const float* bias) {
  const int Gq = (int)((K + group_size - 1) / group_size);
  const TcWorkspace w = tc_layout(M, K, N, Gq);
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  if (!workspace || (size_t)(ws - reinterpret_cast<unsigned char*>(workspace)) + w.total > workspace_bytes) {
    set_error("gptq4_tc: workspace too small");
    return SB200_E_WORKSPACE;
  }
  __half* a_hi = reinterpret_cast<__half*>(ws + w.off_hi);
  __half* a_lo = reinterpret_cast<__half*>(ws + w.off_lo);
  float* xsum = reinterpret_cast<float*>(ws + w.off_xsum);
  float* rowscale = reinterpret_cast<float*>(ws + w.off_rs);
  __half* zint = reinterpret_cast<__half*>(ws + w.off_zint);
  int* flag = reinterpret_cast<int*>(ws + w.off_flag);
  const int G128 = (int)((K + kGroupK - 1) / kGroupK);

  SB_CUDA(cudaMemsetAsync(flag, 0xFF, sizeof(int), st));      // [0] assume integer zero points until disproved
  SB_CUDA(cudaMemsetAsync(flag + 1, 0, sizeof(int), st));     // [1] need_lo: set by the split kernel
  gptq_zero_probe_kernel<<<(unsigned)(((long long)N * Gq + 255) / 256), 256, 0, st>>>(scales, zeros, (long long)N * Gq, zint, flag);
  SB_LAUNCHED();
  if (x_h)  // need_lo stays 0: the lo plane is never loaded
    gptq_permute_f16_kernel<<<(unsigned)M, 256, 0, st>>>(x_h, a_hi, xsum, rowscale, (int)K, G128);
  else
    gptq_split_kernel<<<(unsigned)M, 256, 0, st>>>(x, a_hi, a_lo, xsum, rowscale, flag + 1, (int)K, G128);
  SB_LAUNCHED();

  CUtensorMap map_hi, map_lo, map_q;
  if (!make_wg_maps(&map_hi, &map_lo, &map_q, a_hi, a_lo, qweight, M, K, N, KW)) {
    set_error("gptq4_tc: cuTensorMapEncodeTiled failed (M=%lld K=%lld N=%lld)", M, K, N);
    return SB200_E_CUDA;
  }
  const size_t smem = (size_t)kTcStages * kWgStageBytes + sizeof(StageRing<kTcStages>) + 1024;
  auto* const kernel = x_h ? gptq4_tc_kernel<true> : gptq4_tc_kernel<false>;
  static std::atomic<int> attr_done[2][64];
  SB_CUDA(ensure_dyn_smem(kernel, (int)smem, attr_done[x_h ? 1 : 0]));
  // one CTA per tile, token tile fastest: CTAs running side by side share the packed weight tile through L2
  const long long tiles = ((M + kWgTok - 1) / kWgTok) * ((N + kWgFeat - 1) / kWgFeat);
  kernel<<<(unsigned)tiles, kWgThreads, smem, st>>>(map_hi, map_lo, map_q, out, scales, zeros, xsum, rowscale, zint, flag,
                                                   (int)M, (int)K, (int)N, Gq, G128, group_size, g_tc_backoff_ns, out_h, bias);
  SB_LAUNCHED();
  return SB200_OK;
}

}  // namespace sb200
