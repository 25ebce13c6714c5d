// gptq_ts.cu -- GPTQ int4 group-wise dequant-matmul on wgmma with the SCALED weights as the register operand.
//
// Replaces VecQuant4MatMulKernel (large_language_models/llama/quantization/cuda/cuda_kernel_4bit.cu:88-180) for
// prefill-sized M:   out[m, n] += sum_k (scales[n, k/gs] * q[k, n] - zeros[n, k/gs]) * x[m, k]
//
// Why a second tensor-core kernel.  gptq_tc.cu keeps the int4 values exact in the MMA and applies the per-group fp32
// scale on the accumulator every 128 K.  Here the scale goes INTO the operand instead:
//   w'[n, k] = 2^e[n] * scales[n, g] * (q[k, n] - zero[n, g])  =  w_hi + w_lo     (two fp16 planes, 22 bits)
// built with error-free half2 arithmetic (hi = s_hi * d rounded, t = fma(s_hi, d, -hi) exact, lo = fma(s_lo, d, t)),
// so the accumulator runs over the whole K with no per-group epilogue.  The transposed problem is computed,
//   D[n, m] = sum_k w'[n, k] * x'[m, k],
// the weight planes are the A operand, built by every consumer thread in its own wgmma register fragment; the
// activations x' = x * 2^-ex[m] = x_hi + x_lo (fp16 planes from gptq_split_kernel) are the B operand (tc_common.cuh).
// wgmmas per 64-K stage: w_hi x_hi, w_lo x_hi (+ w_hi x_lo unless the activations are fp16-exact, which is the
// reference's model path, utils/quant.py:262-277), all m64n128k16 into one fp32 register accumulator.
//
// Accumulator rounding.  The tensor core does not round to nearest when it accumulates, so a K = 4096 chain of 512
// MMAs could lose ~1e-5.  The accumulator is therefore restarted every `chunk` 64-K stages (default 8 = 512 K) and
// added into a second fp32 register accumulator with round-to-nearest.
// Zero points.  GPTQ checkpoints store zeros = zero * scale with an integer zero (utils/quant.py:188); the prepare
// kernel verifies that on the device.  If it does not hold, the MMA runs on q - rint(zero) and the epilogue subtracts
// the residual times sum_k x'[m, k in g] (the per-128-K row sums gptq_split_kernel already produces).
#include "tc_common.cuh"

namespace sb200 {

constexpr int kTsStages = 5;
constexpr int kGroup128 = 128;

struct TsSmem {
  uint64_t full[kTsStages];   // TMA data of the stage landed
  uint64_t empty[kTsStages];  // the 8 consumer warps' wgmmas reading the stage completed
};

// ---------------------------------------------------------------------------------- weight-side prepare kernel
// One thread per output feature n.  Splits zeros[n, g] = (zero + delta) * scales[n, g] into the nearest integer
// zero (|zero| <= 1024, goes into the MMA operand as q - zero) and a residual; flag[0] is cleared if any residual
// is not negligible (then the epilogue subtracts residual * row sums).  Picks the power-of-two normalisation e[n]
// so that 2^e * max_g |scale| * max |q - zero| lies in [2^14, 2^15), and writes per (n, g):
//   { fp16 hi | fp16 lo << 16 of 2^e * scale ,  fp16 bits of zero }.
// integer part of the zero point that goes into the MMA operand: rint(zeros / scale) clamped to |.| <= 1024 (so that
// 1024 + zero and q - zero are exact fp16 integers); 0 for non-finite ratios
__device__ __forceinline__ float ts_zero_int(float z, float s) {
  const float r = rintf(z / s);
  return (fabsf(r) <= 1024.f) ? r : (r > 1024.f ? 1024.f : (r < -1024.f ? -1024.f : 0.f));
}

__global__ void gptq_ts_prepare_kernel(const float* __restrict__ scales, const float* __restrict__ zeros, int N, int Gq,
                                       uint2* __restrict__ sz, float* __restrict__ colscale, int* __restrict__ flag) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float smax = 0.f, dmax = 15.f;
  bool all_ok = true;
  for (int g = 0; g < Gq; ++g) {
    const float s = scales[(size_t)n * Gq + g], z = zeros[(size_t)n * Gq + g];
    const float zi = ts_zero_int(z, s);
    all_ok &= fabsf(fmaf(-zi, s, z)) <= fabsf(z) * 0x1p-20f + 1e-30f;
    dmax = fmaxf(dmax, fmaxf(fabsf(zi), fabsf(15.f - zi)));
    if (fabsf(s) < __int_as_float(0x7f800000)) smax = fmaxf(smax, fabsf(s));
  }
  if (!all_ok) atomicAnd(flag, 0);
  int e = 0;
  const float p = smax * dmax;
  if (p > 0.f && p < __int_as_float(0x7f800000)) e = 14 - ilogbf(p);
  e = max(-100, min(100, e));
  colscale[n] = ldexpf(1.f, -e);
  for (int g = 0; g < Gq; ++g) {
    const float s = scales[(size_t)n * Gq + g], z = zeros[(size_t)n * Gq + g];
    const float zi = ts_zero_int(z, s);
    const float sp = ldexpf(s, e);
    const __half hi = __float2half_rn(sp);
    const __half lo = __float2half_rn(sp - __half2float(hi));
    uint2 v;
    v.x = (uint32_t)__half_as_ushort(hi) | ((uint32_t)__half_as_ushort(lo) << 16);
    v.y = (uint32_t)__half_as_ushort(__float2half_rn(zi));
    sz[(size_t)n * Gq + g] = v;
  }
}

// ---------------------------------------------------------------------------------- main kernel
// One CTA per 128-feature x 128-token tile (token tile fastest, so CTAs running side by side share the packed weight
// tile through L2).
__global__ void __launch_bounds__(kWgThreads, 1)
gptq4_ts_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                const __grid_constant__ CUtensorMap map_q, float* __restrict__ out, const float* __restrict__ scales,
                const float* __restrict__ zeros,
                const float* __restrict__ xsum, const float* __restrict__ rowscale, const uint2* __restrict__ sz,
                const float* __restrict__ colscale, const int* __restrict__ flags, int M, int K, int N, int Gq, int G128,
                int group_size, int chunk_kb, __half* __restrict__ out_h, const float* __restrict__ bias, int backoff_ns) {
  // out_h != nullptr: fp16 result  out_h[m, n] = bias[n] + x @ W  (overwrite, no read of `out`); otherwise the fp32
  // accumulate-in-place contract of the reference kernel, out[m, n] += x @ W.
  extern __shared__ unsigned char smem_raw[];
  unsigned char* stage_base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  TsSmem* sm = reinterpret_cast<TsSmem*>(stage_base + (size_t)kTsStages * kWgStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + kWgTok - 1) / kWgTok;
  const int m0 = (int)(blockIdx.x % (unsigned)tiles_m) * kWgTok, n0 = (int)(blockIdx.x / (unsigned)tiles_m) * kWgFeat;
  const int num_kb = (K + kWgBK - 1) / kWgBK;
  const bool int_zero = flags[0] != 0;  // uniform: every zeros[n, g] is an integer multiple of scales[n, g] (no residual)
  const bool need_lo = flags[1] != 0;   // uniform: some activation has a non-zero fp16 low part

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_lo) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
    for (int s = 0; s < kTsStages; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], 8);  // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ================================================================== TMA producer
    reg_dec<40>();
    if (threadIdx.x == 0)
      wg_produce(stage_base, sm->full, sm->empty, kTsStages, &map_hi, &map_lo, &map_q, m0, n0, num_kb, need_lo, backoff_ns);
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
  float acc[64], c[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0.f;
  for (int kb = 0; kb < num_kb;) {
    const int kb_end = min(num_kb, kb + chunk_kb);
    for (bool first = true; kb < kb_end; ++kb, first = false) {
      const int s = kb % kTsStages;
      const uint32_t ph = (uint32_t)(kb / kTsStages) & 1u;
      const int gq = (int)((long long)kb * kWgBK / group_size);
      // {fp16 hi | fp16 lo << 16 of 2^e * scale, fp16 bits of the integer zero} of both rows for this stage's group
      const uint2 pa = live_a ? __ldg(sz + (size_t)na * Gq + gq) : make_uint2(0u, 0u);
      const uint2 pb = live_b ? __ldg(sz + (size_t)nb * Gq + gq) : make_uint2(0u, 0u);
      const __half2 sha = __half2half2(__ushort_as_half((unsigned short)(pa.x & 0xFFFFu)));
      const __half2 sla = __half2half2(__ushort_as_half((unsigned short)(pa.x >> 16)));
      const __half2 shb = __half2half2(__ushort_as_half((unsigned short)(pb.x & 0xFFFFu)));
      const __half2 slb = __half2half2(__ushort_as_half((unsigned short)(pb.x >> 16)));
      const __half2 offa = unpack.offset(__half2float(__ushort_as_half((unsigned short)pa.y)));
      const __half2 offb = unpack.offset(__half2float(__ushort_as_half((unsigned short)pb.y)));
      mbar_wait_relaxed(&sm->full[s], ph, 0);
      const uint32_t* bq = reinterpret_cast<const uint32_t*>(stage_base + (size_t)s * kWgStageBytes + 2 * kWgXBytes);
      uint32_t H[4][4], L[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // 16 K = packed rows 2j (K 0..7) and 2j + 1 (K 8..15)
#pragma unroll
        for (int r = 0; r < 4; ++r) {  // fragment register r: row f0 / f0 + 8 (r & 1), K half (r >> 1)
          const bool rb = (r & 1) != 0;
          const __half2 d = unpack(bq[(2 * j + (r >> 1)) * kWgFeat + f0 + (rb ? 8 : 0)], rb ? offb : offa);  // q - zero
          const __half2 sh = rb ? shb : sha, sl = rb ? slb : sla;
          const __half2 hi = __hmul2(sh, d);               // RN16(s_hi * d)
          const __half2 tt = __hfma2(sh, d, __hneg2(hi));  // s_hi * d - hi, exact
          H[j][r] = h2u(hi);
          L[j][r] = h2u(__hfma2(sl, d, tt));               // + s_lo * d
        }
      }
      const uint32_t xh = stage0 + (uint32_t)s * kWgStageBytes;
      const uint64_t dh = gmma_desc_sw128(xh), dl = gmma_desc_sw128(xh + kWgXBytes);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) wgmma_m64n128k16_rs(c, H[j], dh + 2 * j, !(first && j == 0));
#pragma unroll
      for (int j = 0; j < 4; ++j) wgmma_m64n128k16_rs(c, L[j], dh + 2 * j, 1);
      if (need_lo) {
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_m64n128k16_rs(c, H[j], dl + 2 * j, 1);
      }
      wgmma_commit();
      wgmma_wait_all(c);
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm->empty[s]);
    }
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] += c[j];
  }
  // d[j]: feature f0 + 8 * ((j >> 1) & 1), token m0 + 8 (j >> 2) + 2q + (j & 1)
  const float csa = live_a ? __ldg(colscale + na) : 0.f, csb = live_b ? __ldg(colscale + nb) : 0.f;
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] *= (j & 2) ? csb : csa;
  if (!int_zero) {
    // zero points with a fractional part: the MMA used q - rint(zero); subtract the residual
    //   out = rs * (cs * acc - sum_g (zeros[n, g] - rint(zero) * scales[n, g]) * xsum[m, g])
    for (int g = 0; g < G128; ++g) {
      const int gq = (int)((long long)g * kGroup128 / group_size);
      float zr[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = h ? nb : na;
        if (n < N) {
          const float zi = __half2float(__ushort_as_half((unsigned short)__ldg(&sz[(size_t)n * Gq + gq].y)));
          zr[h] = -fmaf(-zi, __ldg(scales + (size_t)n * Gq + gq), __ldg(zeros + (size_t)n * Gq + gq));
        }
      }
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int m = m0 + 8 * (j >> 2) + 2 * q + (j & 1);
        if (m < M) acc[j] = fmaf(zr[(j >> 1) & 1], __ldg(xsum + (size_t)m * G128 + g), acc[j]);
      }
    }
  }
  const float bna = (out_h && bias && live_a) ? __ldg(bias + na) : 0.f;
  const float bnb = (out_h && bias && live_b) ? __ldg(bias + nb) : 0.f;
#pragma unroll
  for (int j = 0; j < 64; ++j) {
    const int m = m0 + 8 * (j >> 2) + 2 * q + (j & 1);
    const int n = (j & 2) ? nb : na;
    if (m < M && n < N) {
      const float rs = __ldg(rowscale + m);
      if (out_h) {
        out_h[(size_t)m * N + n] = __float2half_rn(fmaf(rs, acc[j], (j & 2) ? bnb : bna));
      } else {
        float* o = out + (size_t)m * N + n;
        *o = fmaf(rs, acc[j], *o);
      }
    }
  }
}

// ---------------------------------------------------------------------------------- host side
int gptq_launch_split(const float* x, __half* a_hi, __half* a_lo, float* xsum, float* rowscale, int* need_lo, long long M,
                      int K, int G, cudaStream_t st);  // gptq_tc.cu
int gptq4_tc_backoff();                                // gptq_tc.cu

struct TsWorkspace {
  size_t off_hi, off_lo, off_xsum, off_rs, off_sz, off_cs, off_flag, total;
};
static TsWorkspace ts_layout(long long M, long long K, long long N, long long Gq) {
  TsWorkspace w;
  const long long G128 = (K + kGroup128 - 1) / kGroup128;
  w.off_hi = 0;
  w.off_lo = align_up((size_t)M * K * 2, 1024);
  w.off_xsum = w.off_lo + align_up((size_t)M * K * 2, 1024);
  w.off_rs = w.off_xsum + align_up((size_t)M * G128 * 4, 1024);
  w.off_sz = w.off_rs + align_up((size_t)M * 4, 1024);
  w.off_cs = w.off_sz + align_up((size_t)N * Gq * 8, 1024);
  w.off_flag = w.off_cs + align_up((size_t)N * 4, 1024);
  w.total = w.off_flag + 1024;
  return w;
}

// fp16 activations: the hi plane IS the input (no row scaling needed: |x| <= 65504 and |w'| < 2^15 keep every product
// inside fp32), copied with every 8 K permuted to (0, 4, 1, 5, 2, 6, 3, 7) to match the nibble pairs one LOP3 extracts;
// xsum[m, g] = sum over the 128-K block (only read when some zero point has a fractional part).
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

size_t gptq4_ts_workspace(long long M, long long K, long long N, int group_size) {
  if (K % 8 != 0 || N % 4 != 0 || group_size % kGroup128 != 0) return 0;
  return ts_layout(M, K, N, (K + group_size - 1) / group_size).total + 1024;
}

// x_h != nullptr: fp16 activations in, fp16 `out_h = bias + x @ W` out (sb200_gptq4_linear_f16); else the fp32 contract.
int gptq4_ts(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
             long long K, long long N, long long KW, int group_size, int chunk_kb, void* workspace, size_t workspace_bytes,
             cudaStream_t st, const __half* x_h, __half* out_h, const float* bias) {
  const int Gq = (int)((K + group_size - 1) / group_size);
  const TsWorkspace w = ts_layout(M, K, N, Gq);
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  if (!workspace || (size_t)(ws - reinterpret_cast<unsigned char*>(workspace)) + w.total > workspace_bytes) {
    set_error("gptq4_ts: workspace too small");
    return SB200_E_WORKSPACE;
  }
  if (chunk_kb <= 0) chunk_kb = 8;
  __half* a_hi = reinterpret_cast<__half*>(ws + w.off_hi);
  __half* a_lo = reinterpret_cast<__half*>(ws + w.off_lo);
  float* xsum = reinterpret_cast<float*>(ws + w.off_xsum);
  float* rowscale = reinterpret_cast<float*>(ws + w.off_rs);
  uint2* sz = reinterpret_cast<uint2*>(ws + w.off_sz);
  float* cs = reinterpret_cast<float*>(ws + w.off_cs);
  int* flag = reinterpret_cast<int*>(ws + w.off_flag);
  const int G128 = (int)((K + kGroup128 - 1) / kGroup128);

  SB_CUDA(cudaMemsetAsync(flag, 0xFF, sizeof(int), st));   // [0] integer zero points until disproved
  SB_CUDA(cudaMemsetAsync(flag + 1, 0, sizeof(int), st));  // [1] need_lo, set by the split kernel
  gptq_ts_prepare_kernel<<<(unsigned)((N + 127) / 128), 128, 0, st>>>(scales, zeros, (int)N, Gq, sz, cs, flag);
  SB_LAUNCHED();
  if (x_h) {
    gptq_permute_f16_kernel<<<(unsigned)M, 256, 0, st>>>(x_h, a_hi, xsum, rowscale, (int)K, G128);
    SB_LAUNCHED();
  } else if (const int rc = gptq_launch_split(x, a_hi, a_lo, xsum, rowscale, flag + 1, M, (int)K, G128, st)) {
    return rc;
  }

  CUtensorMap map_hi, map_lo, map_q;
  if (!make_wg_maps(&map_hi, &map_lo, &map_q, a_hi, a_lo, qweight, M, K, N, KW)) {
    set_error("gptq4_ts: cuTensorMapEncodeTiled failed (M=%lld K=%lld N=%lld)", M, K, N);
    return SB200_E_CUDA;
  }
  const size_t smem = (size_t)kTsStages * kWgStageBytes + sizeof(TsSmem) + 1024;
  static std::atomic<int> attr_done[64];
  SB_CUDA(ensure_dyn_smem(gptq4_ts_kernel, (int)smem, attr_done));
  const long long tiles = ((M + kWgTok - 1) / kWgTok) * ((N + kWgFeat - 1) / kWgFeat);
  gptq4_ts_kernel<<<(unsigned)tiles, kWgThreads, smem, st>>>(map_hi, map_lo, map_q, out, scales, zeros, xsum, rowscale, sz, cs,
                                                            flag, (int)M, (int)K, (int)N, Gq, G128, group_size, chunk_kb,
                                                            out_h, bias, gptq4_tc_backoff());
  SB_LAUNCHED();
  return SB200_OK;
}

}  // namespace sb200
