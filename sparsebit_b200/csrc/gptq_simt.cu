// gptq_simt.cu -- GPTQ 2 / 3 / 4-bit group-wise dequant-matmul, HBM-bound SIMT path (4-bit: decode / small M and
// every shape the decode and tensor-core kernels cannot take; 3 / 2-bit: every shape, SURVEY §8f #3).
//
// Replaces large_language_models/llama/quantization/cuda/cuda_kernel_{4,3,2}bit.cu
// (VecQuant{4,3,2}MatMulKernel) behind the same contract (cuda_kernel.cpp:10-57):
//   out[m, n] += sum_k (scales[n*G + k/gs] * q(k, n) - zeros[n*G + k/gs]) * x[m, k]
//
// Layout facts taken from the reference: qweight int32 [packed rows, N] (gptq_unpack.cuh); scales / zeros are [N, G]
// with zeros = zero*scale (utils/quant.py:188); a K block never straddles a group (gptq_unpack.cuh).
//
// Design: one thread per output column (coalesced 128 B weight rows per warp), a CTA owns a
// [S*kBlockK x 128] slab of the packed matrix, all word loads of a K block are issued before
// the first is used, the activation block lives in shared memory (broadcast float4 reads) and
// the per-group affine is applied once per block on the integer dot product:
//   sum_k (s*q - z) * x  =  s * (sum_k q*x) - z * (sum_k x)
// so the 4-bit inner loop is nibble -> float (3 ALU ops) + MT FMAs.  K is split across CTAs; partial
// results are combined with fp32 atomicAdd exactly like the reference (cuda_kernel_4bit.cu:158,179).
#include "gptq_launch.cuh"
#include "gptq_unpack.cuh"

namespace sb200 {
namespace {

constexpr int kCols = 128;  // threads per CTA == output columns per CTA

// Nibble j (0..3) of `v` WITHOUT shifting it down: masking it in place inside the mantissa of 2^23
// gives the float 2^23 + q * 16^j, and subtracting 2^23 leaves q * 16^j exactly.  The factor 16^j
// is cancelled by staging the activations pre-multiplied by 16^-(k % 4) (exact powers of two), so a
// packed word costs 1 shift (for its upper half) + 8 x (LOP3, FADD, FFMA) instead of 8 extra shifts
// and no I2F at all.  4-bit only: the 2 / 3-bit values do not sit on 4-bit boundaries.
// `magic` (= 0x4B000000, the bits of 2^23) is kept in a register so that (v & mask) | magic is ONE
// LOP3 (a LOP3 takes a single immediate; with two the compiler emits an AND and an OR).
template <int J>
__device__ __forceinline__ float nib_scaled(uint32_t v, uint32_t magic) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(v), "n"(0xFu << (4 * J)), "r"(magic));
  return __uint_as_float(r) - 8388608.0f;
}
__device__ __forceinline__ uint32_t opaque_magic() {
  uint32_t m;
  asm volatile("mov.b32 %0, 0x4B000000;" : "=r"(m));
  return m;
}

// Dynamic shared memory: xs[MT][S * kBlockK] activations of the CTA's whole K slice, then xsum[MT][S].
// 4-bit keeps 8 (MT <= 2) or 5 resident CTAs per SM; 0 leaves 2 / 3-bit to the compiler.
template <int BITS, int MT>
__global__ void __launch_bounds__(kCols, BITS == 4 ? ((MT <= 2) ? 8 : 5) : 0)
gptq_simt_kernel(const float* __restrict__ x, const uint32_t* __restrict__ qw, float* __restrict__ out,
                 const float* __restrict__ scales, const float* __restrict__ zeros, int M, int K, int N, int KW, int G,
                 int group_size, int blocks_per_slice) {
  using F = GptqFmt<BITS>;
  constexpr int kWords = F::kBlockWords, kBlockK = F::kBlockK;
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = blockIdx.x * kCols + tid;
  const bool col_ok = n < N;
  const int nblk = (K + kBlockK - 1) / kBlockK;
  const int b0 = blockIdx.y * blocks_per_slice;
  const int nb = min(b0 + blocks_per_slice, nblk) - b0;
  const int slice_k = blocks_per_slice * kBlockK;
  float* xs = smem_f;                   // [MT][slice_k]
  float* xsum = smem_f + MT * slice_k;  // [MT][blocks_per_slice]
  const uint32_t* wcol = qw + n;
  uint32_t magic;
  if constexpr (BITS == 4) magic = opaque_magic();

  auto load_block = [&](int b, uint32_t (&w)[kWords]) {
    const int row0 = b * kWords;
#pragma unroll
    for (int r = 0; r < kWords; ++r) w[r] = (col_ok && row0 + r < KW) ? __ldcs(wcol + (size_t)(row0 + r) * N) : 0u;
  };

  for (int m0 = 0; m0 < M; m0 += MT) {
    // the first block's packed words are requested before anything else
    uint32_t wa[kWords], wb[kWords];
    load_block(b0, wa);
    // stage x[m0..m0+MT, slice] (zero padded) once, and the per-block row sums
    __syncthreads();  // previous row group is done with xs / xsum
    if constexpr (BITS == 4) {
      // xs holds x * 16^-(k % 4) (see nib_scaled); tid % 4 == k % 4 because every stride is a multiple of 4
      const float down = __uint_as_float((127u - 4u * (tid & 3)) << 23);  // 16^-(tid % 4)
      const float up = __uint_as_float((127u + 4u * (tid & 3)) << 23);
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const float* xrow = x + (size_t)(m0 + m) * K + (size_t)b0 * kBlockK;
        for (int kk = tid; kk < slice_k; kk += kCols) {
          const bool ok = (m0 + m < M) && (b0 * kBlockK + kk < K) && (kk < nb * kBlockK);
          xs[m * slice_k + kk] = ok ? __ldg(xrow + kk) * down : 0.f;
        }
      }
      __syncthreads();
      for (int p = wid; p < MT * blocks_per_slice; p += kCols / 32) {
        const float* src = xs + (size_t)p * kBlockK;  // p = m * blocks_per_slice + b ; lane % 4 == k % 4
        float v = (src[lane] + src[lane + 32] + src[lane + 64] + src[lane + 96]) * up;
        v = warp_sum(v);
        if (lane == 0) xsum[p] = v;
      }
    } else {
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const float* xrow = x + (size_t)(m0 + m) * K + (size_t)b0 * kBlockK;
        for (int kk = tid; kk < slice_k; kk += kCols) {
          const bool ok = (m0 + m < M) && ((long long)b0 * kBlockK + kk < K) && (kk < nb * kBlockK);
          xs[m * slice_k + kk] = ok ? __ldg(xrow + kk) : 0.f;
        }
      }
      __syncthreads();
      for (int p = wid; p < MT * blocks_per_slice; p += kCols / 32) {
        const float* src = xs + (size_t)p * kBlockK;  // p = m * blocks_per_slice + block
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < kBlockK / 32; ++j) v += src[lane + 32 * j];
        v = warp_sum(v);
        if (lane == 0) xsum[p] = v;
      }
    }
    __syncthreads();

    float acc[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m] = 0.f;
    auto compute = [&](int bl, const uint32_t (&w)[kWords]) {
      const int g = ((b0 + bl) * kBlockK) / group_size;
      const float sc = col_ok ? __ldg(scales + (size_t)n * G + g) : 0.f;
      const float zr = col_ok ? __ldg(zeros + (size_t)n * G + g) : 0.f;
      float dot[MT];
#pragma unroll
      for (int m = 0; m < MT; ++m) dot[m] = 0.f;
      if constexpr (BITS == 4) {
        // nibbles decoded in place (nib_scaled), one packed word = 8 k at a time, FMAs in k order
#pragma unroll
        for (int r = 0; r < kWords; ++r) {
          float q[8];
          const uint32_t whi = w[r] >> 16;
          q[0] = nib_scaled<0>(w[r], magic); q[1] = nib_scaled<1>(w[r], magic);
          q[2] = nib_scaled<2>(w[r], magic); q[3] = nib_scaled<3>(w[r], magic);
          q[4] = nib_scaled<0>(whi, magic);  q[5] = nib_scaled<1>(whi, magic);
          q[6] = nib_scaled<2>(whi, magic);  q[7] = nib_scaled<3>(whi, magic);
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            const float* xr = xs + (size_t)m * slice_k + bl * kBlockK + r * 8;
            const float4 xa = *reinterpret_cast<const float4*>(xr);
            const float4 xb = *reinterpret_cast<const float4*>(xr + 4);
            dot[m] = fmaf(q[0], xa.x, dot[m]);
            dot[m] = fmaf(q[1], xa.y, dot[m]);
            dot[m] = fmaf(q[2], xa.z, dot[m]);
            dot[m] = fmaf(q[3], xa.w, dot[m]);
            dot[m] = fmaf(q[4], xb.x, dot[m]);
            dot[m] = fmaf(q[5], xb.y, dot[m]);
            dot[m] = fmaf(q[6], xb.z, dot[m]);
            dot[m] = fmaf(q[7], xb.w, dot[m]);
          }
        }
      } else {
#pragma unroll
        for (int u = 0; u < F::kUnits; ++u) {
          float q[32];
          decode_unit<BITS>(&w[u * F::kUnitWords], q);
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            const float4* xr = reinterpret_cast<const float4*>(xs + (size_t)m * slice_k + bl * kBlockK + u * 32);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 xv = xr[j];
              dot[m] = fmaf(q[4 * j + 0], xv.x, dot[m]);
              dot[m] = fmaf(q[4 * j + 1], xv.y, dot[m]);
              dot[m] = fmaf(q[4 * j + 2], xv.z, dot[m]);
              dot[m] = fmaf(q[4 * j + 3], xv.w, dot[m]);
            }
          }
        }
      }
#pragma unroll
      for (int m = 0; m < MT; ++m) acc[m] += fmaf(sc, dot[m], -zr * xsum[m * blocks_per_slice + bl]);
    };
    // software pipeline over the slice: the next block's words are in flight while this one is used
    for (int bl = 0; bl < nb; bl += 2) {
      if (bl + 1 < nb) load_block(b0 + bl + 1, wb);
      compute(bl, wa);
      if (bl + 1 < nb) {
        if (bl + 2 < nb) load_block(b0 + bl + 2, wa);
        compute(bl + 1, wb);
      }
    }
    if (col_ok) {
#pragma unroll
      for (int m = 0; m < MT; ++m)
        if (m0 + m < M) atomicAdd(out + (size_t)(m0 + m) * N + n, acc[m]);
    }
  }
}

template <int BITS>
int launch_simt(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
                long long K, long long N, long long KW, int group_size, cudaStream_t st) {
  constexpr int kBlockK = GptqFmt<BITS>::kBlockK;
  const int G = (int)((K + group_size - 1) / group_size);
  const int nblk = (int)((K + kBlockK - 1) / kBlockK);
  const int colblocks = (int)((N + kCols - 1) / kCols);
  // enough CTAs for ~8 resident per SM (1024 threads, each with 8-32 packed words in flight)
  int want_slices = (sm_count() * 8 + colblocks - 1) / colblocks;
  want_slices = want_slices < 1 ? 1 : (want_slices > nblk ? nblk : want_slices);
  int S = (nblk + want_slices - 1) / want_slices;
  const int s_cap = 1024 / kBlockK;  // <= 1024 staged activations per row (32 KB at MT = 8)
  if (S > s_cap) S = s_cap;
  const int slices = (nblk + S - 1) / S;
  const dim3 grid((unsigned)colblocks, (unsigned)slices);
  const uint32_t* qw = reinterpret_cast<const uint32_t*>(qweight);
#define SB_GO(MT_)                                                                                               \
  gptq_simt_kernel<BITS, MT_><<<grid, kCols, (size_t)(MT_) * S * (kBlockK + 1) * sizeof(float), st>>>(          \
      x, qw, out, scales, zeros, (int)M, (int)K, (int)N, (int)KW, G, group_size, S)
  if (M == 1) SB_GO(1);
  else if (M == 2) SB_GO(2);
  else if (M <= 4) SB_GO(4);
  else SB_GO(8);
#undef SB_GO
  SB_LAUNCHED();
  return SB200_OK;
}

}  // namespace

int gptq_simt(int bits, const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
              long long M, long long K, long long N, long long KW, int group_size, cudaStream_t st) {
  if (bits == 2) return launch_simt<2>(x, qweight, out, scales, zeros, M, K, N, KW, group_size, st);
  if (bits == 3) return launch_simt<3>(x, qweight, out, scales, zeros, M, K, N, KW, group_size, st);
  return launch_simt<4>(x, qweight, out, scales, zeros, M, K, N, KW, group_size, st);
}

}  // namespace sb200
