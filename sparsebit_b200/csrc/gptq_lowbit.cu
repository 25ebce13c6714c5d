// gptq_lowbit.cu -- GPTQ 3-bit / 2-bit group-wise dequant-matmul (SURVEY §8f #3), HBM-bound SIMT.
//
// Replaces large_language_models/llama/quantization/cuda/cuda_kernel_3bit.cu and cuda_kernel_2bit.cu
// (VecQuant3MatMulKernel / VecQuant2MatMulKernel; bindings cuda_kernel.cpp:26-57) behind the same
// contract:  out[m, n] += sum_k (scales[n*G + k/gs] * q(k, n) - zeros[n*G + k/gs]) * x[m, k].
//
// Packed layouts (QuantLinear.pack, utils/quant.py:210-258), LSB first, rows along K:
//   2-bit: 16 values per int32 word.
//   3-bit: 32 values per 3 words; value 10 straddles words 0/1 (2 + 1 bits), value 21 straddles
//          words 1/2 (1 + 2 bits); the other 30 sit at 3 j (+1, +2 in words 1, 2).
// A "unit" is 32 consecutive k (2 words for 2-bit, 3 words for 3-bit); a K block is 64 (2-bit) or
// 128 (3-bit) values, which never straddles a group because group_size % 64 (% 128) == 0
// (cuda_kernel_2bit.cu:58, cuda_kernel_3bit.cu:60).
//
// Same shape as the 4-bit SIMT kernel (gptq_simt.cu): one thread per output column so that a warp reads
// 128 contiguous bytes of every packed row, the CTA's activation slice sits in shared memory, the next
// block's words are in flight while the current one is decoded, and the per-group affine is applied once
// per block:  sum_k (s q - z) x = s * (sum_k q x) - z * (sum_k x).
#include "common.cuh"
#include "gptq_unpack.cuh"

namespace sb200 {
namespace {

constexpr int kCols = 128;

template <int BITS>
struct Fmt;
template <>
struct Fmt<2> {
  static constexpr int kUnitWords = 2, kUnits = 2;  // block = 64 k, 4 words
};
template <>
struct Fmt<3> {
  static constexpr int kUnitWords = 3, kUnits = 4;  // block = 128 k, 12 words
};

// Dynamic shared memory: xs[MT][S * BK] activations of the CTA's K slice, then xsum[MT][S].
template <int BITS, int MT>
__global__ void __launch_bounds__(kCols) gptq_lowbit_kernel(const float* __restrict__ x, const uint32_t* __restrict__ qw,
                                                            float* __restrict__ out, const float* __restrict__ scales,
                                                            const float* __restrict__ zeros, int M, int K, int N, int KW,
                                                            int G, int group_size, int blocks_per_slice) {
  using F = Fmt<BITS>;
  constexpr int kWords = F::kUnitWords * F::kUnits;
  constexpr int kBlockK = 32 * F::kUnits;
  extern __shared__ __align__(16) float smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = blockIdx.x * kCols + tid;
  const bool col_ok = n < N;
  const int nblk = (K + kBlockK - 1) / kBlockK;
  const int b0 = blockIdx.y * blocks_per_slice;
  const int nb = min(b0 + blocks_per_slice, nblk) - b0;
  const int slice_k = blocks_per_slice * kBlockK;
  float* xs = smem_f;
  float* xsum = smem_f + MT * slice_k;
  const uint32_t* wcol = qw + n;

  auto load_block = [&](int b, uint32_t (&w)[kWords]) {
    const int row0 = b * kWords;
#pragma unroll
    for (int r = 0; r < kWords; ++r) w[r] = (col_ok && row0 + r < KW) ? __ldcs(wcol + (size_t)(row0 + r) * N) : 0u;
  };

  for (int m0 = 0; m0 < M; m0 += MT) {
    uint32_t wa[kWords], wb[kWords];
    load_block(b0, wa);
    __syncthreads();  // previous row group is done with xs / xsum
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
#pragma unroll
      for (int m = 0; m < MT; ++m) acc[m] += fmaf(sc, dot[m], -zr * xsum[m * blocks_per_slice + bl]);
    };
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
int launch_lowbit(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
                  long long K, long long N, long long KW, int group_size, cudaStream_t st) {
  constexpr int kBlockK = 32 * Fmt<BITS>::kUnits;
  const int G = (int)((K + group_size - 1) / group_size);
  const int nblk = (int)((K + kBlockK - 1) / kBlockK);
  const int colblocks = (int)((N + kCols - 1) / kCols);
  int want_slices = (sm_count() * 8 + colblocks - 1) / colblocks;
  want_slices = want_slices < 1 ? 1 : (want_slices > nblk ? nblk : want_slices);
  int S = (nblk + want_slices - 1) / want_slices;
  const int s_cap = 1024 / kBlockK;  // <= 1024 staged activations per row (32 KB at MT = 8)
  if (S > s_cap) S = s_cap;
  const int slices = (nblk + S - 1) / S;
  const dim3 grid((unsigned)colblocks, (unsigned)slices);
  const uint32_t* qw = reinterpret_cast<const uint32_t*>(qweight);
#define SB_GO(MT_)                                                                                                  \
  gptq_lowbit_kernel<BITS, MT_><<<grid, kCols, (size_t)(MT_) * S * (kBlockK + 1) * sizeof(float), st>>>(            \
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

int gptq_lowbit(int bits, const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros,
                long long M, long long K, long long N, long long KW, int group_size, cudaStream_t st) {
  if (bits == 2) return launch_lowbit<2>(x, qweight, out, scales, zeros, M, K, N, KW, group_size, st);
  return launch_lowbit<3>(x, qweight, out, scales, zeros, M, K, N, KW, group_size, st);
}

}  // namespace sb200
