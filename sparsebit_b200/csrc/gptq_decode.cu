// gptq_decode.cu -- GPTQ int4 group-wise dequant-matmul for decode-sized M (1..32 tokens): HBM-bound, so the job is
// to stream the packed weights once at full bandwidth with as few instructions per weight as possible.
//
// Replaces VecQuant4MatMulKernel (large_language_models/llama/quantization/cuda/cuda_kernel_4bit.cu:88-180) behind
// the same contract:  out[m, n] += sum_k (scales[n, k/gs] * q[k, n] - zeros[n, k/gs]) * x[m, k].
//
// The scalar path (gptq_simt.cu) needs 3 instructions per weight (LOP3, FADD, FFMA) and is issue-bound at 0.27 of the
// HBM roofline.  Here the multiply-accumulate goes to the tensor cores through the warp-level mma.sync.m16n8k16
// (HMMA; wgmma needs 64-row warpgroup tiles, pointless for 1..32 tokens):
//   A (16 features x 16 K)  = the int4 values as EXACT fp16 integers (q in [0, 15])
//   B (16 K x 8 tokens)     = the activations x * 2^-e as fp16 hi (+ lo) planes, staged once per CTA in shared memory
//   D (16 x 8 fp32)         = integer dot products of one 128-K group; the group's scale / zero are applied in fp32:
//                             acc += scale * D - zeros * sum_k x        (same factoring as the scalar path)
// which costs ~1.3 instructions per weight: per 32-K chunk a lane issues one LDG.128 (4 packed words = 4 feature
// rows x 8 K), 9 ALU instructions per word to expand it into A fragments, one LDS.128 for the B fragments of both
// K halves and 4 HMMAs (8 with the lo plane; skipped when the activations are fp16-exact, the model path).
//
// Fragment bookkeeping.  K order inside a tile is free as long as A and B agree, and so is the row order.  Lane
// (g = lane / 4, c = lane % 4) loads the packed row kw = 4 * chunk + c for the four features n = nbase + 4 g + {0..3}
// (a warp covers 32 features x 4 packed rows: four full 128-byte lines per load instruction), which become
//   tile T in {0, 1}: row slot g  <-> feature 4 g + 2 T,   row slot g + 8 <-> feature 4 g + 2 T + 1
// and each word feeds two MMAs i in {0, 1}: columns (2c, 2c+1) <-> nibbles (2i, 2i + 4), columns (2c + 8, 2c + 9) <->
// nibbles (2i + 1, 2i + 5) -- exactly the pairs one LOP3 extracts ((w >> 8i) & 0x000F000F, & 0x00F000F0).  The
// activations are stored in shared memory with every 8 K permuted to (0, 4, 1, 5, 2, 6, 3, 7), so one 16-byte load
// returns the B registers of both MMAs.
#include <cuda_fp16.h>

#include "common.cuh"

namespace sb200 {

constexpr int kDecThreads = 128;  // 4 warps x 32 features
constexpr int kDecCols = 128;
constexpr int kDecBlockK = 128;
// SLAB variant: the CTA's whole packed-weight slab ([blocks_per_slice x 16 packed rows] x 128 features) is requested
// with one cp.async.bulk per packed row (thread t <-> row t, all issued in the first microsecond of the CTA's life,
// completion on one mbarrier per 128-K block) instead of 2 x 4 LDG.128 per lane refilled between the MMA groups: every
// byte the CTA will ever need is in flight before it touches the activations, it costs no registers, and a multi-pass
// M (> 8 NB tokens) reads the weights from DRAM once.  Rows are 544 bytes apart in shared memory (512 + 32): the four
// packed rows a quarter-warp reads with one LDS.128 then fall into disjoint bank groups.
constexpr int kSlabRowBytes = kDecCols * 4 + 32;
constexpr int kSlabGroupBytes = (kDecBlockK / 8) * kSlabRowBytes;
__device__ __forceinline__ void dec_mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <uint32_t MASK>
__device__ __forceinline__ uint32_t dec_and_or(uint32_t x, uint32_t c) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(x), "n"(MASK), "r"(c));
  return r;
}
__device__ __forceinline__ void hmma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Several independent linears that share M (q / k / v or gate / up of one decoder layer: same input, different weights)
// run as ONE launch: a decode-sized GEMV lives for a few microseconds, i.e. a handful of DRAM latencies, so launching
// them back to back leaves the memory system idle between kernels.  Passed by value (__grid_constant__).
struct DecProblem {
  const float* x;
  const uint32_t* qw;
  float* out;
  const float* scales;
  const float* zeros;
  int K, N, KW, G, group_size;
  int colblock_begin;  // first blockIdx.x of this problem
  // fp16 linear in ONE launch (sb200_gptq4_linear_f16_ex): fp16 activations in, bias + result out as fp16.  The K
  // slices cannot accumulate into an fp16 tensor, so every slice CTA stores its fp32 partial sums into its own slot of
  // `partial` ([slices][M][N], plain stores), and the LAST slice CTA of a feature block to arrive (ticket from
  // `counters[feature block]`, threadfence-reduction pattern) adds the slots in slice order, adds the bias, writes fp16
  // and resets the counter for the next call: deterministic, no fp32 staging tensors, no cast / bias / cast launches.
  const __half* x_h;   // nullable: fp16 activations (x is ignored)
  __half* out_h;       // nullable: fp16 output (out is ignored)
  const float* bias;   // nullable, fp16 path only
  float* partial;
  int* counters;
};
constexpr int kDecMaxProblems = 4;
struct DecBatch {
  DecProblem p[kDecMaxProblems];
  int count;
};

// NB = number of 8-token blocks (tokens handled per pass = 8 * NB).  Dynamic shared memory:
//   xh[8 NB][stride], xl[8 NB][stride] halves (stride = slice_k + 32: token rows start 64 bytes apart modulo 128, so the
//   8 lanes of an LDS.128 phase hit distinct banks), xsum[8 NB][blocks_per_slice] floats, escale[8 NB] floats,
//   scale / zeros [blocks_per_slice][128] floats each.
//   SLAB: the packed-weight slab [blocks_per_slice][16][544 B] comes first, and only x_rows = min(M, 8 NB) token rows
//   are allocated for xh / xl / xsum (MMA token columns beyond the real tokens re-read the last real row; their results
//   are never written back).
// pdl (bit mask): bit 0 = launched with programmatic stream serialisation: the next kernel of the stream may start
// while this one runs (griddepcontrol.launch_dependents at the top) and this kernel executes griddepcontrol.wait before
// it touches global memory -- plain stream semantics, but the launch latency and CTA ramp-up overlap the predecessor's
// tail.  bit 2 = the caller declared the packed weights, scales and zeros constants of the model (not produced by the
// kernel immediately in front on the stream): they are requested BEFORE the wait, so their DRAM latency overlaps the
// tail of the previous linear too; only the activations and `out` are behind the wait.  bit 1 = L2 prefetch (below).
template <int NB, bool SLAB>
__global__ void __launch_bounds__(kDecThreads) gptq4_decode_kernel(const __grid_constant__ DecBatch batch, int M,
                                                                 int blocks_per_slice, int x_rows, int pdl) {
  extern __shared__ __align__(16) unsigned char dsm[];
  constexpr int MT = 8 * NB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, c = lane & 3;
  int pi = 0;
#pragma unroll
  for (int i = 1; i < kDecMaxProblems; ++i)
    if (i < batch.count && (int)blockIdx.x >= batch.p[i].colblock_begin) pi = i;
  const float* __restrict__ x = batch.p[pi].x;
  const uint32_t* __restrict__ qw = batch.p[pi].qw;
  float* __restrict__ out = batch.p[pi].out;
  const float* __restrict__ scales = batch.p[pi].scales;
  const float* __restrict__ zeros = batch.p[pi].zeros;
  const __half* __restrict__ x_h = batch.p[pi].x_h;
  __half* __restrict__ out_h = batch.p[pi].out_h;
  const int K = batch.p[pi].K, N = batch.p[pi].N, KW = batch.p[pi].KW, G = batch.p[pi].G, group_size = batch.p[pi].group_size;
  const int bx = (int)blockIdx.x - batch.p[pi].colblock_begin;
  const int nblk = (K + kDecBlockK - 1) / kDecBlockK;
  const int b0 = blockIdx.y * blocks_per_slice;
  if (b0 >= nblk) return;  // a problem with a shorter K than the longest one of the batch
  const int nb = min(b0 + blocks_per_slice, nblk) - b0;
  const int slice_k = blocks_per_slice * kDecBlockK;
  const int stride = slice_k + 32;  // halves
  const int x_alloc = SLAB ? x_rows : MT;  // token rows held in shared memory
  const unsigned char* slab = dsm;
  __half* xh = reinterpret_cast<__half*>(dsm + (SLAB ? (size_t)blocks_per_slice * kSlabGroupBytes : 0));
  __half* xl = xh + x_alloc * stride;
  float* xsum = reinterpret_cast<float*>(xl + x_alloc * stride);
  float* escale = xsum + x_alloc * blocks_per_slice;
  float* s_sc = escale + MT;                          // [blocks_per_slice][128] scale of (block, feature of this CTA)
  float* s_zr = s_sc + blocks_per_slice * kDecCols;   // [blocks_per_slice][128] zeros
  __shared__ int s_need_lo;
  __shared__ unsigned int s_amax[32];
  __shared__ __align__(8) uint64_t s_bar[8];  // SLAB: one per 128-K block of the slice (blocks_per_slice <= 8)
  const int nbase = bx * kDecCols + warp * 32 + 4 * g;  // this lane's four features nbase .. nbase + 3
  const bool col_ok = nbase < N;                                  // N % 4 == 0: all four or none
  uint32_t bias;
  asm volatile("mov.b32 %0, 0x64006400;" : "=r"(bias));  // half2(1024, 1024), opaque to constant propagation
  const __half2 k1024 = __float2half2_rn(1024.f), k16 = __float2half2_rn(0.0625f), k64n = __float2half2_rn(-64.f);

  auto load_group = [&](int bl, uint4 (&w)[4]) {  // the four 32-K chunks of one 128-K block
    const int row0 = (b0 + bl) * (kDecBlockK / 8) + c;
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
      const int row = row0 + 4 * ch;
      w[ch] = (col_ok && row < KW) ? __ldcs(reinterpret_cast<const uint4*>(qw + (size_t)row * N + nbase)) : make_uint4(0u, 0u, 0u, 0u);
    }
  };

  uint4 wa[4], wb[4];
  if (pdl & 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if ((pdl & 5) == 1) asm volatile("griddepcontrol.wait;" ::: "memory");  // strict: nothing is read before the predecessor is done
  if (SLAB) {
    if (tid < nb) mbar_init(&s_bar[tid], kDecBlockK / 8);  // every row thread of a block arrives exactly once
    mbar_fence_init();
    __syncthreads();
    const int bl = tid >> 4, r = tid & 15;
    if (bl < nb) {
      const int row = (b0 + bl) * (kDecBlockK / 8) + r;
      unsigned char* dst = dsm + (size_t)(bl * (kDecBlockK / 8) + r) * kSlabRowBytes;
      const int col0 = bx * kDecCols;
      const uint32_t bytes = (uint32_t)min(kDecCols, N - col0) * 4u;  // N % 4 == 0: a multiple of 16
      if (row < KW) {
        mbar_expect_tx(&s_bar[bl], bytes);
        tma_bulk_g2s(dst, qw + (size_t)row * N + col0, bytes, &s_bar[bl]);
      } else {  // K % 128 != 0: rows past the packed matrix contribute nothing
        for (int j = 0; j < kDecCols / 4; ++j) reinterpret_cast<uint4*>(dst)[j] = make_uint4(0u, 0u, 0u, 0u);
        dec_mbar_arrive(&s_bar[bl]);
      }
    }
  } else {
    load_group(0, wa);
    if (nb > 1) load_group(1, wb);
    if (pdl & 2) {
      // The register file holds two 128-K blocks per lane; the blocks after them are requested into L2 right away
      // (one prefetch per 128-byte line: a warp's LDG.128 covers four lines, lanes g == 0 own one each), so that every
      // byte of the CTA's slice is on its way from DRAM before the activations are staged and the refills between the
      // MMA groups hit L2 instead of paying a DRAM round trip in the middle of the CTA's short life.
      if (g == 0 && col_ok) {
        for (int bl = 2; bl < nb; ++bl) {
          const int row0 = (b0 + bl) * (kDecBlockK / 8) + c;
#pragma unroll
          for (int ch = 0; ch < 4; ++ch) {
            const int row = row0 + 4 * ch;
            if (row < KW) asm volatile("prefetch.global.L2 [%0];" ::"l"(qw + (size_t)row * N + nbase));
          }
        }
      }
    }
  }

  // scales / zeros of this CTA's 128 features for every 128-K block of its slice: thread = feature, so the table is
  // read with one request per (feature, block) instead of one per (lane, feature, block) -- the [N, G] checkpoint layout
  // puts consecutive features G floats apart, and fetching them lane by lane inside the group loop cost 4x the sectors
  // of the packed weights themselves
  {
    const int n = bx * kDecCols + tid;
    // quantisation group of each 128-K block, advanced incrementally (one integer division per CTA, not one per block)
    int grp = (b0 * kDecBlockK) / group_size;
    long long kend = (long long)(grp + 1) * group_size;  // first k of group grp + 1
    for (int bl = 0; bl < nb; ++bl) {
      const long long k0 = (long long)(b0 + bl) * kDecBlockK;
      while (k0 >= kend) { ++grp; kend += group_size; }
      s_sc[bl * kDecCols + tid] = n < N ? __ldg(scales + (size_t)n * G + grp) : 0.f;
      s_zr[bl * kDecCols + tid] = n < N ? __ldg(zeros + (size_t)n * G + grp) : 0.f;
    }
  }

  // static-weights form: everything above read constants of the model; from here on the activations and `out` are touched
  if ((pdl & 5) == 5) asm volatile("griddepcontrol.wait;" ::: "memory");

  for (int m0 = 0; m0 < M; m0 += MT) {
    // The kernel lives for a few microseconds, i.e. a handful of DRAM latencies: the packed weights (the whole slab,
    // or the first two 128-K blocks of the register-staged variant) were requested before anything else, so their
    // latency overlaps the staging of the activations.
    if (!SLAB && m0 > 0) {
      load_group(0, wa);
      if (nb > 1) load_group(1, wb);
    }
    __syncthreads();  // the previous pass is done with the staging buffers
    const int tokens = min(MT, M - m0);  // real tokens of this pass; the other token columns of the MMA are never read back
    if (tid < MT) s_amax[tid] = 0u;
    if (tid == 0) s_need_lo = 0;
    __syncthreads();
    // ---- stage the activations of this K slice (work items = (token, 128-K block) pairs spread over the warps):
    // per-token power-of-two scale, fp16 hi / lo planes, 8-K permutation, per-block row sums
    const int pairs = tokens * blocks_per_slice;
    float cache[4];  // the values of this warp's first (token, block) pair: read from global memory once
    // fp16 activations (x_h) are their own hi plane: no per-token power-of-two scale, no lo plane -- the abs-max pass is skipped
    // (token, block) of this warp's pair, advanced by 4 pairs per iteration without a division per iteration
    const int t_first = warp / blocks_per_slice, blk_first = warp - t_first * blocks_per_slice;
    int t = t_first, blk = blk_first;
    auto next_pair = [&]() {
      blk += kDecThreads / 32;
      while (blk >= blocks_per_slice) { blk -= blocks_per_slice; ++t; }
    };
    for (int p = warp, it = 0; p < pairs && !x_h; p += kDecThreads / 32, ++it, next_pair()) {
      const size_t xoff = (size_t)(m0 + t) * K + (size_t)(b0 + blk) * kDecBlockK;
      float amax = 0.f;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int kk = r * 32 + lane;
        const float v = (blk < nb && (b0 + blk) * kDecBlockK + kk < K) ? (x_h ? __half2float(__ldg(x_h + xoff + kk)) : __ldg(x + xoff + kk)) : 0.f;
        if (it == 0) cache[r] = v;
        amax = fmaxf(amax, fabsf(v));
      }
      amax = warp_max(amax);
      if (lane == 0 && amax < __int_as_float(0x7f800000)) atomicMax(&s_amax[t], __float_as_uint(amax));  // non-negative: bit order == value order
    }
    __syncthreads();
    t = t_first;
    blk = blk_first;
    for (int p = warp, it = 0; p < pairs; p += kDecThreads / 32, ++it, next_pair()) {
      const size_t xoff = (size_t)(m0 + t) * K + (size_t)(b0 + blk) * kDecBlockK;
      const uint32_t abits = s_amax[t];
      // 2^-e with e = floor(log2(amax)) - 14, straight from the exponent field: scaled slice max in [2^14, 2^15)
      const int ex = (abits && !x_h) ? (int)(abits >> 23) - 127 - 14 : 0;
      const float down = __uint_as_float((uint32_t)(127 - max(-126, min(127, ex))) << 23);
      if (lane == 0 && blk == 0) escale[t] = __uint_as_float((uint32_t)(127 + max(-126, min(127, ex))) << 23);
      float s = 0.f;
      bool any_lo = false;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int kk = r * 32 + lane;
        const bool ok = blk < nb && ((b0 + blk) * kDecBlockK + kk < K);
        const float v = ((it == 0 && !x_h) ? cache[r] : (ok ? (x_h ? __half2float(__ldg(x_h + xoff + kk)) : __ldg(x + xoff + kk)) : 0.f)) * down;
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        any_lo |= (__half_as_ushort(lo) & 0x7FFFu) != 0;
        const int j = kk & 7, pos = blk * kDecBlockK + (kk & ~7) + ((j & 3) << 1) + (j >> 2);  // (0,4,1,5,2,6,3,7)
        xh[t * stride + pos] = hi;
        xl[t * stride + pos] = lo;
        s += v;
      }
      s = warp_sum(s);
      if (lane == 0) xsum[t * blocks_per_slice + blk] = s;
      if (__any_sync(0xffffffffu, any_lo) && lane == 0) atomicOr(&s_need_lo, 1);
    }
    __syncthreads();
    const bool need_lo = s_need_lo != 0;

    float acc[2][NB][4];
#pragma unroll
    for (int T = 0; T < 2; ++T)
#pragma unroll
      for (int q = 0; q < NB; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[T][q][j] = 0.f;

    // token row of MMA column block q for this lane (SLAB: rows beyond the real tokens alias the last real one)
    auto trow = [&](int r) { return SLAB ? min(r, tokens - 1) : r; };
    auto compute_group = [&](int bl, const uint4 (&w)[4]) {
      if (SLAB) mbar_wait(&s_bar[bl], 0u);  // phase 0 = the slab rows of this block have landed (stays true afterwards)
      float d[2][NB][4];
#pragma unroll
      for (int T = 0; T < 2; ++T)
#pragma unroll
        for (int q = 0; q < NB; ++q)
#pragma unroll
          for (int j = 0; j < 4; ++j) d[T][q][j] = 0.f;
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        // B fragments of this chunk: tokens g (+ 8 q), K = 32 (bl*4 + ch) + 8 c .. + 7 in permuted order
        uint4 bh[NB], bl4[NB];
        const int koff = (bl * 4 + ch) * 32 + 8 * c;
#pragma unroll
        for (int q = 0; q < NB; ++q) {
          bh[q] = *reinterpret_cast<const uint4*>(xh + trow(q * 8 + g) * stride + koff);
          if (need_lo) bl4[q] = *reinterpret_cast<const uint4*>(xl + trow(q * 8 + g) * stride + koff);
        }
        const uint4 wv = SLAB ? *reinterpret_cast<const uint4*>(slab + (size_t)(bl * (kDecBlockK / 8) + 4 * ch + c) * kSlabRowBytes +
                                                                (warp * 32 + 4 * g) * 4)
                              : w[ch];
        const uint32_t words[4] = {wv.x, wv.y, wv.z, wv.w};  // features nbase + 0..3
#pragma unroll
        for (int T = 0; T < 2; ++T) {
          uint32_t a0[4], a1[4];  // A fragments of MMA i = 0 and i = 1
#pragma unroll
          for (int h = 0; h < 2; ++h) {  // row slot g (h = 0) / g + 8 (h = 1)
            const uint32_t wlo = words[2 * T + h], whi = wlo >> 8;
            const uint32_t u0 = dec_and_or<0x000F000Fu>(wlo, bias), u1 = dec_and_or<0x00F000F0u>(wlo, bias);
            const uint32_t u2 = dec_and_or<0x000F000Fu>(whi, bias), u3 = dec_and_or<0x00F000F0u>(whi, bias);
            const __half2 q0 = __hsub2(*reinterpret_cast<const __half2*>(&u0), k1024);        // nibbles (0, 4)
            const __half2 q1 = __hfma2(*reinterpret_cast<const __half2*>(&u1), k16, k64n);    // nibbles (1, 5)
            const __half2 q2 = __hsub2(*reinterpret_cast<const __half2*>(&u2), k1024);        // nibbles (2, 6)
            const __half2 q3 = __hfma2(*reinterpret_cast<const __half2*>(&u3), k16, k64n);    // nibbles (3, 7)
            a0[h] = *reinterpret_cast<const uint32_t*>(&q0);      // columns (2c, 2c + 1)
            a0[2 + h] = *reinterpret_cast<const uint32_t*>(&q1);  // columns (2c + 8, 2c + 9)
            a1[h] = *reinterpret_cast<const uint32_t*>(&q2);
            a1[2 + h] = *reinterpret_cast<const uint32_t*>(&q3);
          }
#pragma unroll
          for (int q = 0; q < NB; ++q) {
            hmma_16816(d[T][q], a0, bh[q].x, bh[q].y);
            hmma_16816(d[T][q], a1, bh[q].z, bh[q].w);
            if (need_lo) {
              hmma_16816(d[T][q], a0, bl4[q].x, bl4[q].y);
              hmma_16816(d[T][q], a1, bl4[q].z, bl4[q].w);
            }
          }
        }
      }
      // group epilogue: acc += scale * D - zeros * sum_k x   (rows: slot g -> feature 2T, slot g + 8 -> feature 2T + 1)
#pragma unroll
      for (int T = 0; T < 2; ++T) {
        const int f = bl * kDecCols + warp * 32 + 4 * g + 2 * T;  // lanes of one g read the same word: conflict-free
        const float sA = s_sc[f], zA = s_zr[f], sB = s_sc[f + 1], zB = s_zr[f + 1];
#pragma unroll
        for (int q = 0; q < NB; ++q) {
          const float xs0 = xsum[trow(q * 8 + 2 * c) * blocks_per_slice + bl], xs1 = xsum[trow(q * 8 + 2 * c + 1) * blocks_per_slice + bl];
          acc[T][q][0] += fmaf(sA, d[T][q][0], -zA * xs0);
          acc[T][q][1] += fmaf(sA, d[T][q][1], -zA * xs1);
          acc[T][q][2] += fmaf(sB, d[T][q][2], -zB * xs0);
          acc[T][q][3] += fmaf(sB, d[T][q][3], -zB * xs1);
        }
      }
    };
    for (int bl = 0; bl < nb; bl += 2) {
      compute_group(bl, wa);
      if (!SLAB && bl + 2 < nb) load_group(bl + 2, wa);
      if (bl + 1 < nb) {
        compute_group(bl + 1, wb);
        if (!SLAB && bl + 3 < nb) load_group(bl + 3, wb);
      }
    }
    if (col_ok) {
#pragma unroll
      for (int T = 0; T < 2; ++T)
#pragma unroll
        for (int q = 0; q < NB; ++q)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int tok = q * 8 + 2 * c + (j & 1), m = m0 + tok;
            const int n = nbase + 2 * T + (j >> 1);
            if (m < M) {
              const float v = acc[T][q][j] * escale[tok];
              if (out_h) batch.p[pi].partial[((size_t)blockIdx.y * M + m) * N + n] = v;  // this slice's own slot
              else atomicAdd(out + (size_t)m * N + n, v);
            }
          }
    }
  }
  if (out_h) {
    // last slice CTA of this feature block adds the slots in slice order (threadfence-reduction pattern)
    __shared__ int s_last;
    const int slices_p = (nblk + blocks_per_slice - 1) / blocks_per_slice;
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(batch.p[pi].counters + bx, 1) == slices_p - 1) ? 1 : 0;
    __syncthreads();
    if (s_last) {
      __threadfence();
      const int n = bx * kDecCols + tid;
      if (n < N) {
        const float* __restrict__ part = batch.p[pi].partial;
        const float bv = batch.p[pi].bias ? __ldg(batch.p[pi].bias + n) : 0.f;
        for (int m = 0; m < M; ++m) {
          float t = 0.f;
          int sl = 0;
          for (; sl + 3 < slices_p; sl += 4) {  // four loads in flight, summed in slice order
            const float v0 = __ldcg(part + ((size_t)sl * M + m) * N + n), v1 = __ldcg(part + ((size_t)(sl + 1) * M + m) * N + n),
                        v2 = __ldcg(part + ((size_t)(sl + 2) * M + m) * N + n), v3 = __ldcg(part + ((size_t)(sl + 3) * M + m) * N + n);
            t = (((t + v0) + v1) + v2) + v3;
          }
          for (; sl < slices_p; ++sl) t += __ldcg(part + ((size_t)sl * M + m) * N + n);
          out_h[(size_t)m * N + n] = __float2half_rn(t + bv);
        }
      }
      if (tid == 0) batch.p[pi].counters[bx] = 0;  // ready for the next call on this state
    }
  }
}

bool gptq4_decode_supported(const int32_t* qweight, long long N) { return (N % 4 == 0) && aligned16(qweight); }

// Decode-kernel variant (process-wide benchmarking / test switch, sb200_gptq4_set_decode): bit 0 = bulk-copy weight
// slab (SLAB), bit 1 = programmatic dependent launch, bit 2 = L2 prefetch of the 128-K blocks beyond the two held in
// registers (register-staged variant only), bit 3 = treat every call as SB200_GPTQ4_STATIC_WEIGHTS,
// bits 4..7 = resident CTAs per SM the K split aims at (0 = 5).
static int g_dec_mode = 6;
void gptq4_decode_set_mode(int mode) { g_dec_mode = mode; }
int gptq4_decode_get_mode() { return g_dec_mode; }

template <int NB, bool SLAB>
static int dec_launch(const DecBatch& batch, dim3 grid, size_t smem, int M, int S, int x_rows, bool pdl, int kflags, cudaStream_t st) {
  static std::atomic<int> attr_done[64];
  if (smem > 48 * 1024) SB_CUDA(ensure_dyn_smem(gptq4_decode_kernel<NB, SLAB>, (int)smem, attr_done));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(kDecThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  SB_CUDA(cudaLaunchKernelEx(&cfg, gptq4_decode_kernel<NB, SLAB>, batch, M, S, x_rows, kflags));
  SB_LAUNCHED();
  return SB200_OK;
}

// `count` problems sharing M in one launch (count == 1: the plain entry point)
int gptq4_decode_batch(const DecProblem* probs, int count, long long M, int flags, cudaStream_t st) {
  DecBatch batch;
  batch.count = count;
  int colblocks = 0, nblk_max = 0;
  for (int i = 0; i < count; ++i) {
    batch.p[i] = probs[i];
    batch.p[i].colblock_begin = colblocks;
    colblocks += (probs[i].N + kDecCols - 1) / kDecCols;
    const int nblk = (probs[i].K + kDecBlockK - 1) / kDecBlockK;
    nblk_max = nblk > nblk_max ? nblk : nblk_max;
  }
  for (int i = count; i < kDecMaxProblems; ++i) batch.p[i] = batch.p[0];
  const int nbk = M <= 8 ? 1 : (M <= 16 ? 2 : 4);
  const bool slab = (g_dec_mode & 1) != 0, pdl = (g_dec_mode & 2) != 0, prefetch = (g_dec_mode & 4) != 0;
  const bool static_w = (g_dec_mode & 8) != 0 || (flags & SB200_GPTQ4_STATIC_WEIGHTS) != 0;
  const int kflags = (pdl ? 1 : 0) | (prefetch ? 2 : 0) | (static_w ? 4 : 0);
  const int per_sm = ((g_dec_mode >> 4) & 15) ? ((g_dec_mode >> 4) & 15) : 5;
  // K slices: ~5 CTAs per SM (what the register file holds: 4 warps x 96 registers), each streaming as long a K
  // range as that allows, bounded by the activation slice held in shared memory
  int want = (sm_count() * per_sm + colblocks - 1) / colblocks;
  if (want < 1) want = 1;
  if (want > nblk_max) want = nblk_max;
  int S = (nblk_max + want - 1) / want;
  const int smax = nbk == 1 ? 8 : (nbk == 2 ? 4 : 2);
  if (S > smax) S = smax;
  const int slices = (nblk_max + S - 1) / S;
  const dim3 grid((unsigned)colblocks, (unsigned)slices);
  const int mt = 8 * nbk;
  const int x_rows = slab ? (int)(M < mt ? M : mt) : mt;
  const size_t smem = (slab ? (size_t)S * kSlabGroupBytes : 0) + (size_t)2 * x_rows * (S * kDecBlockK + 32) * sizeof(__half) +
                      (size_t)x_rows * S * sizeof(float) + (size_t)mt * sizeof(float) + (size_t)2 * S * kDecCols * sizeof(float);
#define SB_GO(NB_) (slab ? dec_launch<NB_, true>(batch, grid, smem, (int)M, S, x_rows, pdl, kflags, st) \
                         : dec_launch<NB_, false>(batch, grid, smem, (int)M, S, x_rows, pdl, kflags, st))
  if (nbk == 1) return SB_GO(1);
  if (nbk == 2) return SB_GO(2);
  return SB_GO(4);
#undef SB_GO
}

int gptq4_decode(const float* x, const int32_t* qweight, float* out, const float* scales, const float* zeros, long long M,
                 long long K, long long N, long long KW, int group_size, int flags, cudaStream_t st) {
  DecProblem p;
  p.x = x;
  p.qw = reinterpret_cast<const uint32_t*>(qweight);
  p.out = out;
  p.scales = scales;
  p.zeros = zeros;
  p.K = (int)K;
  p.N = (int)N;
  p.KW = (int)KW;
  p.G = (int)((K + group_size - 1) / group_size);
  p.group_size = group_size;
  p.colblock_begin = 0;
  p.x_h = nullptr;
  p.out_h = nullptr;
  p.bias = nullptr;
  p.partial = nullptr;
  p.counters = nullptr;
  return gptq4_decode_batch(&p, 1, M, flags, st);
}

// fp16 in / fp16 out in one launch; `partial` holds ceil(K / 128) * M * N floats, `counters` ceil(N / 128) zeroed ints
size_t gptq4_decode_f16_partial_bytes(long long M, long long K, long long N) {
  return (size_t)((K + kDecBlockK - 1) / kDecBlockK) * (size_t)M * (size_t)N * sizeof(float);
}
int gptq4_decode_f16(const __half* x_h, const int32_t* qweight, __half* out_h, const float* bias, const float* scales,
                     const float* zeros, long long M, long long K, long long N, long long KW, int group_size, float* partial,
                     int* counters, int flags, cudaStream_t st) {
  DecProblem p;
  p.x = nullptr;
  p.qw = reinterpret_cast<const uint32_t*>(qweight);
  p.out = nullptr;
  p.scales = scales;
  p.zeros = zeros;
  p.K = (int)K;
  p.N = (int)N;
  p.KW = (int)KW;
  p.G = (int)((K + group_size - 1) / group_size);
  p.group_size = group_size;
  p.colblock_begin = 0;
  p.x_h = x_h;
  p.out_h = out_h;
  p.bias = bias;
  p.partial = partial;
  p.counters = counters;
  return gptq4_decode_batch(&p, 1, M, flags, st);
}

}  // namespace sb200

using namespace sb200;

extern "C" int sb200_gptq4_matmul_batch_ex(const sb200_gptq4_problem* problems, int count, int64_t m, int flags, void* stream);
extern "C" int sb200_gptq4_matmul_batch(const sb200_gptq4_problem* problems, int count, int64_t m, void* stream) {
  return sb200_gptq4_matmul_batch_ex(problems, count, m, 0, stream);
}
extern "C" int sb200_gptq4_matmul_batch_ex(const sb200_gptq4_problem* problems, int count, int64_t m, int flags, void* stream) {
  SB_REQUIRE((flags & ~SB200_GPTQ4_STATIC_WEIGHTS) == 0, "sb200_gptq4_matmul_batch_ex: unknown flags 0x%x", flags);
  SB_REQUIRE(problems && count >= 1 && count <= kDecMaxProblems, "sb200_gptq4_matmul_batch: 1 .. %d problems (got %d)", kDecMaxProblems, count);
  SB_REQUIRE(m >= 1 && m <= 32, "sb200_gptq4_matmul_batch: decode-sized M only (1 .. 32, got %lld)", (long long)m);
  DecProblem p[kDecMaxProblems];
  for (int i = 0; i < count; ++i) {
    const sb200_gptq4_problem& q = problems[i];
    SB_REQUIRE(q.x && q.qweight && q.out && q.scales && q.zeros, "sb200_gptq4_matmul_batch: null pointer in problem %d", i);
    SB_REQUIRE(q.k > 0 && q.n > 0 && q.k < (1LL << 31) && q.n < (1LL << 31), "sb200_gptq4_matmul_batch: bad shape in problem %d", i);
    SB_REQUIRE(q.qweight_rows >= (q.k + 7) / 8, "sb200_gptq4_matmul_batch: qweight of problem %d has too few rows", i);
    SB_REQUIRE(q.group_size == 0 || (q.group_size > 0 && q.group_size % 128 == 0),
               "only group_size divisible by 128 is supported in 4-bit quantization (got %d)", q.group_size);
    SB_REQUIRE(gptq4_decode_supported(q.qweight, q.n), "sb200_gptq4_matmul_batch: problem %d needs N %% 4 == 0 and a 16-byte aligned qweight", i);
    const int gs = q.group_size ? q.group_size : (int)q.k;
    p[i].x = q.x;
    p[i].qw = reinterpret_cast<const uint32_t*>(q.qweight);
    p[i].out = q.out;
    p[i].scales = q.scales;
    p[i].zeros = q.zeros;
    p[i].K = (int)q.k;
    p[i].N = (int)q.n;
    p[i].KW = (int)q.qweight_rows;
    p[i].G = (int)((q.k + gs - 1) / gs);
    p[i].group_size = gs;
    p[i].colblock_begin = 0;
    p[i].x_h = nullptr;
    p[i].out_h = nullptr;
    p[i].bias = nullptr;
    p[i].partial = nullptr;
    p[i].counters = nullptr;
  }
  return gptq4_decode_batch(p, count, m, flags, (cudaStream_t)stream);
}
