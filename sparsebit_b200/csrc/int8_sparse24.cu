// int8_sparse24.cu -- 2:4 structured sparsity: the 2:4 L1 sparser's mask, and integer-grid inference of a calibrated
// QLinear whose weight is 2:4-sparse on the grid, on the sparse tensor cores (wgmma.mma_async.sp).
//
// Mask.  Each row of weight.reshape(C_out, -1) is walked in aligned groups of 4 from k = 0; a group keeps its two
// largest |w| (ties to the lower index, NaN above every number, +-0 as 0), a tail group of r < 4 keeps min(2, r).
//
// Centred weight grid.  With w_q / w_zero as sb200_int8_quantize_rows stores them, d_w = w_q - w_zero = g_w - rint(zp_w)
// is 0 exactly where the fake-quant weight is 0, so a 2:4-sparse fake-quant weight is 2:4-sparse in d_w and
//   I = sum_k a[m, k] d_w[n, k] - Z_x sum_k d_w[n, k]      (a, Z_x on the stored activation grid, as int8_linear.cu)
// is the integer sb200_int8_linear's epilogue forms.  The epilogue applies the same float operations to it:
// y = fp32(fp64(I) * (fp64(s_x) * fp64(s_w[n]))) (+ bias[n] in fp32), NaN for rows of x holding a NaN.
// |a| <= 128 and |d_w| <= 128, so the s32 accumulator is exact for K < 2^17 as in the dense kernel.
//
// Pack (once, at conversion).  The compressed operand of the header's format: vals (the two kept centred values of
// every group), meta (their 2-bit indices in the per-thread order the sparse wgmma reads), dsum = sum_k d_w and bad
// (groups with more than two nonzeros or a centred value outside s8).
//
// GEMM.  The sparse operand of wgmma.sp is A, so the roles of the dense kernel swap: D[feature, token] = W_c x^T with
// wgmma.m64n128k64.sp.s32.s8.s8.  CTA = 128 features x 128 tokens: warpgroup 0 = TMA producer (one thread),
// warpgroups 1 and 2 = 64 features each.  A stage holds 256 K: the activation grid (two 128-token x 128-byte
// SWIZZLE_128B boxes of the row quantizer's output), the compressed weights (128 features x 128 bytes, SWIZZLE_128B:
// 256 K at two stored bytes per group of 4) and the metadata words of both warpgroups (4 steps x 2 x 128 words), all TMA-
// loaded; a consumer thread reads one metadata word per 64-feature x 64-K step from shared memory.  The accumulator
// rows are features, so the epilogue stages the tile through shared memory (the ring, free once both warpgroups are
// done) and stores rows of out [M, N] whole.
//
// Conv2d.  launch_im2col (int8_linear.cu) lowers the input into the same workspace, one s8 row per output pixel in the K
// order (c, kh, kw) of weight.reshape(C_out, -1), the order the 2:4 groups of a pruned conv weight follow; the same GEMM
// (kNchw = true) then writes NCHW: out[(img N + n) P + p] for token m = img P + p, P = OH OW.  The epilogue stages the
// tile as [feature][token] (rows of kSpTok + 4 floats), the mirror of the row-major staging; warp c of the consumers
// stores feature rows c, c + 8, ..., lane l tokens 4 l .. 4 l + 3, whose image / pixel split and NaN flags it computes
// once.  Four tokens at consecutive out addresses (one image, or N = 1) leave as one 16-byte store when the first is
// 16-byte aligned, others one by one,
// so a tile spanning images (P < 128, P = 1 at a 1 x 1 output) is stored correctly.
#include "int8_grid.cuh"
#include "tc_common.cuh"
namespace sb200 {
namespace {

constexpr int kSpFeat = 128;                       // features per CTA (two consumer warpgroups x 64)
constexpr int kSpTok = 128;                        // tokens per CTA = wgmma N
constexpr int kSpBK = 256;                         // K per stage
constexpr int kSpStages = 4;
constexpr int kSpThreads = 384;
constexpr int kSpXBox = kSpTok * 128;              // 16 KB: 128 tokens x 128 K of the activation grid
constexpr int kSpWBytes = kSpFeat * (kSpBK / 2);   // 16 KB: 128 features x 128 stored bytes
constexpr int kSpEWords = (kSpBK / 64) * 2 * 128;  // metadata words of a stage: [k64 step][warpgroup][thread]
constexpr int kSpStageBytes = 2 * kSpXBox + kSpWBytes + kSpEWords * 4;  // 52 KB, a multiple of 1024
constexpr int kSpLd = kSpFeat + 4;                 // floats per staged token row: conflict-free transposed writes
constexpr int kSpLdT = kSpTok + 4;                 // NCHW: floats per staged feature row
constexpr uint32_t kSpPadMeta = 0x44444444u;       // every group keeps indices (0, 1)
static_assert(kSpStageBytes % 1024 == 0, "stage tiles stay 1024-byte aligned");
static_assert(kSpTok * kSpLd * 4 <= kSpStages * kSpStageBytes, "the output tile fits the ring");
static_assert(kSpFeat * kSpLdT * 4 <= kSpStages * kSpStageBytes, "the NCHW output tile fits the ring");

// ---------------------------------------------------------------------------------- 2:4 mask
// |a| ranks above |b|: NaN above every number, +-0 as 0
__device__ __forceinline__ bool sp_above(float a, float b) {
  const bool na = a != a, nb = b != b;
  if (na || nb) return na && !nb;
  return fabsf(a) > fabsf(b);
}

// One thread per group of 4; mask is uint8 0 / 1 shaped like w.
__global__ void __launch_bounds__(256) sparse24_mask_kernel(const float* __restrict__ w, uint8_t* __restrict__ mask,
                                                            long long rows, long long cols, long long groups_per_row) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= rows * groups_per_row) return;
  const long long row = g / groups_per_row, k0 = (g - row * groups_per_row) * 4;
  const int r = (int)min(4LL, cols - k0);
  const float* wr = w + row * cols + k0;
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = i < r ? __ldg(wr + i) : 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i >= r) continue;
    int beaten = 0;  // elements of the group ranked above v[i]; equal ranks go to the lower index
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < r && j != i && (sp_above(v[j], v[i]) || (j < i && !sp_above(v[i], v[j])))) ++beaten;
    mask[row * cols + k0 + i] = beaten < 2 ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------- pack
// One thread per metadata word: tile b (128 features), k64 step kb, warpgroup h, consumer thread t of the warpgroup.
// The word covers feature n = 128 b + 64 h + 16 (t >> 5) + ((t & 31) >> 2) + 8 (t & 1) and the 32 K from
// 64 kb + 32 ((t >> 1) & 1); group g of those 8 groups has its kept indices i0 < i1 in bits [4 g, 4 g + 4).
// Kept: the nonzero centred values, then the lowest-index zeros up to two.  The thread also writes the group's two
// stored values and adds its share of dsum / bad (integer atomics: the totals do not depend on their order).
__global__ void __launch_bounds__(256) sparse24_pack_kernel(const int8_t* __restrict__ w_q, const int* __restrict__ w_zero,
                                                            const float* __restrict__ w_scale, int8_t* __restrict__ vals,
                                                            uint32_t* __restrict__ meta, int* __restrict__ dsum,
                                                            int* __restrict__ bad, int N, int K, int Kp, int kb64,
                                                            long long words) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= words) return;
  const int t = (int)(idx & 127), h = (int)((idx >> 7) & 1);
  const long long bk = idx >> 8;
  const int b = (int)(bk / kb64), kb = (int)(bk - (long long)b * kb64);
  const int n = 128 * b + 64 * h + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * (t & 1);
  const int k0 = 64 * kb + 32 * ((t >> 1) & 1);
  if (n >= N) {
    meta[idx] = kSpPadMeta;
    return;
  }
  const float sw = __ldg(w_scale + n);
  const bool live = sw == sw;  // a NaN-scale row is packed as zeros: its column is NaN anyway
  const int zw = __ldg(w_zero + n);
  const int8_t* wr = w_q + (long long)n * Kp;
  uint32_t word = 0u, packed[4] = {0u, 0u, 0u, 0u};
  int sum = 0, nbad = 0;
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    int d[4], nz = 0;
    bool range = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + 4 * g + i;
      d[i] = (live && k < K) ? (int)wr[k] - zw : 0;
      nz += d[i] != 0;
      range = range || d[i] < -128 || d[i] > 127;
      sum += d[i];
    }
    nbad += (nz > 2 || range) ? 1 : 0;
    // kept set as bits: the nonzeros, then the lowest zeros up to two (a bad group keeps its first two nonzeros)
    uint32_t keep = (d[0] != 0) | (d[1] != 0) << 1 | (d[2] != 0) << 2 | (d[3] != 0) << 3;
    while (__popc(keep) < 2) keep |= ~keep & (keep + 1);
    if (__popc(keep) > 2) keep = (keep & (0u - keep)) | ((keep & (keep - 1)) & (0u - (keep & (keep - 1))));
    const int i0 = __ffs(keep) - 1, i1 = 31 - __clz(keep);
    word |= (uint32_t)(i0 | (i1 << 2)) << (4 * g);
    const int v0 = i0 == 0 ? d[0] : i0 == 1 ? d[1] : d[2];  // i0 <= 2 < i1 or i0 < i1 <= 3
    const int v1 = i1 == 1 ? d[1] : i1 == 2 ? d[2] : d[3];
    const uint32_t v2 = ((uint32_t)v0 & 0xFFu) | (((uint32_t)v1 & 0xFFu) << 8);
    packed[g >> 1] |= v2 << (16 * (g & 1));
  }
  meta[idx] = word;
  *reinterpret_cast<uint4*>(vals + (long long)n * (kb64 * 32) + k0 / 2) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  if (sum) atomicAdd(dsum + n, sum);
  if (nbad) atomicAdd(bad + n, nbad);
}

// ---------------------------------------------------------------------------------- GEMM
// D[64 x 128] (+)= A[64 x 64, 2:4 sparse] * B[64 x 128], s8 x s8 -> s32.  A: the compressed 64 x 32 bytes, K-major
// SWIZZLE_128B; B: 128 x 64 K-major SWIZZLE_128B; e: this thread's metadata word, sparsity selector 0 (every thread of
// the warpgroup supplies one word for 8-bit types).
__device__ __forceinline__ void wgmma_m64n128k64_sp_s8(int (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t e, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %67, 0;\n\t"
      "wgmma.mma_async.sp.sync.aligned.m64n128k64.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "%64, %65, %66, 0, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(e), "r"(accumulate));
}

// NCHW epilogue of the sparse GEMM (the 256 consumer threads; the ring is free).  Thread (warp w, lane l, q = l & 3)
// holds features f0, f0 + 8 of the tile (per-feature terms cn, sxw, bn) and, in acc[j], tokens 8 (j >> 2) + 2 q +
// (j & 1).  The tile is staged [feature][token]; then consumer warp cw stores feature rows cw, cw + 8, ... < N - n0 and
// lane l tokens t = 4 l .. 4 l + 3 < M - m0 of each: out[(img N + n) P + p] with m = img P + p, split once per token.
__device__ __forceinline__ void sp_store_nchw(const int (&acc)[64], float* tile, const long long (&cn)[2],
                                              const double (&sxw)[2], const float (&bn)[2], bool has_bias, int f0, int q,
                                              int cw, int lane, float* __restrict__ out, const uint8_t* __restrict__ x_nan,
                                              int m0, int n0, int M, int N, int P, int vec4) {
#pragma unroll
  for (int c = 0; c < 16; ++c) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float y[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const long long I = (long long)acc[4 * c + 2 * h + e] + cn[h];
        y[e] = __double2float_rn((double)I * sxw[h]);
        if (has_bias) y[e] = __fadd_rn(y[e], bn[h]);
      }
      *reinterpret_cast<float2*>(tile + (f0 + 8 * h) * kSpLdT + 8 * c + 2 * q) = make_float2(y[0], y[1]);
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  // per token of this lane: the out offset of feature 0, img N P + p, and its NaN flag
  long long base[4];
  bool tnan[4], live[4];
  const int t0 = 4 * lane;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + t0 + i;
    live[i] = m < M;
    const int img = live[i] ? m / P : 0;
    base[i] = (long long)img * N * P + (m - img * P);
    tnan[i] = live[i] && __ldg(x_nan + m) != 0;
  }
  // the four tokens are live and lie in one image: consecutive pixels, consecutive out addresses
  const bool run = live[3] && base[3] - base[0] == 3;
  const float qnan = __int_as_float(0x7fc00000);
  for (int r = cw; r < kSpFeat; r += 8) {
    const int n = n0 + r;
    if (n >= N) break;
    const float4 v4 = *reinterpret_cast<const float4*>(tile + r * kSpLdT + t0);
    float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (tnan[i]) v[i] = qnan;
    const long long o = base[0] + (long long)n * P;
    if (vec4 && run && (o & 3) == 0) {
      *reinterpret_cast<float4*>(out + o) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (live[i]) out[base[i] + (long long)n * P] = v[i];
    }
  }
}

// Load kb of the stage ring (tc_common.cuh) holds K block kb, 256 K of both operands.  Unlike the dense kernel, a consumer
// retires each stage's wgmma group before it loads the next stage's metadata words, and releases the stage then (see the
// loop).  Every stage issues four k64 steps, so that no branch separates the wgmmas (a branch there makes ptxas
// serialise them).  Past K64 the last stage's steps multiply zeros: the weight box is zero-filled beyond the vals, their
// metadata word is the padding word (indices 0, 1), and the second activation box, loaded only when one of the stage's
// steps = min(4, kb64 - 4 kb) real steps reads it, holds whatever an earlier stage left there, which the zero weights
// cancel exactly.  No box lies wholly beyond its operand.
//
// Accumulator layout of a consumer thread (warp w of its warpgroup, lane l, q = l & 3), j = 0 .. 63:
//   acc[j] = D[feature 16 w + l / 4 + 8 ((j >> 1) & 1)][token 8 (j >> 2) + 2 q + (j & 1)]
// kNchw = false: out is row-major [M, N].  kNchw = true: out is NCHW [M / P, N, P] (conv2d, P = OH OW pixels per image).
template <bool kNchw>
__global__ void __launch_bounds__(kSpThreads, 1)
int8_sparse24_gemm_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_v,
                          const __grid_constant__ CUtensorMap map_e, float* __restrict__ out,
                          const uint8_t* __restrict__ x_nan, const float* __restrict__ x_scale,
                          const float* __restrict__ x_zero, int x_off, const int* __restrict__ dsum,
                          const float* __restrict__ w_scale, const float* __restrict__ bias, int M, int N, int kb64,
                          int vec4, int P) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* stage_base = smem_align1024(smem_raw);
  auto& ring = *reinterpret_cast<StageRing<kSpStages>*>(stage_base + (size_t)kSpStages * kSpStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + kSpTok - 1) / kSpTok;
  const int m0 = (int)(blockIdx.x % (unsigned)tiles_m) * kSpTok, n0 = (int)(blockIdx.x / (unsigned)tiles_m) * kSpFeat;
  const int num_kb = (kb64 + 3) / 4;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    prefetch_tensormap(&map_v);
    prefetch_tensormap(&map_e);
    ring.init();
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<40>();
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const bool hi = kb64 - 4 * kb > 2;
        const int s = ring.acquire(kb, (uint32_t)(kSpStageBytes - (hi ? 0 : kSpXBox)));
        unsigned char* st = stage_base + (size_t)s * kSpStageBytes;
        tma_load_2d(st, &map_x, kb * kSpBK, m0, &ring.full[s]);
        if (hi) tma_load_2d(st + kSpXBox, &map_x, kb * kSpBK + 128, m0, &ring.full[s]);
        tma_load_2d(st + 2 * kSpXBox, &map_v, kb * (kSpBK / 2), n0, &ring.full[s]);
        tma_load_3d(st + 2 * kSpXBox + kSpWBytes, &map_e, 0, 4 * kb, n0 / kSpFeat, &ring.full[s]);
      }
    }
    return;
  }
  reg_inc<232>();
  const int wg = (warp - 4) >> 2, wt = threadIdx.x - 128 - 128 * wg;  // consumer warpgroup, thread within it
  const uint32_t stage0 = smem_u32(stage_base);
  // the epilogue's per-feature terms are fetched while the ring fills
  const double sx = (double)__ldg(x_scale);
  const long long zx = (long long)rintf(__ldg(x_zero)) - x_off;
  const int q = lane & 3;
  const int f0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // features f0 and f0 + 8 of the tile
  long long cn[2];
  double sxw[2];
  float bn[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = n0 + f0 + 8 * h;
    const bool ok = n < N;
    cn[h] = ok ? -zx * (long long)__ldg(dsum + n) : 0;
    sxw[h] = ok ? sx * (double)__ldg(w_scale + n) : 0.0;
    bn[h] = (ok && bias) ? __ldg(bias + n) : 0.f;
  }

  int acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0;
  const uint32_t stage_e = smem_u32(stage_base) + 2 * kSpXBox + kSpWBytes + (uint32_t)(wg * 128 + wt) * 4;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = ring.wait(kb);
    const uint32_t st = stage0 + (uint32_t)s * kSpStageBytes;
    const uint64_t da = gmma_desc_sw128(st + 2 * kSpXBox + (uint32_t)wg * (64 * 128));
    const int steps = min(4, kb64 - 4 * kb);
    uint32_t ew[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t w;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w) : "r"(stage_e + (uint32_t)s * kSpStageBytes + 1024u * j));
      ew[j] = j < steps ? w : kSpPadMeta;
    }
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint64_t db = gmma_desc_sw128(st + (uint32_t)(j >> 1) * kSpXBox) + 4 * (j & 1);  // +64 B per k64 in the atom
      wgmma_m64n128k64_sp_s8(acc, da + 2 * j, db, ew[j], kb > 0 || j > 0);                  // +32 stored B per k64
    }
    wgmma_commit();
    // The sparse wgmma reads its metadata register when it executes, not when it issues, and ptxas does not guard
    // that register across the loop's back edge: the group retires before the next stage's words are loaded.
    wgmma_wait_s32<0>(acc);
    ring.release(kb, lane);
  }
  // every wgmma of both warpgroups has read its stage: the ring becomes the output tile, [token][feature] (row-major
  // out) or [feature][token] (NCHW out)
  asm volatile("bar.sync 1, 256;" ::: "memory");
  float* tile = reinterpret_cast<float*>(stage_base);
  if constexpr (kNchw) {
    sp_store_nchw(acc, tile, cn, sxw, bn, bias != nullptr, f0, q, warp - 4, lane, out, x_nan, m0, n0, M, N, P, vec4);
  } else {
#pragma unroll
    for (int c = 0; c < 16; ++c) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const long long I = (long long)acc[4 * c + 2 * h + e] + cn[h];
          float y = __double2float_rn((double)I * sxw[h]);
          if (bias) y = __fadd_rn(y, bn[h]);
          tile[(8 * c + 2 * q + e) * kSpLd + f0 + 8 * h] = y;
        }
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    // warp c of the consumers stores token rows c, c + 8, ...: lane l holds features 4 l .. 4 l + 3
    const int cw = warp - 4, nl = 4 * lane, n = n0 + nl;
    const float qnan = __int_as_float(0x7fc00000);
    for (int r = cw; r < kSpTok; r += 8) {
      const int m = m0 + r;
      if (m >= M) break;
      float4 v = *reinterpret_cast<const float4*>(tile + r * kSpLd + nl);
      if (__ldg(x_nan + m)) v = make_float4(qnan, qnan, qnan, qnan);
      float* o = out + (size_t)m * N + n;
      if (vec4 && n + 3 < N) {
        *reinterpret_cast<float4*>(o) = v;
      } else {
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (n + i < N) o[i] = vv[i];
      }
    }
  }
}

long long k64_of(long long k) { return (k + 63) / 64 * 64; }
long long meta_tiles(long long n) { return (n + kSpFeat - 1) / kSpFeat; }

// The lowered activations in the workspace, written by `lower` (the row quantizer or the conv lowering), then the
// sparse GEMM into `out` (row-major [M, N], or NCHW with P pixels per image).  Arguments are checked by the caller.
template <bool kNchw, typename Lower>
int sp_run(const char* fn, long long m, long long k, long long n, long long P, int qmin_x, const float* x_scale,
           const float* x_zero_point, const int8_t* vals, const uint32_t* meta, const int32_t* dsum, const float* w_scale,
           const float* bias, float* out, void* workspace, cudaStream_t st, Lower lower) {
  const I8Lowered w = i8_lowered(workspace, m, k);
  const long long kp = padded_k(k), kb64 = k64_of(k) / 64;
  CUtensorMap map_x, map_v, map_e;
  if (!make_map_2d(&map_x, CU_TENSOR_MAP_DATA_TYPE_UINT8, w.q, (uint64_t)kp, (uint64_t)m, (uint64_t)kp, 128, kSpTok,
                   CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_map_2d(&map_v, CU_TENSOR_MAP_DATA_TYPE_UINT8, vals, (uint64_t)(kb64 * 32), (uint64_t)n, (uint64_t)(kb64 * 32),
                   128, kSpFeat, CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_map_3d(&map_e, CU_TENSOR_MAP_DATA_TYPE_UINT32, meta, 256, (uint64_t)kb64, (uint64_t)meta_tiles(n), 1024, 256,
                   kSpBK / 64, CU_TENSOR_MAP_SWIZZLE_NONE)) {
    set_error("%s: cuTensorMapEncodeTiled failed (M=%lld K=%lld N=%lld)", fn, m, k, n);
    return SB200_E_CUDA;
  }
  if (const int rc = lower(w.q, w.sum, w.nan, st)) return rc;
  const size_t smem = (size_t)kSpStages * kSpStageBytes + sizeof(StageRing<kSpStages>) + 1024;
  static std::atomic<int> attr_done[64];
  SB_CUDA(ensure_dyn_smem(int8_sparse24_gemm_kernel<kNchw>, (int)smem, attr_done));
  const long long tiles = ((m + kSpTok - 1) / kSpTok) * ((n + kSpFeat - 1) / kSpFeat);
  // row-major: 16-byte stores of 4 features need N % 4 = 0; NCHW: each run of 4 pixels checks its own address
  const int vec4 = (kNchw || n % 4 == 0) && aligned16(out);
  int8_sparse24_gemm_kernel<kNchw><<<(unsigned)tiles, kSpThreads, smem, st>>>(
      map_x, map_v, map_e, out, w.nan, x_scale, x_zero_point, grid_offset(qmin_x), reinterpret_cast<const int*>(dsum),
      w_scale, bias, (int)m, (int)n, (int)kb64, vec4, (int)P);
  SB_LAUNCHED();
  return SB200_OK;
}

}  // namespace
}  // namespace sb200

using namespace sb200;

int sb200_sparse24_mask(const float* w, uint8_t* mask, int64_t rows, int64_t cols, void* stream) {
  const char* fn = "sb200_sparse24_mask";
  SB_REQUIRE(w && mask, "%s: null pointer argument", fn);
  SB_REQUIRE(rows > 0 && cols > 0, "%s: empty tensor (rows=%lld cols=%lld)", fn, (long long)rows, (long long)cols);
  const long long gpr = (cols + 3) / 4;
  SB_REQUIRE((__int128)rows * gpr < (1LL << 40), "%s: tensor too large", fn);
  const long long groups = rows * gpr;
  sparse24_mask_kernel<<<(unsigned)((groups + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, mask, rows, cols, gpr);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_int8_sparse24_pack(const int8_t* w_q, const int32_t* w_zero, const float* w_scale, int8_t* vals,
                             uint32_t* meta, int32_t* dsum, int32_t* bad, int64_t n, int64_t k, void* stream) {
  const char* fn = "sb200_int8_sparse24_pack";
  SB_REQUIRE(w_q && w_zero && w_scale && vals && meta && dsum && bad, "%s: null pointer argument", fn);
  SB_REQUIRE(n > 0 && k > 0, "%s: empty operand (N=%lld K=%lld)", fn, (long long)n, (long long)k);
  SB_REQUIRE(n < (1LL << 31), "%s: dimension too large (N=%lld)", fn, (long long)n);
  SB_REQUIRE(k < kI8MaxK, "%s: K >= 2^17, the integer path supports K < 2^17", fn);
  SB_REQUIRE(aligned16(vals), "%s: vals must be 16-byte aligned", fn);
  cudaStream_t st = (cudaStream_t)stream;
  SB_CUDA(cudaMemsetAsync(dsum, 0, (size_t)n * 4, st));
  SB_CUDA(cudaMemsetAsync(bad, 0, (size_t)n * 4, st));
  const long long kb64 = k64_of(k) / 64, words = meta_tiles(n) * kb64 * 256;
  sparse24_pack_kernel<<<(unsigned)((words + 255) / 256), 256, 0, st>>>(
      w_q, reinterpret_cast<const int*>(w_zero), w_scale, vals, meta, reinterpret_cast<int*>(dsum),
      reinterpret_cast<int*>(bad), (int)n, (int)k, (int)padded_k(k), (int)kb64, words);
  SB_LAUNCHED();
  return SB200_OK;
}

int sb200_int8_sparse24_linear(const float* x, const float* x_scale, const float* x_zero_point, int qmin_x, int qmax_x,
                               const int8_t* vals, const uint32_t* meta, const int32_t* dsum, const float* w_scale,
                               const float* bias, float* out, int64_t m, int64_t k, int64_t n, void* workspace,
                               size_t workspace_bytes, void* stream) {
  const char* fn = "sb200_int8_sparse24_linear";
  SB_REQUIRE(x && x_scale && x_zero_point && vals && meta && dsum && w_scale && out && workspace,
             "%s: null pointer argument", fn);
  SB_REQUIRE(m > 0 && k > 0 && n > 0, "%s: empty operand (M=%lld K=%lld N=%lld)", fn, (long long)m, (long long)k,
             (long long)n);
  SB_REQUIRE(m < (1LL << 31) && n < (1LL << 31), "%s: dimension too large", fn);
  if (const int rc = check_range(fn, qmin_x, qmax_x)) return rc;
  SB_REQUIRE(aligned16(vals) && aligned16(meta), "%s: vals and meta must be 16-byte aligned", fn);
  if (const int rc = check_k(fn, k)) return rc;
  if (const int rc = check_workspace(fn, workspace_bytes, sb200_int8_linear_workspace_bytes(m, k))) return rc;
  return sp_run<false>(fn, m, k, n, 1, qmin_x, x_scale, x_zero_point, vals, meta, dsum, w_scale, bias, out, workspace,
                       (cudaStream_t)stream, [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                         return launch_rows(x, x_scale, x_zero_point, 0, qmin_x, qmax_x, xq, xsum, xnan, m, k, st);
                       });
}

int sb200_int8_sparse24_conv2d(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                               const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* vals,
                               const uint32_t* meta, const int32_t* dsum, const float* w_scale, const float* bias,
                               float* out, int64_t c_out, void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "sb200_int8_sparse24_conv2d";
  SB_REQUIRE(x && geom && x_scale && x_zero_point && vals && meta && dsum && w_scale && out && workspace,
             "%s: null pointer argument", fn);
  SB_REQUIRE(c_out > 0, "%s: empty operand (c_out=%lld)", fn, (long long)c_out);
  SB_REQUIRE(c_out < (1LL << 31), "%s: dimension too large (c_out=%lld)", fn, (long long)c_out);
  ConvDims d;
  if (const int rc = check_conv(fn, geom, &d)) return rc;
  if (const int rc = check_range(fn, qmin_x, qmax_x)) return rc;
  SB_REQUIRE(aligned16(vals) && aligned16(meta), "%s: vals and meta must be 16-byte aligned", fn);
  if (const int rc = check_k(fn, d.K)) return rc;
  if (const int rc = check_workspace(fn, workspace_bytes, sb200_int8_conv2d_workspace_bytes(geom))) return rc;
  return sp_run<true>(fn, d.M, d.K, c_out, d.P, qmin_x, x_scale, x_zero_point, vals, meta, dsum, w_scale, bias, out,
                      workspace, (cudaStream_t)stream, [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                        return launch_im2col(x, d, x_scale, x_zero_point, qmin_x, qmax_x, xq, xsum, xnan, st);
                      });
}

int sb200_int8_sparse24_conv2d_nhwc(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                                    const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* vals,
                                    const uint32_t* meta, const int32_t* dsum, const float* w_scale, const float* bias,
                                    float* out, int64_t c_out, void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "sb200_int8_sparse24_conv2d_nhwc";
  SB_REQUIRE(x && geom && x_scale && x_zero_point && vals && meta && dsum && w_scale && out && workspace,
             "%s: null pointer argument", fn);
  SB_REQUIRE(c_out > 0, "%s: empty operand (c_out=%lld)", fn, (long long)c_out);
  SB_REQUIRE(c_out < (1LL << 31), "%s: dimension too large (c_out=%lld)", fn, (long long)c_out);
  ConvDims d;
  if (const int rc = check_conv(fn, geom, &d)) return rc;
  if (const int rc = check_range(fn, qmin_x, qmax_x)) return rc;
  SB_REQUIRE(aligned16(vals) && aligned16(meta), "%s: vals and meta must be 16-byte aligned", fn);
  if (const int rc = check_k(fn, d.K)) return rc;
  if (const int rc = check_workspace(fn, workspace_bytes, sb200_int8_conv2d_workspace_bytes(geom))) return rc;
  // the row-major [n OH OW, c_out] output of the linear is the NHWC storage of [n, c_out, OH, OW]
  return sp_run<false>(fn, d.M, d.K, c_out, 1, qmin_x, x_scale, x_zero_point, vals, meta, dsum, w_scale, bias, out,
                       workspace, (cudaStream_t)stream, [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                         return launch_im2col_nhwc(x, d, (int)geom->c, x_scale, x_zero_point, qmin_x, qmax_x, xq, xsum,
                                                   xnan, st);
                       });
}
