// int8_linear.cu -- integer-grid inference of a calibrated QLinear (per-tensor activations, per-tensor or
// per-output-channel weights):
//   y[m, n] = s_x * s_w[n] * sum_k v_x[m, k] * v_w[n, k] + bias[n],   v = clamp(round(x / s) + Z, qmin, qmax) - Z
// The fake-quant path computes the same sum as an fp32 SGEMM over v * s; here the integer sum is exact.
//
// Row quantizer.  One warp per row writes the grid value g = clamp(round(x / s) + Z, qmin, qmax) of every element as s8
// (QP / quant_round<0> of common.cuh: bit-identical to the QDQ kernels), stored as g - off with off = 128 for unsigned
// (affine) ranges and 0 otherwise, into rows of Kp = round_up(K, 16) bytes whose padding is zero; plus the int32 sum of
// each stored row and a per-row NaN flag.  NaN inputs make the row's flag 1 (and store 0); +-inf clamp to qmin / qmax.
//
// GEMM.  D[m, n] = sum_k a[m, k] * b[n, k] with wgmma.m64n128k32.s32.s8.s8, both operands K-major in shared memory,
// TMA-loaded as 128-row x 128-byte SWIZZLE_128B boxes into a ring of kI8Stages stages.  CTA = one 128-row x
// 128-feature output tile: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = 64 rows each.  Rows and
// features beyond M / N and K beyond Kp are zero-filled by the TMA; the epilogue masks the partial tiles.  The zero
// points come out exactly in int64,
//   I = sum a b - Z_w sum_k a - Z_x sum_k b + K Z_x Z_w        (Z = the zero points on the stored grid, Z' = rint(zp) - off)
// then y = fp32(fp64(I * (s_x * s_w[n]))) (+ bias[n] in fp32; s_x * s_w is exact in fp64), and NaN for flagged rows.
// |a|, |b| <= 128, so |sum a b| <= K * 2^14 fits the s32 accumulator for K < 2^17.  No atomics, no split-K, no state
// between calls: deterministic and safe under CUDA graph capture.
//
// Conv2d.  A calibrated QConv2d is the same GEMM once its input is lowered: M = N OH OW output pixels, K = C KH KW,
// N = C_out, with the K order (c, kh, kw) of weight.reshape(C_out, -1).  The lowering kernel writes the grid value of
// every tap of every window as one s8 row per output pixel (the same grid as the row quantizer); a padding tap is the
// grid point of the fake-quant input's zero padding, v = 0, i.e. rint(zp) - off on the stored grid, so the epilogue's
// correction stays exact with the real K.  The GEMM then writes NCHW: out[(img N + n) P + p], m = img P + p, P = OH OW.
#include "tc_common.cuh"

namespace sb200 {
namespace {

constexpr int kI8Rows = 128;                      // rows of x per CTA (two consumer warpgroups x 64)
constexpr int kI8Feat = 128;                      // output features per CTA = wgmma N
constexpr int kI8BK = 128;                        // K per stage: one 128-byte swizzle atom of s8
constexpr int kI8Stages = 6;
constexpr int kI8Threads = 384;
constexpr int kI8TileBytes = kI8Rows * kI8BK;     // 16 KB (x tile; the weight tile has the same size)
constexpr int kI8StageBytes = 2 * kI8TileBytes;   // 32 KB
constexpr long long kI8MaxK = 1LL << 17;

// per-feature epilogue terms of the CTA's 128 features, computed once per tile
struct I8Col {
  long long cn;  // K Z_x Z_w - Z_x sum_k b
  double sxw;    // s_x * s_w[n], exact in fp64
  int zw;
  float bias;
};
struct I8Smem {
  uint64_t full[kI8Stages];
  uint64_t empty[kI8Stages];
  I8Col col[kI8Feat];
};

static inline int grid_offset(int qmin) { return qmin >= 0 ? 128 : 0; }
static inline long long padded_k(long long k) { return (k + 15) / 16 * 16; }

// ---------------------------------------------------------------------------------- row quantizer
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

// 8 warps per CTA, one row per warp; lane l handles the 16-element chunks starting at 16 l, 16 (l + 32), ...
__global__ void __launch_bounds__(256) int8_quantize_rows_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                                 const float* __restrict__ zero_point, int per_row, float qmin,
                                                                 float qmax, int off, int8_t* __restrict__ q,
                                                                 int* __restrict__ row_sum, uint8_t* __restrict__ nan_flag,
                                                                 long long rows, int K, int Kp, int vec) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  QP p;
  const long long pi = per_row ? row : 0;
  p.set(__ldg(scale + pi), __ldg(zero_point + pi));
  p.qmin = qmin;
  p.qmax = qmax;
  const float* xr = x + row * K;
  int8_t* qr = q + row * Kp;
  int sum = 0;
  bool nan = false;
  for (int c = lane * 16; c < Kp; c += 32 * 16) {
    float v[16];
    if (vec && c + 16 <= K) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 f = ld_stream4(reinterpret_cast<const float4*>(xr + c) + i);
        v[4 * i] = f.x, v[4 * i + 1] = f.y, v[4 * i + 2] = f.z, v[4 * i + 3] = f.w;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = c + i < K ? ld_stream1(xr + c + i) : 0.f;
    }
    uint32_t packed[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      int e = 0;  // K padding stays zero
      if (c + i < K) e = stored_grid(v[i], p, off, nan);
      sum += e;
      packed[i >> 2] |= ((uint32_t)e & 0xFFu) << (8 * (i & 3));
    }
    *reinterpret_cast<uint4*>(qr + c) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const bool any_nan = __any_sync(0xffffffffu, nan);
  if (lane == 0) {
    row_sum[row] = sum;
    nan_flag[row] = any_nan ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------- conv2d lowering
// Conv geometry on the device; every product is 64-bit (M Kp passes 2^31 at ResNet-50 stem sizes from batch ~1024).
struct ConvDims {
  long long H, W, HW, CHW;     // input plane, image
  long long sh, sw, dh, dw;    // stride, dilation
  long long pt, pl;            // top / left padding
  long long OW, P, M;          // output width, pixels per image, output pixels
  int KH, KW, K, Kp;           // taps, taps padded to 16
};

constexpr int kLowPix = 128;              // output pixels (rows of q) per CTA
constexpr int kLowK = 128;                // taps per chunk: one 128-byte line of each row of q
constexpr int kLowWords = kLowK / 4 + 1;  // words per tile row, padded: the column writes are conflict-free
constexpr int kLowThreads = 256;

// One CTA per 128 consecutive output pixels, K in chunks of 128 taps.  Thread t owns pixel t % 128 and every other
// group of 4 taps of the chunk: a warp reads one tap of 32 consecutive pixels (consecutive ow: coalesced along the
// row of x), packs 4 taps per word into a shared tile, and the tile leaves as whole 16-byte pieces of rows of q.
// Row sums and NaN flags stay in registers across the chunks.
__global__ void __launch_bounds__(kLowThreads) int8_im2col_quantize_kernel(const float* __restrict__ x, ConvDims d,
                                                                           const float* __restrict__ scale,
                                                                           const float* __restrict__ zero_point,
                                                                           float qmin, float qmax, int off,
                                                                           int8_t* __restrict__ q,
                                                                           int* __restrict__ row_sum,
                                                                           uint8_t* __restrict__ nan_flag) {
  __shared__ uint32_t tile[kLowPix * kLowWords];
  __shared__ long long tap_off[kLowK], tap_dh[kLowK], tap_dw[kLowK];  // per tap of the chunk: x offset, row, column
  __shared__ int part_sum[kLowThreads];
  __shared__ bool part_nan[kLowThreads];
  const int t = threadIdx.x, px = t % kLowPix, kq0 = t / kLowPix;
  const long long m = (long long)blockIdx.x * kLowPix + px;
  const bool live = m < d.M;
  long long ih0 = 0, iw0 = 0, org = 0;  // top-left tap of the window and its offset in x
  if (live) {
    const long long img = m / d.P, pix = m - img * d.P;
    const long long oh = pix / d.OW, ow = pix - oh * d.OW;
    ih0 = oh * d.sh - d.pt;
    iw0 = ow * d.sw - d.pl;
    org = img * d.CHW + ih0 * d.W + iw0;
  }
  QP p;
  p.set(__ldg(scale), __ldg(zero_point));
  p.qmin = qmin;
  p.qmax = qmax;
  const int pad = (int)p.zp - off;  // the grid point v = 0 of the fake-quant input's zero padding
  int sum = 0;
  bool nan = false;
  for (int k0 = 0; k0 < d.Kp; k0 += kLowK) {
    const int kc = min(kLowK, d.Kp - k0);
    if (t < kc) {
      const int k = k0 + t;
      long long o = 0, a = 0, b = 0;
      if (k < d.K) {
        const int c = k / (d.KH * d.KW), r = k - c * (d.KH * d.KW), kh = r / d.KW, kw = r - kh * d.KW;
        a = kh * d.dh;
        b = kw * d.dw;
        o = c * d.HW + a * d.W + b;
      }
      tap_off[t] = o, tap_dh[t] = a, tap_dw[t] = b;
    }
    __syncthreads();  // the tap table is written; the previous chunk's tile has been read
#pragma unroll 4
    for (int qd = kq0; qd < kc / 4; qd += kLowThreads / kLowPix) {
      uint32_t packed = 0u;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kl = 4 * qd + i;
        int e = 0;  // K padding stays zero
        if (live && k0 + kl < d.K) {
          const long long ih = ih0 + tap_dh[kl], iw = iw0 + tap_dw[kl];
          if ((unsigned long long)ih < (unsigned long long)d.H && (unsigned long long)iw < (unsigned long long)d.W)
            e = stored_grid(__ldg(x + org + tap_off[kl]), p, off, nan);
          else
            e = pad;
        }
        sum += e;
        packed |= ((uint32_t)e & 0xFFu) << (8 * i);
      }
      tile[px * kLowWords + qd] = packed;
    }
    __syncthreads();
    const int pieces = kc / 16;  // 16-byte pieces per row
    for (int idx = t; idx < kLowPix * pieces; idx += kLowThreads) {
      const int row = idx / pieces, j = idx - row * pieces;
      const long long mr = (long long)blockIdx.x * kLowPix + row;
      if (mr < d.M) {
        const uint32_t* s = tile + row * kLowWords + 4 * j;
        *reinterpret_cast<uint4*>(q + mr * d.Kp + k0 + 16 * j) = make_uint4(s[0], s[1], s[2], s[3]);
      }
    }
  }
  part_sum[t] = sum;
  part_nan[t] = nan;
  __syncthreads();
  if (t < kLowPix && live) {
    for (int h = 1; h < kLowThreads / kLowPix; ++h) {
      sum += part_sum[t + h * kLowPix];
      nan = nan || part_nan[t + h * kLowPix];
    }
    row_sum[m] = sum;
    nan_flag[m] = nan ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------- GEMM
// D[64 x 128] (+)= A[64 x 32] * B[32 x 128], s8 x s8 -> s32, both operands K-major SWIZZLE_128B in shared memory.
__device__ __forceinline__ void wgmma_m64n128k32_s8(int (&d)[64], uint64_t adesc, uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "%64, %65, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// wait until at most N wgmma groups of this warpgroup are outstanding; the accumulators are threaded through the
// statement so that no use of them can be scheduled above the wait
template <int N>
__device__ __forceinline__ void wgmma_wait_s32(int (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// One CTA per 128-row x 128-feature tile of y (row tile fastest: neighbouring CTAs share the weight tile in L2).
// kNchw = false: out is row-major [M, N].  kNchw = true: out is NCHW [M / P, N, P] (conv2d, P = OH OW pixels per image).
template <bool kNchw>
__global__ void __launch_bounds__(kI8Threads, 1)
int8_linear_gemm_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                        float* __restrict__ out, const int* __restrict__ x_sum, const uint8_t* __restrict__ x_nan,
                        const float* __restrict__ x_scale, const float* __restrict__ x_zero, int x_off,
                        const int* __restrict__ w_sum, const float* __restrict__ w_scale, const int* __restrict__ w_zero,
                        const float* __restrict__ bias, int M, int N, int K, int P) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* stage_base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  I8Smem* sm = reinterpret_cast<I8Smem*>(stage_base + (size_t)kI8Stages * kI8StageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + kI8Rows - 1) / kI8Rows;
  const int m0 = (int)(blockIdx.x % (unsigned)tiles_m) * kI8Rows, n0 = (int)(blockIdx.x / (unsigned)tiles_m) * kI8Feat;
  const int num_kb = (K + kI8BK - 1) / kI8BK;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    for (int s = 0; s < kI8Stages; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], 8);  // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<40>();
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % kI8Stages;
        const uint32_t ph = (uint32_t)(kb / kI8Stages) & 1u;
        mbar_wait_relaxed(&sm->empty[s], ph ^ 1u, 0);
        unsigned char* st = stage_base + (size_t)s * kI8StageBytes;
        mbar_expect_tx(&sm->full[s], (uint32_t)kI8StageBytes);
        tma_load_2d(st, &map_x, kb * kI8BK, m0, &sm->full[s]);
        tma_load_2d(st + kI8TileBytes, &map_w, kb * kI8BK, n0, &sm->full[s]);
      }
    }
    return;
  }
  reg_inc<232>();
  const int wg = (warp - 4) >> 2;  // consumer warpgroup: rows 64 wg .. 64 wg + 63 of the tile
  const uint32_t stage0 = smem_u32(stage_base);
  // the epilogue's per-feature and per-row terms are fetched while the ring fills
  const float sx = __ldg(x_scale);
  const long long zx = (long long)rintf(__ldg(x_zero)) - x_off;
  if (threadIdx.x - 128 < (unsigned)kI8Feat) {
    const int i = threadIdx.x - 128, n = n0 + i;
    I8Col c{0, 0.0, 0, 0.f};
    if (n < N) {
      c.zw = __ldg(w_zero + n);
      c.cn = (long long)K * zx * c.zw - zx * (long long)__ldg(w_sum + n);
      c.sxw = (double)sx * (double)__ldg(w_scale + n);
      c.bias = bias ? __ldg(bias + n) : 0.f;
    }
    sm->col[i] = c;
  }
  const int q = lane & 3;
  const int r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
  long long sa[2];
  bool rnan[2];
  size_t obase[2];  // NCHW: out offset of (row, feature 0), img N P + p; one division per row
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = r0 + 8 * h;
    sa[h] = m < M ? (long long)__ldg(x_sum + m) : 0;
    rnan[h] = m < M && __ldg(x_nan + m) != 0;
    if constexpr (kNchw) {
      const int img = m / P;
      obase[h] = (size_t)img * N * P + (size_t)(m - img * P);
    }
  }
  int acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % kI8Stages;
    const uint32_t ph = (uint32_t)(kb / kI8Stages) & 1u;
    mbar_wait_relaxed(&sm->full[s], ph, 0);
    const uint32_t xa = stage0 + (uint32_t)s * kI8StageBytes;
    const uint64_t da = gmma_desc_sw128(xa + (uint32_t)wg * (64 * kI8BK)), db = gmma_desc_sw128(xa + kI8TileBytes);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) wgmma_m64n128k32_s8(acc, da + 2 * j, db + 2 * j, kb > 0 || j > 0);  // +32 B per k32
    wgmma_commit();
    // one group stays in flight: the stage of the previous k block is free once this wait returns
    wgmma_wait_s32<1>(acc);
    __syncwarp();
    if (kb > 0 && lane == 0) mbar_arrive(&sm->empty[(kb + kI8Stages - 1) % kI8Stages]);
  }
  wgmma_wait_s32<0>(acc);
  asm volatile("bar.sync 1, 256;" ::: "memory");  // sm->col written by both consumer warpgroups

  // acc[j]: row r0 + 8 ((j >> 1) & 1), feature n0 + 8 (j >> 2) + 2 q + (j & 1)
#pragma unroll
  for (int c = 0; c < 16; ++c) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int i = 8 * c + 2 * q + e, n = n0 + i;
      if (n >= N) continue;
      const I8Col col = sm->col[i];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = r0 + 8 * h;
        if (m >= M) continue;
        const long long I = (long long)acc[4 * c + 2 * h + e] - (long long)col.zw * sa[h] + col.cn;
        float y = __double2float_rn((double)I * col.sxw);
        if (bias) y = __fadd_rn(y, col.bias);
        if (rnan[h]) y = __int_as_float(0x7fc00000);
        if constexpr (kNchw) out[obase[h] + (size_t)n * P] = y;  // a warp stores 8 consecutive pixels per feature
        else out[(size_t)m * N + n] = y;
      }
    }
  }
}

struct I8Layout {
  size_t off_q, off_sum, off_nan, total;
};
I8Layout i8_layout(long long M, long long K) {
  I8Layout w;
  w.off_q = 0;
  w.off_sum = align_up((size_t)M * (size_t)padded_k(K), 1024);
  w.off_nan = w.off_sum + align_up((size_t)M * 4, 256);
  w.total = w.off_nan + align_up((size_t)M, 256);
  return w;
}

// the integer range [qmin, qmax] must fit s8 after the offset
int check_range(const char* fn, int qmin, int qmax) {
  SB_REQUIRE(qmin <= qmax, "%s: qmin %d > qmax %d", fn, qmin, qmax);
  SB_REQUIRE((long long)qmax - qmin <= 255, "%s: integer range [%d, %d] is wider than 8 bits", fn, qmin, qmax);
  const int off = grid_offset(qmin);
  SB_REQUIRE(qmin - off >= -128 && qmax - off <= 127,
             "%s: integer range [%d, %d] is neither signed 8-bit [-128, 127] nor unsigned 8-bit [0, 255]", fn, qmin, qmax);
  return SB200_OK;
}

int launch_rows(const float* x, const float* scale, const float* zero_point, int per_row, int qmin, int qmax, int8_t* q,
                int* row_sum, uint8_t* nan_flag, long long rows, long long k, cudaStream_t st) {
  const int vec = (k % 4 == 0) && aligned16(x);
  int8_quantize_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(x, scale, zero_point, per_row, (float)qmin, (float)qmax,
                                                                      grid_offset(qmin), q, row_sum, nan_flag, rows, (int)k,
                                                                      (int)padded_k(k), vec);
  SB_LAUNCHED();
  return SB200_OK;
}


// The lowered activations (q, row sums, NaN flags) in the workspace, written by `lower`, then the GEMM into `out`
// (row-major [M, N], or NCHW with P pixels per image).  Arguments are checked by the caller.
template <bool kNchw, typename Lower>
int run_gemm(const char* fn, long long m, long long k, long long n, long long P, int qmin_x, const float* x_scale,
             const float* x_zero_point, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
             const int32_t* w_zero, const float* bias, float* out, void* workspace, cudaStream_t st, Lower lower) {
  const I8Layout w = i8_layout(m, k);
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  int8_t* xq = reinterpret_cast<int8_t*>(ws + w.off_q);
  int* xsum = reinterpret_cast<int*>(ws + w.off_sum);
  uint8_t* xnan = ws + w.off_nan;
  const long long kp = padded_k(k);

  CUtensorMap map_x, map_w;
  if (!make_map_2d(&map_x, CU_TENSOR_MAP_DATA_TYPE_UINT8, xq, (uint64_t)kp, (uint64_t)m, (uint64_t)kp, kI8BK, kI8Rows,
                   CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_map_2d(&map_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, w_q, (uint64_t)kp, (uint64_t)n, (uint64_t)kp, kI8BK, kI8Feat,
                   CU_TENSOR_MAP_SWIZZLE_128B)) {
    set_error("%s: cuTensorMapEncodeTiled failed (M=%lld K=%lld N=%lld)", fn, m, k, n);
    return SB200_E_CUDA;
  }
  if (const int rc = lower(xq, xsum, xnan, st)) return rc;
  const size_t smem = (size_t)kI8Stages * kI8StageBytes + sizeof(I8Smem) + 1024;
  static std::atomic<int> attr_done[64];
  SB_CUDA(ensure_dyn_smem(int8_linear_gemm_kernel<kNchw>, (int)smem, attr_done));
  const long long tiles = ((m + kI8Rows - 1) / kI8Rows) * ((n + kI8Feat - 1) / kI8Feat);
  int8_linear_gemm_kernel<kNchw><<<(unsigned)tiles, kI8Threads, smem, st>>>(
      map_x, map_w, out, xsum, xnan, x_scale, x_zero_point, grid_offset(qmin_x), reinterpret_cast<const int*>(w_rowsum),
      w_scale, reinterpret_cast<const int*>(w_zero), bias, (int)m, (int)n, (int)k, (int)P);
  SB_LAUNCHED();
  return SB200_OK;
}

// Output shape of a conv geometry.  Returns 0, or which rule it breaks: 1 = a size, stride or dilation <= 0, a
// padding < 0, or a dimension >= 2^31; 2 = an empty output; 3 = M >= 2^31.  K is saturated at 2^17.
int conv_shape(const sb200_conv2d_geom& g, ConvDims* d) {
  const int64_t pos[] = {g.n, g.c, g.h, g.w, g.kh, g.kw, g.stride_h, g.stride_w, g.dilation_h, g.dilation_w};
  const int64_t pads[] = {g.pad_top, g.pad_bottom, g.pad_left, g.pad_right};
  for (int64_t v : pos)
    if (v <= 0 || v >= (1LL << 31)) return 1;
  for (int64_t v : pads)
    if (v < 0 || v >= (1LL << 31)) return 1;
  if ((__int128)g.n * g.c * g.h * g.w >= ((__int128)1 << 62)) return 1;
  const long long oh_num = g.h + g.pad_top + g.pad_bottom - g.dilation_h * (g.kh - 1) - 1;
  const long long ow_num = g.w + g.pad_left + g.pad_right - g.dilation_w * (g.kw - 1) - 1;
  if (oh_num < 0 || ow_num < 0) return 2;
  const long long OH = oh_num / g.stride_h + 1, OW = ow_num / g.stride_w + 1;
  if ((__int128)g.n * OH * OW >= ((__int128)1 << 31)) return 3;
  const __int128 K = (__int128)g.c * g.kh * g.kw;
  d->H = g.h, d->W = g.w, d->HW = g.h * g.w, d->CHW = g.c * g.h * g.w;
  d->sh = g.stride_h, d->sw = g.stride_w, d->dh = g.dilation_h, d->dw = g.dilation_w;
  d->pt = g.pad_top, d->pl = g.pad_left;
  d->OW = OW, d->P = OH * OW, d->M = g.n * OH * OW;
  d->KH = (int)g.kh, d->KW = (int)g.kw;
  d->K = K >= kI8MaxK ? (int)kI8MaxK : (int)K;
  d->Kp = (int)padded_k(d->K);
  return 0;
}

// Checks of the conv entry points that come before the range check
int check_conv(const char* fn, const sb200_conv2d_geom* g, ConvDims* d) {
  const int rule = conv_shape(*g, d);
  SB_REQUIRE(rule != 1, "%s: empty or non-positive geometry (n=%lld c=%lld h=%lld w=%lld kernel %lldx%lld stride %lldx%lld "
             "dilation %lldx%lld padding %lld/%lld/%lld/%lld)", fn, (long long)g->n, (long long)g->c, (long long)g->h,
             (long long)g->w, (long long)g->kh, (long long)g->kw, (long long)g->stride_h, (long long)g->stride_w,
             (long long)g->dilation_h, (long long)g->dilation_w, (long long)g->pad_top, (long long)g->pad_bottom,
             (long long)g->pad_left, (long long)g->pad_right);
  SB_REQUIRE(rule != 2, "%s: empty output (the dilated kernel does not fit the padded input)", fn);
  SB_REQUIRE(rule != 3, "%s: too many output pixels (M = n OH OW must be < 2^31)", fn);
  return SB200_OK;
}

int check_conv_k(const char* fn, const ConvDims& d) {
  if (d.K >= kI8MaxK) {
    set_error("%s: K = c kh kw >= 2^17, the integer path supports K < 2^17 (|sum| <= K * 2^14 must fit int32)", fn);
    return SB200_E_UNSUPPORTED;
  }
  return SB200_OK;
}

int launch_im2col(const float* x, const ConvDims& d, const float* scale, const float* zero_point, int qmin, int qmax,
                  int8_t* q, int* row_sum, uint8_t* nan_flag, cudaStream_t st) {
  int8_im2col_quantize_kernel<<<(unsigned)((d.M + kLowPix - 1) / kLowPix), kLowThreads, 0, st>>>(
      x, d, scale, zero_point, (float)qmin, (float)qmax, grid_offset(qmin), q, row_sum, nan_flag);
  SB_LAUNCHED();
  return SB200_OK;
}

}  // namespace
}  // namespace sb200

using namespace sb200;

size_t sb200_int8_linear_workspace_bytes(int64_t m, int64_t k) {
  if (m <= 0 || k <= 0) return 0;
  return i8_layout(m, k).total + 1024;  // + the alignment of the workspace base to 1024 bytes
}

int sb200_int8_quantize_rows(const float* x, const float* scale, const float* zero_point, int per_row, int qmin, int qmax,
                             int8_t* q, int32_t* row_sum, uint8_t* nan_flag, int64_t rows, int64_t k, void* stream) {
  SB_REQUIRE(x && scale && zero_point && q && row_sum && nan_flag, "sb200_int8_quantize_rows: null pointer argument");
  SB_REQUIRE(rows > 0 && k > 0, "sb200_int8_quantize_rows: empty operand (rows=%lld K=%lld)", (long long)rows, (long long)k);
  SB_REQUIRE(rows < (1LL << 31), "sb200_int8_quantize_rows: too many rows (%lld)", (long long)rows);
  if (const int rc = check_range("sb200_int8_quantize_rows", qmin, qmax)) return rc;
  SB_REQUIRE(aligned16(q), "sb200_int8_quantize_rows: q must be 16-byte aligned");
  if (k >= kI8MaxK) {
    set_error("sb200_int8_quantize_rows: K = %lld, the integer path supports K < 2^17", (long long)k);
    return SB200_E_UNSUPPORTED;
  }
  return launch_rows(x, scale, zero_point, per_row != 0, qmin, qmax, q, reinterpret_cast<int*>(row_sum), nan_flag, rows, k,
                     (cudaStream_t)stream);
}

int sb200_int8_linear(const float* x, const float* x_scale, const float* x_zero_point, int qmin_x, int qmax_x,
                      const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero,
                      const float* bias, float* out, int64_t m, int64_t k, int64_t n, void* workspace,
                      size_t workspace_bytes, void* stream) {
  SB_REQUIRE(x && x_scale && x_zero_point && w_q && w_rowsum && w_scale && w_zero && out && workspace,
             "sb200_int8_linear: null pointer argument");
  SB_REQUIRE(m > 0 && k > 0 && n > 0, "sb200_int8_linear: empty operand (M=%lld K=%lld N=%lld)", (long long)m, (long long)k,
             (long long)n);
  SB_REQUIRE(m < (1LL << 31) && n < (1LL << 31), "sb200_int8_linear: dimension too large");
  if (const int rc = check_range("sb200_int8_linear", qmin_x, qmax_x)) return rc;
  SB_REQUIRE(aligned16(w_q), "sb200_int8_linear: w_q must be 16-byte aligned");
  if (k >= kI8MaxK) {
    set_error("sb200_int8_linear: K = %lld, the integer path supports K < 2^17 (|sum| <= K * 2^14 must fit int32)",
              (long long)k);
    return SB200_E_UNSUPPORTED;
  }
  if (workspace_bytes < sb200_int8_linear_workspace_bytes(m, k)) {  // covers any alignment of the base
    set_error("sb200_int8_linear: workspace too small (%zu bytes, need %zu)", workspace_bytes,
              sb200_int8_linear_workspace_bytes(m, k));
    return SB200_E_WORKSPACE;
  }
  return run_gemm<false>("sb200_int8_linear", m, k, n, 1, qmin_x, x_scale, x_zero_point, w_q, w_rowsum, w_scale, w_zero,
                         bias, out, workspace, (cudaStream_t)stream,
                         [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                           return launch_rows(x, x_scale, x_zero_point, 0, qmin_x, qmax_x, xq, xsum, xnan, m, k, st);
                         });
}

size_t sb200_int8_conv2d_workspace_bytes(const sb200_conv2d_geom* geom) {
  ConvDims d;
  if (!geom || conv_shape(*geom, &d) != 0) return 0;
  return sb200_int8_linear_workspace_bytes(d.M, d.K);
}

int sb200_int8_im2col_quantize(const float* x, const sb200_conv2d_geom* geom, const float* scale,
                               const float* zero_point, int qmin, int qmax, int8_t* q, int32_t* row_sum,
                               uint8_t* nan_flag, void* stream) {
  const char* fn = "sb200_int8_im2col_quantize";
  SB_REQUIRE(x && geom && scale && zero_point && q && row_sum && nan_flag, "%s: null pointer argument", fn);
  ConvDims d;
  if (const int rc = check_conv(fn, geom, &d)) return rc;
  if (const int rc = check_range(fn, qmin, qmax)) return rc;
  SB_REQUIRE(aligned16(q), "%s: q must be 16-byte aligned", fn);
  if (const int rc = check_conv_k(fn, d)) return rc;
  return launch_im2col(x, d, scale, zero_point, qmin, qmax, q, reinterpret_cast<int*>(row_sum), nan_flag,
                       (cudaStream_t)stream);
}

int sb200_int8_conv2d(const float* x, const sb200_conv2d_geom* geom, const float* x_scale, const float* x_zero_point,
                      int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                      const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* workspace,
                      size_t workspace_bytes, void* stream) {
  const char* fn = "sb200_int8_conv2d";
  SB_REQUIRE(x && geom && x_scale && x_zero_point && w_q && w_rowsum && w_scale && w_zero && out && workspace,
             "%s: null pointer argument", fn);
  SB_REQUIRE(c_out > 0, "%s: empty operand (c_out=%lld)", fn, (long long)c_out);
  SB_REQUIRE(c_out < (1LL << 31), "%s: dimension too large (c_out=%lld)", fn, (long long)c_out);
  ConvDims d;
  if (const int rc = check_conv(fn, geom, &d)) return rc;
  if (const int rc = check_range(fn, qmin_x, qmax_x)) return rc;
  SB_REQUIRE(aligned16(w_q), "%s: w_q must be 16-byte aligned", fn);
  if (const int rc = check_conv_k(fn, d)) return rc;
  const size_t need = sb200_int8_conv2d_workspace_bytes(geom);
  if (workspace_bytes < need) {
    set_error("%s: workspace too small (%zu bytes, need %zu)", fn, workspace_bytes, need);
    return SB200_E_WORKSPACE;
  }
  return run_gemm<true>(fn, d.M, d.K, c_out, d.P, qmin_x, x_scale, x_zero_point, w_q, w_rowsum, w_scale, w_zero, bias,
                        out, workspace, (cudaStream_t)stream,
                        [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                          return launch_im2col(x, d, x_scale, x_zero_point, qmin_x, qmax_x, xq, xsum, xnan, st);
                        });
}
