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
//
// MatMul.  A calibrated activation x activation matmul a [B, M, K] @ b [B, K, N] has two per-tensor operands and no
// bias: y = s_a s_b I.  Both are quantized on the fly into [rows, Kp] s8: a, and a b that lies K-major in memory
// ([B, N, K], the k^T of attention), by the row quantizer; a b that lies N-major ([B, K, N]) by the column quantizer,
// which transposes through shared memory.  The batched GEMM kernel runs the same ring and wgmma loop as the linear
// (i8_produce / i8_consume below) over 3-D tensor maps (Kp, rows, batch), so that a tile never reaches into the next
// batch entry, with its own epilogue: per-row sum_k a, per-column sum_k b, both NaN flags, one scale product.
#include "int8_grid.cuh"
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

// per-feature epilogue terms of the CTA's 128 features, computed once per tile
struct I8Col {
  long long cn;  // K Z_x Z_w - Z_x sum_k b
  double sxw;    // s_x * s_w[n], exact in fp64
  int zw;
  float bias;
};
struct I8Smem {
  StageRing<kI8Stages> ring;
  I8Col col[kI8Feat];
};
// the matmul's per-column terms: both scales and zero points are scalars
struct I8MmCol {
  long long cn;  // K Z_a Z_b - Z_a sum_k b
  int nan;       // the column of b holds a NaN
};
struct I8MmSmem {
  StageRing<kI8Stages> ring;
  I8MmCol col[kI8Feat];
};

// ---------------------------------------------------------------------------------- row quantizer
// Every kernel of this file stores an element through stored_grid(v, p, off, nan) of int8_grid.cuh, the one
// quantizer of the integer path, which the grouped conv kernel (int8_group_conv.cu) shares:
//   g = clamp(quant_round<0>(v, p) + rint(zp), qmin, qmax)   (QP / quant_round<0> of common.cuh, as the QDQ kernels:
//                                                             half-to-even, +-inf clamp to qmin / qmax)
//   stored value = (int)g - off,   off = 128 for unsigned ranges, 0 otherwise
// A NaN (g != g) sets the caller's `nan` and stores 0.  Because all of them go through this one function, a window
// of the conv2d lowering below and the grouped conv kernel's shared-memory tile hold the same stored values for the
// same input, and a grouped conv's group is bit-identical to this file's conv2d run on that group's channel slice.
// The row quantizer below writes the stored value of every element of a row, its int32 row sum and a NaN flag; the
// column quantizer and the conv2d lowering are the same per element.

// 8 warps per CTA, one row per warp; lane l handles the 16-element chunks starting at 16 l, 16 (l + 32), ...
// kDoReFa: x is a DoReFa input normalised by *x_absmax (input_grid), as in every lowering below.
template <bool kDoReFa>
__global__ void __launch_bounds__(256) int8_quantize_rows_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                                 const float* __restrict__ zero_point, int per_row, float qmin,
                                                                 float qmax, int off, int8_t* __restrict__ q,
                                                                 int* __restrict__ row_sum, uint8_t* __restrict__ nan_flag,
                                                                 long long rows, int K, int Kp, int vec,
                                                                 const float* __restrict__ x_absmax) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const double xm = kDoReFa ? dorefa_rcp(__ldg(x_absmax)) : 0.0;  // 1 / m of a DoReFa input
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
      if (c + i < K) e = input_grid<kDoReFa>(v[i], xm, p, off, nan);
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

// ---------------------------------------------------------------------------------- column quantizer
constexpr int kColN = 64;                 // columns of x (rows of q) per CTA
constexpr int kColK = 128;                // K per chunk: one 128-byte line of each row of q
constexpr int kColWords = kColK / 4 + 1;  // words per tile row, padded: the transposing writes are conflict-free
constexpr int kColThreads = 256;

// x [batch, K, N] -> q [batch, N, Kp]: the row quantizer's grid, transposed.  One CTA per 64 columns of one batch entry,
// K in chunks of 128.  A thread owns 4 neighbouring columns for the whole of K and, per chunk, two groups of 4 k: it
// reads a 4 x 4 block (vec: one 16-byte load per k, 8 lanes covering a 128-byte line of the row; otherwise guarded
// scalar loads), packs the 4 k of each column into one word of a shared tile, and the tile leaves as whole 16-byte
// pieces of rows of q.  Column sums and NaN flags stay in registers across the chunks.
__global__ void __launch_bounds__(kColThreads) int8_quantize_cols_kernel(const float* __restrict__ x, const float* __restrict__ scale,
                                                                         const float* __restrict__ zero_point, float qmin,
                                                                         float qmax, int off, int8_t* __restrict__ q,
                                                                         int* __restrict__ col_sum,
                                                                         uint8_t* __restrict__ nan_flag, int tiles_n, int K,
                                                                         int N, int Kp, int vec) {
  __shared__ uint32_t tile[kColN * kColWords];
  __shared__ int part_sum[kColThreads / 64][kColN];
  __shared__ int part_nan[kColThreads / 64][kColN];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const long long b = blockIdx.x / (unsigned)tiles_n;
  const int n0 = (int)(blockIdx.x % (unsigned)tiles_n) * kColN;
  const int nl = 4 * (8 * (warp & 1) + (lane >> 2));  // first of the thread's 4 columns, within the tile
  const int kslot = 4 * (warp >> 1) + (lane & 3);     // the thread's k groups of a chunk: kslot and kslot + 16
  const int n = n0 + nl;
  const float* xb = x + b * K * N;
  int8_t* qb = q + b * N * Kp;
  QP p;
  p.set(__ldg(scale), __ldg(zero_point));
  p.qmin = qmin;
  p.qmax = qmax;
  int sum[4] = {0, 0, 0, 0};
  bool nan[4] = {false, false, false, false};
  for (int k0 = 0; k0 < Kp; k0 += kColK) {
    const int kc = min(kColK, Kp - k0);
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int kq = kslot + 16 * it, kk = k0 + 4 * kq;
      if (4 * kq >= kc) continue;
      float v[4][4];  // [k][column]
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float* xr = xb + (long long)(kk + i) * N + n;
        if (vec && kk + i < K && n < N) {
          const float4 f = ld_stream4(reinterpret_cast<const float4*>(xr));
          v[i][0] = f.x, v[i][1] = f.y, v[i][2] = f.z, v[i][3] = f.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) v[i][j] = (kk + i < K && n + j < N) ? ld_stream1(xr + j) : 0.f;
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t packed = 0u;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          int e = 0;  // K padding stays zero
          if (kk + i < K && n + j < N) e = stored_grid(v[i][j], p, off, nan[j]);
          sum[j] += e;
          packed |= ((uint32_t)e & 0xFFu) << (8 * i);
        }
        tile[(nl + j) * kColWords + kq] = packed;
      }
    }
    __syncthreads();
    const int pieces = kc / 16;  // 16-byte pieces per row
    for (int idx = t; idx < kColN * pieces; idx += kColThreads) {
      const int row = idx / pieces, j = idx - row * pieces;
      if (n0 + row < N) {
        const uint32_t* s = tile + row * kColWords + 4 * j;
        *reinterpret_cast<uint4*>(qb + (long long)(n0 + row) * Kp + k0 + 16 * j) = make_uint4(s[0], s[1], s[2], s[3]);
      }
    }
    __syncthreads();  // the tile has been read
  }
  // a column's k groups are spread over 4 lanes of 4 warps
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int sj = sum[j], fj = nan[j] ? 1 : 0;
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      sj += __shfl_xor_sync(0xffffffffu, sj, o);
      fj |= __shfl_xor_sync(0xffffffffu, fj, o);
    }
    if ((lane & 3) == 0) part_sum[warp >> 1][nl + j] = sj, part_nan[warp >> 1][nl + j] = fj;
  }
  __syncthreads();
  if (t < kColN && n0 + t < N) {
    int sj = 0, fj = 0;
    for (int h = 0; h < kColThreads / 64; ++h) sj += part_sum[h][t], fj |= part_nan[h][t];
    col_sum[b * N + n0 + t] = sj;
    nan_flag[b * N + n0 + t] = fj ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------- conv2d lowering
constexpr int kLowPix = 128;              // output pixels (rows of q) per CTA
constexpr int kLowK = 128;                // taps per chunk: one 128-byte line of each row of q
constexpr int kLowWords = kLowK / 4 + 1;  // words per tile row, padded: the column writes are conflict-free
constexpr int kLowThreads = 256;

// One CTA per 128 consecutive output pixels, K in chunks of 128 taps.  Thread t owns pixel t % 128 and every other
// group of 4 taps of the chunk: a warp reads one tap of 32 consecutive pixels (consecutive ow: coalesced along the
// row of x), packs 4 taps per word into a shared tile, and the tile leaves as whole 16-byte pieces of rows of q.
// Row sums and NaN flags stay in registers across the chunks.
// kDoReFa: at least 5 CTAs per SM (48 registers).  Left to its own occupancy target ptxas holds the DoReFa instantiation
// at 40 registers and spills a few loop-invariant words; the plain one (minimum 0: no hint) is unchanged.
template <bool kDoReFa>
__global__ void __launch_bounds__(kLowThreads, kDoReFa ? 5 : 0) int8_im2col_quantize_kernel(const float* __restrict__ x, ConvDims d,
                                                                           const float* __restrict__ scale,
                                                                           const float* __restrict__ zero_point,
                                                                           float qmin, float qmax, int off,
                                                                           int8_t* __restrict__ q,
                                                                           int* __restrict__ row_sum,
                                                                           uint8_t* __restrict__ nan_flag,
                                                                           const float* __restrict__ x_absmax) {
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
  const double xm = kDoReFa ? dorefa_rcp(__ldg(x_absmax)) : 0.0;  // 1 / m of a DoReFa input
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
            e = input_grid<kDoReFa>(__ldg(x + org + tap_off[kl]), xm, p, off, nan);
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

// ---------------------------------------------------------------------------------- conv2d lowering, NHWC
constexpr int kNhPix = 64;        // output pixels (rows of q) per CTA
constexpr int kNhMaxKC = 640;     // K bytes per chunk at most: the tile is kNhPix x kc <= 40 KB of dynamic shared memory
constexpr int kNhThreads = 256;
constexpr int kNhRowsMinK = 256;  // a stride-1 unpadded 1 x 1 conv with c >= this runs the row quantizer

// The same q, row sums and NaN flags as int8_im2col_quantize_kernel, read from the NHWC storage of x.  One CTA per 64
// consecutive output pixels; K in chunks [k0, k0 + kc) of a multiple of 16 bytes, normally whole blocks of channels
// (kc = cb KH KW).  A work item is (tap, pixel, channel quad): it reads the quad's 4 channels of one input pixel
// (vec: one 16-byte load; otherwise 4 guarded scalar loads) -- a warp reads 8 pixels x 4 quads, whole 64-byte runs of
// channels -- and stores each element whose k = c KH KW + tap lies in the chunk into the pixel's row of the shared
// tile, adding it to the pixel's row sum (integer, so the order of the shared-memory adds does not matter).  The tile
// then leaves as 16-byte pieces of rows of q, K padding zeroed.
template <bool kDoReFa>
__global__ void __launch_bounds__(kNhThreads) int8_im2col_quantize_nhwc_kernel(const float* __restrict__ x, ConvDims d,
                                                                                int C, int kcmax,
                                                                                const float* __restrict__ scale,
                                                                                const float* __restrict__ zero_point,
                                                                                float qmin, float qmax, int off,
                                                                                int8_t* __restrict__ q,
                                                                                int* __restrict__ row_sum,
                                                                                uint8_t* __restrict__ nan_flag, int vec,
                                                                                const float* __restrict__ x_absmax) {
  extern __shared__ __align__(16) unsigned char nh_tile[];
  __shared__ long long pix_org[kNhPix], pix_ih[kNhPix], pix_iw[kNhPix];  // x offset of the window's top-left, row, col
  __shared__ int rsum[kNhPix];
  __shared__ int rnan[kNhPix];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const long long m0 = (long long)blockIdx.x * kNhPix;
  const int pix = (int)min((long long)kNhPix, d.M - m0);
  if (t < pix) {
    const long long m = m0 + t, img = m / d.P, pp = m - img * d.P;
    const long long oh = pp / d.OW, ow = pp - oh * d.OW;
    pix_ih[t] = oh * d.sh - d.pt;
    pix_iw[t] = ow * d.sw - d.pl;
    pix_org[t] = ((img * d.H + pix_ih[t]) * d.W + pix_iw[t]) * C;
    rsum[t] = 0;
    rnan[t] = 0;
  }
  QP p;
  p.set(__ldg(scale), __ldg(zero_point));
  p.qmin = qmin;
  p.qmax = qmax;
  const int pad = (int)p.zp - off;  // the grid point v = 0 of the fake-quant input's zero padding
  const double xm = kDoReFa ? dorefa_rcp(__ldg(x_absmax)) : 0.0;  // 1 / m of a DoReFa input
  const int taps = d.KH * d.KW;
  __syncthreads();
  for (int k0 = 0; k0 < d.Kp; k0 += kcmax) {
    const int kc = min(kcmax, d.Kp - k0);
    const int klive = min(kc, d.K - k0);  // bytes of the chunk below K
    if (klive > 0) {
      const int q0 = k0 / taps / 4, nq = (k0 + klive - 1) / taps / 4 - q0 + 1;  // channel quads the chunk touches
      const int items = taps * pix * nq;
      for (int i = t; i < items; i += kNhThreads) {
        const int qi = i % nq, r = i / nq, px = r % pix, tap = r / pix;
        const int c = 4 * (q0 + qi), kh = tap / d.KW, kw = tap - kh * d.KW;
        const long long ih = pix_ih[px] + (long long)kh * d.dh, iw = pix_iw[px] + (long long)kw * d.dw;
        const bool in = (unsigned long long)ih < (unsigned long long)d.H && (unsigned long long)iw < (unsigned long long)d.W;
        const float* xp = x + pix_org[px] + ((long long)kh * d.dh * d.W + (long long)kw * d.dw) * C + c;
        float v[4];
        if (in && vec) {
          const float4 f = __ldg(reinterpret_cast<const float4*>(xp));
          v[0] = f.x, v[1] = f.y, v[2] = f.z, v[3] = f.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) v[j] = in && c + j < C ? __ldg(xp + j) : 0.f;
        }
        int s = 0;
        bool nan = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = (c + j) * taps + tap - k0;
          if (c + j < C && k >= 0 && k < klive) {
            const int e = in ? input_grid<kDoReFa>(v[j], xm, p, off, nan) : pad;
            s += e;
            nh_tile[px * kcmax + k] = (unsigned char)e;
          }
        }
        if (s) atomicAdd(&rsum[px], s);
        if (nan) rnan[px] = 1;
      }
    }
    __syncthreads();
    // warp w stores rows w, w + 8, ...; bytes at or past K are the K padding
    const int pieces = kc / 16;
    for (int r = warp; r < pix; r += kNhThreads / 32) {
      int8_t* qr = q + (m0 + r) * d.Kp + k0;
      for (int j = lane; j < pieces; j += 32) {
        uint4 u = *reinterpret_cast<const uint4*>(nh_tile + r * kcmax + 16 * j);
        uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int b = 0; b < 16; ++b)
          if (16 * j + b >= klive) w[b >> 2] &= ~(0xFFu << (8 * (b & 3)));
        *reinterpret_cast<uint4*>(qr + 16 * j) = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
    __syncthreads();  // the tile has been read
  }
  if (t < pix) {
    row_sum[m0 + t] = rsum[t];
    nan_flag[m0 + t] = rnan[t] ? 1 : 0;
  }
}

// ---------------------------------------------------------------------------------- GEMM
// The atom of every GEMM of this file is wgmma_m64n128k32_s8 of tc_common.cuh, which the fused attention kernel
// (int8_attention.cu) shares: D[64 x 128] (+)= A[64 x 32] * B[32 x 128], s8 x s8 -> s32, both operands K-major
// SWIZZLE_128B in shared memory, issued by one consumer warpgroup.  A k32 step inside the 128-byte swizzle atom
// advances both descriptors by 32 bytes (2 in the start-address field of gmma_desc_sw128).  wgmma_wait_s32<N> waits
// until at most N groups of the warpgroup are outstanding and threads the accumulators through the wait, so that no
// use of them is scheduled above it.
//
// Accumulator layout of a consumer thread (warp w of its warpgroup, lane l, q = l & 3), for j = 0 .. 63:
//   acc[j] = D[16 w + l / 4 + 8 ((j >> 1) & 1)][8 (j >> 2) + 2 q + (j & 1)]
// so each thread holds two rows and, per row, 32 of the 128 columns in pairs; the four lanes with the same l / 4 (a
// quad) hold a whole row between them.  The epilogues below walk this layout pair by pair.
//
// Exactness.  |a|, |b| <= 128 on the stored grid, so every product is at most 2^14 in magnitude and the s32 sum over
// K < 2^17 products cannot overflow; the zero points come out afterwards in int64.

// ---- the mainloop shared by the linear / conv2d kernel and the batched matmul kernel
// Load kb of the stage ring (tc_common.cuh) is k block kb: one 128-row tile of each operand.  The consumers keep one
// wgmma group in flight, so they release the previous k block's stage, not the current one.
// TMA producer (one thread): rows m0.. of map_a and n0.. of map_b, 128 K per stage.  kBatched: the maps are
// (Kp, rows, batch) and `batch` picks the matrix.
template <bool kBatched>
__device__ __forceinline__ void i8_produce(unsigned char* stage_base, StageRing<kI8Stages>& ring,
                                           const CUtensorMap* map_a, const CUtensorMap* map_b, int m0, int n0, int batch,
                                           int num_kb) {
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = ring.acquire(kb, (uint32_t)kI8StageBytes);
    unsigned char* st = stage_base + (size_t)s * kI8StageBytes;
    if constexpr (kBatched) {
      tma_load_3d(st, map_a, kb * kI8BK, m0, batch, &ring.full[s]);
      tma_load_3d(st + kI8TileBytes, map_b, kb * kI8BK, n0, batch, &ring.full[s]);
    } else {
      tma_load_2d(st, map_a, kb * kI8BK, m0, &ring.full[s]);
      tma_load_2d(st + kI8TileBytes, map_b, kb * kI8BK, n0, &ring.full[s]);
    }
  }
}
// Consumer warpgroup wg: acc = rows 64 wg .. 64 wg + 63 of the a tile times the 128 rows of the b tile, over all of K.
__device__ __forceinline__ void i8_consume(int (&acc)[64], uint32_t stage0, StageRing<kI8Stages>& ring, int wg, int lane,
                                           int num_kb) {
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = ring.wait(kb);
    const uint32_t xa = stage0 + (uint32_t)s * kI8StageBytes;
    const uint64_t da = gmma_desc_sw128(xa + (uint32_t)wg * (64 * kI8BK)), db = gmma_desc_sw128(xa + kI8TileBytes);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) wgmma_m64n128k32_s8(acc, da + 2 * j, db + 2 * j, kb > 0 || j > 0);  // +32 B per k32
    wgmma_commit();
    // one group stays in flight: the stage of the previous k block is free once this wait returns
    wgmma_wait_s32<1>(acc);
    if (kb > 0) ring.release(kb - 1, lane);
  }
  wgmma_wait_s32<0>(acc);
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
  unsigned char* stage_base = smem_align1024(smem_raw);
  I8Smem* sm = reinterpret_cast<I8Smem*>(stage_base + (size_t)kI8Stages * kI8StageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + kI8Rows - 1) / kI8Rows;
  const int m0 = (int)(blockIdx.x % (unsigned)tiles_m) * kI8Rows, n0 = (int)(blockIdx.x / (unsigned)tiles_m) * kI8Feat;
  const int num_kb = (K + kI8BK - 1) / kI8BK;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    prefetch_tensormap(&map_w);
    sm->ring.init();
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<40>();
    if (threadIdx.x == 0) i8_produce<false>(stage_base, sm->ring, &map_x, &map_w, m0, n0, 0, num_kb);
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
  i8_consume(acc, stage0, sm->ring, wg, lane, num_kb);
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

// One CTA per 128-row x 128-column tile of one batch entry's out [M, N] (row tile fastest, batch slowest).  The maps are
// (Kp, rows, batch): rows past M / N of the entry are zero-filled, never the next entry's.
__global__ void __launch_bounds__(kI8Threads, 1)
int8_matmul_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                        float* __restrict__ out, const int* __restrict__ a_sum, const uint8_t* __restrict__ a_nan,
                        const int* __restrict__ b_sum, const uint8_t* __restrict__ b_nan, const float* __restrict__ a_scale,
                        const float* __restrict__ a_zero, int a_off, const float* __restrict__ b_scale,
                        const float* __restrict__ b_zero, int b_off, int M, int N, int K, int vec2) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* stage_base = smem_align1024(smem_raw);
  I8MmSmem* sm = reinterpret_cast<I8MmSmem*>(stage_base + (size_t)kI8Stages * kI8StageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned tiles_m = (unsigned)(M + kI8Rows - 1) / kI8Rows, tiles_n = (unsigned)(N + kI8Feat - 1) / kI8Feat;
  const unsigned tile_n = blockIdx.x / tiles_m;
  const int m0 = (int)(blockIdx.x % tiles_m) * kI8Rows, n0 = (int)(tile_n % tiles_n) * kI8Feat;
  const int batch = (int)(tile_n / tiles_n);
  const int num_kb = (K + kI8BK - 1) / kI8BK;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    sm->ring.init();
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<40>();
    if (threadIdx.x == 0) i8_produce<true>(stage_base, sm->ring, &map_a, &map_b, m0, n0, batch, num_kb);
    return;
  }
  reg_inc<232>();
  const int wg = (warp - 4) >> 2;
  // the epilogue's per-column and per-row terms are fetched while the ring fills
  const double sab = (double)__ldg(a_scale) * (double)__ldg(b_scale);
  const long long za = (long long)rintf(__ldg(a_zero)) - a_off, zb = (long long)rintf(__ldg(b_zero)) - b_off;
  const size_t arow = (size_t)batch * M, brow = (size_t)batch * N;
  if (threadIdx.x - 128 < (unsigned)kI8Feat) {
    const int i = threadIdx.x - 128, n = n0 + i;
    I8MmCol c{0, 0};
    if (n < N) {
      c.cn = (long long)K * za * zb - za * (long long)__ldg(b_sum + brow + n);
      c.nan = __ldg(b_nan + brow + n);
    }
    sm->col[i] = c;
  }
  const int q = lane & 3;
  const int r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
  long long sa[2];
  bool rnan[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = r0 + 8 * h;
    sa[h] = m < M ? zb * (long long)__ldg(a_sum + arow + m) : 0;
    rnan[h] = m < M && __ldg(a_nan + arow + m) != 0;
  }
  int acc[64];
  i8_consume(acc, smem_u32(stage_base), sm->ring, wg, lane, num_kb);
  asm volatile("bar.sync 1, 256;" ::: "memory");  // sm->col written by both consumer warpgroups

  // acc[j]: row r0 + 8 ((j >> 1) & 1), column n0 + 8 (j >> 2) + 2 q + (j & 1)
  const float qnan = __int_as_float(0x7fc00000);
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const int i = 8 * c + 2 * q, n = n0 + i;
    if (n >= N) continue;
    const I8MmCol c0 = sm->col[i], c1 = sm->col[i + 1];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = r0 + 8 * h;
      if (m >= M) continue;
      float y0 = __double2float_rn((double)((long long)acc[4 * c + 2 * h] - sa[h] + c0.cn) * sab);
      float y1 = __double2float_rn((double)((long long)acc[4 * c + 2 * h + 1] - sa[h] + c1.cn) * sab);
      if (rnan[h] || c0.nan) y0 = qnan;
      if (rnan[h] || c1.nan) y1 = qnan;
      float* o = out + (arow + m) * N + n;
      if (vec2) {  // N is even: the pair is in range and 8-byte aligned
        *reinterpret_cast<float2*>(o) = make_float2(y0, y1);
      } else {
        o[0] = y0;
        if (n + 1 < N) o[1] = y1;
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

// The lowered activations (q, row sums, NaN flags) in the workspace, written by `lower`, then the GEMM into `out`
// (row-major [M, N], or NCHW with P pixels per image).  Arguments are checked by the caller.
template <bool kNchw, typename Lower>
int run_gemm(const char* fn, long long m, long long k, long long n, long long P, int qmin_x, const float* x_scale,
             const float* x_zero_point, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
             const int32_t* w_zero, const float* bias, float* out, void* workspace, cudaStream_t st, Lower lower) {
  const I8Lowered w = i8_lowered(workspace, m, k);
  const long long kp = padded_k(k);

  CUtensorMap map_x, map_w;
  if (!make_map_2d(&map_x, CU_TENSOR_MAP_DATA_TYPE_UINT8, w.q, (uint64_t)kp, (uint64_t)m, (uint64_t)kp, kI8BK, kI8Rows,
                   CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_map_2d(&map_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, w_q, (uint64_t)kp, (uint64_t)n, (uint64_t)kp, kI8BK, kI8Feat,
                   CU_TENSOR_MAP_SWIZZLE_128B)) {
    set_error("%s: cuTensorMapEncodeTiled failed (M=%lld K=%lld N=%lld)", fn, m, k, n);
    return SB200_E_CUDA;
  }
  if (const int rc = lower(w.q, w.sum, w.nan, st)) return rc;
  const size_t smem = (size_t)kI8Stages * kI8StageBytes + sizeof(I8Smem) + 1024;
  static std::atomic<int> attr_done[64];
  SB_CUDA(ensure_dyn_smem(int8_linear_gemm_kernel<kNchw>, (int)smem, attr_done));
  const long long tiles = ((m + kI8Rows - 1) / kI8Rows) * ((n + kI8Feat - 1) / kI8Feat);
  int8_linear_gemm_kernel<kNchw><<<(unsigned)tiles, kI8Threads, smem, st>>>(
      map_x, map_w, out, w.sum, w.nan, x_scale, x_zero_point, grid_offset(qmin_x), reinterpret_cast<const int*>(w_rowsum),
      w_scale, reinterpret_cast<const int*>(w_zero), bias, (int)m, (int)n, (int)k, (int)P);
  SB_LAUNCHED();
  return SB200_OK;
}

// Workspace of the matmul: the lowered a (batch m rows) and, 1024-aligned behind it, the lowered b (batch n rows)
size_t matmul_b_offset(long long batch, long long m, long long k) { return align_up(i8_layout(batch * m, k).total, 1024); }

int launch_cols(const float* x, const float* scale, const float* zero_point, int qmin, int qmax, int8_t* q, int* col_sum,
                uint8_t* nan_flag, long long batch, long long k, long long n, cudaStream_t st) {
  const int vec = (n % 4 == 0) && aligned16(x);
  const long long tiles_n = (n + kColN - 1) / kColN;
  int8_quantize_cols_kernel<<<(unsigned)(batch * tiles_n), kColThreads, 0, st>>>(
      x, scale, zero_point, (float)qmin, (float)qmax, grid_offset(qmin), q, col_sum, nan_flag, (int)tiles_n, (int)k, (int)n,
      (int)padded_k(k), vec);
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

}  // namespace

// ---------------------------------------------------------------------------------- shared through int8_grid.cuh
I8Lowered i8_lowered(void* workspace, long long m, long long k) {
  const I8Layout w = i8_layout(m, k);
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  return {reinterpret_cast<int8_t*>(ws + w.off_q), reinterpret_cast<int*>(ws + w.off_sum), ws + w.off_nan};
}

int check_k(const char* fn, long long k) {
  if (k < kI8MaxK) return SB200_OK;
  set_error("%s: K >= 2^17, the integer path supports K < 2^17 (|sum| <= K * 2^14 must fit int32)", fn);
  return SB200_E_UNSUPPORTED;
}

int launch_rows(const float* x, const float* scale, const float* zero_point, int per_row, int qmin, int qmax, int8_t* q,
                int* row_sum, uint8_t* nan_flag, long long rows, long long k, cudaStream_t st, const float* x_absmax) {
  const int vec = (k % 4 == 0) && aligned16(x);
  const auto kernel = x_absmax ? int8_quantize_rows_kernel<true> : int8_quantize_rows_kernel<false>;
  kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(x, scale, zero_point, per_row, (float)qmin, (float)qmax,
                                                     grid_offset(qmin), q, row_sum, nan_flag, rows, (int)k,
                                                     (int)padded_k(k), vec, x_absmax);
  SB_LAUNCHED();
  return SB200_OK;
}

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

int launch_im2col(const float* x, const ConvDims& d, const float* scale, const float* zero_point, int qmin, int qmax,
                  int8_t* q, int* row_sum, uint8_t* nan_flag, cudaStream_t st, const float* x_absmax) {
  const auto kernel = x_absmax ? int8_im2col_quantize_kernel<true> : int8_im2col_quantize_kernel<false>;
  kernel<<<(unsigned)((d.M + kLowPix - 1) / kLowPix), kLowThreads, 0, st>>>(
      x, d, scale, zero_point, (float)qmin, (float)qmax, grid_offset(qmin), q, row_sum, nan_flag, x_absmax);
  SB_LAUNCHED();
  return SB200_OK;
}

int nhwc_chunk(const ConvDims& d) {
  const int taps = d.KH * d.KW;
  const long long cb = 16LL * max(1, 8 / taps);  // channels per chunk: a multiple of 16, so that c0 KH KW is too
  return (int)min(min(cb * taps, (long long)kNhMaxKC), (long long)d.Kp);
}

int launch_im2col_nhwc(const float* x, const ConvDims& d, int c, const float* scale, const float* zero_point, int qmin,
                       int qmax, int8_t* q, int* row_sum, uint8_t* nan_flag, cudaStream_t st, const float* x_absmax) {
  // a stride-1, unpadded 1 x 1 conv: x is already the [n h w, c] row matrix of the lowering.  The row quantizer gives
  // each row one warp, 16 elements per lane, so it takes rows of c >= kNhRowsMinK; shorter rows would leave most lanes
  // idle, and the NHWC kernel below (one tap, 64 rows per CTA) quantizes them.
  if (d.KH == 1 && d.KW == 1 && d.sh == 1 && d.sw == 1 && d.pt == 0 && d.pl == 0 && d.P == d.HW && d.K >= kNhRowsMinK)
    return launch_rows(x, scale, zero_point, 0, qmin, qmax, q, row_sum, nan_flag, d.M, d.K, st, x_absmax);
  const int kc = nhwc_chunk(d);
  const int vec = (c % 4 == 0) && aligned16(x);
  const auto kernel = x_absmax ? int8_im2col_quantize_nhwc_kernel<true> : int8_im2col_quantize_nhwc_kernel<false>;
  kernel<<<(unsigned)((d.M + kNhPix - 1) / kNhPix), kNhThreads, (size_t)kNhPix * kc, st>>>(
      x, d, c, kc, scale, zero_point, (float)qmin, (float)qmax, grid_offset(qmin), q, row_sum, nan_flag, vec, x_absmax);
  SB_LAUNCHED();
  return SB200_OK;
}

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
  if (const int rc = check_k("sb200_int8_quantize_rows", k)) return rc;
  return launch_rows(x, scale, zero_point, per_row != 0, qmin, qmax, q, reinterpret_cast<int*>(row_sum), nan_flag, rows, k,
                     (cudaStream_t)stream);
}

// sb200_int8_linear (dorefa = false) and sb200_int8_linear_dorefa
static int int8_linear_entry(const char* fn, bool dorefa, const float* x, const float* x_scale, const float* x_zero_point,
                             const float* x_absmax, int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                             const float* w_scale, const int32_t* w_zero, const float* bias, float* out, int64_t m,
                             int64_t k, int64_t n, void* workspace, size_t workspace_bytes, void* stream) {
  SB_REQUIRE(x && x_scale && x_zero_point && w_q && w_rowsum && w_scale && w_zero && out && workspace,
             "%s: null pointer argument", fn);
  SB_REQUIRE(m > 0 && k > 0 && n > 0, "%s: empty operand (M=%lld K=%lld N=%lld)", fn, (long long)m, (long long)k,
             (long long)n);
  SB_REQUIRE(m < (1LL << 31) && n < (1LL << 31), "%s: dimension too large", fn);
  if (const int rc = check_range(fn, qmin_x, qmax_x)) return rc;
  SB_REQUIRE(aligned16(w_q), "%s: w_q must be 16-byte aligned", fn);
  if (const int rc = check_k(fn, k)) return rc;
  if (const int rc = check_workspace(fn, workspace_bytes, sb200_int8_linear_workspace_bytes(m, k))) return rc;
  if (const int rc = check_absmax(fn, dorefa, x_absmax)) return rc;
  return run_gemm<false>(fn, m, k, n, 1, qmin_x, x_scale, x_zero_point, w_q, w_rowsum, w_scale, w_zero, bias, out,
                         workspace, (cudaStream_t)stream, [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                           return launch_rows(x, x_scale, x_zero_point, 0, qmin_x, qmax_x, xq, xsum, xnan, m, k, st,
                                              x_absmax);
                         });
}

int sb200_int8_linear(const float* x, const float* x_scale, const float* x_zero_point, int qmin_x, int qmax_x,
                      const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero,
                      const float* bias, float* out, int64_t m, int64_t k, int64_t n, void* workspace,
                      size_t workspace_bytes, void* stream) {
  return int8_linear_entry("sb200_int8_linear", false, x, x_scale, x_zero_point, nullptr, qmin_x, qmax_x, w_q, w_rowsum,
                           w_scale, w_zero, bias, out, m, k, n, workspace, workspace_bytes, stream);
}

int sb200_int8_linear_dorefa(const float* x, const float* x_scale, const float* x_zero_point, const float* x_absmax,
                             int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                             const int32_t* w_zero, const float* bias, float* out, int64_t m, int64_t k, int64_t n,
                             void* workspace, size_t workspace_bytes, void* stream) {
  return int8_linear_entry("sb200_int8_linear_dorefa", true, x, x_scale, x_zero_point, x_absmax, qmin_x, qmax_x, w_q,
                           w_rowsum, w_scale, w_zero, bias, out, m, k, n, workspace, workspace_bytes, stream);
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
  if (const int rc = check_k(fn, d.K)) return rc;
  return launch_im2col(x, d, scale, zero_point, qmin, qmax, q, reinterpret_cast<int*>(row_sum), nan_flag,
                       (cudaStream_t)stream);
}

// sb200_int8_conv2d{,_nhwc} (dorefa = false) and their _dorefa entry points
template <bool kNhwc>
static int int8_conv2d_entry(const char* fn, bool dorefa, const float* x, const sb200_conv2d_geom* geom,
                             const float* x_scale, const float* x_zero_point, const float* x_absmax, int qmin_x,
                             int qmax_x, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                             const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* workspace,
                             size_t workspace_bytes, void* stream) {
  SB_REQUIRE(x && geom && x_scale && x_zero_point && w_q && w_rowsum && w_scale && w_zero && out && workspace,
             "%s: null pointer argument", fn);
  SB_REQUIRE(c_out > 0, "%s: empty operand (c_out=%lld)", fn, (long long)c_out);
  SB_REQUIRE(c_out < (1LL << 31), "%s: dimension too large (c_out=%lld)", fn, (long long)c_out);
  ConvDims d;
  if (const int rc = check_conv(fn, geom, &d)) return rc;
  if (const int rc = check_range(fn, qmin_x, qmax_x)) return rc;
  SB_REQUIRE(aligned16(w_q), "%s: w_q must be 16-byte aligned", fn);
  if (const int rc = check_k(fn, d.K)) return rc;
  if (const int rc = check_workspace(fn, workspace_bytes, sb200_int8_conv2d_workspace_bytes(geom))) return rc;
  if (const int rc = check_absmax(fn, dorefa, x_absmax)) return rc;
  if constexpr (kNhwc) {
    // the row-major [n OH OW, c_out] output of the linear is the NHWC storage of [n, c_out, OH, OW]
    return run_gemm<false>(fn, d.M, d.K, c_out, 1, qmin_x, x_scale, x_zero_point, w_q, w_rowsum, w_scale, w_zero, bias,
                           out, workspace, (cudaStream_t)stream,
                           [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                             return launch_im2col_nhwc(x, d, (int)geom->c, x_scale, x_zero_point, qmin_x, qmax_x, xq,
                                                       xsum, xnan, st, x_absmax);
                           });
  } else {
    return run_gemm<true>(fn, d.M, d.K, c_out, d.P, qmin_x, x_scale, x_zero_point, w_q, w_rowsum, w_scale, w_zero, bias,
                          out, workspace, (cudaStream_t)stream,
                          [&](int8_t* xq, int* xsum, uint8_t* xnan, cudaStream_t st) {
                            return launch_im2col(x, d, x_scale, x_zero_point, qmin_x, qmax_x, xq, xsum, xnan, st,
                                                 x_absmax);
                          });
  }
}

int sb200_int8_conv2d(const float* x, const sb200_conv2d_geom* geom, const float* x_scale, const float* x_zero_point,
                      int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                      const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* workspace,
                      size_t workspace_bytes, void* stream) {
  return int8_conv2d_entry<false>("sb200_int8_conv2d", false, x, geom, x_scale, x_zero_point, nullptr, qmin_x, qmax_x,
                                  w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, workspace, workspace_bytes, stream);
}

int sb200_int8_conv2d_dorefa(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                             const float* x_zero_point, const float* x_absmax, int qmin_x, int qmax_x, const int8_t* w_q,
                             const int32_t* w_rowsum, const float* w_scale, const int32_t* w_zero, const float* bias,
                             float* out, int64_t c_out, void* workspace, size_t workspace_bytes, void* stream) {
  return int8_conv2d_entry<false>("sb200_int8_conv2d_dorefa", true, x, geom, x_scale, x_zero_point, x_absmax, qmin_x,
                                  qmax_x, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, workspace, workspace_bytes,
                                  stream);
}

int sb200_int8_im2col_quantize_nhwc(const float* x, const sb200_conv2d_geom* geom, const float* scale,
                                    const float* zero_point, int qmin, int qmax, int8_t* q, int32_t* row_sum,
                                    uint8_t* nan_flag, void* stream) {
  const char* fn = "sb200_int8_im2col_quantize_nhwc";
  SB_REQUIRE(x && geom && scale && zero_point && q && row_sum && nan_flag, "%s: null pointer argument", fn);
  ConvDims d;
  if (const int rc = check_conv(fn, geom, &d)) return rc;
  if (const int rc = check_range(fn, qmin, qmax)) return rc;
  SB_REQUIRE(aligned16(q), "%s: q must be 16-byte aligned", fn);
  if (const int rc = check_k(fn, d.K)) return rc;
  return launch_im2col_nhwc(x, d, (int)geom->c, scale, zero_point, qmin, qmax, q, reinterpret_cast<int*>(row_sum),
                            nan_flag, (cudaStream_t)stream);
}

int sb200_int8_conv2d_nhwc(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                           const float* x_zero_point, int qmin_x, int qmax_x, const int8_t* w_q, const int32_t* w_rowsum,
                           const float* w_scale, const int32_t* w_zero, const float* bias, float* out, int64_t c_out,
                           void* workspace, size_t workspace_bytes, void* stream) {
  return int8_conv2d_entry<true>("sb200_int8_conv2d_nhwc", false, x, geom, x_scale, x_zero_point, nullptr, qmin_x,
                                 qmax_x, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, workspace, workspace_bytes,
                                 stream);
}

int sb200_int8_conv2d_nhwc_dorefa(const float* x, const sb200_conv2d_geom* geom, const float* x_scale,
                                  const float* x_zero_point, const float* x_absmax, int qmin_x, int qmax_x,
                                  const int8_t* w_q, const int32_t* w_rowsum, const float* w_scale,
                                  const int32_t* w_zero, const float* bias, float* out, int64_t c_out, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  return int8_conv2d_entry<true>("sb200_int8_conv2d_nhwc_dorefa", true, x, geom, x_scale, x_zero_point, x_absmax,
                                 qmin_x, qmax_x, w_q, w_rowsum, w_scale, w_zero, bias, out, c_out, workspace,
                                 workspace_bytes, stream);
}

size_t sb200_int8_matmul_workspace_bytes(int64_t batch, int64_t m, int64_t k, int64_t n) {
  if (batch <= 0 || m <= 0 || k <= 0 || n <= 0) return 0;
  if ((__int128)batch * m >= (1LL << 31) || (__int128)batch * n >= (1LL << 31) || k >= kI8MaxK) return 0;
  return matmul_b_offset(batch, m, k) + i8_layout(batch * n, k).total + 1024;  // + the alignment of the base
}

int sb200_int8_quantize_cols(const float* x, const float* scale, const float* zero_point, int qmin, int qmax, int8_t* q,
                             int32_t* col_sum, uint8_t* nan_flag, int64_t batch, int64_t k, int64_t n, void* stream) {
  const char* fn = "sb200_int8_quantize_cols";
  SB_REQUIRE(x && scale && zero_point && q && col_sum && nan_flag, "%s: null pointer argument", fn);
  SB_REQUIRE(batch > 0 && k > 0 && n > 0, "%s: empty operand (batch=%lld K=%lld N=%lld)", fn, (long long)batch, (long long)k,
             (long long)n);
  SB_REQUIRE((__int128)batch * n < (1LL << 31), "%s: too many columns (batch N = %lld x %lld must be < 2^31)", fn,
             (long long)batch, (long long)n);
  if (const int rc = check_range(fn, qmin, qmax)) return rc;
  SB_REQUIRE(aligned16(q), "%s: q must be 16-byte aligned", fn);
  if (const int rc = check_k(fn, k)) return rc;
  return launch_cols(x, scale, zero_point, qmin, qmax, q, reinterpret_cast<int*>(col_sum), nan_flag, batch, k, n,
                     (cudaStream_t)stream);
}

int sb200_int8_matmul(const float* a, const float* b, int b_k_major, const float* a_scale, const float* a_zero_point,
                      int qmin_a, int qmax_a, const float* b_scale, const float* b_zero_point, int qmin_b, int qmax_b,
                      float* out, int64_t batch, int64_t m, int64_t k, int64_t n, void* workspace, size_t workspace_bytes,
                      void* stream) {
  const char* fn = "sb200_int8_matmul";
  SB_REQUIRE(a && b && a_scale && a_zero_point && b_scale && b_zero_point && out && workspace, "%s: null pointer argument",
             fn);
  SB_REQUIRE(batch > 0 && m > 0 && k > 0 && n > 0, "%s: empty operand (batch=%lld M=%lld K=%lld N=%lld)", fn,
             (long long)batch, (long long)m, (long long)k, (long long)n);
  SB_REQUIRE((__int128)batch * m < (1LL << 31) && (__int128)batch * n < (1LL << 31),
             "%s: dimension too large (batch M and batch N must be < 2^31)", fn);
  const __int128 tiles = (__int128)batch * ((m + kI8Rows - 1) / kI8Rows) * ((n + kI8Feat - 1) / kI8Feat);
  SB_REQUIRE(tiles < (1LL << 31), "%s: dimension too large (%lld x %lld x %lld output tiles)", fn, (long long)batch,
             (long long)((m + kI8Rows - 1) / kI8Rows), (long long)((n + kI8Feat - 1) / kI8Feat));
  if (const int rc = check_range(fn, qmin_a, qmax_a)) return rc;
  if (const int rc = check_range(fn, qmin_b, qmax_b)) return rc;
  if (const int rc = check_k(fn, k)) return rc;
  if (const int rc = check_workspace(fn, workspace_bytes, sb200_int8_matmul_workspace_bytes(batch, m, k, n))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const I8Lowered la = i8_lowered(workspace, batch * m, k);
  const I8Lowered lb = i8_lowered(la.q + matmul_b_offset(batch, m, k), batch * n, k);
  const long long kp = padded_k(k);
  CUtensorMap map_a, map_b;
  if (!make_map_3d(&map_a, CU_TENSOR_MAP_DATA_TYPE_UINT8, la.q, (uint64_t)kp, (uint64_t)m, (uint64_t)batch, (uint64_t)kp,
                   kI8BK, kI8Rows, CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_map_3d(&map_b, CU_TENSOR_MAP_DATA_TYPE_UINT8, lb.q, (uint64_t)kp, (uint64_t)n, (uint64_t)batch, (uint64_t)kp, kI8BK,
                   kI8Feat, CU_TENSOR_MAP_SWIZZLE_128B)) {
    set_error("%s: cuTensorMapEncodeTiled failed (batch=%lld M=%lld K=%lld N=%lld)", fn, (long long)batch, (long long)m,
              (long long)k, (long long)n);
    return SB200_E_CUDA;
  }
  if (const int rc = launch_rows(a, a_scale, a_zero_point, 0, qmin_a, qmax_a, la.q, la.sum, la.nan, batch * m, k, st))
    return rc;
  if (const int rc = b_k_major ? launch_rows(b, b_scale, b_zero_point, 0, qmin_b, qmax_b, lb.q, lb.sum, lb.nan, batch * n, k,
                                             st)
                               : launch_cols(b, b_scale, b_zero_point, qmin_b, qmax_b, lb.q, lb.sum, lb.nan, batch, k, n, st))
    return rc;
  const size_t smem = (size_t)kI8Stages * kI8StageBytes + sizeof(I8MmSmem) + 1024;
  static std::atomic<int> attr_done[64];
  SB_CUDA(ensure_dyn_smem(int8_matmul_gemm_kernel, (int)smem, attr_done));
  const int vec2 = (n % 2 == 0) && (reinterpret_cast<uintptr_t>(out) & 7u) == 0;
  int8_matmul_gemm_kernel<<<(unsigned)tiles, kI8Threads, smem, st>>>(
      map_a, map_b, out, la.sum, la.nan, lb.sum, lb.nan, a_scale, a_zero_point, grid_offset(qmin_a), b_scale,
      b_zero_point, grid_offset(qmin_b), (int)m, (int)n, (int)k, vec2);
  SB_LAUNCHED();
  return SB200_OK;
}
