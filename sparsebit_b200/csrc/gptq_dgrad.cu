// gptq_dgrad.cu -- input gradient of the GPTQ dequant-matmul (2 / 3 / 4-bit), the backward of QuantLinear:
//   grad_in[m, k] += sum_n grad_out[m, n] * (scales[n, k/gs] * q(k, n) - zeros[n, k/gs])
// grad_out [M, N] fp32, grad_in [M, K] fp32 (accumulated in place), qweight / scales / zeros exactly the tensors the
// forward reads (gptq.cu, gptq_simt.cu).  Both kernels are deterministic: no float atomics, fixed reduction orders.
//
// SIMT kernel (any bit width, any shape).  A CTA owns one 32-k unit of packed rows, MT rows of grad_out and one slice
// of N.  Each thread walks the columns n = tid, tid + 128, ... of the slice (a warp reads 128 contiguous bytes of every
// packed row), decodes the unit and applies the per-group affine the way the forward SIMT kernel does, here with the
// scale folded into the gradient:  sum_n g (s q - z) = sum_n (g s) q - sum_n g z.  The 128 per-thread partials are
// summed through shared memory in a fixed order; with more than one N slice every slice writes its own partial and a
// finish kernel adds them in slice order.
//
// Tensor-core kernel (4-bit, wgmma, sm_90a).  The transposed problem  D[k, m] = sum_n W[k, n] * g'[m, n]  has the
// forward's structure with K and N swapped (tc_common.cuh):
//   * the packed weights are repacked per call into qT[N/8, K] (8 nibbles along n) in the workspace;
//   * g' = grad_out * 2^-e[m] = g_hi + g_lo (fp16 planes, every 8 n permuted 0,4,1,5,2,6,3,7) comes from the
//     unchanged gptq_split_kernel, the TMA ring and NibblePair are the forward's;
//   * the scale varies along the reduction index n, so it cannot be folded into the accumulator once per group.  It goes
//     into the operand instead: every consumer thread builds w' = 2^c[g] * (s q - z) = fmaf(s', q, -z') in fp32 for its
//     fragment pair (n, n + 4) and splits it into fp16 planes w_hi + w_lo (22 significant bits).  Fractional zero points
//     therefore need no correction term.  The CTA's 128-k tile lies in one group (group_size % 128 == 0), so it reads one
//     [N] slice of a per-call table { s'[n], s'[n+4], z'[n], z'[n+4] } per fragment pair;
//   * the power-of-two c[g] must be uniform along the reduction, so it is per group: 2^c max_n |s q - z| lies in
//     [2^14, 2^15).  An element w of the group keeps its 22 bits while |w| >= 2^-17 max_group |w|; below that its w_lo
//     is an fp16 subnormal and its absolute error stays under 2^-40 max_group |w|;
//   * three m64n128k16 passes per 16 n (w_hi g_hi, w_lo g_hi, w_hi g_lo -- the last only when some g_lo != 0), into a
//     register accumulator restarted every 512 n and added into a second one with round-to-nearest: the tensor core
//     truncates instead of rounding to nearest when it accumulates, so one chain over all of N could lose ~1e-5;
//   * epilogue grad_in[m, k] = fmaf(2^e[m], 2^-c[g] * acc, grad_in[m, k]).
// Limits: N % 8 == 0 (16-byte rows of g' and the 8-wide permutation), K % 4 == 0 (16-byte rows of qT), grad_out 16-byte
// aligned, group_size a multiple of 128 or one group.  Everything else runs the SIMT kernel.
#include "gptq_launch.cuh"
#include "gptq_unpack.cuh"
#include "tc_common.cuh"

namespace sb200 {
namespace {

// ---------------------------------------------------------------------------------- SIMT kernel
constexpr int kDgCols = 128;        // threads per CTA; the columns n one pass of the CTA reads
constexpr int kDgUnitK = 32;        // k per CTA (one unit)
constexpr long long kDgTargetCtas = 1024;  // N is split until the grid has about this many CTAs (~8 per SM)
constexpr long long kDgMaxGridY = 65535;   // CUDA's limit on gridDim.y

// scales / zeros [N, G] -> sz[g, n] = (s, z): the SIMT kernel reads them along n, coalesced
__global__ void __launch_bounds__(256) dgrad_sz_kernel(const float* __restrict__ scales, const float* __restrict__ zeros,
                                                        float2* __restrict__ sz, int N, int G) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * G) return;
  const int g = (int)(i / N), n = (int)(i % N);
  sz[i] = make_float2(scales[(size_t)n * G + g], zeros[(size_t)n * G + g]);
}

// grid (units, M tiles, N slices); partial == nullptr: one slice, the CTA adds into grad_in itself.  gridDim.y is capped
// at 65535 (kDgMaxGridY), so a CTA walks the M tiles blockIdx.y, blockIdx.y + gridDim.y, ...; each tile is reduced as if
// it had a CTA of its own.  Only LOOP kernels (M > 262,140, so MT = 4) walk; the others run their one tile with the code
// and registers they had before the cap (the loop in every kernel cost ~3% at M = 65536, K = 4096, N = 128 on an H100).
// The loop's bound of three CTAs per SM keeps it at 168 registers without spills; ptxas gives it ~200 without the bound,
// room for two CTAs of 128 threads per SM.
template <int BITS, int MT, bool LOOP>
__global__ void __launch_bounds__(kDgCols, LOOP ? 3 : 0) gptq_dgrad_simt_kernel(const float* __restrict__ go, const uint32_t* __restrict__ qw,
                                                                   float* __restrict__ grad_in, const float2* __restrict__ sz,
                                                                   float* __restrict__ partial, int M, int K, int N, int KW,
                                                                   int group_size, int slice_n) {
  constexpr int kWords = GptqFmt<BITS>::kUnitWords;
  __shared__ float red[kDgUnitK][kDgCols + 1];
  const int tid = threadIdx.x;
  const int u = blockIdx.x;
  const int n_begin = blockIdx.z * slice_n, n_end = min(N, n_begin + slice_n);
  const int g = (u * kDgUnitK) / group_size;
  const float2* szg = sz + (size_t)g * N;
  const int m_tiles = LOOP ? (int)(((long long)M + MT - 1) / MT) : 0;  // M + MT - 1 passes INT_MAX for M near 2^31
  for (int tile = blockIdx.y; !LOOP || tile < m_tiles; tile += gridDim.y) {  // uniform across the CTA
    const int m0 = tile * MT;
    float acc[MT][kDgUnitK], zacc[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      zacc[m] = 0.f;
#pragma unroll
      for (int j = 0; j < kDgUnitK; ++j) acc[m][j] = 0.f;
    }
    for (int n = n_begin + tid; n < n_end; n += kDgCols) {
      uint32_t w[kWords];
#pragma unroll
      for (int r = 0; r < kWords; ++r) {
        const int row = u * kWords + r;
        w[r] = row < KW ? __ldg(qw + (size_t)row * N + n) : 0u;
      }
      const float2 p = __ldg(szg + n);
      float gs[MT];
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const float gv = (m0 + m < M) ? __ldg(go + (size_t)(m0 + m) * N + n) : 0.f;
        gs[m] = gv * p.x;
        zacc[m] = fmaf(gv, p.y, zacc[m]);
      }
      float q[32];
      decode_unit<BITS>(w, q);
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int j = 0; j < kDgUnitK; ++j) acc[m][j] = fmaf(gs[m], q[j], acc[m][j]);
    }
    // fixed-order sum over the 128 threads: thread t adds red[t / 4][32 (t % 4) ...] and the 4 quarters meet in shuffles
    const int jr = tid >> 2, part = tid & 3;
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      __syncthreads();
#pragma unroll
      for (int j = 0; j < kDgUnitK; ++j) red[j][tid] = acc[m][j] - zacc[m];
      __syncthreads();
      float v = 0.f;
#pragma unroll 8
      for (int i = 0; i < kDgCols / 4; ++i) v += red[jr][part * (kDgCols / 4) + i];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      const int k = u * kDgUnitK + jr;
      if (part == 0 && m0 + m < M && k < K) {
        if (partial) {
          partial[((size_t)blockIdx.z * M + m0 + m) * K + k] = v;
        } else {
          float* o = grad_in + (size_t)(m0 + m) * K + k;
          *o += v;
        }
      }
    }
    if (!LOOP) break;
  }
}

// grad_in += sum over the N slices in slice order
__global__ void __launch_bounds__(256) dgrad_finish_kernel(const float* __restrict__ partial, float* __restrict__ grad_in,
                                                           long long mk, int slices) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < mk; i += (long long)gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int s = 0; s < slices; ++s) v += partial[(size_t)s * mk + i];
    grad_in[i] += v;
  }
}

struct SimtPlan {
  int mt, slices, slice_n;
  size_t sz_bytes, partial_bytes;
};
// a pure function of the shape (the workspace query must not touch the device)
SimtPlan simt_plan(long long M, long long K, long long N, int group_size) {
  SimtPlan p;
  p.mt = M == 1 ? 1 : (M == 2 ? 2 : 4);
  const long long base = ((K + kDgUnitK - 1) / kDgUnitK) * ((M + p.mt - 1) / p.mt);
  long long s = (kDgTargetCtas + base - 1) / base;
  const long long s_max = (N + 4 * kDgCols - 1) / (4 * kDgCols);  // at least 4 columns per thread and slice
  s = s < 1 ? 1 : (s > s_max ? s_max : s);
  p.slice_n = (int)(((N + s - 1) / s + kDgCols - 1) / kDgCols * kDgCols);
  p.slices = (int)((N + p.slice_n - 1) / p.slice_n);
  const long long G = (K + group_size - 1) / group_size;
  p.sz_bytes = align_up((size_t)N * G * sizeof(float2), 1024);
  p.partial_bytes = p.slices > 1 ? (size_t)p.slices * M * K * sizeof(float) : 0;
  return p;
}

template <int BITS>
int launch_simt(const float* go, const int32_t* qweight, float* grad_in, const float* scales, const float* zeros, long long M,
                long long K, long long N, long long KW, int group_size, unsigned char* ws, cudaStream_t st) {
  const SimtPlan p = simt_plan(M, K, N, group_size);
  const int G = (int)((K + group_size - 1) / group_size);
  float2* sz = reinterpret_cast<float2*>(ws);
  float* partial = p.slices > 1 ? reinterpret_cast<float*>(ws + p.sz_bytes) : nullptr;
  dgrad_sz_kernel<<<(unsigned)(((long long)N * G + 255) / 256), 256, 0, st>>>(scales, zeros, sz, (int)N, G);
  SB_LAUNCHED();
  const long long m_tiles = (M + p.mt - 1) / p.mt;
  const dim3 grid((unsigned)((K + kDgUnitK - 1) / kDgUnitK), (unsigned)(m_tiles < kDgMaxGridY ? m_tiles : kDgMaxGridY),
                  (unsigned)p.slices);
  const uint32_t* qw = reinterpret_cast<const uint32_t*>(qweight);
#define SB_GO(MT_, LOOP_)                                                                                         \
  gptq_dgrad_simt_kernel<BITS, MT_, LOOP_><<<grid, kDgCols, 0, st>>>(go, qw, grad_in, sz, partial, (int)M, (int)K,  \
                                                                     (int)N, (int)KW, group_size, p.slice_n)
  if (m_tiles > kDgMaxGridY) SB_GO(4, true);  // M > 4 * 65535: mt = 4
  else if (p.mt == 1) SB_GO(1, false);
  else if (p.mt == 2) SB_GO(2, false);
  else SB_GO(4, false);
#undef SB_GO
  SB_LAUNCHED();
  if (partial) {
    const long long mk = M * K;
    long long b = (mk + 255) / 256, cap = (long long)sm_count() * 16;
    dgrad_finish_kernel<<<(unsigned)(b < cap ? b : cap), 256, 0, st>>>(partial, grad_in, mk, p.slices);
    SB_LAUNCHED();
  }
  return SB200_OK;
}

// ---------------------------------------------------------------------------------- tensor-core kernel
constexpr int kDgStages = 5;
constexpr int kDgChunk = 8;  // 64-n stages per restart of the MMA accumulator (512 n)

// qweight[KW, N] (8 nibbles along k) -> qT[N/8, K] (8 nibbles along n).  CTA = 64 k x 64 n.
__global__ void __launch_bounds__(256) dgrad_repack_kernel(const uint32_t* __restrict__ qw, uint32_t* __restrict__ qT, int K,
                                                           int N, int KW) {
  __shared__ uint32_t w[8][65];
  const int tid = threadIdx.x;
  const int kw0 = blockIdx.x * 8, n0 = blockIdx.y * 64;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = tid + 256 * i, row = idx >> 6, col = idx & 63;
    w[row][col] = (kw0 + row < KW && n0 + col < N) ? __ldg(qw + (size_t)(kw0 + row) * N + n0 + col) : 0u;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = tid + 256 * i, r = idx >> 6, kk = idx & 63;
    const int k = kw0 * 8 + kk, rr = n0 / 8 + r;
    const uint32_t sh = 4u * (uint32_t)(kk & 7);
    uint32_t v = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) v |= ((w[kk >> 3][8 * r + j] >> sh) & 15u) << (4 * j);
    if (k < K && rr < N / 8) qT[(size_t)rr * K + k] = v;
  }
}

// One CTA per group g: c[g] from max_n |s q - z| over q in [0, 15], then the table of fragment pairs
//   tab[g, n8, q] = { s'[8 n8 + q], s'[8 n8 + q + 4], z'[8 n8 + q], z'[8 n8 + q + 4] },  s' = 2^c s, z' = 2^c z,
// zero for n >= N (the padding of the last 64-n stage), and gscale[g] = 2^-c.
__global__ void __launch_bounds__(256) dgrad_table_kernel(const float* __restrict__ scales, const float* __restrict__ zeros,
                                                          float4* __restrict__ tab, float* __restrict__ gscale, int N, int G,
                                                          int N8p) {
  __shared__ float red[8];
  const int g = blockIdx.x, tid = threadIdx.x;
  float wmax = 0.f;
  for (int n = tid; n < N; n += 256) {
    const float s = scales[(size_t)n * G + g], z = zeros[(size_t)n * G + g];
    const float b = fmaxf(fabsf(z), fabsf(fmaf(15.f, s, -z)));
    if (b < __int_as_float(0x7f800000)) wmax = fmaxf(wmax, b);
  }
  wmax = warp_max(wmax);
  if ((tid & 31) == 0) red[tid >> 5] = wmax;
  __syncthreads();
  wmax = red[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) wmax = fmaxf(wmax, red[i]);
  int c = 0;
  if (wmax > 0.f) c = 14 - ilogbf(wmax);
  c = max(-100, min(100, c));
  if (tid == 0) gscale[g] = ldexpf(1.f, -c);
  for (int i = tid; i < N8p * 4; i += 256) {
    const int n = 8 * (i >> 2) + (i & 3);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < N) {
      v.x = ldexpf(scales[(size_t)n * G + g], c);
      v.z = ldexpf(zeros[(size_t)n * G + g], c);
    }
    if (n + 4 < N) {
      v.y = ldexpf(scales[(size_t)(n + 4) * G + g], c);
      v.w = ldexpf(zeros[(size_t)(n + 4) * G + g], c);
    }
    tab[(size_t)g * N8p * 4 + i] = v;
  }
}

// One CTA per 128-k x 128-m tile of grad_in (m tile fastest: CTAs side by side share the repacked weight tile in L2).
// Roles as in tc_common.cuh with K (features) and N (reduction) swapped.
__global__ void __launch_bounds__(kWgThreads, 1)
gptq4_dgrad_tc_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                      const __grid_constant__ CUtensorMap map_q, float* __restrict__ grad_in, const float* __restrict__ rowscale,
                      const float4* __restrict__ tab, const float* __restrict__ gscale, const int* __restrict__ need_lo_flag,
                      int M, int K, int N, int group_size, int N8p, int backoff_ns) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* stage_base = smem_align1024(smem_raw);
  auto& ring = *reinterpret_cast<StageRing<kDgStages>*>(stage_base + (size_t)kDgStages * kWgStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + kWgTok - 1) / kWgTok;
  const int m0 = (int)(blockIdx.x % (unsigned)tiles_m) * kWgTok, k0 = (int)(blockIdx.x / (unsigned)tiles_m) * kWgFeat;
  const int num_nb = (N + kWgBK - 1) / kWgBK;
  const bool need_lo = need_lo_flag[0] != 0;  // uniform: some gradient has a non-zero fp16 low part

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_hi);
    prefetch_tensormap(&map_lo);
    prefetch_tensormap(&map_q);
    ring.init();
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<40>();
    if (threadIdx.x == 0)
      wg_produce(stage_base, ring, &map_hi, &map_lo, &map_q, m0, k0, num_nb, need_lo, backoff_ns);
    return;
  }
  reg_inc<232>();
  const int q = lane & 3;
  const int f0 = ((warp - 4) >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);  // k rows f0, f0 + 8 of the tile
  const int g = k0 / group_size;                                         // the whole 128-k tile lies in group g
  const float4* tg = tab + (size_t)g * N8p * 4 + q;
  const NibblePair unpack(q);
  const __half2 off = unpack.offset(0.f);
  const uint32_t stage0 = smem_u32(stage_base);
  float acc[64], c[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0.f;
  for (int nb = 0; nb < num_nb;) {
    const int nb_end = min(num_nb, nb + kDgChunk);
    for (bool first = true; nb < nb_end; ++nb, first = false) {
      // the stage's 8 packed rows p -> fragment pairs (n, n + 4) = 64 nb + 8 p + (q, q + 4)
      float4 t[8];
#pragma unroll
      for (int p = 0; p < 8; ++p) t[p] = __ldg(tg + (size_t)(nb * 8 + p) * 4);
      const int s = ring.wait(nb);
      const uint32_t* bq = reinterpret_cast<const uint32_t*>(stage_base + (size_t)s * kWgStageBytes + 2 * kWgXBytes);
      uint32_t H[4][4], L[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // 16 n = packed rows 2j (n 0..7) and 2j + 1 (n 8..15)
#pragma unroll
        for (int r = 0; r < 4; ++r) {  // fragment register r: k row f0 / f0 + 8 (r & 1), n half (r >> 1)
          const int p = 2 * j + (r >> 1);
          const float2 d = __half22float2(unpack(bq[p * kWgFeat + f0 + ((r & 1) ? 8 : 0)], off));  // q, exact
          const float2 wv = make_float2(fmaf(t[p].x, d.x, -t[p].z), fmaf(t[p].y, d.y, -t[p].w));
          const __half2 hi = __float22half2_rn(wv);
          const float2 hf = __half22float2(hi);
          H[j][r] = h2u(hi);
          L[j][r] = h2u(__float22half2_rn(make_float2(wv.x - hf.x, wv.y - hf.y)));
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
      ring.release(nb, lane);
    }
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] += c[j];
  }
  // d[j]: k row f0 + 8 * ((j >> 1) & 1), m = m0 + 8 (j >> 2) + 2q + (j & 1)
  const float cs = __ldg(gscale + g);
  const int ka = k0 + f0, kb = ka + 8;
#pragma unroll
  for (int j = 0; j < 64; ++j) {
    const int m = m0 + 8 * (j >> 2) + 2 * q + (j & 1);
    const int k = (j & 2) ? kb : ka;
    if (m < M && k < K) {
      float* o = grad_in + (size_t)m * K + k;
      *o = fmaf(__ldg(rowscale + m), acc[j] * cs, *o);
    }
  }
}

struct TcLayout {
  size_t off_qt, off_hi, off_lo, off_xsum, off_rs, off_tab, off_gs, off_flag, total;
};
TcLayout tc_layout(long long M, long long K, long long N, long long G) {
  TcLayout w;
  const long long N8p = (N + kWgBK - 1) / kWgBK * 8;
  w.off_qt = 0;
  w.off_hi = align_up((size_t)(N / 8) * K * 4, 1024);
  w.off_lo = w.off_hi + align_up((size_t)M * N * 2, 1024);
  w.off_xsum = w.off_lo + align_up((size_t)M * N * 2, 1024);
  w.off_rs = w.off_xsum + align_up((size_t)M * ((N + 127) / 128) * 4, 1024);
  w.off_tab = w.off_rs + align_up((size_t)M * 4, 1024);
  w.off_gs = w.off_tab + align_up((size_t)G * N8p * 4 * sizeof(float4), 1024);  // 4 fragment pairs per 8 n
  w.off_flag = w.off_gs + align_up((size_t)G * 4, 1024);
  w.total = w.off_flag + 1024;
  return w;
}

bool tc_shape_ok(long long K, long long N, int group_size) {
  return N % 8 == 0 && K % 4 == 0 && (group_size % 128 == 0 || group_size == K);
}

}  // namespace

size_t gptq_dgrad_simt_workspace(long long M, long long K, long long N, int group_size) {
  const SimtPlan p = simt_plan(M, K, N, group_size);
  return p.sz_bytes + p.partial_bytes + 256;
}

size_t gptq_dgrad_tc_workspace(long long M, long long K, long long N, int group_size) {
  if (!tc_shape_ok(K, N, group_size)) return 0;
  return tc_layout(M, K, N, (K + group_size - 1) / group_size).total + 1024;
}

bool gptq_dgrad_tc_supported(const float* grad_out, long long K, long long N, int group_size) {
  return get_encode() && tc_shape_ok(K, N, group_size) && aligned16(grad_out);
}

int gptq_dgrad_simt(int bits, const float* go, const int32_t* qweight, float* grad_in, const float* scales, const float* zeros,
                    long long M, long long K, long long N, long long KW, int group_size, void* workspace,
                    size_t workspace_bytes, cudaStream_t st) {
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 256));
  if (!workspace || workspace_bytes < gptq_dgrad_simt_workspace(M, K, N, group_size)) {
    set_error("sb200_gptq_matmul_dgrad: workspace too small (%zu bytes, need %zu)", workspace_bytes,
              gptq_dgrad_simt_workspace(M, K, N, group_size));
    return SB200_E_WORKSPACE;
  }
  if (bits == 2) return launch_simt<2>(go, qweight, grad_in, scales, zeros, M, K, N, KW, group_size, ws, st);
  if (bits == 3) return launch_simt<3>(go, qweight, grad_in, scales, zeros, M, K, N, KW, group_size, ws, st);
  return launch_simt<4>(go, qweight, grad_in, scales, zeros, M, K, N, KW, group_size, ws, st);
}

int gptq4_dgrad_tc(const float* go, const int32_t* qweight, float* grad_in, const float* scales, const float* zeros,
                   long long M, long long K, long long N, long long KW, int group_size, void* workspace, size_t workspace_bytes,
                   cudaStream_t st) {
  const int G = (int)((K + group_size - 1) / group_size);
  const TcLayout w = tc_layout(M, K, N, G);
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  if (!workspace || (size_t)(ws - reinterpret_cast<unsigned char*>(workspace)) + w.total > workspace_bytes) {
    set_error("sb200_gptq_matmul_dgrad: workspace too small (%zu bytes)", workspace_bytes);
    return SB200_E_WORKSPACE;
  }
  uint32_t* qT = reinterpret_cast<uint32_t*>(ws + w.off_qt);
  __half* g_hi = reinterpret_cast<__half*>(ws + w.off_hi);
  __half* g_lo = reinterpret_cast<__half*>(ws + w.off_lo);
  float* xsum = reinterpret_cast<float*>(ws + w.off_xsum);
  float* rowscale = reinterpret_cast<float*>(ws + w.off_rs);
  float4* tab = reinterpret_cast<float4*>(ws + w.off_tab);
  float* gscale = reinterpret_cast<float*>(ws + w.off_gs);
  int* flag = reinterpret_cast<int*>(ws + w.off_flag);
  const int N8p = (int)((N + kWgBK - 1) / kWgBK * 8);

  SB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));  // need_lo, set by the split kernel
  dgrad_repack_kernel<<<dim3((unsigned)((KW + 7) / 8), (unsigned)((N + 63) / 64)), 256, 0, st>>>(
      reinterpret_cast<const uint32_t*>(qweight), qT, (int)K, (int)N, (int)KW);
  SB_LAUNCHED();
  dgrad_table_kernel<<<(unsigned)G, 256, 0, st>>>(scales, zeros, tab, gscale, (int)N, G, N8p);
  SB_LAUNCHED();
  if (const int rc = gptq_launch_split(go, g_hi, g_lo, xsum, rowscale, flag, M, (int)N, (int)((N + 127) / 128), st)) return rc;

  // the forward's maps with (features, reduction) = (K, N): g' planes [M, N], repacked words [N/8, K]
  CUtensorMap map_hi, map_lo, map_q;
  if (!make_wg_maps(&map_hi, &map_lo, &map_q, g_hi, g_lo, reinterpret_cast<const int32_t*>(qT), M, N, K, N / 8)) {
    set_error("sb200_gptq_matmul_dgrad: cuTensorMapEncodeTiled failed (M=%lld K=%lld N=%lld)", M, K, N);
    return SB200_E_CUDA;
  }
  const size_t smem = (size_t)kDgStages * kWgStageBytes + sizeof(StageRing<kDgStages>) + 1024;
  static std::atomic<int> attr_done[64];
  SB_CUDA(ensure_dyn_smem(gptq4_dgrad_tc_kernel, (int)smem, attr_done));
  const long long tiles = ((M + kWgTok - 1) / kWgTok) * ((K + kWgFeat - 1) / kWgFeat);
  gptq4_dgrad_tc_kernel<<<(unsigned)tiles, kWgThreads, smem, st>>>(map_hi, map_lo, map_q, grad_in, rowscale, tab, gscale, flag,
                                                                  (int)M, (int)K, (int)N, group_size, N8p, gptq4_tc_backoff());
  SB_LAUNCHED();
  return SB200_OK;
}

}  // namespace sb200
