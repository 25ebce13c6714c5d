// int8_attention_cache.cu -- the fused integer-grid attention (int8_attention.cu) over an int8 key/value cache, for
// generation: each key and value is quantized once, when it is appended, and every later step reads 1 byte per cached
// element instead of re-quantizing the whole fp32 past.
//
// Cache.  Per entry e (one element of the flattened leading dimensions, e.g. one (batch, head)), capacity C:
//   k_q [E, C, dp]  row j = the grid of key j as int8_quantize_rows_kernel stores it (dp = round_up(d, 16), pad 0)
//   k_sum, k_nan    [E, C] that row's sum and NaN flag
//   v_t [E, dv, Cp] v^T key-major as int8_quantize_cols_kernel stores it (Cp = round_up(C, 16))
//   v_sum, v_nan    [E, dv] the column sums over the L stored keys and a sticky NaN flag
// Every byte at a key position >= L is 0 (the buffers start zeroed), as the quantizers' padding is.  So the first L
// keys of the cache hold exactly what the workspace of sb200_int8_attention holds for the same L keys.
//
// Append (int8_kv_append_kernel, one launch): t new keys and values at positions [L, L + t), every element through
// stored_grid (int8_grid.cuh); v_sum and v_nan are updated.  One CTA per entry, so the column sums need no atomics.
//
// Attention, Tq > kDecRows: q is quantized into the workspace and int8_attention_kernel runs over the cache through TMA
// maps that view its first L keys (k: (dp, L, E) with entry stride C dp; v^T: (round_up(L, 16), dv, E) with row
// stride Cp): the output and p_q are bit-identical to sb200_int8_attention[_masked] on the appended fp32 keys and
// values.
//
// Attention, Tq <= kDecRows (decode: one token, a few speculative tokens, a short chunk).  p is quantized, so it must be
// final -- global max m and sum l -- before its grid exists, and the partial outputs of flash-decoding cannot be
// rescaled afterwards.  Two passes over key splits instead, with exact integer partials:
//   pass 1 (int8_attention_decode_scores_kernel)  work item = (entry, split of the keys): the exact int8 scores of the
//          split's keys (dp4a), the score epilogue, scale, causal band and mask (at_score / at_masked), written to the
//          workspace as fp32 (4 B per key, against the dp bytes a second read of k would cost); per row the split's
//          max and fp64 sum of exp_diff, and whether the row sees a NaN key.
//   pass 2 (int8_attention_decode_pv_kernel)  each work item combines every split's (m, l) of its rows in split order
//          (at_rescale), then p = exp_diff(s, m) RN32(1 / l) on its grid (at_p_grid), p_q, and the int32 partials
//          sum_j g_p v (cached v^T, dp4a) and sum_j g_p of its split: exact, |products| <= 2^14 and L < 2^17.
//   combine (int8_attention_decode_out_kernel)  the partials summed in int64, the zero-point terms with v_sum (every
//          key is visited and a hidden key carries the grid of p = 0, so no prefix sums are needed), the NaN rules
//          (at_row_nan) and out = RN32(fp64(I_pv) fp64(s_p) fp64(s_v)) (at_out).
// The scores are bit-identical to sb200_int8_matmul(q, k^T); only l's fp64 summation order differs from the fused
// kernel, so a p grid value differs from its grid there only when RN32(1 / l) does, by at most one step.  The split
// size depends on the shape alone (kDecWork), no atomics, no state between calls: the result is deterministic.
#include "int8_attention.cuh"

namespace sb200 {
namespace {

constexpr int kDecRows = 16;          // the largest Tq of the decode kernels: one m16 row tile
constexpr int kDecThreads = 256;
constexpr int kDecWarps = kDecThreads / 32;
constexpr int kDecMaxSplit = 2048;    // keys per split at most: pass 2 keeps 16 x split bytes of p grid in shared memory
constexpr long long kDecWork = 4 * 132;  // work items that fill the 132 SMs of an H100 SXM four CTAs deep; a constant,
                                         // so that the splits (and l's summation order) depend on the shape only
constexpr int kAppThreads = 256;

// ---------------------------------------------------------------------------------- append
// One CTA per entry.  k: a warp per new key, lane l stores bytes [4 l, 4 l + 4) of the row (dp <= 128), the row sum
// and NaN flag as int8_quantize_rows_kernel.  v: thread (n, half) quantizes column n of the new tokens i = half,
// half + 2, ... into v^T[n, L + i]; the two halves' sums and NaN flags are added to v_sum / v_nan by half 0.
__global__ void __launch_bounds__(kAppThreads) int8_kv_append_kernel(
    const float* __restrict__ k, const float* __restrict__ v, const float* __restrict__ k_scale,
    const float* __restrict__ k_zero, float k_qmin, float k_qmax, int k_off, const float* __restrict__ v_scale,
    const float* __restrict__ v_zero, float v_qmin, float v_qmax, int v_off, int8_t* __restrict__ k_q,
    int* __restrict__ k_sum, uint8_t* __restrict__ k_nan, int8_t* __restrict__ v_t, int* __restrict__ v_sum,
    uint8_t* __restrict__ v_nan, int C, int L, int t, int d, int dp, int dv, int Cp) {
  __shared__ int part_sum[kAppThreads];
  __shared__ int part_nan[kAppThreads];
  const long long e = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  QP pk, pv;
  pk.set(__ldg(k_scale), __ldg(k_zero));
  pk.qmin = k_qmin, pk.qmax = k_qmax;
  pv.set(__ldg(v_scale), __ldg(v_zero));
  pv.qmin = v_qmin, pv.qmax = v_qmax;
  for (int i = warp; i < t; i += kAppThreads / 32) {
    const float* src = k + (e * t + i) * d;
    const long long row = e * C + L + i;
    int sum = 0;
    bool nan = false;
    uint32_t word = 0u;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int c = 4 * lane + b;
      const int g = c < d ? stored_grid(__ldg(src + c), pk, k_off, nan) : 0;  // padding stays zero
      sum += g;
      word |= ((uint32_t)g & 0xFFu) << (8 * b);
    }
    if (4 * lane < dp) *reinterpret_cast<uint32_t*>(k_q + row * dp + 4 * lane) = word;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const bool any_nan = __any_sync(0xffffffffu, nan);
    if (lane == 0) {
      k_sum[row] = sum;
      k_nan[row] = any_nan ? 1 : 0;
    }
  }
  const int n = threadIdx.x % kAtMaxDim, half = threadIdx.x / kAtMaxDim;
  int sum = 0;
  bool nan = false;
  if (n < dv) {
    int8_t* dst = v_t + (e * dv + n) * Cp + L;
    for (int i = half; i < t; i += 2) {
      const int g = stored_grid(__ldg(v + (e * t + i) * dv + n), pv, v_off, nan);
      dst[i] = (int8_t)g;
      sum += g;
    }
  }
  part_sum[threadIdx.x] = sum;
  part_nan[threadIdx.x] = nan ? 1 : 0;
  __syncthreads();
  if (half == 0 && n < dv) {
    v_sum[e * dv + n] += part_sum[n] + part_sum[n + kAtMaxDim];
    v_nan[e * dv + n] |= (uint8_t)(part_nan[n] | part_nan[n + kAtMaxDim]);
  }
}

// ---------------------------------------------------------------------------------- decode
struct DecParams {
  const int8_t* q_q;     // [E, Tq, dp] the stored grid of q (workspace)
  const int8_t* k_q;     // the cache
  const int8_t* v_t;
  float* s;              // [E, Tq, L] the masked fp32 scores
  float* part_m;         // [E, ns, Tq] per split: the row max,
  double* part_l;        //   the fp64 sum of exp_diff(s, max),
  uint8_t* part_kn;      //   a NaN key the row sees,
  int* part_pv;          //   [E, ns, Tq, dv] sum_j g_p v
  int* part_ps;          //   sum_j g_p
  uint8_t* part_pn;      //   a NaN p
  int C, Cp, L, Lp, split, ns;
};

// Pass 1.  Lanes in groups of gl = pow2ceil(dp / 16) share a key, each taking 16 of its bytes: per row r < Tq the group
// sums its dp4a products by shuffles, and lane r % gl of the group finishes rows r, r + gl, ...: the score, its max and
// the NaN flag.  The second sweep reads back only the scores the thread wrote itself.  The block reductions run in a
// fixed order.
template <bool kMasked>
__global__ void __launch_bounds__(kDecThreads) int8_attention_decode_scores_kernel(const __grid_constant__ AtParams a,
                                                                                   const __grid_constant__ AtMask mk,
                                                                                   const __grid_constant__ DecParams dc) {
  __shared__ uint32_t sq[kDecRows][kAtMaxDim / 4];
  __shared__ long long rterm[kDecRows];
  __shared__ float red_m[kDecWarps][kDecRows];
  __shared__ double red_l[kDecWarps][kDecRows];
  __shared__ int red_k[kDecWarps][kDecRows];
  __shared__ float row_m[kDecRows];
  const int e = (int)(blockIdx.x / (unsigned)dc.ns), sp = (int)(blockIdx.x % (unsigned)dc.ns);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Tq = a.Tq, L = dc.L, dw = a.dp / 4;
  const long long zq = (long long)rintf(__ldg(a.q_zero)) - a.q_off, zk = (long long)rintf(__ldg(a.k_zero)) - a.k_off;
  const double sqk = (double)__ldg(a.q_scale) * (double)__ldg(a.k_scale);
  for (int i = threadIdx.x; i < Tq * dw; i += kDecThreads)
    sq[i / dw][i % dw] = __ldg(reinterpret_cast<const uint32_t*>(dc.q_q + ((size_t)e * Tq + i / dw) * a.dp) + i % dw);
  if (threadIdx.x < Tq)
    rterm[threadIdx.x] = (long long)a.d * zq * zk - zk * (long long)__ldg(a.q_sum + (size_t)e * Tq + threadIdx.x);
  __syncthreads();
  const int gl = a.dp <= 16 ? 1 : a.dp <= 32 ? 2 : a.dp <= 64 ? 4 : 8;  // lanes per key
  const int sub = lane & (gl - 1), kpw = 32 / gl;
  const int j0 = sp * dc.split, j1 = min(j0 + dc.split, L);
  const long long mbase = kMasked && mk.mask != nullptr ? at_mask_base(mk, e) : 0;
  const size_t krow0 = (size_t)e * a.ks, srow0 = (size_t)e * Tq;
  float mloc[kDecRows];
  bool kn[kDecRows];
#pragma unroll
  for (int r = 0; r < kDecRows; ++r) mloc[r] = -INFINITY, kn[r] = false;
  for (int jb = j0; jb < j1; jb += kDecWarps * kpw) {
    const int j = jb + warp * kpw + lane / gl;
    const bool live = j < j1;
    uint4 kw = make_uint4(0u, 0u, 0u, 0u);
    if (live && 16 * sub < a.dp) kw = __ldg(reinterpret_cast<const uint4*>(dc.k_q + ((size_t)e * dc.C + j) * a.dp) + sub);
    int acc[kDecRows];
#pragma unroll
    for (int r = 0; r < kDecRows; ++r) {
      acc[r] = 0;
      if (r < Tq && 16 * sub < a.dp) {
        acc[r] = __dp4a((int)kw.x, (int)sq[r][4 * sub], acc[r]);
        acc[r] = __dp4a((int)kw.y, (int)sq[r][4 * sub + 1], acc[r]);
        acc[r] = __dp4a((int)kw.z, (int)sq[r][4 * sub + 2], acc[r]);
        acc[r] = __dp4a((int)kw.w, (int)sq[r][4 * sub + 3], acc[r]);
      }
      if (r < Tq)
        for (int o = 1; o < gl; o <<= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
    }
    if (!live) continue;
    const long long kz = zq * (long long)__ldg(a.k_sum + krow0 + j);
    const bool knan = __ldg(a.k_nan + krow0 + j) != 0;
#pragma unroll
    for (int r = 0; r < kDecRows; ++r) {
      if (r >= Tq || (r & (gl - 1)) != sub) continue;
      float sc = at_score((long long)acc[r] + rterm[r] - kz, sqk, a.has_scale, a.scale);
      bool seen = true;
      if constexpr (kMasked) {
        seen = !mk.causal || (long long)j <= (long long)r + L - Tq;
        const float* mrow = mk.mask != nullptr ? mk.mask + mbase + (long long)r * mk.stride_row : nullptr;
        sc = at_masked(sc, seen, mrow, j);
      }
      kn[r] |= seen && knan;
      dc.s[(srow0 + r) * L + j] = sc;
      mloc[r] = fmaxf(mloc[r], sc);
    }
  }
  // the split's row max
#pragma unroll
  for (int r = 0; r < kDecRows; ++r) {
    if (r >= Tq) continue;
    float m = mloc[r];
    int k = kn[r] ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      k |= __shfl_xor_sync(0xffffffffu, k, o);
    }
    if (lane == 0) red_m[warp][r] = m, red_k[warp][r] = k;
  }
  __syncthreads();
  if (threadIdx.x < Tq) {
    float m = -INFINITY;
    for (int w = 0; w < kDecWarps; ++w) m = fmaxf(m, red_m[w][threadIdx.x]);
    row_m[threadIdx.x] = m;
  }
  __syncthreads();
  // the split's sum of exp_diff(s, m), over the scores this thread wrote
  double lloc[kDecRows];
#pragma unroll
  for (int r = 0; r < kDecRows; ++r) lloc[r] = 0.0;
  for (int jb = j0; jb < j1; jb += kDecWarps * kpw) {
    const int j = jb + warp * kpw + lane / gl;
    if (j >= j1) continue;
#pragma unroll
    for (int r = 0; r < kDecRows; ++r)
      if (r < Tq && (r & (gl - 1)) == sub) lloc[r] += (double)exp_diff(dc.s[(srow0 + r) * L + j], row_m[r]);
  }
#pragma unroll
  for (int r = 0; r < kDecRows; ++r) {
    if (r >= Tq) continue;
    double l = lloc[r];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
    if (lane == 0) red_l[warp][r] = l;
  }
  __syncthreads();
  if (threadIdx.x < Tq) {
    const int r = threadIdx.x;
    double l = 0.0;
    int k = 0;
    for (int w = 0; w < kDecWarps; ++w) l += red_l[w][r], k |= red_k[w][r];
    const size_t o = ((size_t)e * dc.ns + sp) * Tq + r;
    dc.part_m[o] = row_m[r];
    dc.part_l[o] = l;
    dc.part_kn[o] = (uint8_t)k;
  }
}

// Pass 2.  Rows r < Tq first combine the splits' (m, l) in split order; then each thread puts p's grid of keys j0 + t,
// j0 + t + 256, ... of every row into a shared tile [Tq][split] (and p_q); then warp w takes the columns n = w, w + 8,
// ... of v^T, lane l the 4-key words l, l + 32, ... of the split, and the warp sums the dp4a partials of each row.
__global__ void __launch_bounds__(kDecThreads) int8_attention_decode_pv_kernel(const __grid_constant__ AtParams a,
                                                                               const __grid_constant__ DecParams dc) {
  extern __shared__ uint32_t gp[];  // [Tq][split / 4] words of p's grid
  __shared__ float row_m[kDecRows], row_inv[kDecRows];
  __shared__ int red_s[kDecWarps][kDecRows], red_n[kDecWarps][kDecRows];
  const int e = (int)(blockIdx.x / (unsigned)dc.ns), sp = (int)(blockIdx.x % (unsigned)dc.ns);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Tq = a.Tq, L = dc.L;
  const size_t srow0 = (size_t)e * Tq;
  if (threadIdx.x < Tq) {
    const size_t o = (size_t)e * dc.ns * Tq + threadIdx.x;
    float m = -INFINITY;
    for (int s = 0; s < dc.ns; ++s) m = fmaxf(m, dc.part_m[o + (size_t)s * Tq]);
    double l = 0.0;
    for (int s = 0; s < dc.ns; ++s) l += at_rescale(dc.part_l[o + (size_t)s * Tq], dc.part_m[o + (size_t)s * Tq], m);
    row_m[threadIdx.x] = m;
    row_inv[threadIdx.x] = __double2float_rn(1.0 / l);
  }
  __syncthreads();
  QP pp;
  pp.set(__ldg(a.p_scale), __ldg(a.p_zero));
  pp.qmin = a.p_qmin;
  pp.qmax = a.p_qmax;
  const int j0 = sp * dc.split, jp = min(j0 + dc.split, dc.Lp);  // keys [L, Lp) are p_q's padding: 0
  const int words = dc.split / 4;
  int8_t* g8 = reinterpret_cast<int8_t*>(gp);
  int psum[kDecRows];
  bool pnan[kDecRows];
#pragma unroll
  for (int r = 0; r < kDecRows; ++r) psum[r] = 0, pnan[r] = false;
  for (int j = j0 + threadIdx.x; j < jp; j += kDecThreads) {
#pragma unroll
    for (int r = 0; r < kDecRows; ++r) {
      if (r >= Tq) continue;
      const int g = j < L ? at_p_grid(dc.s[(srow0 + r) * L + j], row_m[r], row_inv[r], pp, a.p_off, pnan[r]) : 0;
      psum[r] += g;
      g8[r * dc.split + (j - j0)] = (int8_t)g;
      if (a.p_q != nullptr) a.p_q[(srow0 + r) * (size_t)a.Tkp + j] = (int8_t)g;
    }
  }
#pragma unroll
  for (int r = 0; r < kDecRows; ++r) {
    if (r >= Tq) continue;
    int s = psum[r], n = pnan[r] ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o), n |= __shfl_xor_sync(0xffffffffu, n, o);
    if (lane == 0) red_s[warp][r] = s, red_n[warp][r] = n;
  }
  __syncthreads();
  const size_t part0 = ((size_t)e * dc.ns + sp) * Tq;
  if (threadIdx.x < Tq) {
    int s = 0, n = 0;
    for (int w = 0; w < kDecWarps; ++w) s += red_s[w][threadIdx.x], n |= red_n[w][threadIdx.x];
    dc.part_ps[part0 + threadIdx.x] = s;
    dc.part_pn[part0 + threadIdx.x] = (uint8_t)n;
  }
  const int nw = (jp - j0) / 4;  // Lp is a multiple of 16: whole words, all inside the row of v^T
  for (int n = warp; n < a.dv; n += kDecWarps) {
    const uint32_t* vrow = reinterpret_cast<const uint32_t*>(dc.v_t + ((size_t)e * a.dv + n) * dc.Cp + j0);
    int acc[kDecRows];
#pragma unroll
    for (int r = 0; r < kDecRows; ++r) acc[r] = 0;
    for (int w = lane; w < nw; w += 32) {
      const int vw = (int)__ldg(vrow + w);
#pragma unroll
      for (int r = 0; r < kDecRows; ++r)
        if (r < Tq) acc[r] = __dp4a((int)gp[r * words + w], vw, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < kDecRows; ++r) {
      if (r >= Tq) continue;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
      if (lane == r) dc.part_pv[(part0 + r) * a.dv + n] = acc[r];
    }
  }
}

// Combine: thread (r, n) of entry e sums the splits' partials in int64 and writes out[e, r, n].
__global__ void __launch_bounds__(kDecThreads) int8_attention_decode_out_kernel(const __grid_constant__ AtParams a,
                                                                                const __grid_constant__ DecParams dc) {
  const int e = blockIdx.x, Tq = a.Tq, dv = a.dv;
  const long long zp = (long long)rintf(__ldg(a.p_zero)) - a.p_off, zv = (long long)rintf(__ldg(a.v_zero)) - a.v_off;
  const double spv = (double)__ldg(a.p_scale) * (double)__ldg(a.v_scale);
  for (int i = threadIdx.x; i < Tq * dv; i += kDecThreads) {
    const int r = i / dv, n = i % dv;
    float m = -INFINITY;
    bool kn = false, pn = false;
    long long ps = 0, o = 0;
    for (int s = 0; s < dc.ns; ++s) {
      const size_t p = ((size_t)e * dc.ns + s) * Tq + r;
      m = fmaxf(m, dc.part_m[p]);
      kn |= dc.part_kn[p] != 0;
      pn |= dc.part_pn[p] != 0;
      ps += dc.part_ps[p];
      o += dc.part_pv[p * dv + n];
    }
    const bool bad = at_row_nan(__ldg(a.q_nan + (size_t)e * Tq + r) != 0, kn, pn, m == -INFINITY);
    const long long I = o + (long long)dc.L * zp * zv - zv * ps - zp * (long long)__ldg(a.v_sum + (size_t)e * dv + n);
    a.out[((size_t)e * Tq + r) * dv + n] = at_out(I, spv, bad || __ldg(a.v_nan + (size_t)e * dv + n) != 0);
  }
}

// ---------------------------------------------------------------------------------- host
// The split of the decode kernels: keys per split (a multiple of 128, at most kDecMaxSplit) and the split count.
void dec_split(long long batch, long long length, int* split, int* ns) {
  const long long want = std::max(1LL, (kDecWork + batch - 1) / batch);  // splits per entry that fill the SMs
  long long s = ((length + want - 1) / want + kAtKeys - 1) / kAtKeys * kAtKeys;
  s = std::min<long long>(std::max<long long>(s, kAtKeys), kDecMaxSplit);
  *split = (int)s;
  *ns = (int)((length + s - 1) / s);
}

// Workspace: q's stored grid, sums and NaN flags; then for Tq > kDecRows under causal the column sums of v^T, for
// Tq <= kDecRows the scores and the split partials, each 1024-aligned.
struct CaLayout {
  size_t q, q_sum, q_nan, s, m, l, kn, pv, ps, pn, total;
};
CaLayout ca_layout(long long batch, long long tq, long long length, long long d, long long dv, int causal) {
  CaLayout w = {};
  size_t o = 0;
  auto take = [&o](size_t bytes) {
    const size_t at = o;
    o = align_up(o + bytes, 1024);
    return at;
  };
  w.q = take((size_t)(batch * tq * padded_k(d)));
  w.q_sum = take((size_t)(batch * tq) * 4);
  w.q_nan = take((size_t)(batch * tq));
  if (tq > kDecRows) {
    w.s = o;
    if (causal) o += at_vpre_bytes(batch, length, dv);
  } else {
    int split, ns;
    dec_split(batch, length, &split, &ns);
    const size_t parts = (size_t)(batch * ns * tq);
    w.s = take((size_t)(batch * tq * length) * 4);
    w.m = take(parts * 4);
    w.l = take(parts * 8);
    w.kn = take(parts);
    w.pv = take(parts * (size_t)dv * 4);
    w.ps = take(parts * 4);
    w.pn = take(parts);
  }
  w.total = o;
  return w;
}

// The checks the append and the attention share: the cache pointers, its geometry (length of the attention / after
// the append <= capacity < 2^17, batch capacity < 2^31), d and dv.
int check_cache(const char* fn, const int8_t* k_q, const int8_t* v_t, int64_t batch, int64_t capacity, int64_t length,
                int64_t d, int64_t dv) {
  SB_REQUIRE(aligned16(k_q) && aligned16(v_t), "%s: k_q and v_t must be 16-byte aligned", fn);
  if (capacity >= kAtMaxTk || d > kAtMaxDim || dv > kAtMaxDim) {
    set_error("%s: capacity = %lld, d = %lld, dv = %lld; the cache supports capacity < 2^17, d <= 128 and dv <= 128", fn,
              (long long)capacity, (long long)d, (long long)dv);
    return SB200_E_UNSUPPORTED;
  }
  SB_REQUIRE(length <= capacity, "%s: %lld keys do not fit a cache of capacity %lld", fn, (long long)length,
             (long long)capacity);
  SB_REQUIRE((__int128)batch * capacity < (1LL << 31), "%s: dimension too large (batch capacity must be < 2^31)", fn);
  return SB200_OK;
}

size_t cached_workspace_bytes(int64_t batch, int64_t tq, int64_t capacity, int64_t length, int64_t d, int64_t dv,
                              int causal) {
  if (batch <= 0 || tq <= 0 || capacity <= 0 || length <= 0 || d <= 0 || dv <= 0 || length > capacity ||
      capacity >= kAtMaxTk || d > kAtMaxDim || dv > kAtMaxDim || (causal != 0 && causal != 1))
    return 0;
  if ((__int128)batch * tq >= (1LL << 31) || (__int128)batch * capacity >= (1LL << 31)) return 0;
  if ((__int128)batch * ((tq + kAtRows - 1) / kAtRows) >= (1LL << 31)) return 0;
  return ca_layout(batch, tq, length, d, dv, causal).total + 1024;  // + the alignment of the base
}

}  // namespace
}  // namespace sb200

using namespace sb200;

int sb200_int8_kv_append(const float* k, const float* v, const float* k_scale, const float* k_zero_point, int qmin_k,
                         int qmax_k, const float* v_scale, const float* v_zero_point, int qmin_v, int qmax_v,
                         int8_t* k_q, int32_t* k_sum, uint8_t* k_nan, int8_t* v_t, int32_t* v_sum, uint8_t* v_nan,
                         int64_t batch, int64_t capacity, int64_t length, int64_t t, int64_t d, int64_t dv,
                         void* stream) {
  const char* fn = "sb200_int8_kv_append";
  SB_REQUIRE(k && v && k_scale && k_zero_point && v_scale && v_zero_point && k_q && k_sum && k_nan && v_t && v_sum &&
                 v_nan,
             "%s: null pointer argument", fn);
  SB_REQUIRE(batch > 0 && capacity > 0 && t > 0 && d > 0 && dv > 0 && length >= 0,
             "%s: empty operand or negative length (batch=%lld capacity=%lld length=%lld t=%lld d=%lld dv=%lld)", fn,
             (long long)batch, (long long)capacity, (long long)length, (long long)t, (long long)d, (long long)dv);
  if (const int rc = check_cache(fn, k_q, v_t, batch, capacity, length + t, d, dv)) return rc;
  if (const int rc = check_range(fn, qmin_k, qmax_k)) return rc;
  if (const int rc = check_range(fn, qmin_v, qmax_v)) return rc;
  int8_kv_append_kernel<<<(unsigned)batch, kAppThreads, 0, (cudaStream_t)stream>>>(
      k, v, k_scale, k_zero_point, (float)qmin_k, (float)qmax_k, grid_offset(qmin_k), v_scale, v_zero_point,
      (float)qmin_v, (float)qmax_v, grid_offset(qmin_v), k_q, reinterpret_cast<int*>(k_sum), k_nan, v_t,
      reinterpret_cast<int*>(v_sum), v_nan, (int)capacity, (int)length, (int)t, (int)d, (int)padded_k(d), (int)dv,
      (int)padded_k(capacity));
  SB_LAUNCHED();
  return SB200_OK;
}

size_t sb200_int8_attention_cached_workspace_bytes(int64_t batch, int64_t tq, int64_t capacity, int64_t length,
                                                   int64_t d, int64_t dv, int causal) {
  return cached_workspace_bytes(batch, tq, capacity, length, d, dv, causal);
}

int sb200_int8_attention_cached(const float* q, const float* q_scale, const float* q_zero_point, int qmin_q, int qmax_q,
                                const float* k_scale, const float* k_zero_point, int qmin_k, int qmax_k,
                                const float* p_scale, const float* p_zero_point, int qmin_p, int qmax_p,
                                const float* v_scale, const float* v_zero_point, int qmin_v, int qmax_v, int has_scale,
                                float scale, const float* mask, int64_t mask_stride_outer, int64_t mask_stride_inner,
                                int64_t mask_inner, int64_t mask_stride_row, int causal, const int8_t* k_q,
                                const int32_t* k_sum, const uint8_t* k_nan, const int8_t* v_t, const int32_t* v_sum,
                                const uint8_t* v_nan, int64_t capacity, int64_t length, float* out, int8_t* p_q,
                                int64_t batch, int64_t tq, int64_t d, int64_t dv, void* workspace,
                                size_t workspace_bytes, void* stream) {
  const char* fn = "sb200_int8_attention_cached";
  SB_REQUIRE(q && q_scale && q_zero_point && k_scale && k_zero_point && p_scale && p_zero_point && v_scale &&
                 v_zero_point && k_q && k_sum && k_nan && v_t && v_sum && v_nan && out && workspace,
             "%s: null pointer argument", fn);
  SB_REQUIRE(capacity > 0, "%s: empty cache (capacity=%lld)", fn, (long long)capacity);
  if (const int rc = at_check_dims(fn, batch, tq, length, d, dv)) return rc;
  if (const int rc = check_cache(fn, k_q, v_t, batch, capacity, length, d, dv)) return rc;
  const int ranges[4][2] = {{qmin_q, qmax_q}, {qmin_k, qmax_k}, {qmin_p, qmax_p}, {qmin_v, qmax_v}};
  if (const int rc = at_check_args(fn, ranges, has_scale, scale, p_q, causal, mask, mask_stride_outer, mask_stride_inner,
                                   mask_inner, mask_stride_row, batch, tq, length))
    return rc;
  if (const int rc = check_workspace(fn, workspace_bytes,
                                     cached_workspace_bytes(batch, tq, capacity, length, d, dv, causal)))
    return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const CaLayout w = ca_layout(batch, tq, length, d, dv, causal);
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  int8_t* qq = reinterpret_cast<int8_t*>(ws + w.q);
  const long long dp = padded_k(d), cp = padded_k(capacity), lp = padded_k(length);
  AtParams a;
  a.q_sum = reinterpret_cast<const int*>(ws + w.q_sum), a.q_nan = ws + w.q_nan;
  a.k_sum = reinterpret_cast<const int*>(k_sum), a.k_nan = k_nan;
  a.v_sum = reinterpret_cast<const int*>(v_sum), a.v_nan = v_nan;
  const float* const qparams[8] = {q_scale, q_zero_point, k_scale, k_zero_point, p_scale, p_zero_point, v_scale,
                                   v_zero_point};
  at_set_qparams(a, qparams, ranges, has_scale, scale);
  a.out = out, a.p_q = p_q;
  a.Tq = (int)tq, a.Tk = (int)length, a.Tkp = (int)lp, a.d = (int)d, a.dp = (int)dp, a.dv = (int)dv;
  a.ks = (int)capacity;
  a.vec2 = (dv % 2 == 0) && (reinterpret_cast<uintptr_t>(out) & 7u) == 0;
  const AtMask mk = {mask, mask_stride_outer, mask_stride_inner, mask_stride_row, nullptr, (int)(mask ? mask_inner : 1),
                     causal, (int)batch};
  if (tq > kDecRows) {
    CUtensorMap map_q, map_k, map_v;
    if (!make_map_3d(&map_q, CU_TENSOR_MAP_DATA_TYPE_UINT8, qq, (uint64_t)dp, (uint64_t)tq, (uint64_t)batch,
                     (uint64_t)dp, 128, kAtRows, CU_TENSOR_MAP_SWIZZLE_128B) ||
        !make_map_3d(&map_k, CU_TENSOR_MAP_DATA_TYPE_UINT8, k_q, (uint64_t)dp, (uint64_t)length, (uint64_t)batch,
                     (uint64_t)dp, 128, kAtKeys, CU_TENSOR_MAP_SWIZZLE_128B, (uint64_t)(capacity * dp)) ||
        !make_map_3d(&map_v, CU_TENSOR_MAP_DATA_TYPE_UINT8, v_t, (uint64_t)lp, (uint64_t)dv, (uint64_t)batch,
                     (uint64_t)cp, kAtKeys, 128, CU_TENSOR_MAP_SWIZZLE_128B, (uint64_t)(dv * cp))) {
      set_error("%s: cuTensorMapEncodeTiled failed (batch=%lld Tq=%lld capacity=%lld length=%lld d=%lld dv=%lld)", fn,
                (long long)batch, (long long)tq, (long long)capacity, (long long)length, (long long)d, (long long)dv);
      return SB200_E_CUDA;
    }
    if (const int rc = launch_rows(q, q_scale, q_zero_point, 0, qmin_q, qmax_q, qq, reinterpret_cast<int*>(ws + w.q_sum),
                                   ws + w.q_nan, batch * tq, d, st))
      return rc;
    return at_launch(map_q, map_k, map_v, a, mk, v_t, cp, reinterpret_cast<int*>(ws + w.s), batch, st);
  }
  if (const int rc = launch_rows(q, q_scale, q_zero_point, 0, qmin_q, qmax_q, qq, reinterpret_cast<int*>(ws + w.q_sum),
                                 ws + w.q_nan, batch * tq, d, st))
    return rc;
  DecParams dc;
  dc.q_q = qq, dc.k_q = k_q, dc.v_t = v_t;
  dc.s = reinterpret_cast<float*>(ws + w.s);
  dc.part_m = reinterpret_cast<float*>(ws + w.m), dc.part_l = reinterpret_cast<double*>(ws + w.l);
  dc.part_kn = ws + w.kn, dc.part_pv = reinterpret_cast<int*>(ws + w.pv), dc.part_ps = reinterpret_cast<int*>(ws + w.ps);
  dc.part_pn = ws + w.pn;
  dc.C = (int)capacity, dc.Cp = (int)cp, dc.L = (int)length, dc.Lp = (int)lp;
  dec_split(batch, length, &dc.split, &dc.ns);
  const unsigned items = (unsigned)(batch * dc.ns);
  if (mask == nullptr && !causal)
    int8_attention_decode_scores_kernel<false><<<items, kDecThreads, 0, st>>>(a, mk, dc);
  else
    int8_attention_decode_scores_kernel<true><<<items, kDecThreads, 0, st>>>(a, mk, dc);
  SB_LAUNCHED();
  int8_attention_decode_pv_kernel<<<items, kDecThreads, (size_t)tq * dc.split, st>>>(a, dc);
  SB_LAUNCHED();
  int8_attention_decode_out_kernel<<<(unsigned)batch, kDecThreads, 0, st>>>(a, dc);
  SB_LAUNCHED();
  return SB200_OK;
}
