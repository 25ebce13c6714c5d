// int8_attention.cu -- integer-grid inference of a calibrated QAttention: softmax(q k^T [* scale]) v with q, k, the
// softmax output p and v each on its own per-tensor int8 grid, in one kernel that never writes the [Tq, Tk] scores.
//
// Operands.  q [B, Tq, d] and k [B, Tk, d] go through int8_quantize_rows_kernel, v [B, Tk, dv] through
// int8_quantize_cols_kernel (v^T K-major, [B, dv, Tkp]), all into the workspace with their sums and NaN flags
// (int8_linear.cu, unchanged).  Everything after that is int8_attention_kernel.
//
// CTA = 128 query rows of one batch entry: warpgroup 0 is the TMA producer (one thread), warpgroups 1 and 2 own 64
// rows each.  The q tile is loaded once; k blocks (128 keys) and v^T blocks (128 keys of all dv <= 128 columns) stream
// through the stage ring of tc_common.cuh.  The key blocks are walked twice, with one load index running over both:
//   pass 1  (k only)   s = the scores of the block; per row a running max m and sum l = sum exp(s - m) in fp64
//   pass 2  (k and v)  the same scores again; p = exp(s - m) * RN32(1 / l) in fp32, quantized by the QDQ rule
//                      (stored_grid, int8_grid.cuh) into a SWIZZLE_128B s8 tile in shared memory, which is the K-major
//                      A operand of the p @ v wgmma accumulating into s32 over all key blocks.
// Both passes read k from global (L2) memory; nothing of size O(Tq Tk) is written unless the caller asks for p_q.
//
// Scores.  I = sum (v_q - Z_q)(v_k - Z_k) exactly (wgmma s32.s8.s8, zero points in int64), s = RN32(fp64(I) *
// (fp64(s_q) fp64(s_k))): operation for operation the epilogue of int8_matmul_gemm_kernel, so s is bit-identical to
// sb200_int8_matmul(q, k^T).  With a scale, s = RN32(s * scale).
// Softmax.  exp(s - m) is expf of the rounded difference corrected by its exact rounding error (exp_diff); l is
// summed in fp64 and rescaled with the fp64 exp.  DESIGN §4 derives |p - p64| <= 13 2^-24 p64 + 2^-125, p64 the fp64
// softmax of the same fp32 scores.
// p @ v.  I_pv = sum_j (g_p - Z_p)(v_v - Z_v) exactly (|products| <= 2^14, Tk < 2^17), out = RN32(fp64(I_pv) *
// (fp64(s_p) fp64(s_v))), the epilogue of int8_matmul_gemm_kernel with p as the left operand.
// NaN.  A NaN in row i of q makes row i NaN; a NaN anywhere in k of an entry makes the entry NaN; a NaN in column n of
// v makes column n NaN; a NaN p (only from non-finite scores) makes its row NaN.  No atomics, no state between calls.
//
// Masks (int8_attention_kernel<true>).  After the scale, s = -inf where key j is hidden from row i by the causal band
// (j > i + Tk - Tq, aligned bottom-right), then s = RN32(s + mask[i, j]): the composition of QAttention, score for
// score, in both passes.  Under causal a key block that no row of the CTA can see is neither loaded nor computed
// (at_visible_blocks, the same count in the producer and the consumers), so a CTA visits a prefix of the key blocks.
// Its skipped keys have p = 0, whose grid is Z_p, so their products vanish; the epilogue's sum of v covers the visited
// prefix only (int8_attention_vprefix_kernel: per-block column sums of v^T, accumulated), and a zero point off the
// range adds its exact (g_0 - Z_p) sum (v - Z_v) over the skipped keys.  p_q receives the grid of 0 * RN32(1 / l)
// at skipped keys, as at a hidden key the kernel visits.  A NaN in k poisons only the rows that see its key; a row
// without a visible key is NaN.
#include "int8_attention.cuh"

namespace sb200 {
namespace {

constexpr int kAtStages = 4;
constexpr int kAtThreads = 384;
constexpr int kAtTile = 128 * 128;              // 16 KB: the q tile, a k block, a v^T block (128 rows x 128 bytes)
constexpr int kAtStageBytes = 2 * kAtTile;      // k block | v^T block
constexpr int kAtPBytes = 64 * 128;             // one warpgroup's p tile (64 rows x 128 keys)
constexpr size_t kAtSmem = 1024 + kAtTile + (size_t)kAtStages * kAtStageBytes + 2 * kAtPBytes + 128;

// Key blocks a CTA of rows [m0, m0 + 128) visits: all of them, or under causal those up to the last key its last row
// sees (0 when no row sees a key).
__device__ __forceinline__ int at_visible_blocks(int m0, int Tq, int Tk, int nkb, int causal) {
  if (!causal) return nkb;
  const long long last = (long long)min(m0 + kAtRows, Tq) - 1 + Tk - Tq;  // the last key the CTA's last row sees
  return last < 0 ? 0 : min(nkb, (int)(last / kAtKeys) + 1);
}

// acc = the q tile rows of this warpgroup times the 128 keys of a k block, over nk32 steps of 32 d
__device__ __forceinline__ void qk_mma(int (&acc)[64], uint64_t dq, uint64_t dk, int nk32) {
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (j < nk32) wgmma_m64n128k32_s8(acc, dq + 2 * j, dk + 2 * j, j > 0);
  wgmma_commit();
  wgmma_wait_s32<0>(acc);
}

__device__ __forceinline__ void bar_wg(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

// One CTA per 128 query rows of one batch entry (row tile fastest; under causal batch fastest, the last row tiles,
// which visit the most key blocks, first).  Maps: q (dp, Tq, B), k (dp, Tk, B), v^T (Tkp, dv, B), boxes of 128 x 128
// bytes: rows past Tq / Tk / dv and bytes past dp / Tkp are zero-filled.  kMasked = false ignores mk.  kCache: k_sum /
// k_nan of entry b start at b ks (a key/value cache), not at b Tk; a template flag, so that the kernels of the
// concatenated operands keep their code.
template <bool kMasked, bool kCache>
__global__ void __launch_bounds__(kAtThreads, 1)
int8_attention_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                      const __grid_constant__ CUtensorMap map_v, const __grid_constant__ AtParams a,
                      const __grid_constant__ AtMask mk) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* q_tile = smem_align1024(smem_raw);
  unsigned char* stages = q_tile + kAtTile;
  unsigned char* p_tiles = stages + (size_t)kAtStages * kAtStageBytes;
  auto& ring = *reinterpret_cast<StageRing<kAtStages>*>(p_tiles + 2 * kAtPBytes);
  uint64_t* qbar = reinterpret_cast<uint64_t*>(&ring + 1);  // the q tile's barrier
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned tiles_q = (unsigned)(a.Tq + kAtRows - 1) / kAtRows;
  int m0 = (int)(blockIdx.x % tiles_q) * kAtRows, batch = (int)(blockIdx.x / tiles_q);
  const int nkb = (a.Tk + kAtKeys - 1) / kAtKeys;
  int nvb = nkb;  // the key blocks this CTA visits
  if constexpr (kMasked) {
    if (mk.causal) {
      m0 = (int)(tiles_q - 1 - blockIdx.x / (unsigned)mk.batch) * kAtRows, batch = (int)(blockIdx.x % (unsigned)mk.batch);
      nvb = at_visible_blocks(m0, a.Tq, a.Tk, nkb, 1);
    }
  }

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_k);
    prefetch_tensormap(&map_v);
    ring.init();
    mbar_init(qbar, 1);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(qbar, (uint32_t)kAtTile);
      tma_load_3d(q_tile, &map_q, 0, m0, batch, qbar);
      // block i < nvb: pass 1 (k block i); i >= nvb: pass 2 (k and v^T block i - nvb)
      for (int i = 0; i < 2 * nvb; ++i) {
        const int kb = i < nvb ? i : i - nvb;
        const int s = ring.acquire(i, (uint32_t)(i < nvb ? kAtTile : kAtStageBytes));
        unsigned char* st = stages + (size_t)s * kAtStageBytes;
        tma_load_3d(st, &map_k, 0, kb * kAtKeys, batch, &ring.full[s]);
        if (i >= nvb) tma_load_3d(st + kAtTile, &map_v, kb * kAtKeys, 0, batch, &ring.full[s]);
      }
    }
    return;
  }
  reg_inc<232>();
  const int wg = (warp - 4) >> 2, q4 = lane & 3;
  const int rl = 16 * (warp & 3) + (lane >> 2);  // the thread's first row within the warpgroup's 64; the second is +8
  const size_t qrow0 = (size_t)batch * a.Tq, krow0 = (size_t)batch * (kCache ? a.ks : a.Tk), vrow0 = (size_t)batch * a.dv;
  const double sqk = (double)__ldg(a.q_scale) * (double)__ldg(a.k_scale);
  const long long zq = (long long)rintf(__ldg(a.q_zero)) - a.q_off, zk = (long long)rintf(__ldg(a.k_zero)) - a.k_off;
  const long long zv = (long long)rintf(__ldg(a.v_zero)) - a.v_off;
  QP pp;
  pp.set(__ldg(a.p_scale), __ldg(a.p_zero));
  pp.qmin = a.p_qmin;
  pp.qmax = a.p_qmax;
  const long long zp = (long long)pp.zp - a.p_off;
  int row[2];
  long long rterm[2];  // d Z_q Z_k - Z_k sum_k v_q of the row
  bool bad[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row[h] = m0 + 64 * wg + rl + 8 * h;
    const bool live = row[h] < a.Tq;
    rterm[h] = (long long)a.d * zq * zk - (live ? zk * (long long)__ldg(a.q_sum + qrow0 + row[h]) : 0);
    bad[h] = live && __ldg(a.q_nan + qrow0 + row[h]) != 0;
  }
  const float* mrow[2] = {nullptr, nullptr};  // the mask row of each of the thread's rows (none past Tq)
  long long vis[2] = {0, 0};                  // causal: the last key each row sees
  if constexpr (kMasked) {
    const long long base = at_mask_base(mk, batch);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (mk.mask != nullptr && row[h] < a.Tq) mrow[h] = mk.mask + base + (long long)row[h] * mk.stride_row;
      vis[h] = mk.causal ? (long long)row[h] + a.Tk - a.Tq : (long long)a.Tk;
    }
  }
  const int nk32 = (a.dp + 31) / 32;
  mbar_wait_relaxed(qbar, 0, 0);
  const uint64_t dq = gmma_desc_sw128(smem_u32(q_tile) + (uint32_t)wg * (64 * 128));
  const uint32_t stage0 = smem_u32(stages);
  int acc[64];

  // ---- pass 1: row max and sum.  Each thread keeps (m, l) of its 32 keys per block; the quad combines them.
  float mx[2] = {-INFINITY, -INFINITY};
  double l[2] = {0.0, 0.0};
  bool knan = false, knr[2] = {false, false};  // knr: the masked kernel's per-row NaN key
  for (int kb = 0; kb < nvb; ++kb) {
    const int s = ring.wait(kb);
    qk_mma(acc, dq, gmma_desc_sw128(stage0 + (uint32_t)s * kAtStageBytes), nk32);
    ring.release(kb, lane);
    float bm[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 64; j += 2) {  // acc[j], acc[j + 1]: keys 8 (j >> 2) + 2 q4 + {0, 1}, row h = (j >> 1) & 1
      const int h = (j >> 1) & 1;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = kb * kAtKeys + 8 * (j >> 2) + 2 * q4 + e;
        float sc = -INFINITY;
        if (key < a.Tk) {
          const long long I = (long long)acc[j + e] + rterm[h] - zq * (long long)__ldg(a.k_sum + krow0 + key);
          sc = at_score(I, sqk, a.has_scale, a.scale);
          if constexpr (kMasked) {
            const bool seen = key <= vis[h];
            sc = at_masked(sc, seen, mrow[h], key);
            knr[h] |= seen && __ldg(a.k_nan + krow0 + key) != 0;
          } else {
            if (h == 0) knan |= __ldg(a.k_nan + krow0 + key) != 0;
          }
        }
        acc[j + e] = __float_as_int(sc);
        bm[h] = fmaxf(bm[h], sc);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
      if (bm[h] > mx[h]) {
        l[h] *= exp((double)mx[h] - (double)bm[h]);
        mx[h] = bm[h];
      }
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      const int h = (j >> 1) & 1;
      l[h] += (double)exp_diff(__int_as_float(acc[j]), mx[h]);
    }
  }
  float inv[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float m = mx[h];
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    double lh = at_rescale(l[h], mx[h], m);
    lh += __shfl_xor_sync(0xffffffffu, lh, 1);
    lh += __shfl_xor_sync(0xffffffffu, lh, 2);
    mx[h] = m;
    inv[h] = __double2float_rn(1.0 / lh);
  }
  const bool kbad = __any_sync(0xffffffffu, knan);  // the quad's keys are all keys; every quad saw them
  if constexpr (kMasked) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // the quad's keys are all keys of the row
      knr[h] = __shfl_xor_sync(0xffffffffu, (int)knr[h], 1) | knr[h];
      knr[h] = __shfl_xor_sync(0xffffffffu, (int)knr[h], 2) | knr[h];
    }
  }

  // ---- pass 2: p on its grid into shared memory, then p @ v
  unsigned char* my_p = p_tiles + wg * kAtPBytes;
  const uint64_t dp_desc = gmma_desc_sw128(smem_u32(my_p));
  int o[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) o[j] = 0;
  int psum[2] = {0, 0};
  bool pnan[2] = {false, false};
  for (int kb = 0; kb < nvb; ++kb) {
    const int s = ring.wait(nvb + kb);
    const uint32_t st = stage0 + (uint32_t)s * kAtStageBytes;
    qk_mma(acc, dq, gmma_desc_sw128(st), nk32);
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const int kl = 8 * c + 2 * q4, key = kb * kAtKeys + kl;  // the pair kl, kl + 1 of the block
      long long kz[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) kz[e] = key + e < a.Tk ? zq * (long long)__ldg(a.k_sum + krow0 + key + e) : 0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t pair = 0u;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (key + e >= a.Tk) continue;  // masked keys store 0: with v^T zero there, they add nothing
          const long long I = (long long)acc[4 * c + 2 * h + e] + rterm[h] - kz[e];
          float sc = at_score(I, sqk, a.has_scale, a.scale);
          if constexpr (kMasked) sc = at_masked(sc, key + e <= vis[h], mrow[h], key + e);
          const int g = at_p_grid(sc, mx[h], inv[h], pp, a.p_off, pnan[h]);
          psum[h] += g;
          pair |= ((uint32_t)g & 0xFFu) << (8 * e);
        }
        const int r = rl + 8 * h;  // SWIZZLE_128B: 16-byte chunk kl / 16 of row r sits at chunk (kl / 16) ^ (r % 8)
        *reinterpret_cast<uint16_t*>(my_p + r * 128 + ((((kl >> 4) ^ (r & 7))) << 4) + (kl & 15)) = (uint16_t)pair;
        if (a.p_q != nullptr && row[h] < a.Tq && key < a.Tkp)
          *reinterpret_cast<uint16_t*>(a.p_q + (qrow0 + row[h]) * (size_t)a.Tkp + key) = (uint16_t)pair;
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the p tile is visible to the wgmma
    bar_wg(wg);
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) wgmma_m64n128k32_s8(o, dp_desc + 2 * j, gmma_desc_sw128(st + kAtTile) + 2 * j, 1);
    wgmma_commit();
    wgmma_wait_s32<0>(o);  // the stage and the p tile are free again
    ring.release(nvb + kb, lane);
  }
  if constexpr (kMasked) {  // the skipped keys' p is 0 (NaN in a row without a visible key): its grid into p_q
    if (a.p_q != nullptr) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (row[h] >= a.Tq) continue;
        bool unused = false;
        const uint32_t g0 = (uint32_t)stored_grid(__fmul_rn(0.f, inv[h]), pp, a.p_off, unused) & 0xFFu;
        int8_t* dst = a.p_q + (qrow0 + row[h]) * (size_t)a.Tkp;
        for (int key = nvb * kAtKeys + 2 * q4; key < a.Tkp; key += 8)
          *reinterpret_cast<uint16_t*>(dst + key) = (uint16_t)((key < a.Tk ? g0 : 0u) | (key + 1 < a.Tk ? g0 << 8 : 0u));
      }
    }
  }

  // ---- epilogue: I_pv = sum g_p v - Z_v sum g_p - Z_p sum v + Tk Z_p Z_v, out = RN32(fp64(I_pv) s_p s_v)
  const double spv = (double)__ldg(a.p_scale) * (double)__ldg(a.v_scale);
  // the masked kernel over a visited prefix of nvis keys: - Z_p sum v over the prefix, and (g_0 - Z_p) (v - Z_v) for
  // each skipped key, g_0 the grid of p = 0 (the products of the skipped keys vanish when Z_p lies in the range)
  const int nvis = kMasked ? min(nvb * kAtKeys, a.Tk) : a.Tk;
  long long d0 = 0;
  if constexpr (kMasked) {
    bool unused = false;
    d0 = (long long)stored_grid(0.f, pp, a.p_off, unused) - zp;
  }
  long long rp[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int ps = psum[h], pn = pnan[h] ? 1 : 0;
    ps += __shfl_xor_sync(0xffffffffu, ps, 1);
    pn |= __shfl_xor_sync(0xffffffffu, pn, 1);
    ps += __shfl_xor_sync(0xffffffffu, ps, 2);
    pn |= __shfl_xor_sync(0xffffffffu, pn, 2);
    rp[h] = (long long)nvis * zp * zv - zv * (long long)ps;
    if constexpr (kMasked) {
      rp[h] -= d0 * (long long)(a.Tk - nvis) * zv;
      bad[h] = at_row_nan(bad[h], knr[h], pn != 0, mx[h] == -INFINITY);  // a NaN key the row sees; no visible key
    } else {
      bad[h] = at_row_nan(bad[h], kbad, pn != 0, false);
    }
  }
#pragma unroll
  for (int c = 0; c < 16; ++c) {
    const int n = 8 * c + 2 * q4;
    if (n >= a.dv) continue;
    long long cn[2];
    bool cnan[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool live = n + e < a.dv;
      cn[e] = live ? zp * (long long)__ldg(a.v_sum + vrow0 + n + e) : 0;
      if constexpr (kMasked) {
        if (live && nvis < a.Tk) {  // causal: the column's sum over the visited prefix
          const long long all = __ldg(a.v_sum + vrow0 + n + e);
          const long long pre = nvb > 0 ? __ldg(mk.v_pre + (vrow0 + n + e) * (size_t)nkb + nvb - 1) : 0;
          cn[e] = zp * pre - d0 * (all - pre);
        }
      }
      cnan[e] = live && __ldg(a.v_nan + vrow0 + n + e) != 0;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (row[h] >= a.Tq) continue;
      float y[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        y[e] = at_out((long long)o[4 * c + 2 * h + e] + rp[h] - cn[e], spv, bad[h] || cnan[e]);
      }
      float* dst = a.out + (qrow0 + row[h]) * (size_t)a.dv + n;
      if (a.vec2) {  // dv is even: the pair is in range and 8-byte aligned
        *reinterpret_cast<float2*>(dst) = make_float2(y[0], y[1]);
      } else {
        dst[0] = y[0];
        if (n + 1 < a.dv) dst[1] = y[1];
      }
    }
  }
}

// Causal: pre[r, kb] = the sum of the stored v^T row r (one column of v) over key blocks 0 .. kb (|sum| < 2^24).
// One warp per row, each lane 4 of a block's 128 bytes; Tkp is a multiple of 16, so a lane's 4 bytes are all in range
// or all past it.
__global__ void __launch_bounds__(256) int8_attention_vprefix_kernel(const int8_t* __restrict__ vq, int* __restrict__ pre,
                                                                     long long rows, int tkp, int nkb) {
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const int8_t* src = vq + r * tkp;
  int run = 0;
  for (int kb = 0; kb < nkb; ++kb) {
    const int c = kb * kAtKeys + 4 * lane;
    int x = c < tkp ? __dp4a(*reinterpret_cast<const int*>(src + c), 0x01010101, 0) : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    run += x;
    if (lane == 0) pre[r * nkb + kb] = run;
  }
}

// Workspace: the three stored operands, each 1024-aligned and followed by its int32 sums and NaN flags
struct AtLayout {
  size_t q, q_sum, q_nan, k, k_sum, k_nan, v, v_sum, v_nan, total;
};
AtLayout at_layout(long long batch, long long tq, long long tk, long long d, long long dv) {
  AtLayout w;
  size_t o = 0;
  const long long rows[3] = {batch * tq, batch * tk, batch * dv}, width[3] = {padded_k(d), padded_k(d), padded_k(tk)};
  size_t* q[3][3] = {{&w.q, &w.q_sum, &w.q_nan}, {&w.k, &w.k_sum, &w.k_nan}, {&w.v, &w.v_sum, &w.v_nan}};
  for (int i = 0; i < 3; ++i) {
    *q[i][0] = o;
    o = align_up(o + (size_t)rows[i] * (size_t)width[i], 256);
    *q[i][1] = o;
    o = align_up(o + (size_t)rows[i] * 4, 256);
    *q[i][2] = o;
    o = align_up(o + (size_t)rows[i], 1024);
  }
  w.total = o;
  return w;
}

template <bool kMasked, bool kCache>
int at_run(const CUtensorMap& map_q, const CUtensorMap& map_k, const CUtensorMap& map_v, const AtParams& a,
           const AtMask& mk, long long ctas, cudaStream_t st) {
  static std::atomic<int> attr_done[64];
  SB_CUDA(ensure_dyn_smem(int8_attention_kernel<kMasked, kCache>, (int)kAtSmem, attr_done));
  int8_attention_kernel<kMasked, kCache><<<(unsigned)ctas, kAtThreads, kAtSmem, st>>>(map_q, map_k, map_v, a, mk);
  SB_LAUNCHED();
  return SB200_OK;
}

size_t at_workspace_bytes(int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv, int causal) {
  if (batch <= 0 || tq <= 0 || tk <= 0 || d <= 0 || dv <= 0 || d > kAtMaxDim || dv > kAtMaxDim || tk >= kAtMaxTk)
    return 0;
  if ((__int128)batch * tq >= (1LL << 31) || (__int128)batch * tk >= (1LL << 31)) return 0;
  return at_layout(batch, tq, tk, d, dv).total + (causal ? at_vpre_bytes(batch, tk, dv) : 0) +
         1024;  // + the alignment of the base
}

// The shared host code of both entry points; mask == null and causal == 0 runs int8_attention_kernel<false>.
int attention_run(const char* fn, const float* q, const float* k, const float* v, const float* q_scale,
                  const float* q_zero_point, int qmin_q, int qmax_q, const float* k_scale, const float* k_zero_point,
                  int qmin_k, int qmax_k, const float* p_scale, const float* p_zero_point, int qmin_p, int qmax_p,
                  const float* v_scale, const float* v_zero_point, int qmin_v, int qmax_v, int has_scale, float scale,
                  const float* mask, int64_t mask_stride_outer, int64_t mask_stride_inner, int64_t mask_inner,
                  int64_t mask_stride_row, int causal, float* out, int8_t* p_q, int64_t batch, int64_t tq, int64_t tk,
                  int64_t d, int64_t dv, void* workspace, size_t workspace_bytes, void* stream) {
  SB_REQUIRE(q && k && v && q_scale && q_zero_point && k_scale && k_zero_point && p_scale && p_zero_point && v_scale &&
                 v_zero_point && out && workspace,
             "%s: null pointer argument", fn);
  if (const int rc = at_check_dims(fn, batch, tq, tk, d, dv)) return rc;
  const int ranges[4][2] = {{qmin_q, qmax_q}, {qmin_k, qmax_k}, {qmin_p, qmax_p}, {qmin_v, qmax_v}};
  if (const int rc = at_check_args(fn, ranges, has_scale, scale, p_q, causal, mask, mask_stride_outer, mask_stride_inner,
                                   mask_inner, mask_stride_row, batch, tq, tk))
    return rc;
  if (const int rc = check_workspace(fn, workspace_bytes, at_workspace_bytes(batch, tq, tk, d, dv, causal))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const AtLayout w = at_layout(batch, tq, tk, d, dv);
  unsigned char* ws = reinterpret_cast<unsigned char*>(align_up(reinterpret_cast<uintptr_t>(workspace), 1024));
  int8_t *qq = reinterpret_cast<int8_t*>(ws + w.q), *kq = reinterpret_cast<int8_t*>(ws + w.k);
  int8_t* vq = reinterpret_cast<int8_t*>(ws + w.v);
  const long long dp = padded_k(d), tkp = padded_k(tk);
  CUtensorMap map_q, map_k, map_v;
  if (!make_map_3d(&map_q, CU_TENSOR_MAP_DATA_TYPE_UINT8, qq, (uint64_t)dp, (uint64_t)tq, (uint64_t)batch, (uint64_t)dp,
                   128, kAtRows, CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_map_3d(&map_k, CU_TENSOR_MAP_DATA_TYPE_UINT8, kq, (uint64_t)dp, (uint64_t)tk, (uint64_t)batch, (uint64_t)dp,
                   128, kAtKeys, CU_TENSOR_MAP_SWIZZLE_128B) ||
      !make_map_3d(&map_v, CU_TENSOR_MAP_DATA_TYPE_UINT8, vq, (uint64_t)tkp, (uint64_t)dv, (uint64_t)batch,
                   (uint64_t)tkp, kAtKeys, 128, CU_TENSOR_MAP_SWIZZLE_128B)) {
    set_error("%s: cuTensorMapEncodeTiled failed (batch=%lld Tq=%lld Tk=%lld d=%lld dv=%lld)", fn, (long long)batch,
              (long long)tq, (long long)tk, (long long)d, (long long)dv);
    return SB200_E_CUDA;
  }
  if (const int rc = sb200_int8_quantize_rows(q, q_scale, q_zero_point, 0, qmin_q, qmax_q, qq,
                                              reinterpret_cast<int32_t*>(ws + w.q_sum), ws + w.q_nan, batch * tq, d,
                                              stream))
    return rc;
  if (const int rc = sb200_int8_quantize_rows(k, k_scale, k_zero_point, 0, qmin_k, qmax_k, kq,
                                              reinterpret_cast<int32_t*>(ws + w.k_sum), ws + w.k_nan, batch * tk, d,
                                              stream))
    return rc;
  if (const int rc = sb200_int8_quantize_cols(v, v_scale, v_zero_point, qmin_v, qmax_v, vq,
                                              reinterpret_cast<int32_t*>(ws + w.v_sum), ws + w.v_nan, batch, tk, dv,
                                              stream))
    return rc;
  const AtMask mk = {mask, mask_stride_outer, mask_stride_inner, mask_stride_row, nullptr, (int)(mask ? mask_inner : 1),
                     causal, (int)batch};
  AtParams a;
  a.q_sum = reinterpret_cast<const int*>(ws + w.q_sum), a.q_nan = ws + w.q_nan;
  a.k_sum = reinterpret_cast<const int*>(ws + w.k_sum), a.k_nan = ws + w.k_nan;
  a.v_sum = reinterpret_cast<const int*>(ws + w.v_sum), a.v_nan = ws + w.v_nan;
  const float* const qparams[8] = {q_scale, q_zero_point, k_scale, k_zero_point, p_scale, p_zero_point, v_scale,
                                   v_zero_point};
  at_set_qparams(a, qparams, ranges, has_scale, scale);
  a.out = out, a.p_q = p_q;
  a.Tq = (int)tq, a.Tk = (int)tk, a.Tkp = (int)tkp, a.d = (int)d, a.dp = (int)dp, a.dv = (int)dv, a.ks = (int)tk;
  a.vec2 = (dv % 2 == 0) && (reinterpret_cast<uintptr_t>(out) & 7u) == 0;
  return at_launch(map_q, map_k, map_v, a, mk, vq, tkp, reinterpret_cast<int*>(ws + w.total), batch, st);
}

}  // namespace

// ---------------------------------------------------------------------------------- shared through int8_attention.cuh
int at_check_dims(const char* fn, int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv) {
  SB_REQUIRE(batch > 0 && tq > 0 && tk > 0 && d > 0 && dv > 0,
             "%s: empty operand (batch=%lld Tq=%lld Tk=%lld d=%lld dv=%lld)", fn, (long long)batch, (long long)tq,
             (long long)tk, (long long)d, (long long)dv);
  if (d > kAtMaxDim || dv > kAtMaxDim || tk >= kAtMaxTk) {
    set_error("%s: d = %lld, dv = %lld, Tk = %lld; the fused attention supports d <= 128, dv <= 128 and Tk < 2^17",
              fn, (long long)d, (long long)dv, (long long)tk);
    return SB200_E_UNSUPPORTED;
  }
  SB_REQUIRE((__int128)batch * tq < (1LL << 31) && (__int128)batch * tk < (1LL << 31) &&
                 (__int128)batch * ((tq + kAtRows - 1) / kAtRows) < (1LL << 31),
             "%s: dimension too large (batch Tq and batch Tk must be < 2^31)", fn);
  return SB200_OK;
}

int at_check_args(const char* fn, const int (&ranges)[4][2], int has_scale, float scale, const int8_t* p_q, int causal,
                  const float* mask, int64_t mask_stride_outer, int64_t mask_stride_inner, int64_t mask_inner,
                  int64_t mask_stride_row, int64_t batch, int64_t tq, int64_t tk) {
  for (const auto& r : ranges)
    if (const int rc = check_range(fn, r[0], r[1])) return rc;
  SB_REQUIRE(!has_scale || (scale == scale && scale - scale == 0.f), "%s: the scale %g is not finite", fn, (double)scale);
  SB_REQUIRE(p_q == nullptr || aligned16(p_q), "%s: p_q must be 16-byte aligned", fn);
  SB_REQUIRE(causal == 0 || causal == 1, "%s: causal must be 0 or 1, got %d", fn, causal);
  if (mask != nullptr) {
    SB_REQUIRE(mask_stride_outer >= 0 && mask_stride_inner >= 0 && mask_stride_row >= 0,
               "%s: negative mask stride (outer %lld, inner %lld, row %lld)", fn, (long long)mask_stride_outer,
               (long long)mask_stride_inner, (long long)mask_stride_row);
    SB_REQUIRE(mask_inner > 0 && batch % mask_inner == 0, "%s: mask_inner = %lld must be positive and divide batch = %lld",
               fn, (long long)mask_inner, (long long)batch);
    SB_REQUIRE((reinterpret_cast<uintptr_t>(mask) & 3u) == 0, "%s: the mask must be 4-byte aligned", fn);
    const __int128 last = (__int128)(batch / mask_inner - 1) * mask_stride_outer +
                          (__int128)(mask_inner - 1) * mask_stride_inner + (__int128)(tq - 1) * mask_stride_row + tk - 1;
    SB_REQUIRE(last < ((__int128)1 << 62), "%s: the mask's offsets exceed 2^62 elements", fn);
  }
  return SB200_OK;
}

void at_set_qparams(AtParams& a, const float* const (&qparams)[8], const int (&ranges)[4][2], int has_scale,
                    float scale) {
  a.q_scale = qparams[0], a.q_zero = qparams[1], a.k_scale = qparams[2], a.k_zero = qparams[3];
  a.p_scale = qparams[4], a.p_zero = qparams[5], a.v_scale = qparams[6], a.v_zero = qparams[7];
  a.q_off = grid_offset(ranges[0][0]), a.k_off = grid_offset(ranges[1][0]);
  a.p_off = grid_offset(ranges[2][0]), a.v_off = grid_offset(ranges[3][0]);
  a.p_qmin = (float)ranges[2][0], a.p_qmax = (float)ranges[2][1];
  a.has_scale = has_scale != 0, a.scale = has_scale ? scale : 1.f;
}

size_t at_vpre_bytes(long long batch, long long tk, long long dv) {
  return align_up((size_t)(batch * dv) * (size_t)((tk + kAtKeys - 1) / kAtKeys) * 4, 1024);
}

int at_launch(const CUtensorMap& map_q, const CUtensorMap& map_k, const CUtensorMap& map_v, const AtParams& a, AtMask mk,
              const int8_t* vt, long long vt_stride, int* v_pre, long long batch, cudaStream_t st) {
  if (mk.causal) {
    const long long rows = batch * a.dv;
    int8_attention_vprefix_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(vt, v_pre, rows, (int)vt_stride,
                                                                              (a.Tk + kAtKeys - 1) / kAtKeys);
    SB_LAUNCHED();
    mk.v_pre = v_pre;
  }
  const long long ctas = batch * ((a.Tq + kAtRows - 1) / kAtRows);
  const bool masked = mk.mask != nullptr || mk.causal, cache = a.ks != a.Tk;
  if (!masked && !cache)
    return at_run<false, false>(map_q, map_k, map_v, a, mk, ctas, st);
  if (masked && !cache)
    return at_run<true, false>(map_q, map_k, map_v, a, mk, ctas, st);
  if (!masked)
    return at_run<false, true>(map_q, map_k, map_v, a, mk, ctas, st);
  return at_run<true, true>(map_q, map_k, map_v, a, mk, ctas, st);
}

}  // namespace sb200

using namespace sb200;

size_t sb200_int8_attention_workspace_bytes(int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv) {
  return at_workspace_bytes(batch, tq, tk, d, dv, 0);
}

size_t sb200_int8_attention_masked_workspace_bytes(int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv,
                                                   int causal) {
  return causal == 0 || causal == 1 ? at_workspace_bytes(batch, tq, tk, d, dv, causal) : 0;
}

int sb200_int8_attention(const float* q, const float* k, const float* v, const float* q_scale,
                         const float* q_zero_point, int qmin_q, int qmax_q, const float* k_scale,
                         const float* k_zero_point, int qmin_k, int qmax_k, const float* p_scale,
                         const float* p_zero_point, int qmin_p, int qmax_p, const float* v_scale,
                         const float* v_zero_point, int qmin_v, int qmax_v, int has_scale, float scale, float* out,
                         int8_t* p_q, int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv, void* workspace,
                         size_t workspace_bytes, void* stream) {
  return attention_run("sb200_int8_attention", q, k, v, q_scale, q_zero_point, qmin_q, qmax_q, k_scale, k_zero_point,
                       qmin_k, qmax_k, p_scale, p_zero_point, qmin_p, qmax_p, v_scale, v_zero_point, qmin_v, qmax_v,
                       has_scale, scale, nullptr, 0, 0, 1, 0, 0, out, p_q, batch, tq, tk, d, dv, workspace,
                       workspace_bytes, stream);
}

int sb200_int8_attention_masked(const float* q, const float* k, const float* v, const float* q_scale,
                                const float* q_zero_point, int qmin_q, int qmax_q, const float* k_scale,
                                const float* k_zero_point, int qmin_k, int qmax_k, const float* p_scale,
                                const float* p_zero_point, int qmin_p, int qmax_p, const float* v_scale,
                                const float* v_zero_point, int qmin_v, int qmax_v, int has_scale, float scale,
                                const float* mask, int64_t mask_stride_outer, int64_t mask_stride_inner,
                                int64_t mask_inner, int64_t mask_stride_row, int causal, float* out, int8_t* p_q,
                                int64_t batch, int64_t tq, int64_t tk, int64_t d, int64_t dv, void* workspace,
                                size_t workspace_bytes, void* stream) {
  return attention_run("sb200_int8_attention_masked", q, k, v, q_scale, q_zero_point, qmin_q, qmax_q, k_scale,
                       k_zero_point, qmin_k, qmax_k, p_scale, p_zero_point, qmin_p, qmax_p, v_scale, v_zero_point,
                       qmin_v, qmax_v, has_scale, scale, mask, mask_stride_outer, mask_stride_inner, mask_inner,
                       mask_stride_row, causal, out, p_q, batch, tq, tk, d, dv, workspace, workspace_bytes, stream);
}
